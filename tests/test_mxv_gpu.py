"""mxv / vxm entry by entry on every pull and push route, against mxv_reference.py.

Two value regimes throughout:
  int    weights and u in -8..8 without 0 (unless a case is about 0): every
         partial sum is exact, so every route must agree with the reference BIT
         FOR BIT, long rows included;
  float  arbitrary floats of both signs with magnitude in [0.5, 2): plus-adds
         within the float64 bound of mxv_reference.pull, min / max exactly.

Routes and the limits the designed shapes sit on (test_mxv_reference_cpu.py
checks these numbers against the #defines):
  merge pull   spmvMergeKernelT, tiles of TILE = SPMV_NT * SPMV_IPT = 1152 merge
               items (rows + entries); LaneMajor when colind or val is not 32-byte
               aligned (arrays adopted one element past an aligned address)
  hub pull     spmvHubKernel, nnz >= 2^22 and hub coverage >= 30 % (R-MAT-20 here;
               designed shapes in a child process with both thresholds at 0),
               weighted tiles of HUB_TILE = 1008 items, a row end weighs HUB_RW = 4,
               HUB_CAPACITY = 32768 hub columns, HUB_GROUPS = 8 tile groups a CTA
  Boolean pull spmvMaskedOrPullBitsKernel (identity 0: LogicalOrAnd) and
               spmvMaskedOrPullKernel (CustomLessPlus, NotEqualToPlus,
               CustomLessLess), scmp x earlyexit x opreuse; warps take PULL_WPI = 4
               mask words a step
  push         spmspvPushKernel<StructOnly, MaskMode>; one-CTA degree scan up to
               DEGSCAN_MAX = 8192 frontier entries + 1, cub beyond; PUSH_TILE = 2048
               edges a tile, unstaged search when a tile spans more than
               PUSH_SEG = 2050 frontier entries; edge-share hand-back to the pull
               from 4096 frontier entries under mxvmode 0
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import mxm_reference as mref
import mxv_reference as ref
from support import Csr, csr, device_matrix, gb, launch_count

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SPMV_NT, SPMV_IPT = 128, 9
TILE = SPMV_NT*SPMV_IPT
HUB_RW, HUB_TILE, HUB_CAPACITY, HUB_GROUPS = 4, 1008, 32768, 8
HUB_ROWEND_LIMIT = HUB_TILE//HUB_RW
PUSH_TILE, PUSH_SEG = 2048, 2050
DEGSCAN_MAX = 8192
PULL_WPI = 4

# child processes of this file run with these set (the knobs are read once a process)
HUB_FORCED = (os.environ.get("GB200_SPMV_HUB_MIN_NNZ") == "0" and
              os.environ.get("GB200_SPMV_HUB_MIN_PCT") == "0")
MERGE_FORCED = os.environ.get("GB200_SPMV_HUB") == "0"

PLUS, MINPLUS, MAXMUL = 1, 2, 3
PULL_SEMIRINGS = [PLUS, MINPLUS, MAXMUL]
LOR, CLESS_PLUS, NE_PLUS, CLESS_LESS = 0, 9, 12, 15
MINMUL, MINSECOND = 10, 13
FLT_MAX = mref.FLT_MAX
INTS = np.float32([v for v in range(-8, 9) if v != 0])


def values(rng, regime, n):
    if regime == "int":
        return rng.choice(INTS, n).astype(np.float32)
    sign = np.where(rng.rand(n) < 0.5, -1, 1)
    return (sign*rng.uniform(0.5, 2.0, n)).astype(np.float32)


# ---------------------------------------------------------------------------
# host-side structures
# ---------------------------------------------------------------------------

_PRIMES = [7919, 104729, 15485863, 32452843]


def structure(rng, lengths, ncols, regime="int"):
    """Csr with the given row lengths; each row's columns distinct and sorted."""
    lengths = np.asarray(lengths, np.int64)
    assert lengths.max(initial=0) <= ncols
    nrows = len(lengths)
    rows = np.repeat(np.arange(nrows), lengths)
    pos = np.arange(len(rows)) - np.repeat(np.cumsum(lengths) - lengths, lengths)
    stride = np.array([p for p in _PRIMES if np.gcd(p, ncols) == 1][:2], np.int64)
    start = rng.randint(0, ncols, nrows)
    step = rng.choice(stride, nrows)
    cols = (start[rows] + pos*step[rows]) % ncols
    return csr(nrows, ncols, rows, cols, values(rng, regime, len(rows)), np.float32)


def lengths_hitting(targets):
    """Row lengths whose row-end merge items land on the given diagonals."""
    out, pos = [], 0
    for t in targets:
        assert t >= pos
        out.append(t - pos)
        pos = t + 1
    return out


def merge_cases():
    """(name, ncols, row lengths) of the designed merge-pull shapes."""
    T = TILE
    cases = []
    # one long row starting at a tile boundary and one item either side of it:
    # 127 rows of 8 (9 items each) plus one row of 7, 8 or 9
    for span in (1, 2, 3, 40):
        for delta in (-1, 0, 1):
            lens = [8]*127 + [8 + delta, span*T, 3, 0, 5]
            cases.append(("span%d_%+d" % (span, delta), span*T + 17, lens))
    targets = [c*T + d for c in range(1, 10) for d in (0, -1, 1)]
    targets = sorted(set(targets))
    cases.append(("rowends_on_tiles", 2*T, lengths_hitting(targets) + [4]))
    cases.append(("empty_runs", 300, [5] + [0]*(T + 1) + [7] + [0]*(2*T) + [3, 0]))
    for L, ncols in ((1, 29), (8, 29), (9, 1000)):
        cases.append(("all_len%d_n%d" % (L, ncols), ncols, [L]*3001))
    for k, d in ((4, 0), (4, -1), (4, 1)):
        lens = [8]*(k*SPMV_NT)                # 9 items a row: k*T in all
        lens[-1] += d
        cases.append(("total_%dT%+d" % (k, d), 64, lens))
    # a row from mid-warp 0 to warp 3 of tile 0 (warps take 288 items each)
    cases.append(("cross_warp", 1000, [99, 900, 2, 2, 1, 0, 300]))
    cases.append(("nnz_lt_8", 5, [2, 0, 3]))
    cases.append(("nnz_mod8", 77, [7]*143 + [2]))
    cases.append(("one_by_one", 1, [1]))
    cases.append(("one_row", 3001, [3001]))
    cases.append(("nnz0", 40, [0]*37))
    return cases


MERGE_CASES = merge_cases()


# ---------------------------------------------------------------------------
# device side
# ---------------------------------------------------------------------------

def dense_vector(gb, x):
    v = gb.Vector(len(x))
    v.build(np.asarray(x, np.float32))
    return v


def pull(gb, M, orient, semiring, u, mask=None, scmp=False, w_old=None, desc=None,
         count=False):
    """One pull through mxv (CSR rows) or vxm (CSC columns); returns w (and the
    launches of a second, warm call when count is set)."""
    desc = gb.Descriptor(mxvmode=2) if desc is None else desc
    if scmp:
        desc.toggle(gb.Desc_field.GrB_MASK)
    n_out = M.nrows() if orient == "mxv" else M.ncols()
    uv = dense_vector(gb, u)
    w = gb.Vector(n_out)
    if w_old is not None:
        w.build(np.asarray(w_old, np.float32))
    m = None
    if mask is not None:
        m = mask if isinstance(mask, gb.Vector) else dense_vector(gb, mask)
    accum = None if w_old is None else "accum"

    def call():
        if orient == "mxv":
            gb.mxv(w, m, accum, semiring, M, uv, desc)
        else:
            gb.vxm(w, m, accum, semiring, uv, M, desc)
    call()
    assert desc.lastmxv == gb.Desc_value.GrB_PULLONLY
    got = w.extractTuples()
    if not count:
        return got
    before = launch_count(gb)
    call()
    launches = launch_count(gb) - before
    assert np.array_equal(w.extractTuples().view(np.uint32), got.view(np.uint32))
    return got, launches


def check_pull(got, want, bound, where=""):
    """bound None: equal entry by entry (NaN equal to NaN, -0 equal to +0);
    otherwise |got - want| <= bound (bound 0: exact)."""
    got = np.asarray(got)
    assert got.shape == want.shape, where
    if bound is None:
        ok = (got == want) | (np.isnan(got) & np.isnan(want))
    else:
        ok = np.abs(got.astype(np.float64) - want) <= bound
    if not ok.all():
        i = int(np.argmin(ok))
        pytest.fail("%s: %d of %d differ, first at %d: got %r want %r" % (
            where, int((~ok).sum()), len(ok), i, got[i], want[i]))


def reference_pull(semiring, S, u, regime, **kw):
    want, bound = ref.pull(semiring, S.ptr, S.ind, S.val, u, **kw)
    if bound is not None and regime == "int":
        bound = np.zeros_like(bound)       # integer sums below 2^24 are exact
    return want, bound


def expected_launches(S, offset):
    """Warm pull launches without mask or accum: 3 on the hub route (pre-pass,
    SpMV, carry fix-up), 2 on the merge route (SpMV, carry fix-up)."""
    if S.nrows == 0:
        return 0
    aligned = offset == 0 or S.nnz == 0           # an empty matrix adopts nothing
    hub = (not MERGE_FORCED and aligned and
           (S.nnz >= (0 if HUB_FORCED else 1 << 22)))
    return 3 if hub else 2


def run_pull_case(gb, S, regime, seed, semirings=PULL_SEMIRINGS, offsets=(0, 1)):
    """Every semiring, both orientations, aligned and lane-major arrays: each must
    match the reference, and the two alignments each other bit for bit."""
    rng = np.random.RandomState(seed)
    u = values(rng, regime, S.ncols)
    mats = {}
    for off in offsets:
        mats[("mxv", off)] = device_matrix(gb, S, offset=off)       # pulls over its CSR
        mats[("vxm", off)] = device_matrix(gb, S.T, offset=off)     # pulls over its CSC
    for sem in semirings:
        want, bound = reference_pull(sem, S, u, regime)
        for orient in ("mxv", "vxm"):
            outs = []
            for off in offsets:
                got, launches = pull(gb, mats[(orient, off)], orient, sem, u,
                                     count=True)
                where = "semiring %d %s offset %d" % (sem, orient, off)
                check_pull(got, want, bound, where)
                assert launches == expected_launches(S, off), where
                outs.append(got.view(np.uint32))
            # the same route, or an exact fold: the two forms agree in every bit
            same_route = len({expected_launches(S, off) for off in offsets}) == 1
            if same_route or sem != PLUS or regime == "int":
                for o in outs[1:]:
                    assert np.array_equal(o, outs[0]), "aligned and lane-major differ"


# ---------------------------------------------------------------------------
# merge pull
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["int", "float"])
@pytest.mark.parametrize("case", MERGE_CASES, ids=[c[0] for c in MERGE_CASES])
def test_merge_pull_designed(gb, case, regime):
    name, ncols, lens = case
    S = structure(np.random.RandomState(len(lens)), lens, ncols, regime)
    run_pull_case(gb, S, regime, seed=ncols + len(lens))


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["int", "float"])
@pytest.mark.parametrize("shape", [(3000, 29), (29, 3000), (1000, 4097), (5000, 1)])
def test_merge_pull_rectangular(gb, shape, regime):
    m, n = shape
    rng = np.random.RandomState(m*7 + n)
    lens = np.minimum(rng.randint(0, 40, m), n)
    lens[rng.rand(m) < 0.1] = 0
    S = structure(rng, lens, n, regime)
    run_pull_case(gb, S, regime, seed=m + n)


# ---------------------------------------------------------------------------
# hub pull: designed shapes (forced in a child), natural selection at R-MAT-20
# ---------------------------------------------------------------------------

def hub_cases():
    out = []
    out.append(("len1_packed", 4000, [1]*20000))
    out.append(("len2_packed", 4000, [2]*20000))
    out.append(("len12_mixed", 4000, [1, 2]*10000 + [0, 0, 1]))
    out.append(("long_row", 30000, [3, 20*HUB_TILE + 5, 0, 1, 7]))
    # > capacity columns, every one referenced exactly twice: ties at the threshold
    out.append(("ties_above_capacity", 40000, [2]*40000))
    out.append(("few_hubs", 1000, [5]*3000))
    out.append(("all_hubs", 5000, [40]*500))
    out.append(("nnz_mod8", 3001, [7]*1001 + [3]))
    out.append(("rect_narrow", 100, [9]*7000))
    out.append(("rect_wide", 50000, [30]*700))
    return out


HUB_CASES = hub_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["int", "float"])
@pytest.mark.parametrize("case", HUB_CASES, ids=[c[0] for c in HUB_CASES])
def test_hub_designed(gb, case, regime):
    """In process these run the merge kernel; under the forced thresholds
    (test_hub_forced_in_a_child) the aligned forms run the hub kernel."""
    name, ncols, lens = case
    rng = np.random.RandomState(len(lens) + ncols)
    if name == "ties_above_capacity":
        # row i holds columns i and i + 1 (mod ncols): every column exactly twice
        rows = np.repeat(np.arange(ncols), 2)
        cols = (rows + np.tile([0, 1], ncols)) % ncols
        S = csr(ncols, ncols, rows, cols, values(rng, regime, len(rows)), np.float32)
        assert np.all(np.bincount(S.ind, minlength=ncols) == 2)
    else:
        S = structure(rng, lens, ncols, regime)
    run_pull_case(gb, S, regime, seed=ncols)


@pytest.mark.gpu
def test_hub_many_tiles_per_group(gb):
    """At least 4 weighted tiles for every tile group of the persistent grid (one
    CTA per SM): each group goes round its staging ring several times."""
    m, ncols, lens = 300000, 6000, [12]*300000
    tiles = (HUB_RW*m + sum(lens) + HUB_TILE - 1)//HUB_TILE
    assert tiles >= 4*HUB_GROUPS*gb.sm_count()
    S = structure(np.random.RandomState(4), lens, ncols, "int")
    run_pull_case(gb, S, "int", seed=4, semirings=[PLUS, MINPLUS], offsets=(0,))


@pytest.fixture(scope="module")
def rmat20(gb):
    """Symmetrised R-MAT-20 (edge factor 16) with unsymmetric values, so that
    mxv and vxm traverse different matrices: returns (Csr of A, Csr of A's CSC,
    Matrix)."""
    import torch
    from graphblast_b200 import graphs
    n = 1 << 20
    src, dst = graphs.rmat_edges(20, 16, seed=3)
    rowptr, colind = graphs.build_csr(n, src, dst, undirected=True)
    del src, dst
    rng = torch.Generator(device="cuda")
    rng.manual_seed(5)
    ints = torch.randint(1, 9, (colind.numel(),), generator=rng, device="cuda",
                         dtype=torch.int32)
    sign = torch.randint(0, 2, (colind.numel(),), generator=rng, device="cuda",
                         dtype=torch.int32)*2 - 1
    val = (ints*sign).to(torch.float32)
    cscval = graphs.transpose_values(n, rowptr, colind, val)
    M = graphs.matrix_from_csr(n, rowptr, colind, val, symmetric=True, cscval=cscval)
    M._keep.append(cscval)
    ptr = rowptr.cpu().numpy().astype(np.int64)
    ind = colind.cpu().numpy().astype(np.int64)
    A = Csr(n, n, ptr, ind, val.cpu().numpy())
    At = Csr(n, n, ptr, ind, cscval.cpu().numpy())
    assert A.nnz >= 1 << 22
    return A, At, M


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["int", "float"])
def test_hub_natural_rmat20(gb, rmat20, regime):
    """R-MAT-20 takes the hub route on its own (about 30 tiles per tile group:
    the staging ring wraps many times).  Weights are integers in -8..8; with an
    integer u every route is exact, with a float u the plus-add is held to the
    float64 bound and to scipy's float64 product."""
    A, At, M = rmat20
    rng = np.random.RandomState(20)
    u = values(rng, regime, A.nrows)
    for orient, S in (("mxv", A), ("vxm", At)):
        for sem in PULL_SEMIRINGS:
            want, bound = reference_pull(sem, S, u, regime)
            got, launches = pull(gb, M, orient, sem, u, count=True)
            check_pull(got, want, bound, "semiring %d %s" % (sem, orient))
            assert launches == (2 if MERGE_FORCED else 3)
            if sem == PLUS and regime == "float":
                import scipy.sparse as sp
                sp_w = S.scipy() @ u.astype(np.float64)
                assert np.allclose(want, sp_w, rtol=0, atol=1e-6*np.abs(sp_w).max())


def _child(env, kexpr):
    full = dict(os.environ)
    full.update(env)
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider",
           os.path.abspath(__file__), "-k", kexpr]
    r = subprocess.run(cmd, env=full, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=1500, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:]
    assert " passed" in r.stdout


@pytest.mark.gpu
@pytest.mark.skipif(HUB_FORCED or MERGE_FORCED, reason="already a child")
def test_hub_forced_in_a_child():
    """The designed merge, hub and cache cases with the hub thresholds at 0: the
    aligned forms of every shape take the hub kernel."""
    _child({"GB200_SPMV_HUB": "1", "GB200_SPMV_HUB_MIN_NNZ": "0",
            "GB200_SPMV_HUB_MIN_PCT": "0"},
           "merge_pull or hub_designed or hub_many or caches")


@pytest.mark.gpu
@pytest.mark.skipif(HUB_FORCED or MERGE_FORCED, reason="already a child")
def test_merge_forced_in_a_child_on_rmat20():
    """The same R-MAT-20 pulls through the merge kernel (GB200_SPMV_HUB=0): both
    routes are held to the same exact reference on the same big inputs."""
    _child({"GB200_SPMV_HUB": "0"}, "hub_natural")


# ---------------------------------------------------------------------------
# generic pull with mask and accum
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("accum", [False, True])
@pytest.mark.parametrize("masking", ["none", "mask", "scmp"])
@pytest.mark.parametrize("semiring", [PLUS, MINPLUS])
@pytest.mark.parametrize("orient", ["mxv", "vxm"])
def test_generic_pull_mask_and_accum(gb, orient, semiring, masking, accum):
    """Masked-out rows hold the semiring's identity (FLT_MAX for MinimumPlus),
    then accum folds with the semiring's add."""
    rng = np.random.RandomState(semiring*10 + len(masking))
    S = structure(rng, np.minimum(rng.randint(0, 30, 1500), 700), 700, "int")
    M = device_matrix(gb, S if orient == "mxv" else S.T)
    u = values(rng, "int", S.ncols)
    mask = rng.choice(np.float32([0, 0, -0.0, 1, -3, 0.25]), S.nrows)
    w_old = values(rng, "int", S.nrows) if accum else None
    kw = {} if masking == "none" else {"mask": mask, "scmp": masking == "scmp"}
    want, bound = reference_pull(semiring, S, u, "int", w_old=w_old, **kw)
    got = pull(gb, M, orient, semiring, u, w_old=w_old, **kw)
    check_pull(got, want, bound, "%s %s" % (orient, masking))
    if masking != "none" and semiring == MINPLUS and not accum:
        assert np.all(got[~ref._kept(mask, masking == "scmp")] == FLT_MAX)


@pytest.mark.gpu
@pytest.mark.parametrize("accum", [False, True])
def test_generic_pull_sparse_mask_is_refused_and_leaves_w(gb, accum):
    rng = np.random.RandomState(1)
    S = structure(rng, rng.randint(1, 10, 300), 300, "int")
    M = device_matrix(gb, S)
    u = dense_vector(gb, values(rng, "int", 300))
    w_old = values(rng, "int", 300)
    w = dense_vector(gb, w_old)
    m = gb.Vector(300)
    m.build(np.array([3, 7], np.int32), np.float32([1, 1]))
    with pytest.raises(gb.GraphBLASError) as e:
        gb.mxv(w, m, "accum" if accum else None, MINPLUS, M, u,
               gb.Descriptor(mxvmode=2))
    assert e.value.info == gb.Info.GrB_NOT_IMPLEMENTED
    assert np.array_equal(w.extractTuples(), w_old)


@pytest.mark.gpu
def test_pull_and_push_disagree_on_identity_valued_u(gb):
    """MinimumPlus with u = FLT_MAX on a negative weight: the pull has no identity
    short-circuit (FLT_MAX + -2^127 is finite), the push has one (the product is
    the identity).  Each route follows its own reference."""
    big = np.float32(-2.0**127)
    S = csr(2, 3, [0, 0, 1], [0, 1, 2], np.float32([big, 1, 2]), np.float32)
    At = device_matrix(gb, S)                 # vxm over A: pull over CSC, push over CSR
    u = np.float32([FLT_MAX, 1])
    want, _ = ref.pull(MINPLUS, S.T.ptr, S.T.ind, S.T.val, u)
    got = pull(gb, At, "vxm", MINPLUS, u)
    check_pull(got, want, None, "pull")
    assert got[0] == np.float32(FLT_MAX) + big
    w_ind, w_val = run_push(gb, At, "vxm", MINPLUS, [0, 1], u)
    r_ind, r_val = ref.push(MINPLUS, S.ptr, S.ind, S.val, [0, 1], u, 3)
    assert np.array_equal(w_ind, r_ind) and np.array_equal(w_val, r_val)
    assert w_val[0] == FLT_MAX


# ---------------------------------------------------------------------------
# fused Boolean pull
# ---------------------------------------------------------------------------

def square(rng, n, maxlen=12):
    return structure(rng, np.minimum(rng.randint(0, maxlen, n), n), n, "int")


def mask_values(rng, kind, n):
    if kind == "01":
        return rng.choice(np.float32([0, 1]), n)
    return rng.choice(np.float32([0, -0.0, 2.5, -1, FLT_MAX]), n)


def make_mask(gb, x, shadow):
    """Dense mask vector of values x.  shadow 'current': its bitmap shadow is kept
    by fill() + assign(); 'none': only values (the kernel builds the shadow)."""
    if shadow == "none":
        return dense_vector(gb, x)
    nz = np.nonzero(x != 0)[0].astype(np.int32)
    assert np.all(x[nz] == 1), "a current shadow is built for 0/1 masks"
    m = gb.Vector(len(x))
    m.fill(0.0)
    if len(nz):
        sel = gb.Vector(len(x))
        sel.build(nz, np.ones(len(nz), np.float32))
        gb.assign(m, sel, None, 1.0, None, 0, gb.Descriptor())
    return m


def bool_pull(gb, M, orient, semiring, u, mask, scmp, earlyexit, opreuse):
    desc = gb.Descriptor(mxvmode=2, fusedmask=1, earlyexit=int(earlyexit),
                         opreuse=int(opreuse))
    if scmp:
        desc.toggle(gb.Desc_field.GrB_MASK)
    n_out = M.nrows() if orient == "mxv" else M.ncols()
    w = gb.Vector(n_out)
    uv = u if isinstance(u, gb.Vector) else dense_vector(gb, u)
    if orient == "mxv":
        gb.mxv(w, mask, None, semiring, M, uv, desc)
    else:
        gb.vxm(w, mask, None, semiring, uv, M, desc)
    assert desc.lastmxv == gb.Desc_value.GrB_PULLONLY
    return w


BOOL_SIZES = [1, 31, 33, 127, 129, 1003]
VARIANTS = [(s, e, o) for s in (False, True) for e in (False, True) for o in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("shadow", ["none", "current"])
@pytest.mark.parametrize("variant", VARIANTS,
                         ids=["scmp%d_ee%d_or%d" % tuple(map(int, v)) for v in VARIANTS])
def test_bool_pull_bits_form(gb, variant, shadow):
    scmp, earlyexit, opreuse = variant
    for n in BOOL_SIZES:
        rng = np.random.RandomState(n)
        S = square(rng, n)
        for orient in ("mxv", "vxm"):
            M = device_matrix(gb, S if orient == "mxv" else S.T)
            mk = mask_values(rng, "01" if shadow == "current" else "any", n)
            u = rng.choice(np.float32([0, 0, -0.0, 1, 3.5]), n)
            w = bool_pull(gb, M, orient, LOR, u, make_mask(gb, mk, shadow), scmp,
                          earlyexit, opreuse)
            want = ref.bool_pull(S.ptr, S.ind, mk, u, 0.0, scmp, opreuse)
            got = w.extractTuples()
            assert np.array_equal(got, want), (n, orient)


@pytest.mark.gpu
@pytest.mark.parametrize("semiring", [CLESS_PLUS, NE_PLUS, CLESS_LESS])
@pytest.mark.parametrize("variant", VARIANTS,
                         ids=["scmp%d_ee%d_or%d" % tuple(map(int, v)) for v in VARIANTS])
def test_bool_pull_value_form(gb, variant, semiring):
    scmp, earlyexit, opreuse = variant
    for n in (1, 33, 129, 1003):
        rng = np.random.RandomState(n + semiring)
        S = square(rng, n)
        M = device_matrix(gb, S)
        mk = mask_values(rng, "any", n)
        u = rng.choice(np.float32([FLT_MAX, FLT_MAX, 0, -0.0, 1, -2]), n)
        w = bool_pull(gb, M, "mxv", semiring, u, dense_vector(gb, mk), scmp,
                      earlyexit, opreuse)
        want = ref.bool_pull(S.ptr, S.ind, mk, u, FLT_MAX, scmp, opreuse)
        assert np.array_equal(w.extractTuples(), want), n


@pytest.mark.gpu
def test_bool_pull_rmat16_and_chained(gb):
    """A 2^16-row R-MAT; the lazily held result is read, used as the next mask
    and as the next push frontier."""
    import oracle_binding as orc
    rp, ci = orc.rmat_csr(16)
    n = len(rp) - 1
    S = Csr(n, n, rp, ci, np.ones(len(ci), np.float32))
    M = device_matrix(gb, S)
    rng = np.random.RandomState(16)
    mk = (rng.rand(n) < 0.7).astype(np.float32)
    u = (rng.rand(n) < 0.05).astype(np.float32)
    for scmp, ee, opr in VARIANTS:
        w = bool_pull(gb, M, "mxv", LOR, u, make_mask(gb, mk, "current"), scmp, ee, opr)
        want = ref.bool_pull(S.ptr, S.ind, mk, u, 0.0, scmp, opr)
        assert np.array_equal(w.extractTuples(), want)
    # chain: w1 = pull(!visited, u); w2 = pull(mask=w1, u=w1); push from w2
    w1 = bool_pull(gb, M, "mxv", LOR, u, make_mask(gb, mk, "current"), True, True, False)
    want1 = ref.bool_pull(S.ptr, S.ind, mk, u, 0.0, True, False)
    w2 = bool_pull(gb, M, "mxv", LOR, w1, w1, False, False, False)
    want2 = ref.bool_pull(S.ptr, S.ind, want1, want1, 0.0, False, False)
    desc = gb.Descriptor(mxvmode=1)
    w2.dense2sparse(0.0, desc)
    f_ind, f_val = w2.extractTuples(sparse=True)
    assert np.array_equal(f_ind, np.nonzero(want2)[0]) and np.all(f_val == 1)
    w3 = gb.Vector(n)
    gb.vxm(w3, None, None, LOR, w2, M, desc)
    assert desc.lastmxv == gb.Desc_value.GrB_PUSHONLY
    r_ind, r_val = ref.push(LOR, S.ptr, S.ind, S.val, f_ind, f_val, n)
    g_ind, g_val = w3.extractTuples(sparse=True)
    assert np.array_equal(g_ind, r_ind) and np.array_equal(g_val, r_val)
    assert np.array_equal(w1.extractTuples(), want1)


# ---------------------------------------------------------------------------
# push
# ---------------------------------------------------------------------------

def run_push(gb, M, orient, semiring, f_ind, f_val, mask=None, scmp=False,
             struconly=False, mode=1, switchpoint=None):
    knobs = dict(mxvmode=mode, struconly=int(struconly))
    if switchpoint is not None:
        knobs["switchpoint"] = switchpoint
    desc = gb.Descriptor(**knobs)
    if scmp:
        desc.toggle(gb.Desc_field.GrB_MASK)
    n_in = M.nrows() if orient == "vxm" else M.ncols()
    n_out = M.ncols() if orient == "vxm" else M.nrows()
    u = gb.Vector(n_in)
    u.build(np.asarray(f_ind, np.int32), np.asarray(f_val, np.float32))
    w = gb.Vector(n_out)
    if orient == "vxm":
        gb.vxm(w, mask, None, semiring, u, M, desc)
    else:
        gb.mxv(w, mask, None, semiring, M, u, desc)
    if mode == 1:
        assert desc.lastmxv == gb.Desc_value.GrB_PUSHONLY
        assert w.getStorage() == gb.Storage.GrB_SPARSE
        return w.extractTuples(sparse=True)
    return w, desc.lastmxv


def check_push(got, want, where=""):
    g_ind, g_val = got
    r_ind, r_val = want
    assert np.array_equal(g_ind, r_ind), where
    assert np.array_equal(g_val, r_val), where


PUSH_MASKS = [("none", "none"), ("mask", "none"), ("mask", "current"),
              ("scmp", "none"), ("scmp", "current")]


@pytest.mark.gpu
@pytest.mark.parametrize("masking,shadow", PUSH_MASKS)
@pytest.mark.parametrize("struconly", [False, True])
def test_push_instantiations(gb, struconly, masking, shadow):
    """<StructOnly, MaskMode> x mask read as values or as its bitmap shadow, on a
    rectangular matrix both ways (vxm: CSR of A, mxv: CSC of A)."""
    rng = np.random.RandomState(int(struconly)*7 + len(masking))
    m, n = 3000, 1234
    S = structure(rng, np.minimum(rng.randint(0, 40, m), n), n, "int")
    M = device_matrix(gb, S)
    for orient, T, n_out in (("vxm", S, n), ("mxv", S.T, m)):
        f = np.sort(rng.choice(T.nrows, T.nrows//5, replace=False))
        fv = values(rng, "int", len(f))
        mk = mask_values(rng, "01" if shadow == "current" else "any", n_out)
        mask = None if masking == "none" else make_mask(gb, mk, shadow)
        for sem in (PLUS, MINPLUS):
            got = run_push(gb, M, orient, sem, f, fv, mask, masking == "scmp",
                           struconly)
            want = ref.push(sem, T.ptr, T.ind, T.val, f, fv, n_out,
                            None if masking == "none" else mk, masking == "scmp",
                            struconly)
            check_push(got, want, "%s semiring %d" % (orient, sem))


@pytest.mark.gpu
@pytest.mark.parametrize("nf", [1, DEGSCAN_MAX - 1, DEGSCAN_MAX, DEGSCAN_MAX + 1, 20000])
def test_push_frontier_sizes(gb, nf):
    rng = np.random.RandomState(nf)
    n = 30000
    S_int = structure(rng, rng.randint(0, 7, n), n, "int")
    f = np.sort(rng.choice(n, nf, replace=False))
    for regime in ("int", "float"):
        S = S_int if regime == "int" else S_int.with_values(values(rng, regime, S_int.nnz))
        M = device_matrix(gb, S)
        fv = values(rng, regime, nf)
        for sem in (PLUS, MINPLUS, MAXMUL):
            got = run_push(gb, M, "vxm", sem, f, fv)
            r_ind, r_val = ref.push(sem, S.ptr, S.ind, S.val, f, fv, n)
            if sem == PLUS and regime == "float":
                # atomics add in any order: within the fold's bound
                assert np.array_equal(got[0], r_ind)
                w64, bound = ref.pull(PLUS, *_gather_rows(S, f, fv, n))
                assert np.all(np.abs(got[1] - w64[r_ind]) <= bound[r_ind])
            else:
                check_push(got, (r_ind, r_val), "semiring %d %s" % (sem, regime))


def _gather_rows(S, f, fv, n):
    """The push of frontier (f, fv) restated as a pull: (ptr, ind, val, u) over
    the transpose of the frontier's rows, u = fv."""
    sub_rows = np.repeat(np.arange(len(f)), S.ptr[f + 1] - S.ptr[f])
    edge = np.concatenate([np.arange(S.ptr[r], S.ptr[r + 1]) for r in f]) \
        if len(f) else np.zeros(0, np.int64)
    T = csr(n, len(f), S.ind[edge], sub_rows, S.val[edge], np.float32)
    return T.ptr, T.ind, T.val, fv


@pytest.mark.gpu
def test_push_unstaged_search(gb):
    """A frontier of 5000 where vertex 0 (10 edges) and vertex 4001 (3000 edges)
    are separated by 4000 isolated vertices: the first tile spans 4002 frontier
    entries, more than PUSH_SEG, and takes the unstaged search."""
    rng = np.random.RandomState(50)
    n = 6000
    lens = np.zeros(n, np.int64)
    lens[0] = 10
    lens[4001] = 3000
    lens[4002:5000] = rng.randint(0, 4, 998)
    S = structure(rng, lens, 5000, "int")
    M = device_matrix(gb, S)
    f = np.arange(5000)
    assert 4002 > PUSH_SEG and lens[0] + lens[4001] > PUSH_TILE
    fv = values(rng, "int", len(f))
    for sem in (PLUS, MINPLUS, MAXMUL):
        got = run_push(gb, M, "vxm", sem, f, fv)
        check_push(got, ref.push(sem, S.ptr, S.ind, S.val, f, fv, 5000))


@pytest.mark.gpu
def test_push_hands_back_to_pull(gb):
    """A 4096+ frontier owning more than a third of the entries under mxvmode 0:
    the push hands the call to the pull, whose result equals the forced push's."""
    rng = np.random.RandomState(60)
    n = 20000
    lens = rng.randint(0, 3, n)
    lens[:5000] = rng.randint(5, 12, 5000)
    S = structure(rng, lens, n, "int")
    M = device_matrix(gb, S)
    f = np.arange(5000)
    fv = values(rng, "int", len(f))
    r_ind, r_val = ref.push(PLUS, S.ptr, S.ind, S.val, f, fv, n)
    assert S.ptr[5000] > S.nnz/3
    w, last = run_push(gb, M, "vxm", PLUS, f, fv, mode=0, switchpoint=0.9)
    assert last == gb.Desc_value.GrB_PULLONLY
    dense = np.zeros(n, np.float32)
    dense[r_ind] = r_val
    assert np.array_equal(w.extractTuples(), dense)
    check_push(run_push(gb, M, "vxm", PLUS, f, fv), (r_ind, r_val))


@pytest.mark.gpu
def test_push_negative_and_identity_values(gb):
    """Negative weights and frontier values, and values equal to the identity
    (the push's short-circuit: the product is the identity, the entry present)."""
    rng = np.random.RandomState(70)
    n = 2000
    S = structure(rng, rng.randint(0, 8, n), n, "int")
    for sem, ident in ((MINPLUS, FLT_MAX), (PLUS, 0.0), (MAXMUL, 0.0), (MINMUL, FLT_MAX)):
        vals = S.val.copy()
        vals[rng.rand(len(vals)) < 0.2] = ident
        T = S.with_values(vals)
        M = device_matrix(gb, T)
        f = np.sort(rng.choice(n, 300, replace=False))
        fv = values(rng, "int", len(f))
        fv[rng.rand(len(f)) < 0.2] = ident
        got = run_push(gb, M, "vxm", sem, f, fv)
        check_push(got, ref.push(sem, T.ptr, T.ind, T.val, f, fv, n), "semiring %d" % sem)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["minmul", "minmul_mirrored", "minsecond",
                                  "minsecond_mirrored"])
def test_push_min_of_negative_and_negative_zero(gb, case):
    """Each of 4 columns gets 64 in-edges from 64 frontier vertices of degree 1;
    products alternate -4 and -0.0 in edge order.  min is -4: an integer atomicMin
    of -0.0 (INT_MIN as an int) must not overwrite the cell."""
    ncols, per = 4, 64
    rows = np.arange(ncols*per)
    cols = rows % ncols
    k = rows // ncols                              # position among the column's edges
    first = (k % 2 == 0) if not case.endswith("mirrored") else (k % 2 == 1)
    if case.startswith("minmul"):
        sem = MINMUL
        weights = np.where(first, -4, -1).astype(np.float32)
        u = np.where(first, 1, 0).astype(np.float32)
    else:
        sem = MINSECOND
        weights = np.ones(len(rows), np.float32)
        u = np.where(first, -4, -0.0).astype(np.float32)
    S = csr(len(rows), ncols, rows, cols, weights, np.float32)
    M = device_matrix(gb, S)
    got = run_push(gb, M, "vxm", sem, rows, u)
    want = ref.push(sem, S.ptr, S.ind, S.val, rows, u, ncols)
    assert list(want[1]) == [-4]*ncols
    check_push(got, want)
    # the pull over the same products
    w, _ = ref.pull(sem, S.T.ptr, S.T.ind, S.T.val, u)
    assert np.array_equal(pull(gb, M, "vxm", sem, u), w)


# ---------------------------------------------------------------------------
# caches follow a rebuilt structure
# ---------------------------------------------------------------------------

@pytest.mark.gpu
def test_caches_follow_a_rebuilt_structure(gb):
    """One Matrix object rebuilt with the same n and nnz but another structure:
    merge tile partition, first-neighbour summary and hub index (under the forced
    thresholds) must be recomputed."""
    n = 4000
    rng = np.random.RandomState(80)
    lens1 = rng.randint(0, 20, n)
    lens2 = lens1[::-1].copy()                       # same nnz, other row lengths
    S1 = structure(rng, lens1, n, "int")
    S2 = structure(rng, lens2, n, "int")
    assert S1.nnz == S2.nnz and not np.array_equal(S1.ptr, S2.ptr)
    M = gb.Matrix(n, n)
    u = values(rng, "int", n)
    mk = mask_values(rng, "any", n)
    ub = rng.choice(np.float32([0, 1]), n)
    for S in (S1, S2, S1):
        device_matrix(gb, S, into=M)
        for sem in (PLUS, MINPLUS):
            want, bound = reference_pull(sem, S, u, "int")
            got, launches = pull(gb, M, "mxv", sem, u, count=True)
            check_pull(got, want, bound, "semiring %d" % sem)
            assert launches == expected_launches(S, 0)
        w = bool_pull(gb, M, "mxv", LOR, ub, dense_vector(gb, mk), True, True, False)
        assert np.array_equal(w.extractTuples(),
                              ref.bool_pull(S.ptr, S.ind, mk, ub, 0.0, True, False))
