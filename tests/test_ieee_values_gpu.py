"""Every FP32 route entry by entry with NaN of both signs, infinities, signed zeros,
subnormals and FLT_MAX, against the contract of ieee_reference.py.

The other suites use small integers or +-uniform(0.5, 2): nothing there would
notice a route that flushes subnormals, fuses a multiply into an add, or lets a NaN
through a min or max.  Here the operands are designed so that every fold rounds
the same in any order, which makes every plus fold comparable bit for bit:

  * fixed-point folds: values k 2^-149 (mostly subnormal) against units +-1, 2, 4,
    every partial sum below 2^-125, where the multiples of 2^-149 are exact; an
    atomic or a kernel that flushes subnormals gives 0 there;
  * specials planted in those folds: a NaN, +-inf, -0.0 and FLT_MAX decide a fold
    whatever its order (inf + -inf is NaN, FLT_MAX + a subnormal is FLT_MAX);
  * pair folds of two terms, which commute: (1 + 2^-12)^2 - (1 + 2^-12)^2 is 0
    unless one product is fused into the add (+-2^-24), -FLT_MAX + 2^64 * 2^64 is
    inf unless fused (2^104), 2^-149 + 2^-149 and the largest subnormal + 2^-149.

min and max folds are exact in any order; with fmin / fmax a NaN product is
ignored, which the push's ordered-integer atomics have to respect.  Semirings
whose products or folds round order-dependently on these operands (PlusMinus,
MultipliesMultiplies) and the order-dependent adds are left to the other suites, as
is the masked mxm, which takes INT32 operands only (test_int32_values_gpu.py).
test_ieee_reference_cpu.py checks that the designed operands hold what they are
meant to hold, and that the comparison rejects an FTZ, a fused and a ternary-min
reference on them.
"""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import ewise_matrix_reference
import ewise_reference as eref
import ieee_reference as ieee
import mxm_reference as mref
import mxv_reference as vref
from ieee_reference import (BIG, FLT_MAX, INF, MAX_SUB, NAN, NEG_NAN, NEG_ZERO, ONE_EPS,
                            PAYLOAD_NAN, TINY)
from support import Csr, csr, device_matrix, gb  # noqa: F401
from test_ewise_matrix_gpu import overlap, straddling
from test_mxm_unmasked_gpu import DESIGNED
from test_mxm_unmasked_gpu import designed_rows as mxm_designed_rows
from test_mxv_gpu import (PUSH_MASKS, TILE, VARIANTS, bool_pull, dense_vector, pull,
                          run_push, square)
from test_spmm_gpu import designed_rows as spmm_designed_rows
from test_spmm_gpu import dense_matrix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
HUB_FORCED = (os.environ.get("GB200_SPMV_HUB_MIN_NNZ") == "0" and
              os.environ.get("GB200_SPMV_HUB_MIN_PCT") == "0")

LOR, PLUS, MINPLUS, MAXMUL, PLUSDIV, PLUSGT = 0, 1, 2, 3, 4, 5
PLUSLT, MINMUL, MINSECOND, PLUSNE, MINNE = 8, 10, 13, 14, 16
# every accepted semiring whose folds round alike in any order on these operands
SEMIRINGS = [LOR, PLUS, MINPLUS, MAXMUL, PLUSDIV, PLUSGT, PLUSLT, MINMUL, MINSECOND,
             PLUSNE, MINNE]
UNITS = F32([-4, -2, -1, 1, 2, 4])
ARITH_SPECIALS = [NAN, NEG_NAN, PAYLOAD_NAN, INF, -INF, NEG_ZERO, FLT_MAX]
MASK_VALUES = F32([0, 0, NEG_ZERO, NAN, NEG_NAN, TINY, MAX_SUB, 1, -2, FLT_MAX])


def fixed(rng, n, kmax=63):
    """k 2^-149, 1 <= |k| <= kmax, one in twenty -0.0, some 2^-149 itself."""
    k = rng.randint(1, kmax + 1, n)*np.where(rng.rand(n) < 0.5, -1, 1)
    k[rng.rand(n) < 0.1] = 1
    v = (k.astype(np.float64)*2.0**-149).astype(F32)
    v[rng.rand(n) < 0.05] = NEG_ZERO
    return v


# ---------------------------------------------------------------------------
# the designed pull / push operand: S (rows of fixed-point, special and pair
# folds) and u (a unit block, special columns, pair columns)
# ---------------------------------------------------------------------------

N_UNIT = 4000
SPECIAL_U = [NAN, NEG_NAN, PAYLOAD_NAN, INF, -INF, NEG_ZERO]
# pair columns: (-FLT_MAX * 1) + (2^64 * 2^64); (1+e)(1+e) - (1+e)(1+e);
# 2^-149 + 2^-149; MAX_SUB + 2^-149; FLT_MAX + FLT_MAX
PAIR_U = [F32(1), BIG, ONE_EPS, ONE_EPS, TINY, TINY, F32(1), F32(1)]
PAIRS = [((0, -FLT_MAX), (1, BIG)),
         ((2, ONE_EPS), (3, -ONE_EPS)),
         ((4, F32(1)), (5, F32(1))),
         ((6, MAX_SUB), (7, TINY)),
         ((6, FLT_MAX), (7, FLT_MAX)),
         ((6, INF), (7, -INF))]


@functools.lru_cache(None)
def pull_operands():
    rng = np.random.RandomState(31)
    sp0 = N_UNIT
    pr0 = N_UNIT + len(SPECIAL_U)
    u = np.concatenate([rng.choice(UNITS, N_UNIT), F32(SPECIAL_U), F32(PAIR_U)])
    rows = []

    def unit_row(length):
        cols = np.sort(rng.choice(N_UNIT, length, replace=False))
        return list(zip(cols.tolist(), fixed(rng, length)))

    # fixed-point rows: short, across the merge tile and longer than it
    for length in [0, 1, 2, 3, 7, 8, 9, 31, 33, 0, 5, TILE - 1, TILE, TILE + 1, 3*TILE + 5]:
        rows.append(unit_row(length))
    for _ in range(300):
        rows.append(unit_row(rng.randint(0, 40)))
    # a special u column in a fixed-point row
    for j in range(len(SPECIAL_U)):
        for length in (0, 4, 60):
            r = unit_row(length) + [(sp0 + j, fixed(rng, 1)[0] or TINY)]
            rows.append(sorted(r))
    rows.append(sorted(unit_row(6) + [(sp0 + 3, TINY), (sp0 + 4, TINY)]))     # inf - inf
    # a special A value in a fixed-point row
    for a in ARITH_SPECIALS:
        for length in (0, 5, 50):
            r = unit_row(length + 1)
            r[length // 2] = (r[length // 2][0], a)
            rows.append(r)
    for p in PAIRS:
        rows.append([(pr0 + c, F32(a)) for c, a in p])
    order = rng.permutation(len(rows))              # mix the kinds across tiles
    rows = [rows[i] for i in order]
    r = np.concatenate([np.full(len(x), i) for i, x in enumerate(rows)])
    c = np.concatenate([[e[0] for e in x] for x in rows if x])
    v = np.concatenate([[e[1] for e in x] for x in rows if x]).astype(F32)
    S = Csr(len(rows), len(u), *_csr_arrays(len(rows), r, c, v))
    return S, u


def _csr_arrays(nrows, r, c, v):
    order = np.lexsort((c, r))
    ptr = np.zeros(nrows + 1, np.int64)
    np.add.at(ptr, np.asarray(r, np.int64)[order] + 1, 1)
    return np.cumsum(ptr), np.asarray(c, np.int64)[order], np.asarray(v, F32)[order]


def pull_want(semiring, S, u, **kw):
    return ieee.pull(semiring, S.ptr, S.ind, S.val, u, **kw)


def push_frontier(u):
    f = np.arange(len(u))
    return f, u


def push_want(semiring, S, u, mask=None, scmp=False, struconly=False):
    f, fv = push_frontier(u)
    T = S.T
    return vref.push(semiring, T.ptr, T.ind, T.val, f, fv, S.nrows, mask, scmp, struconly)


# ---------------------------------------------------------------------------
# mxm / SpMM / eWise matrix operands
# ---------------------------------------------------------------------------

B1 = F32([-FLT_MAX, ONE_EPS, TINY, MAX_SUB, NAN, NEG_NAN, INF, -INF, NEG_ZERO, FLT_MAX])
B2 = F32([BIG, ONE_EPS, TINY, TINY, 1, 1, -INF, 1, NEG_ZERO, FLT_MAX])
PAIR_A = [(F32(1), BIG), (ONE_EPS, -ONE_EPS), (F32(1), F32(1)), (F32(2), NEG_ZERO),
          (MAX_SUB, FLT_MAX)]


def plant(rng, v, share=0.002):
    """A few of v replaced by NaN of both signs, +-inf and -0.0."""
    v = v.copy()
    at = np.nonzero(rng.rand(len(v)) < share)[0]
    v[at] = np.resize(F32([NAN, NEG_NAN, INF, -INF, NEG_ZERO]), len(at))
    return v


def with_pairs(A, B):
    """A and B with two more B rows (B1, B2 from column 0) that only the appended
    rows of A read, one per PAIR_A."""
    nb = A.ncols
    ncols = max(B.ncols, len(B1))
    br = np.concatenate([B.rows(), np.full(len(B1), nb), np.full(len(B2), nb + 1)])
    bc = np.concatenate([B.ind, np.arange(len(B1)), np.arange(len(B2))])
    bv = np.concatenate([B.val, B1, B2])
    B2_ = Csr(nb + 2, ncols, *_csr_arrays(nb + 2, br, bc, bv))
    m = A.nrows
    ar = np.concatenate([A.rows(), np.repeat(np.arange(m, m + len(PAIR_A)), 2)])
    ac = np.concatenate([A.ind, np.tile([nb, nb + 1], len(PAIR_A))])
    av = np.concatenate([A.val, F32(PAIR_A).ravel()])
    A2 = Csr(m + len(PAIR_A), nb + 2, *_csr_arrays(m + len(PAIR_A), ar, ac, av))
    return A2, B2_


@functools.lru_cache(None)
def unmasked_operands():
    rng = np.random.RandomState(41)
    A, B = mxm_designed_rows(DESIGNED)
    A = A.with_values(plant(rng, rng.choice(UNITS, A.nnz)))
    B = B.with_values(fixed(rng, B.nnz, kmax=15))
    return with_pairs(A, B)


def mxm_want(semiring, A, B):
    rp, ci, val = mref.mxm(semiring, A.ptr, A.ind, A.val, B.ptr, B.ind, B.val, B.ncols)
    return Csr(A.nrows, B.ncols, rp, ci, val)


SPMM_WIDTHS = [1, 4, 33, 64, 65, 129]


@functools.lru_cache(None)
def spmm_operands(n):
    rng = np.random.RandomState(47 + n)
    A, _ = spmm_designed_rows(rng, 3000, F32([1]))
    A = A.with_values(plant(rng, fixed(rng, A.nnz, kmax=15)))
    Bd = rng.choice(UNITS, (A.ncols, n)).astype(F32)
    Bs = csr(A.ncols, n, np.repeat(np.arange(A.ncols), n), np.tile(np.arange(n), A.ncols),
             Bd.ravel(), F32)
    Bs = Csr(Bs.nrows, max(n, len(B1)), Bs.ptr, Bs.ind, Bs.val)
    A2, B2_ = with_pairs(A, Bs)
    B = np.ones((A2.ncols, n), F32)
    B[:A.ncols] = Bd
    k = min(n, len(B1))
    B[A.ncols, :k], B[A.ncols + 1, :k] = B1[:k], B2[:k]
    return A2, B


def spmm_want(semiring, A, B):
    k, n = B.shape
    Bs = Csr(k, n, np.arange(k + 1, dtype=np.int64)*n, np.tile(np.arange(n), k), B.ravel())
    C = mxm_want(semiring, A, Bs)
    out = np.full((A.nrows, n), mref.SEMIRINGS[semiring][2], F32)
    out[C.rows(), C.ind] = C.val
    return out


EWISE_POOL = F32([NAN, NEG_NAN, PAYLOAD_NAN, INF, -INF, NEG_ZERO, TINY, MAX_SUB, FLT_MAX,
                  -FLT_MAX, -TINY, 1, -2.5, 0])


def ewise_operands(name):
    rng = np.random.RandomState(len(name))
    if name.startswith("straddling"):
        A, B = straddling(int(name[-1]))
    else:
        A, B = overlap(len(name), name, PLUS)
    return (A.with_values(rng.choice(EWISE_POOL, A.nnz)),
            B.with_values(rng.choice(EWISE_POOL, B.nnz)))


def ewise_want(add, semiring, A, B):
    rp, ci, val = ewise_matrix_reference.ewise(add, semiring, A.ptr, A.ind, A.val, B.ptr,
                                               B.ind, B.val, A.ncols)
    return Csr(A.nrows, A.ncols, rp, ci, val)


def only_one(A, B, want):
    """Entries of want that come from A alone or B alone (eWiseAdd's carried ones)."""
    key = lambda S: S.rows().astype(np.int64)*S.ncols + S.ind
    ka, kb, kw = key(A), key(B), key(want)
    return ~(np.isin(kw, ka) & np.isin(kw, kb))


REDUCE_SETS = {
    "subnormal": lambda rng, n: fixed(rng, n, kmax=3),
    "nan": lambda rng, n: np.where(rng.rand(n) < 0.01, NAN, fixed(rng, n, 3)).astype(F32),
    "-nan": lambda rng, n: np.where(rng.rand(n) < 0.01, NEG_NAN, fixed(rng, n, 3)).astype(F32),
    "inf": lambda rng, n: np.where(rng.rand(n) < 0.01, INF, fixed(rng, n, 3)).astype(F32),
    "-inf": lambda rng, n: np.where(rng.rand(n) < 0.01, -INF, fixed(rng, n, 3)).astype(F32),
    "infs": lambda rng, n: rng.choice(F32([INF, -INF, TINY, MAX_SUB, FLT_MAX]), n),
}
REDUCE_LENGTHS = [1, 255, 257, 600_001]


def reduce_input(name, n):
    rng = np.random.RandomState(n + len(name))
    x = REDUCE_SETS[name](rng, n)
    if name != "subnormal" and n > 1:
        x[0] = {"nan": NAN, "-nan": NEG_NAN, "inf": INF, "-inf": -INF, "infs": INF}[name]
    return x


def reduce_want(monoid, x):
    op, ident = eref.MONOIDS[monoid]
    if op == "plus":
        with np.errstate(all="ignore"):
            return F32(np.sum(x.astype(np.float64)) + 0.0)
    return eref.reduce(monoid, x)[0]


# ---------------------------------------------------------------------------
# GPU: mxv / vxm
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("semiring", SEMIRINGS)
def test_pull_every_form(gb, semiring):
    """mxv over the CSR and vxm over the CSC, aligned and lane-major; under the
    forced hub thresholds (test_pull_on_the_hub_in_a_child) the aligned forms run
    spmvHubKernel."""
    S, u = pull_operands()
    want = pull_want(semiring, S, u)
    for off in (0, 1):
        for orient, T in (("mxv", S), ("vxm", S.T)):
            got = pull(gb, device_matrix(gb, T, offset=off), orient, semiring, u)
            ieee.check(got, want, ieee.is_minmax(semiring),
                       "%s offset %d semiring %d" % (orient, off, semiring))


@pytest.mark.gpu
@pytest.mark.skipif(HUB_FORCED, reason="already a child")
def test_pull_on_the_hub_in_a_child():
    full = dict(os.environ, GB200_SPMV_HUB="1", GB200_SPMV_HUB_MIN_NNZ="0",
                GB200_SPMV_HUB_MIN_PCT="0")
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider",
           os.path.abspath(__file__), "-k", "pull_every_form or generic_pull"]
    r = subprocess.run(cmd, env=full, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=1500, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:]
    assert " passed" in r.stdout


@pytest.mark.gpu
def test_pull_on_the_hub_as_it_selects_itself(gb):
    """A power-law matrix of 2^22+ entries takes the hub route on its own: fixed-point
    weights, a unit u with NaN, -NaN, +-inf and -0.0 in a few of its columns."""
    import torch
    from graphblast_b200 import graphs
    n = 1 << 20
    src, dst = graphs.rmat_edges(20, 16, seed=3)
    rowptr, colind = graphs.build_csr(n, src, dst, undirected=True)
    del src, dst
    ptr = rowptr.cpu().numpy().astype(np.int64)
    ind = colind.cpu().numpy().astype(np.int64)
    rng = np.random.RandomState(20)
    val = fixed(rng, len(ind), kmax=7)
    M = graphs.matrix_from_csr(n, rowptr, colind, torch.from_numpy(val).cuda(),
                               symmetric=True)
    u = rng.choice(F32([-2, -1, 1, 2]), n)
    at = rng.choice(n, 40, replace=False)
    u[at] = np.resize(F32(SPECIAL_U), len(at))
    for sem in (PLUS, MINPLUS, MAXMUL, MINSECOND):
        want = ieee.pull(sem, ptr, ind, val, u)
        got, launches = pull(gb, M, "mxv", sem, u, count=True)
        assert launches == 3, "not the hub route"
        ieee.check(got, want, ieee.is_minmax(sem), "semiring %d" % sem)


@pytest.mark.gpu
@pytest.mark.parametrize("masking,shadow", PUSH_MASKS)
@pytest.mark.parametrize("struconly", [False, True])
def test_push_every_instantiation(gb, struconly, masking, shadow):
    """spmspvPushKernel<StructOnly, MaskMode>, the mask read as values (NaN nonzero,
    -0.0 zero) or as its bitmap shadow; every semiring, frontier = all of u."""
    from test_mxv_gpu import make_mask
    S, u = pull_operands()
    M = device_matrix(gb, S.T)
    rng = np.random.RandomState(len(masking) + 2*struconly)
    mk = rng.choice(F32([0, 1]) if shadow == "current" else MASK_VALUES, S.nrows)
    f, fv = push_frontier(u)
    for sem in SEMIRINGS:
        mask = None if masking == "none" else make_mask(gb, mk, shadow)
        g_ind, g_val = run_push(gb, M, "vxm", sem, f, fv, mask, masking == "scmp", struconly)
        r_ind, r_val = push_want(sem, S, u, None if masking == "none" else mk,
                                 masking == "scmp", struconly)
        where = "semiring %d" % sem
        assert np.array_equal(g_ind, r_ind), where
        ieee.check(g_val, r_val, ieee.is_minmax(sem), where)


@pytest.mark.gpu
def test_push_agrees_with_the_pull(gb):
    """Where no product meets the push's identity short-circuit (no zero in u or A
    under a zero identity, no FLT_MAX under a FLT_MAX one), push and pull define the
    same entries."""
    S, u = pull_operands()
    M = device_matrix(gb, S.T)
    for sem in (PLUS, MAXMUL, MINSECOND, MINPLUS):
        ident = mref.SEMIRINGS[sem][2]
        keep = (S.val != ident) & (u[S.ind] != ident)
        T = Csr(S.nrows, S.ncols, *_csr_arrays(S.nrows, S.rows()[keep], S.ind[keep],
                                               S.val[keep]))
        f = np.nonzero(u != ident)[0]
        g_ind, g_val = run_push(gb, device_matrix(gb, T.T), "vxm", sem, f, u[f])
        dense = pull(gb, device_matrix(gb, T), "mxv", sem, u)
        ieee.check(g_val, dense[g_ind], ieee.is_minmax(sem), "semiring %d" % sem)
        assert np.array_equal(g_ind, np.nonzero(np.diff(T.ptr))[0])
    del M


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS,
                         ids=["scmp%d_ee%d_or%d" % tuple(map(int, v)) for v in VARIANTS])
def test_bool_pull_both_forms(gb, variant):
    """NaN (set), -0.0 (clear) and subnormals (set) in u and in the mask."""
    scmp, earlyexit, opreuse = variant
    for n in (33, 1003):
        rng = np.random.RandomState(n)
        S = square(rng, n)
        M = device_matrix(gb, S)
        mk = rng.choice(MASK_VALUES, n)
        u = rng.choice(F32([0, 0, NEG_ZERO, NAN, NEG_NAN, TINY, -TINY, 1]), n)
        w = bool_pull(gb, M, "mxv", LOR, u, dense_vector(gb, mk), scmp, earlyexit, opreuse)
        assert np.array_equal(w.extractTuples(),
                              vref.bool_pull(S.ptr, S.ind, mk, u, 0.0, scmp, opreuse)), n
        uv = rng.choice(F32([FLT_MAX, FLT_MAX, NAN, NEG_NAN, NEG_ZERO, TINY, INF]), n)
        for sem in (9, 12, 15):
            w = bool_pull(gb, M, "mxv", sem, uv, dense_vector(gb, mk), scmp, earlyexit,
                          opreuse)
            assert np.array_equal(w.extractTuples(), vref.bool_pull(
                S.ptr, S.ind, mk, uv, FLT_MAX, scmp, opreuse)), (n, sem)


@pytest.mark.gpu
@pytest.mark.parametrize("masking", ["none", "mask", "scmp"])
@pytest.mark.parametrize("semiring", [PLUS, MINPLUS, MAXMUL])
def test_generic_pull_mask_and_accum(gb, semiring, masking):
    S, u = pull_operands()
    rng = np.random.RandomState(semiring + len(masking))
    mask = rng.choice(MASK_VALUES, S.nrows)
    w_old = rng.choice(F32([TINY, -TINY, MAX_SUB, NAN, NEG_ZERO, INF, 1]), S.nrows)
    kw = {} if masking == "none" else {"mask": mask, "scmp": masking == "scmp"}
    for orient, T in (("mxv", S), ("vxm", S.T)):
        got = pull(gb, device_matrix(gb, T), orient, semiring, u, w_old=w_old, **kw)
        want = pull_want(semiring, S, u, w_old=w_old, **kw)
        ieee.check(got, want, ieee.is_minmax(semiring), orient)


# ---------------------------------------------------------------------------
# GPU: mxm, SpMM, matrix eWise
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("semiring", [PLUS, MINPLUS, MAXMUL, MINSECOND])
def test_unmasked_mxm_every_bin(gb, semiring):
    """Rows on every hash bin and on the dense accumulator (its float atomics)."""
    A, B = unmasked_operands()
    C = gb.Matrix(A.nrows, B.ncols)
    gb.mxm(C, None, None, semiring, device_matrix(gb, A), device_matrix(gb, B),
           gb.Descriptor())
    ieee.check_csr(C, mxm_want(semiring, A, B), ieee.is_minmax(semiring))


@pytest.mark.gpu
@pytest.mark.parametrize("n", SPMM_WIDTHS)
def test_spmm_every_class_and_segment(gb, n):
    A, B = spmm_operands(n)
    for sem in (PLUS, MINPLUS, MAXMUL, PLUSDIV):
        Cm = gb.Matrix(A.nrows, n)
        gb.mxm(Cm, None, None, sem, device_matrix(gb, A), dense_matrix(gb, B),
               gb.Descriptor())
        ieee.check(Cm.extract_dense(), spmm_want(sem, A, B), ieee.is_minmax(sem),
                   "semiring %d" % sem)


EWISE_CASES = ["disjoint", "identical", "nested", "partial", "straddling_1",
               "straddling_3"]


@pytest.mark.gpu
@pytest.mark.parametrize("add", [True, False])
@pytest.mark.parametrize("name", EWISE_CASES)
def test_matrix_ewise(gb, name, add):
    A, B = ewise_operands(name)
    for sem in (PLUS, MINPLUS, MAXMUL):
        want = ewise_want(add, sem, A, B)
        C = gb.Matrix(A.nrows, A.ncols)
        (gb.eWiseAdd if add else gb.eWiseMult)(C, None, None, sem, device_matrix(gb, A),
                                               device_matrix(gb, B), gb.Descriptor())
        ieee.check_csr(C, want, ieee.is_minmax(sem), "semiring %d" % sem)
        if add:
            carried = only_one(A, B, want)
            ieee.check_bits(C.extract_csr()[2][carried], want.val[carried], "carried")


# ---------------------------------------------------------------------------
# GPU: vector operations and reduce
# ---------------------------------------------------------------------------

def vector_operands(n):
    rng = np.random.RandomState(n)
    pool = EWISE_POOL
    u, v = rng.choice(pool, n), rng.choice(pool, n)
    ind = np.sort(rng.choice(n, max(1, n//3), replace=False)).astype(np.int32)
    return u, v, ind, rng.choice(pool, len(ind))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [33, 2049, 16385])
def test_vector_ewise_every_storage(gb, n):
    from test_ewise_gpu import dense, sparse
    u, v, ind, val = vector_operands(n)
    desc = gb.Descriptor()
    for s in (PLUS, MINPLUS, MAXMUL, MINSECOND):
        mm = ieee.is_minmax(s)
        w = gb.Vector(n)
        gb.eWiseAdd(w, None, None, s, dense(gb, u), dense(gb, v), desc)
        ieee.check(w.extractTuples(), eref.ewise_add_dense(s, u, v), mm, "add dd %d" % s)
        w = gb.Vector(n)
        gb.eWiseAdd(w, None, None, s, sparse(gb, n, ind, val), dense(gb, v), desc)
        ieee.check(w.extractTuples(), eref.ewise_add_sparse_dense(s, ind, val, v), mm,
                   "add sd %d" % s)
        w = gb.Vector(n)
        gb.eWiseMult(w, None, None, s, dense(gb, u), dense(gb, v), desc)
        ieee.check(w.extractTuples(), eref.ewise_mult_dense(s, u, v), mm, "mult dd %d" % s)
        w = gb.Vector(n)
        gb.eWiseMult(w, None, None, s, sparse(gb, n, ind, val), dense(gb, v), desc)
        g_ind, g_val = w.extractTuples(sparse=True)
        r_ind, r_val = eref.ewise_mult_sparse_dense(s, ind, val, v)
        assert np.array_equal(g_ind, r_ind)
        ieee.check(g_val, r_val, mm, "mult sd %d" % s)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(REDUCE_SETS))
def test_reduce_vector_matrix_and_rows(gb, name):
    from test_ewise_gpu import dense, reduce_val, sparse
    for n in REDUCE_LENGTHS:
        x = reduce_input(name, n)
        for monoid, mono in ((0, gb.Monoid.Plus), (2, gb.Monoid.Minimum),
                             (3, gb.Monoid.Maximum)):
            want = reduce_want(monoid, x)
            where = "%s n %d monoid %d" % (name, n, monoid)
            ieee.check(F32([reduce_val(gb, mono, dense(gb, x))]), F32([want]),
                       monoid != 0, where + " dense")
            ind = np.arange(0, n, 2, dtype=np.int32)
            ieee.check(F32([reduce_val(gb, mono, sparse(gb, n, ind, x[ind]))]),
                       F32([reduce_want(monoid, x[ind])]), monoid != 0, where + " sparse")
            cols = 1000
            rows = -(-n // cols)
            S = csr(rows, cols, np.arange(n) // cols, np.arange(n) % cols, x, F32)
            A = device_matrix(gb, S, csc=False)
            ieee.check(F32([reduce_val(gb, mono, A)]), F32([want]), monoid != 0,
                       where + " matrix")
            w = gb.Vector(rows)
            gb.reduce(None, mono, A, gb.Descriptor(), out=w)
            want_rows = np.array([reduce_want(monoid, x[S.ptr[i]:S.ptr[i + 1]])
                                  for i in range(rows)], F32)
            ieee.check(w.extractTuples(), want_rows, monoid != 0, where + " rows")


# ---------------------------------------------------------------------------
# GPU: values carried without arithmetic keep their bits
# ---------------------------------------------------------------------------

CARRIED = F32([NAN, NEG_NAN, PAYLOAD_NAN, -PAYLOAD_NAN, INF, -INF, NEG_ZERO, TINY, -TINY,
               MAX_SUB, FLT_MAX, -FLT_MAX, 1.5])


@functools.lru_cache(None)
def carried_matrix():
    rng = np.random.RandomState(61)
    m, n = 150, 110
    flat = np.sort(rng.choice(m*n, 2000, replace=False))
    return csr(m, n, flat // n, flat % n, rng.choice(CARRIED, len(flat)), F32)


@pytest.mark.gpu
def test_carried_matrix_values_keep_their_bits(gb):
    """Host build from shuffled tuples, extract_csr, transpose, extract and assign
    without accum."""
    S = carried_matrix()
    rng = np.random.RandomState(62)
    order = rng.permutation(S.nnz)
    M = gb.Matrix(S.nrows, S.ncols)
    M.build(S.rows()[order].astype(np.int32), S.ind[order].astype(np.int32), S.val[order])
    rp, ci, val = M.extract_csr()
    assert np.array_equal(rp, S.ptr) and np.array_equal(ci, S.ind)
    ieee.check_bits(val, S.val, "build")
    T = gb.Matrix(S.ncols, S.nrows)
    gb.transpose(T, None, None, device_matrix(gb, S), gb.Descriptor())
    ieee.check_bits(T.extract_csr()[2], S.T.val, "transpose")
    I = np.sort(rng.choice(S.nrows, 60, replace=False))
    J = rng.permutation(S.ncols)[:50]
    X = gb.Matrix(len(I), len(J))
    gb.extract(X, None, None, device_matrix(gb, S), I, len(I), J, len(J), gb.Descriptor())
    import extract_reference
    rp, ci, val = extract_reference.extract_matrix(S.ptr, S.ind, S.val, S.nrows, S.ncols, I, J)
    got = X.extract_csr()
    assert np.array_equal(got[0], rp) and np.array_equal(got[1], ci)
    ieee.check_bits(got[2], val, "extract")
    import assign_reference
    C = carried_matrix()
    src = Csr(len(I), len(J), rp, ci, val)
    dC = device_matrix(gb, C)
    gb.assign(dC, None, None, device_matrix(gb, src), I, len(I), J, len(J), gb.Descriptor())
    rp2, ci2, val2 = assign_reference.assign_matrix((C.ptr, C.ind, C.val), C.nrows, C.ncols,
                                                    (rp, ci, val, len(I), len(J)), I, J)
    got = dC.extract_csr()
    assert np.array_equal(got[0], rp2) and np.array_equal(got[1], ci2)
    ieee.check_bits(got[2], val2, "assign")


@pytest.mark.gpu
def test_carried_vector_values_keep_their_bits(gb):
    """Vector build (dense and sparse), dup, sparse2dense and dense2sparse, and a
    dense -> sparse -> dense round trip."""
    rng = np.random.RandomState(63)
    n = 5000
    x = rng.choice(CARRIED, n)
    v = dense_vector(gb, x)
    ieee.check_bits(v.extractTuples(), x, "dense build")
    d = gb.Vector(n)
    d.dup(v)
    ieee.check_bits(d.extractTuples(), x, "dup")
    v.dense2sparse(0.0, gb.Descriptor())
    ind, val = v.extractTuples(sparse=True)
    r_ind, r_val = eref.dense2sparse(x, 0.0)
    assert np.array_equal(ind, r_ind)          # -0.0 is the identity 0: dropped
    ieee.check_bits(val, r_val, "dense2sparse")
    v.sparse2dense(0.0)
    ieee.check_bits(v.extractTuples(), eref.sparse2dense(n, r_ind, r_val, 0.0),
                    "sparse2dense")
    ind = np.sort(rng.choice(n, 700, replace=False)).astype(np.int32)
    s = gb.Vector(n)
    s.build(ind, x[ind])
    g_ind, g_val = s.extractTuples(sparse=True)
    assert np.array_equal(g_ind, ind)
    ieee.check_bits(g_val, x[ind], "sparse build")
    s.sparse2dense(FLT_MAX)
    ieee.check_bits(s.extractTuples(), eref.sparse2dense(n, ind, x[ind], FLT_MAX),
                    "sparse2dense FLT_MAX")


# ---------------------------------------------------------------------------
# GPU: the cooperative algorithms read only the pattern; SSSP on inf / subnormals
# ---------------------------------------------------------------------------

def _pattern_outputs(gb, A, n):
    from graphblast_b200 import algorithm
    desc = gb.Descriptor
    out = {}
    for name, f in (("cc", algorithm.cc), ("scc", algorithm.scc)):
        v = gb.Vector(n)
        k, _ = f(v, A, desc())
        out[name] = (k, v.extractTuples().tobytes())
    for name, f in (("mis", algorithm.mis), ("gc", algorithm.gc)):
        v = gb.Vector(n)
        k, _ = f(v, A, 7, desc())
        out[name] = (k, v.extractTuples().tobytes())
    K = gb.Matrix(n, n)
    k, _ = algorithm.ktruss(K, A, 4, desc())
    out["ktruss"] = (k,) + tuple(x.tobytes() for x in K.extract_csr())
    K = gb.Matrix(n, n)
    k, _ = algorithm.trussness(K, A, desc())
    out["trussness"] = (k,) + tuple(x.tobytes() for x in K.extract_csr())
    v = gb.Vector(n)
    algorithm.bc(v, A, desc(), sources=range(0, n, 7))
    out["bc"] = v.extractTuples().tobytes()
    v = gb.Vector(n)
    k, it, _ = algorithm.cdlp(v, A, 10, desc())
    out["cdlp"] = (k, it, v.extractTuples().tobytes())
    return out


@pytest.mark.gpu
def test_cooperative_algorithms_read_no_values(gb):
    import oracle_binding as orc
    rp, ci = orc.rmat_csr(9)
    n = len(rp) - 1
    odd = np.resize(F32([NAN, NEG_ZERO, TINY, NEG_NAN, MAX_SUB]), len(ci))
    got = _pattern_outputs(gb, device_matrix(gb, Csr(n, n, rp, ci, odd)), n)
    want = _pattern_outputs(gb, device_matrix(gb, Csr(n, n, rp, ci,
                                                      np.ones(len(ci), F32))), n)
    assert sorted(got) == sorted(want)
    for name in want:
        assert got[name] == want[name], name


@pytest.mark.gpu
def test_sssp_on_infinite_and_subnormal_weights(gb):
    from graphblast_b200 import algorithm
    import oracle_binding as orc
    rp, ci = orc.rmat_csr(10)
    n = len(rp) - 1
    rng = np.random.RandomState(71)
    w = rng.choice(F32([INF, TINY, MAX_SUB, 2*TINY, 2.0**-130, 1]), len(ci))
    A = device_matrix(gb, Csr(n, n, rp, ci, w))
    s = int(np.argmax(np.diff(rp)))
    want = orc.sssp(rp, ci, w, s)          # float32 Bellman-Ford
    assert ieee.is_subnormal(want).any()
    for mode in (0, 1, 2):
        v = gb.Vector(n)
        algorithm.sssp(v, A, s, gb.Descriptor(mxvmode=mode))
        ieee.check_bits(v.extractTuples(), want, "mode %d" % mode)
