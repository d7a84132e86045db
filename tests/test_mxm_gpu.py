"""The masked SpGEMM C<M> = A*B (gb.mxm, int plus-times) entry by entry against
the oracle's exact per-entry product (orc_mxm_masked), on every kernel route.

Operand values are small nonzero integers (-3..7), so a value read from the
wrong array or the wrong position changes the result; C is compared in full:
its pattern must be the mask's and every value must be bit-exact.

Routes of backend/cuda/spgemm.hpp (spgemmMasked), both run by every GPU test:
  * hash kernels (kernels/spgemm_hash.cuh): a mask with a CSC side ("hash"
    cases below);
  * search kernels spgemmMaskedEdgeKernel + spgemmMaskedHeavyKernel
    (kernels/spgemm_masked.cuh): a mask without a CSC side ("search" cases).

The designed operands put list lengths and partner counts at, below and one past
every boundary of the hash kernels.  The boundaries (kernels/spgemm_hash.cuh,
kernels/spgemm_masked.cuh; test_kernel_constants_match_the_table checks them):

  owner list length  class  group             table                  partners/item
  0 .. 64            S      one warp          256 slots              256
  65 .. 1024         M      256-thread CTA    2048 slots             1024
  > 1024             L      1024-thread CTA   16384 slots, 8192 keys 2048
                                              per segment
  The owner of mask entry (i,j) is row i of A in pass 1 (|B(:,j)| <= |A(i,:)|,
  ties included) and column j of B in pass 2 (|A(i,:)| < |B(:,j)|); its partners
  are all entries of mask row i (pass 1) or mask column j (pass 2).
  Search route: an entry whose shorter list holds more than 32 keys goes to the
  warp-per-entry heavy kernel.
"""
import collections
import os
import re

import numpy as np
import pytest

import oracle_binding as orc
from support import Csr, csr, device_matrix, gb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = os.path.join(ROOT, "graphblast_b200", "csrc", "graphblas", "backend",
                       "cuda", "kernels")

CAP_S, CAP_M, SEG_L = 64, 1024, 8192
CHUNK = {"S": 256, "M": 1024, "L": 2048}
HEAVY = 32

# list lengths at and one past every class / segment boundary, 1..3 segments
LENS = [0, 1, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 8191, 8192, 8193, 16384,
        16385, 20000]
K = 45000            # inner dimension: every list is a subset of 0..K-1
POOL = 5000          # short rows / columns that serve as partners
VALUES = np.array([-3, -2, -1, 1, 2, 3, 4, 5, 6, 7], np.int32)


# ---------------------------------------------------------------------------
# host-side sparse matrices
# ---------------------------------------------------------------------------

def padded(S, nrows, ncols):
    """The same entries in a larger nrows x ncols matrix."""
    assert nrows >= S.nrows and ncols >= S.ncols
    ptr = np.concatenate([S.ptr, np.full(nrows - S.nrows, S.ptr[-1], np.int32)])
    return Csr(nrows, ncols, ptr, S.ind, S.val)


def random_keys(rng, length, universe=K):
    """`length` distinct sorted keys out of 0..universe-1."""
    if length == 0:
        return np.zeros(0, np.int32)
    got = np.unique(rng.randint(0, universe, 2*length + 16))
    while len(got) < length:
        got = np.union1d(got, rng.randint(0, universe, length))
    return np.sort(rng.choice(got, length, replace=False)).astype(np.int32)


class Lists(object):
    """Sorted index lists with values: the rows of A or the columns of B."""

    def __init__(self, rng):
        self.rng = rng
        self.keys = []

    def add(self, length=None, keys=None, universe=K):
        if keys is None:
            keys = random_keys(self.rng, length, universe)
        self.keys.append(np.asarray(keys, np.int32))
        return len(self.keys) - 1

    def matrix(self, universe=K):
        """CSR whose row r is list r (for B: the CSC, i.e. the CSR of B^T)."""
        rows = np.repeat(np.arange(len(self.keys)), [len(k) for k in self.keys])
        cols = np.concatenate(self.keys) if self.keys else np.zeros(0, np.int32)
        vals = self.rng.choice(VALUES, len(cols))
        return csr(len(self.keys), universe, rows, cols, vals, np.int32)


Problem = collections.namedtuple("Problem", "A Bt M")   # A m x k, B^T n x k, M m x n


def mask_values(rng, n):
    """Mostly 1, about one in eight an explicit 0, some other nonzero values."""
    return rng.choice(np.array([0, 1, 1, 1, 1, 1, 1, 3], np.int32), n)


def designed_problem(seed=7):
    rng = np.random.RandomState(seed)
    rows, cols = Lists(rng), Lists(rng)
    entries = []
    # every length at and around a boundary, each row against the column one
    # shorter, of equal length (the tie decides the pass) and one longer; keys
    # from a range twice the length, so that the lists share about half of them
    lens = sorted({max(0, x + d) for x in LENS for d in (-1, 0, 1)})
    rid = {n: rows.add(n, universe=2*n + 64) for n in lens}
    cid = {n: cols.add(n, universe=2*n + 64) for n in lens}
    for n in lens:
        for d in (-1, 0, 1):
            if n + d in cid:
                entries.append((rid[n], cid[n + d]))
    # partners per owner: one less than, exactly and one more than a work item,
    # and enough for several items, for an owner of every class in both passes
    # (keys of the short partners from 0..99, of the owners from twice their length)
    pool_cols = [cols.add(rng.randint(0, 41), universe=100) for _ in range(POOL)]
    pool_rows = [rows.add(rng.randint(0, 40), universe=100) for _ in range(POOL)]
    for cls, own in (("S", 40), ("M", 600), ("L", 9000)):
        c = CHUNK[cls]
        for count in (c - 1, c, c + 1, 4500):
            i = rows.add(own, universe=max(100, 2*own))
            entries += [(i, j) for j in rng.choice(pool_cols, count, replace=False)]
            j = cols.add(own, universe=max(100, 2*own))
            entries += [(i, j) for i in rng.choice(pool_rows, count, replace=False)]
    # lists that do not meet (even keys against odd keys), in every class
    even = lambda n: np.arange(0, 2*n, 2)
    odd = lambda n: np.arange(1, 2*n + 1, 2)
    for a, b in ((20, 10), (10, 20), (600, 700), (700, 600), (9000, 9000),
                 (17000, 16500)):
        entries.append((rows.add(keys=even(a)), cols.add(keys=odd(b))))
    # long lists that no mask entry uses: empty mask rows and columns
    rows.add(3000)
    cols.add(3000)
    rows.add(0)                 # and two more rows than columns: m != n
    rows.add(0)
    A = rows.matrix()
    Bt = cols.matrix()
    r, c = zip(*entries)
    M = csr(A.nrows, Bt.nrows, r, c, mask_values(rng, len(entries)), np.int32)
    return Problem(A, Bt, M)


def random_problem(seed, m, k, n, da, db, dm):
    """Uniform random operands; rows and columns without entries included."""
    rng = np.random.RandomState(seed)

    def rand(nr, nc, d, vals):
        cnt = rng.binomial(nr*nc, d)
        flat = np.unique(rng.randint(0, nr*nc, cnt)) if cnt else np.zeros(0, int)
        return csr(nr, nc, flat // nc, flat % nc, vals(len(flat)), np.int32)

    A = rand(m, k, da, lambda s: rng.choice(VALUES, s))
    Bt = rand(n, k, db, lambda s: rng.choice(VALUES, s))
    M = rand(m, n, dm, lambda s: mask_values(rng, s))
    return Problem(A, Bt, M)


def oracle(p):
    return orc.mxm_masked(p.A.ptr, p.A.ind, p.A.val, p.Bt.ptr, p.Bt.ind, p.Bt.val,
                          p.M.ptr, p.M.ind, p.M.val)


def tc_lower(scale=14):
    """L = tril of an R-MAT: operand, mask and output pattern of the triangle count
    (L * L^T) .* L."""
    rp, ci = orc.rmat_csr(scale)
    lr, lc = orc.tril(rp, ci)
    return Csr(len(lr) - 1, len(lr) - 1, lr, lc, np.ones(len(lc), np.int32))


def routes(p):
    """Where the hash kernels take every mask entry: a per-entry table."""
    i, j = p.M.rows(), p.M.ind
    a_len = np.diff(p.A.ptr).astype(np.int64)[i]
    b_len = np.diff(p.Bt.ptr).astype(np.int64)[j]
    pass1 = b_len <= a_len
    own = np.where(pass1, a_len, b_len)
    cls = np.where(own <= CAP_S, "S", np.where(own <= CAP_M, "M", "L"))
    row_cnt = np.diff(p.M.ptr)[i]
    col_cnt = np.bincount(p.M.ind, minlength=p.M.ncols)[j]
    partners = np.where(pass1, row_cnt, col_cnt)
    chunk = np.array([CHUNK[c] for c in cls]) if len(cls) else np.zeros(0)
    return dict(pass_=np.where(pass1, 1, 2), cls=cls, a_len=a_len, b_len=b_len,
                owner_len=own, nseg=np.maximum(1, -(-own // SEG_L)),
                partners=partners, items=-(-partners // chunk), mval=p.M.val)


# ---------------------------------------------------------------------------
# device side
# ---------------------------------------------------------------------------

def check_entries(C, M, want):
    """C's pattern is M's and its values equal `want` bit for bit."""
    rp, ci, val = C.extract_csr()
    assert np.array_equal(rp, M.ptr), "C's row offsets differ from the mask's"
    assert np.array_equal(ci, M.ind), "C's column indices differ from the mask's"
    assert np.abs(want).max(initial=0) < 2**31
    bad = np.nonzero(val.astype(np.int64) != want)[0]
    if len(bad):
        rows = M.rows()
        shown = ["(%d,%d) got %d want %d" % (rows[e], ci[e], val[e], want[e])
                 for e in bad[:8]]
        pytest.fail("%d of %d entries differ: %s" % (len(bad), len(want),
                                                     "; ".join(shown)))


def run_mxm(gb, C, p, route, A=None, B=None, mask=None, desc=None):
    A = device_matrix(gb, p.A, integer=True) if A is None else A
    B = device_matrix(gb, p.Bt.T, integer=True) if B is None else B
    if mask is None:
        mask = device_matrix(gb, p.M, csc=(route == "hash"), integer=True)
    gb.mxm(C, mask, None, gb.Semiring.PlusMultiplies, A, B,
           gb.Descriptor() if desc is None else desc)
    return C


# ---------------------------------------------------------------------------
# CPU: the designed operands reach what they are meant to reach
# ---------------------------------------------------------------------------

def test_kernel_constants_match_the_table():
    """A change to a kernel boundary must come with a change to the designed
    shapes; this fails first."""
    src = open(os.path.join(KERNELS, "spgemm_hash.cuh")).read()
    src += open(os.path.join(KERNELS, "spgemm_masked.cuh")).read()
    got = dict(re.findall(r"#define\s+(GB_\w+)\s+(\d+)", src))
    want = {"GB_HASH_CAP_S": CAP_S, "GB_HASH_CAP_M": CAP_M, "GB_HASH_SEG_L": SEG_L,
            "GB_HASH_CHUNK_S": CHUNK["S"], "GB_HASH_CHUNK_M": CHUNK["M"],
            "GB_HASH_CHUNK_L": CHUNK["L"], "GB_SPGEMM_HEAVY": HEAVY}
    assert {k: int(got[k]) for k in want} == want


def test_designed_operands_reach_every_class_pass_and_split():
    p = designed_problem()
    r = routes(p)
    want = oracle(p)
    meets_not = (want == 0) & (r["mval"] != 0) & (r["a_len"] > 0) & (r["b_len"] > 0)
    for ps in (1, 2):
        in_pass = r["pass_"] == ps
        # owners of every boundary length
        assert set(LENS) - {0} <= set(r["owner_len"][in_pass].tolist()), ps
        for cls in "SML":
            sel = in_pass & (r["cls"] == cls)
            c = CHUNK[cls]
            parts = set(r["partners"][sel].tolist())
            assert {c - 1, c, c + 1} <= parts, (ps, cls)       # one item or two
            assert r["items"][sel].max() >= 3, (ps, cls)        # several items
            assert (r["mval"][sel] == 0).any(), (ps, cls)       # explicit-zero mask
            assert (meets_not & sel).any(), (ps, cls)           # lists do not meet
            if ps == 1:                                         # the tie rule
                assert (sel & (r["a_len"] == r["b_len"])).any(), cls
        segs = set(r["nseg"][in_pass & (r["cls"] == "L")].tolist())
        assert segs == {1, 2, 3}, (ps, segs)
    # empty lists on either side, empty mask rows and columns of nonempty lists
    assert (r["a_len"] == 0).any() and (r["b_len"] == 0).any()
    assert ((np.diff(p.M.ptr) == 0) & (np.diff(p.A.ptr) > 0)).any()
    col_cnt = np.bincount(p.M.ind, minlength=p.M.ncols)
    assert ((col_cnt == 0) & (np.diff(p.Bt.ptr) > 0)).any()
    # search route: entries for the thread-per-entry and for the heavy kernel, at
    # the threshold and one past it
    shorter = np.minimum(r["a_len"], r["b_len"])
    assert {HEAVY, HEAVY + 1} <= set(shorter.tolist())
    assert (shorter > HEAVY).sum() > 100
    assert np.count_nonzero(want) > len(want) // 2
    # the triangle count's entry (i, j) meets rows i and j of L: on the search
    # route too it reaches both kernels
    L = tc_lower()
    deg = np.diff(L.ptr)
    shorter = np.minimum(deg[L.rows()], deg[L.ind])
    assert (shorter > HEAVY).any() and (shorter <= HEAVY).any()


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------

ROUTES = ["hash", "search"]


@pytest.fixture(scope="module")
def designed():
    p = designed_problem()
    return p, oracle(p)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
def test_designed_shapes_rectangular(gb, designed, route):
    """A (m x k) times B (k x n), no transposes, m != n != k."""
    p, want = designed
    assert len({p.A.nrows, p.Bt.nrows, K}) == 3
    C = gb.Matrix(p.M.nrows, p.M.ncols, dtype=gb.api.INT32)
    run_mxm(gb, C, p, route)
    check_entries(C, p.M, want)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("tran", ["inp1", "inp0"])
def test_designed_shapes_transposed_operand(gb, designed, route, tran):
    """Square operands with GrB_INP1 = GrB_TRAN (the triangle-count
    configuration: B is stored as B^T) and with GrB_INP0 = GrB_TRAN (A is stored
    as A^T).  The oracle is fed the explicit transposes."""
    p, want = designed
    N = K
    P = Problem(padded(p.A, N, N), padded(p.Bt, N, N), padded(p.M, N, N))
    desc = gb.Descriptor()
    if tran == "inp1":
        A = device_matrix(gb, P.A, integer=True)
        B = device_matrix(gb, P.Bt, integer=True)                 # B^T stored
        desc.set(gb.Desc_field.GrB_INP1, gb.Desc_value.GrB_TRAN)
    else:
        A = device_matrix(gb, P.A.T, integer=True)                # A^T stored
        B = device_matrix(gb, P.Bt.T, integer=True)
        desc.set(gb.Desc_field.GrB_INP0, gb.Desc_value.GrB_TRAN)
    C = gb.Matrix(N, N, dtype=gb.api.INT32)
    run_mxm(gb, C, P, route, A=A, B=B, desc=desc)
    check_entries(C, P.M, oracle(P))
    assert np.array_equal(oracle(P), want)


RANDOM_CASES = [(1, 1, 1, 1.0, 1.0, 1.0), (5, 3, 7, 0.6, 0.5, 0.8),
                (33, 100, 65, 0.2, 0.3, 0.3), (300, 2000, 250, 0.05, 0.4, 0.05),
                (257, 64, 1025, 0.7, 0.2, 0.02), (2000, 3000, 40, 0.01, 0.5, 0.5)]


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("case", range(len(RANDOM_CASES)))
def test_random_rectangular(gb, route, case):
    p = random_problem(case, *RANDOM_CASES[case])
    C = gb.Matrix(p.M.nrows, p.M.ncols, dtype=gb.api.INT32)
    run_mxm(gb, C, p, route)
    check_entries(C, p.M, oracle(p))


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
def test_output_matrix_reuse(gb, designed, route):
    """One C through four calls: new operand values under the same mask (the
    buffers are reused: nothing of the first result may remain), a mask with the
    same number of entries in another pattern, then one with fewer entries."""
    p, want = designed
    rng = np.random.RandomState(11)
    C = gb.Matrix(p.M.nrows, p.M.ncols, dtype=gb.api.INT32)
    B = device_matrix(gb, p.Bt.T, integer=True)
    run_mxm(gb, C, p, route, B=B)
    check_entries(C, p.M, want)

    p2 = p._replace(A=p.A.with_values(rng.choice(VALUES, p.A.nnz)))
    want2 = oracle(p2)
    assert np.count_nonzero(want2 != want) > len(want) // 2
    run_mxm(gb, C, p2, route, B=B)
    check_entries(C, p2.M, want2)

    perm = rng.permutation(p.M.ncols)                  # same count, new pattern
    M3 = csr(p.M.nrows, p.M.ncols, p.M.rows(), perm[p.M.ind], p.M.val, np.int32)
    p3 = p2._replace(M=M3)
    assert not np.array_equal(M3.ind, p.M.ind)
    run_mxm(gb, C, p3, route, B=B)
    check_entries(C, M3, oracle(p3))

    keep = rng.rand(p.M.nnz) < 0.5                     # fewer entries
    rows = p.M.rows()
    M4 = csr(p.M.nrows, p.M.ncols, rows[keep], p.M.ind[keep], p.M.val[keep], np.int32)
    p4 = p2._replace(M=M4)
    run_mxm(gb, C, p4, route, B=B)
    check_entries(C, M4, oracle(p4))


def tc_per_entry(rp, ci):
    """(L * L^T) .* L of a lower triangle L, one value per entry of L."""
    ones = np.ones(len(ci), np.int32)
    return orc.mxm_masked(rp, ci, ones, rp, ci, ones, rp, ci, ones)


@pytest.mark.gpu
def test_triangle_count_twice_on_the_same_output(gb):
    """algorithm.tc twice into one B, per entry both times (B keeps its buffers
    between the calls), on both routes: L is the mask, so L with a CSC side takes
    the hash kernels and L without one the search kernels."""
    from graphblast_b200 import algorithm
    L = tc_lower()
    want = tc_per_entry(L.ptr, L.ind)
    desc = gb.Descriptor(mxvmode=0)
    for route in ROUTES:
        dL = device_matrix(gb, L, csc=(route == "hash"), integer=True)
        B = gb.Matrix(L.nrows, L.nrows, dtype=gb.api.INT32)
        for _ in range(2):
            ntris, _ = algorithm.tc(dL, B, desc)
            assert ntris == int(want.sum()) == orc.tc(L.ptr, L.ind), route
            check_entries(B, L, want)

