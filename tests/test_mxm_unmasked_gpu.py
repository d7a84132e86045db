"""The unmasked product C = A (+.x) B (gb.mxm with no mask) against the CPU
reference (mxm_reference.mxm): C's row offsets, column indices and values, all
bit for bit (NaN equal to NaN, -0 equal to +0).

Operand values are drawn so that every fold is exact in any order (+-{0.5, 1, 2,
4} and stored zeros; +-1 for MultipliesMultiplies), so the device's unordered
hash accumulation must give exactly the reference's ascending-k fold.

Bins of kernels/spgemm_unmasked.cuh (test_mxm_unmasked_oracle.py checks the
constants below against its #defines).  A row's bound is
min(sum_k |B(k,:)|, ncols); its count the distinct columns of C(i,:):

  bin  group            symbolic: bound  table         numeric: count  table
  S    one warp         1 .. 1024        <= 2048       1 .. 256        <= 512
  M    256-thread CTA   .. 4096          <= 8192       .. 2048         <= 4096
  L    1024-thread CTA  .. 16384         <= 32768      .. 8192         <= 16384
  D    1024-thread CTA  beyond           bitmap        beyond          dense
  Rows of A with one entry skip the symbolic count (their bound is exact).

The designed operands put bounds and counts at, one below and one past every
limit, with a hub-like row (bound >> count) and a row whose output is all ncols
columns, ncols larger than the largest table.
"""
import numpy as np
import pytest

import mxm_reference as ref
import oracle_binding as orc
from support import Csr, check_csr, csr, device_matrix, gb, random_csr

SYM = (1024, 4096, 16384)
NUM = (256, 2048, 8192)
VALUES = np.array([-4, -2, -1, -0.5, 0.5, 1, 2, 4], np.float32)
ACCEPTED = [s for s in range(17) if s not in ref.ORDER_DEPENDENT]


# ---------------------------------------------------------------------------
# host-side operands
# ---------------------------------------------------------------------------

def reference(semiring, A, B, integer=False):
    rp, ci, val = ref.mxm(semiring, A.ptr, A.ind, A.val, B.ptr, B.ind, B.val,
                          B.ncols, integer=integer)
    return Csr(A.nrows, B.ncols, rp, ci, val)


def designed_rows(bound_count):
    """A (m x k) and B (k x ncols) with row i of A*B having the (bound, count) of
    bound_count[i]: B rows are column sets inside one random set of `count`
    columns, the first covering all of it."""
    rng = np.random.RandomState(5)
    ncols = 20000
    a_rows, a_cols, b_rows, b_cols = [], [], [], []
    nb = 0
    for i, (u, d) in enumerate(bound_count):
        cols = rng.choice(ncols, d, replace=False)
        left = u
        first = True
        while left > 0:
            take = d if first else min(left, d)
            part = cols if first else rng.choice(cols, take, replace=False)
            b_rows.append(np.full(take, nb))
            b_cols.append(part)
            a_rows.append(i)
            a_cols.append(nb)
            nb += 1
            left -= take
            first = False
    A = csr(len(bound_count), nb, a_rows, a_cols,
            rng.choice(VALUES, len(a_cols)), np.float32)
    bc = np.concatenate(b_cols)
    B = csr(nb, ncols, np.concatenate(b_rows), bc, rng.choice(VALUES, len(bc)), np.float32)
    return A, B


def _around(x):
    return [x - 1, x, x + 1]


DESIGNED = ([(u, 100) for u in _around(SYM[0])] +
            [(u, 300) for u in _around(SYM[1])] +
            [(u, 1000) for u in _around(SYM[2])] +
            [(max(c, 300), c) for c in _around(NUM[0])] +
            [(3000, c) for c in _around(NUM[1])] +
            [(12000, c) for c in _around(NUM[2])] +
            [(c, c) for c in _around(SYM[2])] +          # one B row: exact bound
            [(100000, 3000),                             # hub-like: bound >> count
             (30000, 20000),                             # all ncols columns
             (5, 3), (1, 1)])


# ---------------------------------------------------------------------------
# device side
# ---------------------------------------------------------------------------

def run(gb, semiring, A, B, C=None, desc=None, integer=False):
    dA = device_matrix(gb, A, integer=integer)
    dB = device_matrix(gb, B, integer=integer)
    if C is None:
        C = gb.Matrix(A.nrows, B.ncols, dtype=gb.api.INT32 if integer else gb.api.FP32)
    gb.mxm(C, None, None, semiring, dA, dB, gb.Descriptor() if desc is None else desc)
    return C


def operands(seed, semiring):
    rng = np.random.RandomState(seed)
    vals = np.array([-1, 1], np.float32) if semiring == 11 else VALUES
    A = random_csr(rng, 300, 500, 0.02, vals)
    B = random_csr(rng, 500, 200, 0.03, vals)
    return A, B


# ---------------------------------------------------------------------------
# CPU: the designed operands reach every limit
# ---------------------------------------------------------------------------

def test_designed_operands_reach_every_limit():
    A, B = designed_rows(DESIGNED)
    blen = np.diff(B.ptr).astype(np.int64)
    bound = np.minimum(np.add.reduceat(blen[A.ind], A.ptr[:-1]), B.ncols)
    want = reference(1, A, B)
    count = np.diff(want.ptr)
    got = list(zip(bound.tolist(), count.tolist()))
    assert got == [(min(u, B.ncols), d) for u, d in DESIGNED]
    for lim in SYM + NUM:
        assert {lim - 1, lim, lim + 1} <= set(bound.tolist()) | set(count.tolist())
    assert count.max() == B.ncols > 2*NUM[2]


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("semiring", ACCEPTED)
def test_every_float_semiring_rectangular(gb, semiring):
    A, B = operands(semiring, semiring)
    assert (np.diff(A.ptr) == 0).any() and (A.val == 0).any()
    check_csr(run(gb, semiring, A, B), reference(semiring, A, B))


@pytest.mark.gpu
@pytest.mark.parametrize("semiring", ref.ORDER_DEPENDENT)
def test_order_dependent_semirings_refused(gb, semiring):
    A, B = operands(1, 1)
    want = reference(1, A, B)
    C = run(gb, 1, A, B)
    with pytest.raises(gb.api.GraphBLASError) as err:
        run(gb, semiring, A, B, C=C)
    assert err.value.info == gb.api.Info.GrB_NOT_IMPLEMENTED
    check_csr(C, want)


@pytest.mark.gpu
def test_int_plus_times(gb):
    rng = np.random.RandomState(3)
    ivals = np.array([-3, -2, -1, 1, 2, 3, 5, 7], np.int32)
    A = random_csr(rng, 310, 470, 0.03, ivals)
    B = random_csr(rng, 470, 190, 0.04, ivals)
    check_csr(run(gb, 1, A, B, integer=True), reference(1, A, B, integer=True))


@pytest.mark.gpu
@pytest.mark.parametrize("semiring", [1, 2])
def test_every_bin_limit(gb, semiring):
    A, B = designed_rows(DESIGNED)
    check_csr(run(gb, semiring, A, B), reference(semiring, A, B))


@pytest.mark.gpu
@pytest.mark.parametrize("tran", ["inp0", "inp1", "both"])
def test_transposed_operands(gb, tran):
    rng = np.random.RandomState(9)
    A = random_csr(rng, 257, 257, 0.03, VALUES)
    B = random_csr(rng, 257, 257, 0.03, VALUES)
    desc = gb.Descriptor()
    sA, sB = A, B
    if tran in ("inp0", "both"):
        sA = A.T
        desc.set(gb.Desc_field.GrB_INP0, gb.Desc_value.GrB_TRAN)
    if tran in ("inp1", "both"):
        sB = B.T
        desc.set(gb.Desc_field.GrB_INP1, gb.Desc_value.GrB_TRAN)
    check_csr(run(gb, 1, sA, sB, desc=desc), reference(1, A, B))


@pytest.mark.gpu
@pytest.mark.parametrize("tran", ["inp0", "inp1", "both"])
def test_transposed_rectangular_operands(gb, tran):
    """op(A) 40 x 60 times op(B) 60 x 30 with the transposed operand stored as
    such; then the operands as stored without transposing, under the same
    descriptor, whose op() shapes do not fit: GrB_DIMENSION_MISMATCH, C unchanged."""
    rng = np.random.RandomState(21)
    A = random_csr(rng, 40, 60, 0.1, VALUES)
    B = random_csr(rng, 60, 30, 0.1, VALUES)
    desc = gb.Descriptor()
    sA, sB = A, B
    if tran in ("inp0", "both"):
        sA = A.T
        desc.set(gb.Desc_field.GrB_INP0, gb.Desc_value.GrB_TRAN)
    if tran in ("inp1", "both"):
        sB = B.T
        desc.set(gb.Desc_field.GrB_INP1, gb.Desc_value.GrB_TRAN)
    want = reference(1, A, B)
    C = gb.Matrix(40, 30)
    gb.mxm(C, None, None, 1, device_matrix(gb, sA), device_matrix(gb, sB), desc)
    check_csr(C, want)
    with pytest.raises(gb.api.GraphBLASError) as err:
        gb.mxm(C, None, None, 1, device_matrix(gb, A), device_matrix(gb, B), desc)
    assert err.value.info == gb.api.Info.GrB_DIMENSION_MISMATCH
    check_csr(C, want)


@pytest.mark.gpu
def test_aliasing(gb):
    rng = np.random.RandomState(4)
    A = random_csr(rng, 200, 200, 0.03, VALUES)
    X = random_csr(rng, 200, 200, 0.03, VALUES)
    dA = device_matrix(gb, A)
    gb.mxm(dA, None, None, 1, dA, dA, gb.Descriptor())           # A = A*A
    AA = reference(1, A, A)
    check_csr(dA, AA)
    dA2 = device_matrix(gb, A)
    dC = device_matrix(gb, X)
    gb.mxm(dC, None, None, 1, dA2, dC, gb.Descriptor())          # C = A*C
    check_csr(dC, reference(1, A, X))


def _dense(S):
    out = np.zeros((S.nrows, S.ncols), np.float64)
    out[S.rows(), S.ind] = S.val
    return out


@pytest.mark.gpu
def test_result_as_operand_and_mask(gb):
    """C feeds vxm / mxv (push and pull) and serves as the mask of a masked mxm
    (hash route, which needs C's CSC); then C is recomputed with another pattern
    into the same object and everything is checked again (no stale caches)."""
    rng = np.random.RandomState(8)
    n = 300
    C = gb.Matrix(n, n, dtype=gb.api.INT32)
    ivals = np.array([-2, -1, 1, 2, 3], np.int32)
    for density in (0.02, 0.035):
        A = random_csr(rng, n, n, density, ivals, zeros=0)
        B = random_csr(rng, n, n, density, ivals, zeros=0)
        gb.mxm(C, None, None, 1, device_matrix(gb, A, integer=True),
               device_matrix(gb, B, integer=True), gb.Descriptor())
        want = reference(1, A, B, integer=True)
        check_csr(C, want)
        # masked mxm with C as the mask
        X = random_csr(rng, n, n, 0.05, ivals, zeros=0)
        Y = random_csr(rng, n, n, 0.05, ivals, zeros=0)
        M = gb.Matrix(n, n, dtype=gb.api.INT32)
        gb.mxm(M, C, None, 1, device_matrix(gb, X, integer=True),
               device_matrix(gb, Y, integer=True), gb.Descriptor())
        Yt = Y.T
        got = M.extract_csr()
        exp = orc.mxm_masked(X.ptr, X.ind, X.val, Yt.ptr, Yt.ind, Yt.val,
                             want.ptr, want.ind, want.val.astype(np.int32))
        assert np.array_equal(got[1], want.ind)
        assert np.array_equal(got[2].astype(np.int64), exp)
    # float C through vxm / mxv, push and pull; then recomputed into the same C
    # from a sparser A (another pattern) and checked again
    Bf = random_csr(rng, n, n, 0.03, VALUES, zeros=0)
    Cf = gb.Matrix(n, n)
    for density in (0.03, 0.01):
        Af = random_csr(rng, n, n, density, VALUES, zeros=0)
        gb.mxm(Cf, None, None, 1, device_matrix(gb, Af), device_matrix(gb, Bf),
               gb.Descriptor())
        want = reference(1, Af, Bf)
        check_csr(Cf, want)
        u = rng.choice(np.array([1, 2, -1], np.float32), n)
        D = _dense(want)
        for mode in (gb.Desc_value.GrB_PUSHONLY, gb.Desc_value.GrB_PULLONLY):
            desc = gb.Descriptor()
            desc.set(gb.Desc_field.GrB_MXVMODE, mode)
            for op, exp in (("vxm", u @ D), ("mxv", D @ u)):
                uv = gb.Vector(n)
                uv.build(u)
                w = gb.Vector(n)
                if op == "vxm":
                    gb.vxm(w, None, None, 1, uv, Cf, desc)
                else:
                    gb.mxv(w, None, None, 1, Cf, uv, desc)
                assert np.array_equal(w.extractTuples().astype(np.float64), exp), (op, mode)


@pytest.mark.gpu
def test_chain_is_associative_on_integers(gb):
    rng = np.random.RandomState(12)
    ivals = np.array([-2, -1, 1, 2], np.int32)
    A = random_csr(rng, 150, 150, 0.04, ivals, zeros=0)
    dA = device_matrix(gb, A, integer=True)
    AA = gb.Matrix(150, 150, dtype=gb.api.INT32)
    gb.mxm(AA, None, None, 1, dA, dA, gb.Descriptor())
    left = gb.Matrix(150, 150, dtype=gb.api.INT32)
    right = gb.Matrix(150, 150, dtype=gb.api.INT32)
    gb.mxm(left, None, None, 1, AA, dA, gb.Descriptor())
    gb.mxm(right, None, None, 1, dA, AA, gb.Descriptor())
    l, r = left.extract_csr(), right.extract_csr()
    for x, y in zip(l, r):
        assert np.array_equal(x, y)
    AAA = reference(1, reference(1, A, A, integer=True), A, integer=True)
    check_csr(left, AAA)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["nnzA0", "nnzB0", "1x1", "odd"])
def test_edge_shapes(gb, shape):
    rng = np.random.RandomState(2)
    if shape == "1x1":
        A = csr(1, 1, [0], [0], np.float32([2]), np.float32)
        B = csr(1, 1, [0], [0], np.float32([-0.5]), np.float32)
    else:
        m, k, n = (33, 65, 97) if shape == "odd" else (40, 50, 60)
        A = random_csr(rng, m, k, 0.1, VALUES)
        B = random_csr(rng, k, n, 0.1, VALUES)
        if shape == "nnzA0":
            A = csr(m, k, [], [], np.zeros(0, np.float32), np.float32)
        if shape == "nnzB0":
            B = csr(k, n, [], [], np.zeros(0, np.float32), np.float32)
    check_csr(run(gb, 1, A, B), reference(1, A, B))


def too_large(case):
    """Operands whose product has more than INT32_MAX entries.
    outer:   50 000 x 1 times 1 x 50 000 (2.5e9 entries); every row of A has one
             entry, so the bound is exact and the call stops before counting;
    counted: 131 073 x 2 (all ones) times 2 x 16 384 whose two rows cover disjoint
             halves of the columns (2^31 + 16 384 entries); two entries per row of
             A, so the rows are counted (L bin) and the total is checked after."""
    ones = lambda k: np.ones(k, np.float32)
    if case == "outer":
        m = n = 50000
        A = csr(m, 1, np.arange(m), np.zeros(m), ones(m), np.float32)
        B = csr(1, n, np.zeros(n), np.arange(n), ones(n), np.float32)
    else:
        m, n = 131073, 16384
        A = csr(m, 2, np.repeat(np.arange(m), 2), np.tile([0, 1], m), ones(2*m), np.float32)
        B = csr(2, n, np.repeat([0, 1], n // 2), np.arange(n), ones(n), np.float32)
    return A, B


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["outer", "counted"])
def test_size_limit(gb, case):
    """GrB_OUT_OF_MEMORY, quickly; the C it was called on keeps its previous
    result and multiplies correctly afterwards."""
    import time
    A, B = too_large(case)
    m, k, n = A.nrows, A.ncols, B.ncols
    assert m * n > 2**31 - 1                 # every row of A*B is full
    X = csr(m, k, [0, 5, m - 1], [0, 0, k - 1], np.float32([2, -1, 4]), np.float32)
    Y = csr(k, n, [0, 0, k - 1], [0, 7, n - 1], np.float32([0.5, 1, -2]), np.float32)
    want = reference(1, X, Y)
    C = run(gb, 1, X, Y)
    check_csr(C, want)
    dA, dB = device_matrix(gb, A), device_matrix(gb, B)
    t0 = time.time()
    with pytest.raises(gb.api.GraphBLASError) as err:
        gb.mxm(C, None, None, 1, dA, dB, gb.Descriptor())
    assert err.value.info == gb.api.Info.GrB_OUT_OF_MEMORY
    assert time.time() - t0 < 10
    check_csr(C, want)
    run(gb, 1, X, Y, C=C)
    check_csr(C, want)


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [12, 14])
def test_rmat_square(gb, scale):
    import scipy.sparse as sp
    import torch
    from graphblast_b200 import graphs
    rp, ci = orc.rmat_csr(scale)
    n = len(rp) - 1
    R = graphs.matrix_from_csr(n, torch.from_numpy(rp).cuda(), torch.from_numpy(ci).cuda())
    S = sp.csr_matrix((np.ones(len(ci), np.float64), ci, rp), shape=(n, n))
    want = (S @ S).tocsr()
    want.sort_indices()
    C = gb.Matrix(n, n)
    gb.mxm(C, None, None, 1, R, R, gb.Descriptor())
    grp, gci, gval = C.extract_csr()
    assert np.array_equal(grp, want.indptr) and np.array_equal(gci, want.indices)
    assert np.array_equal(gval.astype(np.float64), want.data)
    gb.mxm(C, None, None, 0, R, R, gb.Descriptor())              # LogicalOrAnd
    grp, gci, gval = C.extract_csr()
    assert np.array_equal(grp, want.indptr) and np.array_equal(gci, want.indices)
    assert np.all(gval == 1)
