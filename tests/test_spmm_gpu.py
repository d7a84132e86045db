"""SpMM: gb.mxm with a sparse A and a dense B, C = op(A) (+.x) B, dense m x N.

Unless a test says otherwise, C is compared bit for bit (NaN equal to NaN, -0
equal to +0) with the CPU product reference (mxm_reference.mxm) with B given as a
CSR whose every entry is stored, densified with the identity (rows of op(A) with
no entries are the identity).  Operand values are +-{0.5, 1, 2, 4} and stored
zeros (+-1 for MultipliesMultiplies), so every fold is exact in any order.

Classes of kernels/spmm.cuh (test_spmm_constants checks them against its
#defines).  A CTA takes one merge tile of GB_SPMV_TILE rows + entries, split
evenly between groups of L lanes, each lane holding 4 columns:
  N <= GROUP_N (64)      L = the power of two >= ceil(N/4), several groups a warp
  N <= COL_TILE (128)    L = 32, a warp per segment
  N >  COL_TILE          L = 32, columns tiled over the grid
The designed operand has rows at, one below and one past each group's share of a
tile (1152 / (128 / L) items for every L) and the tile itself.
"""
import ctypes as C
import os
import re
import time

import numpy as np
import pytest

import mxm_reference as ref
from support import Csr, csr, device_matrix, gb, launch_count

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = os.path.join(ROOT, "graphblast_b200", "csrc", "graphblas", "backend",
                       "cuda", "kernels")

NT = 128                 # GB_SPMM_NT
GROUP_N = 64             # GB_SPMM_GROUP_N
COL_TILE = 128           # GB_SPMM_COL_TILE
TILE = 128*9             # GB_SPMV_TILE = GB_SPMV_NT * GB_SPMV_IPT
LANES = (1, 2, 4, 8, 16, 32)
SEGMENTS = sorted({TILE//(NT//l) for l in LANES} | {TILE})

WIDTHS = [1, 3, 4, 31, 32, 33, 128, 129, 300]
DESIGNED_WIDTHS = [GROUP_N - 1, GROUP_N, GROUP_N + 1, COL_TILE - 1, COL_TILE,
                   COL_TILE + 1]
VALUES = np.array([-4, -2, -1, -0.5, 0.5, 1, 2, 4], np.float32)
ACCEPTED = [s for s in range(17) if s not in ref.ORDER_DEPENDENT]
PROF_SPMM = 4


def lanes_for(n):
    """spmmLanes of kernels/spmm.cuh."""
    if n > GROUP_N:
        return 32
    lanes = 1
    while lanes < (n + 3)//4:
        lanes *= 2
    return lanes


# ---------------------------------------------------------------------------
# host-side operands
# ---------------------------------------------------------------------------

def values_for(semiring):
    return np.array([-1, 1], np.float32) if semiring == 11 else VALUES


def random_csr(rng, nrows, ncols, density, values, zeros=0.1, empty=0.1):
    d = np.full(nrows, density)
    d[rng.rand(nrows) < 0.05] *= 10
    d[rng.rand(nrows) < empty] = 0
    mask = rng.rand(nrows, ncols) < d[:, None]
    rows, cols = np.nonzero(mask)
    vals = rng.choice(values, len(cols)).astype(np.float32)
    vals[rng.rand(len(vals)) < zeros] = 0
    return csr(nrows, ncols, rows, cols, vals, np.float32)


def dense_values(rng, shape, values, zeros=0.1):
    b = rng.choice(values, shape).astype(np.float32)
    b[rng.rand(*shape) < zeros] = 0
    return b


def designed_rows(rng, ncols, values):
    """Rows of every segment length +-1, separated by empty and short rows."""
    lengths = []
    for s in SEGMENTS:
        lengths += [0, 3, s - 1, s, s + 1]
    lengths += [0, 0, 2*TILE + 5, 1]
    rows, cols = [], []
    for i, n in enumerate(lengths):
        rows.append(np.full(n, i))
        cols.append(np.sort(rng.choice(ncols, n, replace=False)))
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    vals = rng.choice(values, len(cols)).astype(np.float32)
    vals[rng.rand(len(vals)) < 0.05] = 0
    return csr(len(lengths), ncols, rows, cols, vals, np.float32), lengths


def reference(semiring, A, B):
    """mxm_reference.mxm with B (k x N dense) as a CSR of every entry."""
    k, n = B.shape
    b_ptr = np.arange(k + 1, dtype=np.int64)*n
    b_ind = np.tile(np.arange(n, dtype=np.int64), k)
    rp, ci, val = ref.mxm(semiring, A.ptr, A.ind, A.val, b_ptr, b_ind,
                          B.reshape(-1), n)
    out = np.full((A.nrows, n), ref.SEMIRINGS[semiring][2], np.float32)
    out[np.repeat(np.arange(A.nrows), np.diff(rp)), ci] = val
    return out


def check(got, want):
    assert got.shape == want.shape
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    if not same.all():
        bad = np.argwhere(~same)
        i, j = bad[0]
        pytest.fail("%d of %d values differ, first at (%d, %d): got %r want %r" % (
            len(bad), got.size, i, j, got[i, j], want[i, j]))


# ---------------------------------------------------------------------------
# device side
# ---------------------------------------------------------------------------

def dense_matrix(gb, B):
    M = gb.Matrix(B.shape[0], B.shape[1])
    M.build_dense(B)
    return M


def spmm(gb, semiring, A, B, desc=None):
    dA = device_matrix(gb, A)
    dB = dense_matrix(gb, B)
    Cm = gb.Matrix(A.nrows, B.shape[1])
    gb.mxm(Cm, None, None, semiring, dA, dB, gb.Descriptor() if desc is None else desc)
    assert Cm.getStorage() == gb.api.Storage.GrB_DENSE
    return Cm.extract_dense()


def refused(gb, code, fn):
    with pytest.raises(gb.api.GraphBLASError) as err:
        fn()
    assert err.value.info == code


# ---------------------------------------------------------------------------
# CPU: constants and designed operands
# ---------------------------------------------------------------------------

def _defines(path):
    text = open(path).read()
    return {m.group(1): m.group(2) for m in
            re.finditer(r"^#define\s+(\w+)\s+(\S+)", text, re.M)}


def test_spmm_constants():
    d = _defines(os.path.join(KERNELS, "spmm.cuh"))
    assert int(d["GB_SPMM_NT"]) == NT
    assert int(d["GB_SPMM_GROUP_N"]) == GROUP_N
    assert int(d["GB_SPMM_COL_TILE"]) == COL_TILE
    p = _defines(os.path.join(KERNELS, "spmv_pull.cuh"))
    assert int(p["GB_SPMV_NT"])*int(p["GB_SPMV_IPT"]) == TILE
    # 32 lanes x 4 columns fill a column tile; every group count divides a tile
    assert 32*4 == COL_TILE and all(TILE % (NT//l) == 0 for l in LANES)


def test_designed_operands_reach_every_limit():
    widths = set(WIDTHS) | set(DESIGNED_WIDTHS)
    for lim in (GROUP_N, COL_TILE):
        assert {lim - 1, lim, lim + 1} <= widths
    # every lane count and both load paths occur
    assert {lanes_for(n) for n in widths} >= {1, 8, 16, 32}
    assert any(n % 4 for n in WIDTHS) and any(n % 4 == 0 for n in WIDTHS)
    assert lanes_for(GROUP_N) < 32 <= lanes_for(GROUP_N + 1)
    A, lengths = designed_rows(np.random.RandomState(1), 3000, VALUES)
    got = set(np.diff(A.ptr).tolist())
    for s in SEGMENTS:
        assert {s - 1, s, s + 1} <= got
    assert 0 in got and max(got) > 2*TILE


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("n", WIDTHS)
@pytest.mark.parametrize("semiring", ACCEPTED)
def test_every_semiring_every_width(gb, semiring, n):
    rng = np.random.RandomState(semiring*1000 + n)
    vals = values_for(semiring)
    A = random_csr(rng, 300, 170, 0.04, vals)
    assert (np.diff(A.ptr) == 0).any() and (A.val == 0).any()
    B = dense_values(rng, (A.ncols, n), vals)
    check(spmm(gb, semiring, A, B), reference(semiring, A, B))


@pytest.mark.gpu
@pytest.mark.parametrize("n", DESIGNED_WIDTHS + [4, 8, 33])
@pytest.mark.parametrize("semiring", [1, 2])
def test_every_class_and_segment_limit(gb, semiring, n):
    rng = np.random.RandomState(n)
    A, _ = designed_rows(rng, 3000, VALUES)
    B = dense_values(rng, (A.ncols, n), VALUES)
    check(spmm(gb, semiring, A, B), reference(semiring, A, B))


def _operands(seed=1, n=8):
    rng = np.random.RandomState(seed)
    A = random_csr(rng, 60, 50, 0.1, VALUES)
    return A, dense_values(rng, (50, n), VALUES)


@pytest.mark.gpu
@pytest.mark.parametrize("semiring", ref.ORDER_DEPENDENT)
def test_order_dependent_semirings_refused(gb, semiring):
    A, B = _operands()
    dA, dB = device_matrix(gb, A), dense_matrix(gb, B)
    Cm = gb.Matrix(A.nrows, B.shape[1])
    gb.mxm(Cm, None, None, 1, dA, dB, gb.Descriptor())
    want = reference(1, A, B)
    refused(gb, gb.api.Info.GrB_NOT_IMPLEMENTED,
            lambda: gb.mxm(Cm, None, None, semiring, dA, dB, gb.Descriptor()))
    check(Cm.extract_dense(), want)


@pytest.mark.gpu
def test_refusals_leave_c_unchanged(gb):
    A, B = _operands(n=50)             # B square: GrB_INP1 = GrB_TRAN fits the shapes
    dA, dB = device_matrix(gb, A), dense_matrix(gb, B)
    Cm = gb.Matrix(A.nrows, 50)
    gb.mxm(Cm, None, None, 1, dA, dB, gb.Descriptor())
    want = reference(1, A, B)
    NI = gb.api.Info.GrB_NOT_IMPLEMENTED
    # a mask beside a dense operand
    mask = device_matrix(gb, random_csr(np.random.RandomState(2), A.nrows, 50, 0.1,
                                        VALUES))
    refused(gb, NI, lambda: gb.mxm(Cm, mask, None, 1, dA, dB, gb.Descriptor()))
    # a dense A (dense x sparse, dense x dense)
    dAd = dense_matrix(gb, reference(1, A, np.eye(50, dtype=np.float32)))
    refused(gb, NI, lambda: gb.mxm(Cm, None, None, 1, dAd, dB, gb.Descriptor()))
    S50 = device_matrix(gb, random_csr(np.random.RandomState(3), 50, 50, 0.1, VALUES))
    refused(gb, NI, lambda: gb.mxm(Cm, None, None, 1, dAd, S50, gb.Descriptor()))
    # a transposed dense B
    desc = gb.Descriptor()
    desc.set(gb.Desc_field.GrB_INP1, gb.Desc_value.GrB_TRAN)
    refused(gb, NI, lambda: gb.mxm(Cm, None, None, 1, dA, dB, desc))
    # shapes that do not fit
    wrong = dense_matrix(gb, np.ones((49, 50), np.float32))
    refused(gb, gb.api.Info.GrB_DIMENSION_MISMATCH,
            lambda: gb.mxm(Cm, None, None, 1, dA, wrong, gb.Descriptor()))
    assert Cm.getStorage() == gb.api.Storage.GrB_DENSE
    check(Cm.extract_dense(), want)


@pytest.mark.gpu
def test_csr_only_a_under_transpose(gb):
    A, B = _operands(n=8)
    AT_rows = A.ncols
    dA = device_matrix(gb, A, csc=False)
    dB = dense_matrix(gb, np.ones((A.nrows, 8), np.float32))
    Cm = gb.Matrix(AT_rows, 8)
    desc = gb.Descriptor()
    desc.set(gb.Desc_field.GrB_INP0, gb.Desc_value.GrB_TRAN)
    refused(gb, gb.api.Info.GrB_UNINITIALIZED_OBJECT,
            lambda: gb.mxm(Cm, None, None, 1, dA, dB, desc))
    assert Cm.getStorage() == gb.api.Storage.GrB_SPARSE


def hub_operand(rng, values, hub=300000):
    """One row of `hub` entries among short and empty rows."""
    m, k = 3000, hub
    lens = rng.randint(0, 9, m)
    lens[rng.rand(m) < 0.2] = 0
    lens[m//2] = hub
    cols = [np.arange(k) if n == k else np.unique(rng.randint(0, k, n)) for n in lens]
    lens = np.array([len(c) for c in cols])
    rows = np.repeat(np.arange(m), lens)
    cols = np.concatenate(cols)
    if values is None:
        vals = rng.uniform(-1, 1, len(cols)).astype(np.float32)
    else:
        vals = rng.choice(values, len(cols)).astype(np.float32)
        vals[rng.rand(len(vals)) < 0.05] = 0
    return csr(m, k, rows, cols, vals, np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4, 64, 256])
def test_hub_row_exact(gb, n):
    """Plus-times with exact values: the fp64 product is the exact one, which is
    every order's fp32 result (partial sums stay far below 2^24 units)."""
    rng = np.random.RandomState(n)
    A = hub_operand(rng, VALUES)
    assert np.diff(A.ptr).max() >= 300000
    B = dense_values(rng, (A.ncols, n), VALUES)
    want = (A.scipy() @ B.astype(np.float64)).astype(np.float32)
    check(spmm(gb, 1, A, B), want)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4, 64, 256])
def test_hub_row_arbitrary_floats(gb, n):
    """Arbitrary floats against the fp64 product within the fp32 fold bound: a
    sum of L products in any order is within (L + 1) u sum |a b| (u = 2^-24)."""
    rng = np.random.RandomState(100 + n)
    A = hub_operand(rng, None)
    B = rng.uniform(-1, 1, (A.ncols, n)).astype(np.float32)
    got = spmm(gb, 1, A, B).astype(np.float64)
    want = A.scipy() @ B.astype(np.float64)
    absA = Csr(A.nrows, A.ncols, A.ptr, A.ind, np.abs(A.val))
    scale = absA.scipy() @ np.abs(B).astype(np.float64)
    lens = np.diff(A.ptr)[:, None].astype(np.float64)
    bound = (lens + 1)*2.0**-24*scale*1.0001 + 1e-30
    assert (np.abs(got - want) <= bound).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [8, 33, 64, 300])
def test_two_calls_identical_bytes(gb, n):
    import oracle_binding as orc
    rp, ci = orc.rmat_csr(14)
    rng = np.random.RandomState(n)
    A = Csr(len(rp) - 1, len(rp) - 1, rp, ci,
            rng.uniform(-1, 1, len(ci)).astype(np.float32))
    B = rng.uniform(-1, 1, (A.ncols, n)).astype(np.float32)
    dA, dB = device_matrix(gb, A), dense_matrix(gb, B)
    C1, C2 = gb.Matrix(A.nrows, n), gb.Matrix(A.nrows, n)
    gb.mxm(C1, None, None, 1, dA, dB, gb.Descriptor())
    gb.mxm(C2, None, None, 1, dA, dB, gb.Descriptor())
    one, two = C1.extract_dense(), C2.extract_dense()
    assert one.tobytes() == two.tobytes()
    want = A.scipy() @ B.astype(np.float64)
    assert np.allclose(one, want, rtol=1e-4, atol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("tran", [False, True])
@pytest.mark.parametrize("semiring", [1, 2, 3])
def test_columns_equal_pull_mxv(gb, semiring, tran):
    rng = np.random.RandomState(semiring + 10*tran)
    A = random_csr(rng, 230, 190, 0.05, VALUES)
    op_a = A.T if tran else A
    n = 33
    B = dense_values(rng, (op_a.ncols, n), VALUES)
    desc = gb.Descriptor()
    if tran:
        desc.set(gb.Desc_field.GrB_INP0, gb.Desc_value.GrB_TRAN)
    dA, dB = device_matrix(gb, A), dense_matrix(gb, B)
    Cm = gb.Matrix(op_a.nrows, n)
    gb.mxm(Cm, None, None, semiring, dA, dB, desc)
    got = Cm.extract_dense()
    dT = device_matrix(gb, op_a)           # the transposed operand, stored as such
    for j in range(n):
        u = gb.Vector(op_a.ncols)
        u.build(B[:, j])
        w = gb.Vector(op_a.nrows)
        d = gb.Descriptor(mxvmode=2)
        gb.mxv(w, None, None, semiring, dT, u, d)
        assert d.lastmxv == gb.Desc_value.GrB_PULLONLY
        check(got[:, j:j + 1], w.extractTuples()[:, None])


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [64, 1])
def test_adopted_b_read_in_place(gb, offset):
    """offset in floats from a 256-byte aligned allocation: 64 keeps the 16-byte
    loads, 1 (4 bytes) takes the scalar path; both give the same bytes."""
    import torch
    A, B = _operands(seed=4, n=64)
    buf = torch.zeros(offset + B.size, dtype=torch.float32, device="cuda")
    view = buf[offset:]
    view.copy_(torch.from_numpy(B.reshape(-1)))
    dA = device_matrix(gb, A)
    dB = gb.Matrix(B.shape[0], B.shape[1])
    dB.build_dense_device(view)
    assert dB.dense_ptr() == view.data_ptr()
    Cm = gb.Matrix(A.nrows, 64)
    gb.mxm(Cm, None, None, 1, dA, dB, gb.Descriptor())
    check(Cm.extract_dense(), reference(1, A, B))
    view.mul_(2)                       # read in place: the next product sees it
    gb.mxm(Cm, None, None, 1, dA, dB, gb.Descriptor())
    check(Cm.extract_dense(), reference(1, A, 2*B))
    assert np.array_equal(dB.extract_dense(), 2*B)


@pytest.mark.gpu
@pytest.mark.parametrize("semiring", [1, 2])
def test_power_iteration_in_place(gb, semiring):
    rng = np.random.RandomState(semiring)
    A = random_csr(rng, 200, 200, 0.02, VALUES)
    X = dense_values(rng, (200, 12), VALUES)
    dA, dX = device_matrix(gb, A), dense_matrix(gb, X)
    want = X
    for _ in range(3):
        gb.mxm(dX, None, None, semiring, dA, dX, gb.Descriptor())
        want = reference(semiring, A, want)
        check(dX.extract_dense(), want)


@pytest.mark.gpu
def test_c_is_a(gb):
    rng = np.random.RandomState(7)
    A = random_csr(rng, 90, 70, 0.1, VALUES)
    B = dense_values(rng, (70, 70), VALUES)
    dA, dB = device_matrix(gb, A), dense_matrix(gb, B)
    gb.mxm(dA, None, None, 1, dA, dB, gb.Descriptor())
    assert dA.getStorage() == gb.api.Storage.GrB_DENSE
    check(dA.extract_dense(), reference(1, A, B))


@pytest.mark.gpu
def test_storage_switches(gb):
    rng = np.random.RandomState(8)
    A = random_csr(rng, 120, 80, 0.08, VALUES)
    S = random_csr(rng, 80, 60, 0.08, VALUES)
    B = dense_values(rng, (80, 60), VALUES)
    dA, dS, dB = device_matrix(gb, A), device_matrix(gb, S), dense_matrix(gb, B)
    Cm = gb.Matrix(120, 60)
    UI = gb.api.Info.GrB_UNINITIALIZED_OBJECT

    def sparse_step():
        gb.mxm(Cm, None, None, 1, dA, dS, gb.Descriptor())
        assert Cm.getStorage() == gb.api.Storage.GrB_SPARSE
        rp, ci, val = Cm.extract_csr()
        dense = np.zeros((120, 60), np.float32)
        dense[np.repeat(np.arange(120), np.diff(rp)), ci] = val
        want = (A.scipy() @ S.scipy()).toarray().astype(np.float32)
        assert np.array_equal(dense, want)
        refused(gb, UI, lambda: Cm.extract_dense())
        # the sparse C serves a pull mxv: no cache of an earlier structure survives
        u = rng.choice(VALUES, 60).astype(np.float32)
        uv, w = gb.Vector(60), gb.Vector(120)
        uv.build(u)
        gb.mxv(w, None, None, 1, Cm, uv, gb.Descriptor(mxvmode=2))
        assert np.array_equal(w.extractTuples(),
                              (want.astype(np.float64) @ u).astype(np.float32))

    sparse_step()
    gb.mxm(Cm, None, None, 1, dA, dB, gb.Descriptor())
    assert Cm.getStorage() == gb.api.Storage.GrB_DENSE
    check(Cm.extract_dense(), reference(1, A, B))
    refused(gb, UI, lambda: Cm.extract_csr())
    sparse_step()
    gb.mxm(Cm, None, None, 1, dA, dB, gb.Descriptor())
    # the dense C as B of a further SpMM
    P = random_csr(rng, 40, 120, 0.1, VALUES)
    dP = device_matrix(gb, P)
    D = gb.Matrix(40, 60)
    gb.mxm(D, None, None, 2, dP, Cm, gb.Descriptor())
    check(D.extract_dense(), reference(2, P, reference(1, A, B)))


@pytest.mark.gpu
@pytest.mark.parametrize("semiring", [1, 2])
def test_no_entries_gives_identity(gb, semiring):
    A = Csr(50, 40, np.zeros(51), [], np.float32([]))
    B = dense_values(np.random.RandomState(1), (40, 9), VALUES)
    got = spmm(gb, semiring, A, B)
    assert (got == ref.SEMIRINGS[semiring][2]).all()
    check(got, reference(semiring, A, B))


@pytest.mark.gpu
def test_one_by_one(gb):
    A = Csr(1, 1, [0, 1], [0], np.float32([-2]))
    check(spmm(gb, 1, A, np.array([[4]], np.float32)), np.array([[-8]], np.float32))


@pytest.mark.gpu
def test_dense_size_limits(gb):
    """m*N > INT32_MAX is refused before anything is allocated, C unchanged."""
    import torch
    m, n = 65536, 32769
    A = Csr(m, 1, np.r_[0, np.arange(1, m + 1) <= 3].cumsum(), [0, 0, 0],
            np.float32([1, 2, 4]))
    S = Csr(1, n, [0, 2], [0, n - 1], np.float32([1, -1]))
    dA, dS = device_matrix(gb, A), device_matrix(gb, S)
    Cm = gb.Matrix(m, n)
    gb.mxm(Cm, None, None, 1, dA, dS, gb.Descriptor())
    before = Cm.extract_csr()
    dB = dense_matrix(gb, np.ones((1, n), np.float32))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.time()
    refused(gb, gb.api.Info.GrB_OUT_OF_MEMORY,
            lambda: gb.mxm(Cm, None, None, 1, dA, dB, gb.Descriptor()))
    assert time.time() - t0 < 1.0
    assert free0 - torch.cuda.mem_get_info()[0] < (1 << 28)
    assert Cm.getStorage() == gb.api.Storage.GrB_SPARSE
    after = Cm.extract_csr()
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    # a dense matrix of more than INT32_MAX elements is refused the same way
    big = gb.Matrix(m, n)
    refused(gb, gb.api.Info.GrB_OUT_OF_MEMORY,
            lambda: big.build_dense(np.zeros(4, np.float32)))


@pytest.mark.gpu
def test_dense_build_and_extract(gb):
    M = gb.Matrix(3, 4)
    M.build_dense(np.arange(5, dtype=np.float32))       # fewer values: rest 0
    assert M.getStorage() == gb.api.Storage.GrB_DENSE and M.nvals() == 12
    want = np.zeros(12, np.float32)
    want[:5] = np.arange(5)
    assert np.array_equal(M.extract_dense(), want.reshape(3, 4))
    refused(gb, gb.api.Info.GrB_DIMENSION_MISMATCH,
            lambda: M.build_dense(np.zeros(13, np.float32)))
    lib, out = M._lib, np.zeros(20, np.float32)
    P = out.ctypes.data_as(C.c_void_p)
    assert lib.gb200_matrix_extract_dense(M._h, P, 20) == gb.api.Info.GrB_UNINITIALIZED_OBJECT
    assert np.array_equal(out[:12], want) and not out[12:].any()
    assert lib.gb200_matrix_extract_dense(M._h, P, 5) == gb.api.Info.GrB_INSUFFICIENT_SPACE
    I = gb.Matrix(3, 4, dtype=gb.api.INT32)
    assert lib.gb200_matrix_build_dense(I._h, P, 12) == gb.api.Info.GrB_NOT_IMPLEMENTED


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4, 33, 256])
def test_warm_call_launches_and_bytes(gb, n):
    A, B = _operands(seed=5, n=n)
    dA, dB = device_matrix(gb, A), dense_matrix(gb, B)
    Cm = gb.Matrix(A.nrows, n)
    desc = gb.Descriptor()
    gb.mxm(Cm, None, None, 1, dA, dB, desc)
    before = launch_count(gb)
    gb.mxm(Cm, None, None, 1, dA, dB, desc)
    assert launch_count(gb) - before <= 3
    lib = gb.api._lib.load()
    lib.gb200_profile_enable(1)
    lib.gb200_profile_reset()
    gb.mxm(Cm, None, None, 1, dA, dB, desc)
    ms, launches, nbytes = C.c_double(), C.c_longlong(), C.c_double()
    lib.gb200_profile_read(PROF_SPMM, C.byref(ms), C.byref(launches), C.byref(nbytes))
    lib.gb200_profile_enable(0)
    m, k = A.nrows, A.ncols
    assert launches.value == 1 and ms.value > 0
    assert nbytes.value == 4*(m + 1) + 8*A.nnz + 4*k*n + 4*m*n
    check(Cm.extract_dense(), reference(1, A, B))
