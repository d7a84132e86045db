"""eWiseAdd / eWiseMult of two sparse matrices and transpose (gb.eWiseAdd,
gb.eWiseMult, gb.transpose with Matrix operands) against the CPU reference
(ewise_matrix_reference.ewise): C's row offsets, column indices and values, all
bit for bit (NaN equal to NaN, -0 equal to +0).

The device splits the merged item stream of the two operands into tiles of
TILE items (GB_EWM_TILE of kernels/ewise_matrix.cuh, checked below) and each
tile into runs of IPT items per thread, whatever the row lengths; the balance
cases put a hub row over many tiles, and matched pairs across every tile and
thread boundary.
"""
import os
import re

import numpy as np
import pytest

import ewise_matrix_reference as ref
from support import Csr, check_csr, csr, device_matrix, gb, random_csr

TILE = 2048            # GB_EWM_TILE
IPT = 16               # GB_EWM_IPT
# zeros and infinities among the values: divides give inf and NaN
VALUES = np.array([-4, -2, -1, -0.5, 0, 0.5, 1, 2, 4, np.inf], np.float32)
KINDS = ["disjoint", "identical", "nested", "partial"]
HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "graphblast_b200",
                      "csrc", "graphblas", "backend", "cuda", "kernels", "ewise_matrix.cuh")


def reference(add, semiring, A, B, integer=False):
    rp, ci, val = ref.ewise(add, semiring, A.ptr, A.ind, A.val, B.ptr, B.ind, B.val,
                            A.ncols, integer=integer)
    return Csr(A.nrows, A.ncols, rp, ci, val)


def op(gb, add):
    return gb.eWiseAdd if add else gb.eWiseMult


def run(gb, add, semiring, A, B, desc=None, integer=False):
    dA = device_matrix(gb, A, integer=integer)
    dB = dA if B is A else device_matrix(gb, B, integer=integer)
    C = gb.Matrix(A.nrows, A.ncols, dtype=gb.api.INT32 if integer else gb.api.FP32)
    op(gb, add)(C, None, None, semiring, dA, dB, gb.Descriptor() if desc is None else desc)
    return C


def csr_only(gb, S):
    """A Matrix holding device copies of S's CSR only (no CSC).  Unlike
    device_matrix(csc=False) it never calls the CSC adoption, which even without
    arrays marks the CSC side initialised."""
    import torch
    dev = lambda a, dt=np.int32: torch.from_numpy(np.ascontiguousarray(a, dt)).cuda()
    M = gb.Matrix(S.nrows, S.ncols)
    M._keep = [dev(S.ptr), dev(S.ind), dev(S.val, np.float32)]
    gb.api._check(M._lib.gb200_matrix_adopt_csr(M._h, gb.api._dev(M._keep[0]),
                                                gb.api._dev(M._keep[1]),
                                                gb.api._dev(M._keep[2]), S.nnz),
                  "adopt CSR")
    return M


def overlap(seed, kind, semiring, m=120, n=170):
    rng = np.random.RandomState(seed)
    vals = np.array([-1, 1, 0], np.float32) if semiring == 11 else VALUES
    A = random_csr(rng, m, n, 0.08, vals)
    if kind == "identical":
        return A, A
    if kind == "partial":
        return A, random_csr(rng, m, n, 0.08, vals)
    if kind == "nested":
        keep = rng.rand(A.nnz) < 0.5
        return A, csr(m, n, A.rows()[keep], A.ind[keep], rng.choice(vals, keep.sum()),
                      np.float32)
    B = random_csr(rng, m, n, 0.08, vals)
    taken = set(zip(A.rows().tolist(), A.ind.tolist()))
    keep = np.array([(r, c) not in taken for r, c in zip(B.rows().tolist(), B.ind.tolist())],
                    bool)
    return A, csr(m, n, B.rows()[keep], B.ind[keep], B.val[keep], np.float32)


# ---------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------

def test_tile_constants_match_header():
    text = open(HEADER).read()
    nt = int(re.search(r"#define GB_EWM_NT\s+(\d+)", text).group(1))
    ipt = int(re.search(r"#define GB_EWM_IPT\s+(\d+)", text).group(1))
    assert "#define GB_EWM_TILE (GB_EWM_NT*GB_EWM_IPT)" in text
    assert (ipt, nt*ipt) == (IPT, TILE)


def straddling(lead):
    """Row 0 holds `lead` merged items (A only), row 1 equal columns in A and B:
    with lead odd every matched pair of row 1 straddles a boundary at an even
    item, which every tile and thread boundary is."""
    rng = np.random.RandomState(lead)
    n = 3*TILE
    cols = np.sort(rng.choice(n, 5*TILE // 2, replace=False))
    ar = np.concatenate([np.zeros(lead, int), np.ones(len(cols), int)])
    ac = np.concatenate([np.arange(lead), cols])
    A = csr(3, n, ar, ac, rng.choice(VALUES[:-1], len(ac)), np.float32)
    B = csr(3, n, np.ones(len(cols), int), cols, rng.choice(VALUES[:-1], len(cols)),
            np.float32)
    return A, B


@pytest.mark.parametrize("lead", [1, 3])
def test_straddling_pairs_cross_every_boundary(lead):
    A, B = straddling(lead)
    # merged position of each B item of row 1: lead + 2k + 1 (after its A partner)
    k = np.arange(B.nnz)
    a_pos, b_pos = lead + 2*k, lead + 2*k + 1
    crossing = (a_pos // IPT) != (b_pos // IPT)
    assert crossing.sum() >= B.nnz // IPT - 1
    assert ((a_pos // TILE) != (b_pos // TILE)).sum() >= 2


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("add", [True, False])
@pytest.mark.parametrize("semiring", range(17))
def test_every_semiring_and_overlap(gb, semiring, add, kind):
    A, B = overlap(semiring*7 + KINDS.index(kind), kind, semiring)
    assert (np.diff(A.ptr) == 0).any() and (A.val == 0).any()
    check_csr(run(gb, add, semiring, A, B), reference(add, semiring, A, B))


@pytest.mark.gpu
@pytest.mark.parametrize("add", [True, False])
@pytest.mark.parametrize("semiring", [1, 2])
def test_hub_row_over_many_tiles(gb, add, semiring):
    """Row 2 holds 1.2 M merged items, next to rows of 0 and 1 entries."""
    rng = np.random.RandomState(31)
    n = 1 << 20
    hub_a = np.sort(rng.choice(n, 600000, replace=False))
    hub_b = np.sort(rng.choice(n, 600000, replace=False))
    ar = np.concatenate([[0], np.full(len(hub_a), 2), [4]])
    ac = np.concatenate([[5], hub_a, [n - 1]])
    br = np.concatenate([[1], np.full(len(hub_b), 2), [4], [6]])
    bc = np.concatenate([[7], hub_b, [n - 1], [0]])
    A = csr(8, n, ar, ac, rng.choice(VALUES[:-1], len(ac)), np.float32)
    B = csr(8, n, br, bc, rng.choice(VALUES[:-1], len(bc)), np.float32)
    assert A.nnz + B.nnz > 1000000
    check_csr(run(gb, add, semiring, A, B), reference(add, semiring, A, B))


@pytest.mark.gpu
@pytest.mark.parametrize("lead", [1, 3])
@pytest.mark.parametrize("add", [True, False])
def test_straddling_pairs(gb, lead, add):
    A, B = straddling(lead)
    check_csr(run(gb, add, 1, A, B), reference(add, 1, A, B))
    check_csr(run(gb, add, 1, B, A), reference(add, 1, B, A))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["nnzA0", "nnzB0", "both0", "one_row", "one_col"])
@pytest.mark.parametrize("add", [True, False])
def test_edge_shapes(gb, shape, add):
    rng = np.random.RandomState(2)
    m, n = {"one_row": (1, 5000), "one_col": (5000, 1)}.get(shape, (40, 60))
    A = random_csr(rng, m, n, 0.3, VALUES)
    B = random_csr(rng, m, n, 0.3, VALUES)
    empty = csr(m, n, [], [], np.zeros(0, np.float32), np.float32)
    if shape in ("nnzA0", "both0"):
        A = empty
    if shape in ("nnzB0", "both0"):
        B = empty
    check_csr(run(gb, add, 1, A, B), reference(add, 1, A, B))


@pytest.mark.gpu
@pytest.mark.parametrize("tran", ["inp0", "inp1", "both"])
@pytest.mark.parametrize("add", [True, False])
def test_transposed_operands(gb, tran, add):
    """op(A), op(B) 70 x 110, the transposed operand stored as such; then the same
    call with the transposed operand CSR-only: GrB_UNINITIALIZED_OBJECT, C
    unchanged; then mis-shaped: GrB_DIMENSION_MISMATCH, C unchanged."""
    rng = np.random.RandomState(17)
    A = random_csr(rng, 70, 110, 0.1, VALUES)
    B = random_csr(rng, 70, 110, 0.1, VALUES)
    desc = gb.Descriptor()
    sA, sB = A, B
    if tran in ("inp0", "both"):
        sA = A.T
        desc.set(gb.Desc_field.GrB_INP0, gb.Desc_value.GrB_TRAN)
    if tran in ("inp1", "both"):
        sB = B.T
        desc.set(gb.Desc_field.GrB_INP1, gb.Desc_value.GrB_TRAN)
    want = reference(add, 2, A, B)
    C = gb.Matrix(70, 110)
    op(gb, add)(C, None, None, 2, device_matrix(gb, sA), device_matrix(gb, sB), desc)
    check_csr(C, want)
    plain_A = csr_only(gb, sA) if tran != "inp1" else device_matrix(gb, sA)
    plain_B = csr_only(gb, sB) if tran != "inp0" else device_matrix(gb, sB)
    with pytest.raises(gb.api.GraphBLASError) as err:
        op(gb, add)(C, None, None, 2, plain_A, plain_B, desc)
    assert err.value.info == gb.api.Info.GrB_UNINITIALIZED_OBJECT
    check_csr(C, want)
    with pytest.raises(gb.api.GraphBLASError) as err:
        op(gb, add)(C, None, None, 2, device_matrix(gb, A), device_matrix(gb, B), desc)
    assert err.value.info == gb.api.Info.GrB_DIMENSION_MISMATCH
    check_csr(C, want)


def _dense(S):
    out = np.zeros((S.nrows, S.ncols), np.float64)
    out[S.rows(), S.ind] = S.val
    return out


def check_csc(gb, C, want):
    """C's CSC, read through gb.transpose (which copies it into T's CSR), and a
    pull vxm over C (which reads the CSC)."""
    T = gb.Matrix(want.ncols, want.nrows)
    gb.transpose(T, None, None, C, gb.Descriptor())
    check_csr(T, want.T)
    u = np.array([1, 2, -1, 0.5], np.float32)[np.arange(want.nrows) % 4]
    uv = gb.Vector(want.nrows)
    uv.build(u)
    w = gb.Vector(want.ncols)
    desc = gb.Descriptor()
    desc.set(gb.Desc_field.GrB_MXVMODE, gb.Desc_value.GrB_PULLONLY)
    gb.vxm(w, None, None, 1, uv, C, desc)
    assert np.array_equal(w.extractTuples().astype(np.float64), u.astype(np.float64) @ _dense(want))


@pytest.mark.gpu
@pytest.mark.parametrize("alias", ["C_is_A", "C_is_B", "C_is_both"])
@pytest.mark.parametrize("add", [True, False])
def test_aliasing(gb, alias, add):
    rng = np.random.RandomState(4)
    vals = np.array([-2, -1, 1, 2, 4], np.float32)
    A = random_csr(rng, 150, 130, 0.05, vals, zeros=0)
    B = random_csr(rng, 150, 130, 0.05, vals, zeros=0)
    dA, dB = device_matrix(gb, A), device_matrix(gb, B)
    if alias == "C_is_A":
        op(gb, add)(dA, None, None, 1, dA, dB, gb.Descriptor())
        C, want = dA, reference(add, 1, A, B)
    elif alias == "C_is_B":
        op(gb, add)(dB, None, None, 1, dA, dB, gb.Descriptor())
        C, want = dB, reference(add, 1, A, B)
    else:
        op(gb, add)(dA, None, None, 1, dA, dA, gb.Descriptor())
        C, want = dA, reference(add, 1, A, A)
    check_csr(C, want)
    check_csc(gb, C, want)


@pytest.mark.gpu
@pytest.mark.parametrize("add", [True, False])
def test_int_plus_times(gb, add):
    rng = np.random.RandomState(3)
    ivals = np.array([-3, -2, -1, 0, 1, 2, 3, 5, 7], np.int32)
    A = random_csr(rng, 110, 90, 0.1, ivals)
    B = random_csr(rng, 110, 90, 0.1, ivals)
    check_csr(run(gb, add, 1, A, B, integer=True), reference(add, 1, A, B, integer=True))


@pytest.mark.gpu
@pytest.mark.parametrize("add", [True, False])
def test_refusals_leave_c_unchanged(gb, add):
    rng = np.random.RandomState(6)
    A = random_csr(rng, 50, 40, 0.1, VALUES)
    B = random_csr(rng, 50, 40, 0.1, VALUES)
    want = reference(add, 1, A, B)
    C = run(gb, add, 1, A, B)
    dA, dB = device_matrix(gb, A), device_matrix(gb, B)
    f = op(gb, add)
    Err, Info = gb.api.GraphBLASError, gb.api.Info

    def refused(code, *args):
        with pytest.raises(Err) as err:
            f(*args)
        assert err.value.info == code
        check_csr(C, want)
        assert C.getStorage() == gb.Storage.GrB_SPARSE

    refused(Info.GrB_NOT_IMPLEMENTED, C, dA, None, 1, dA, dB, gb.Descriptor())  # mask
    D = gb.Matrix(50, 40)
    D.build_dense(np.ones((50, 40), np.float32))
    refused(Info.GrB_NOT_IMPLEMENTED, C, None, None, 1, D, dB, gb.Descriptor())
    refused(Info.GrB_NOT_IMPLEMENTED, C, None, None, 1, dA, D, gb.Descriptor())
    refused(Info.GrB_DIMENSION_MISMATCH, C, None, None, 1, dA,
            device_matrix(gb, random_csr(rng, 50, 41, 0.1, VALUES)), gb.Descriptor())
    refused(Info.GrB_DIMENSION_MISMATCH, gb.Matrix(50, 41), None, None, 1, dA, dB,
            gb.Descriptor())
    # INT32 operands: another semiring, then mixed element types
    ivals = np.array([-2, 1, 3], np.int32)
    iA = device_matrix(gb, random_csr(rng, 50, 40, 0.1, ivals), integer=True)
    iB = device_matrix(gb, random_csr(rng, 50, 40, 0.1, ivals), integer=True)
    iC = gb.Matrix(50, 40, dtype=gb.api.INT32)
    with pytest.raises(Err) as err:
        f(iC, None, None, 2, iA, iB, gb.Descriptor())
    assert err.value.info == Info.GrB_NOT_IMPLEMENTED
    refused(Info.GrB_DOMAIN_MISMATCH, C, None, None, 1, iA, dB, gb.Descriptor())
    refused(Info.GrB_DOMAIN_MISMATCH, C, None, None, 1, dA, iB, gb.Descriptor())
    # a dense C refused stays dense; a dense C that succeeds turns sparse
    Cd = gb.Matrix(50, 40)
    Cd.build_dense(np.full((50, 40), 3, np.float32))
    with pytest.raises(Err):
        f(Cd, dA, None, 1, dA, dB, gb.Descriptor())
    assert Cd.getStorage() == gb.Storage.GrB_DENSE
    assert np.all(Cd.extract_dense() == 3)
    f(Cd, None, None, 1, dA, dB, gb.Descriptor())
    assert Cd.getStorage() == gb.Storage.GrB_SPARSE
    check_csr(Cd, want)


@pytest.mark.gpu
@pytest.mark.parametrize("add", [True, False])
def test_deterministic_with_fixed_launches(gb, add):
    import ctypes
    rng = np.random.RandomState(13)
    A = random_csr(rng, 3000, 2000, 0.01, VALUES)
    B = random_csr(rng, 3000, 2000, 0.01, VALUES)
    dA, dB = device_matrix(gb, A), device_matrix(gb, B)
    lib = dA._lib
    count = ctypes.c_ulonglong(0)
    out, launches = [], []
    for _ in range(3):
        C = gb.Matrix(3000, 2000)
        lib.gb200_launch_count(ctypes.byref(count))
        before = count.value
        op(gb, add)(C, None, None, 4, dA, dB, gb.Descriptor())
        lib.gb200_launch_count(ctypes.byref(count))
        launches.append(count.value - before)
        out.append([x.tobytes() for x in C.extract_csr()])
    assert out[0] == out[1] == out[2]
    assert launches[1] == launches[2]
    check_csr(C, reference(add, 4, A, B))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["square", "rect", "rect_csr_only", "symmetric",
                                  "in_place", "inp0_tran"])
def test_transpose(gb, case):
    rng = np.random.RandomState(23)
    m, n = (90, 90) if case in ("square", "symmetric", "in_place") else (70, 130)
    A = random_csr(rng, m, n, 0.08, VALUES[:-1])       # finite: vxm sums are exact
    if case == "symmetric":
        D = _dense(A)
        D = np.triu(D) + np.triu(D, 1).T
        r, c = np.nonzero(D != 0)
        A = csr(m, n, r, c, D[r, c].astype(np.float32), np.float32)
    if case == "rect_csr_only":
        dA = csr_only(gb, A)
    elif case == "symmetric":
        dA = device_matrix(gb, A, symmetric=True)
    else:
        dA = device_matrix(gb, A)
    desc = gb.Descriptor()
    if case == "inp0_tran":
        desc.set(gb.Desc_field.GrB_INP0, gb.Desc_value.GrB_TRAN)
        C, want = gb.Matrix(m, n), A
    elif case == "in_place":
        C, want = dA, A.T
    else:
        C, want = gb.Matrix(n, m), A.T
    gb.transpose(C, None, None, dA, desc)
    check_csr(C, want)
    check_csc(gb, C, want)
    with pytest.raises(gb.api.GraphBLASError) as err:
        gb.transpose(C, C, None, dA, desc)                # C as a mask of its shape
    assert err.value.info == gb.api.Info.GrB_NOT_IMPLEMENTED
    check_csr(C, want)
    if m != n:
        with pytest.raises(gb.api.GraphBLASError) as err:
            gb.transpose(gb.Matrix(m + 1, n + 1), None, None, dA, desc)
        assert err.value.info == gb.api.Info.GrB_DIMENSION_MISMATCH


@pytest.mark.gpu
def test_size_limit(gb):
    """A (even columns) + B (odd columns), 2^15 x 2^16, 2^30 entries each: the union
    has 2^31 > INT32_MAX entries.  GrB_OUT_OF_MEMORY, and C keeps its result."""
    import torch
    m, n = 1 << 15, 1 << 16
    X = csr(m, n, [0, 5, m - 1], [0, 3, n - 1], np.float32([2, -1, 4]), np.float32)
    Y = csr(m, n, [0, 7], [0, 9], np.float32([0.5, 1]), np.float32)
    want = reference(True, 1, X, Y)
    C = run(gb, True, 1, X, Y)
    check_csr(C, want)
    rowptr = torch.arange(0, m + 1, dtype=torch.int32, device="cuda")*(n // 2)
    even = torch.arange(0, n, 2, dtype=torch.int32, device="cuda").repeat(m)
    ones = torch.ones(m*(n // 2), dtype=torch.float32, device="cuda")
    dA = gb.Matrix(m, n)
    dA._keep = [rowptr, even, ones]
    gb.api._check(dA._lib.gb200_matrix_adopt_csr(dA._h, gb.api._dev(rowptr),
                                                 gb.api._dev(even), gb.api._dev(ones),
                                                 m*(n // 2)), "adopt A")
    odd = even + 1
    dB = gb.Matrix(m, n)
    dB._keep = [rowptr, odd, ones]
    gb.api._check(dB._lib.gb200_matrix_adopt_csr(dB._h, gb.api._dev(rowptr),
                                                 gb.api._dev(odd), gb.api._dev(ones),
                                                 m*(n // 2)), "adopt B")
    with pytest.raises(gb.api.GraphBLASError) as err:
        gb.eWiseAdd(C, None, None, 1, dA, dB, gb.Descriptor())
    assert err.value.info == gb.api.Info.GrB_OUT_OF_MEMORY
    check_csr(C, want)
    # the intersection of the two is empty
    E = gb.Matrix(m, n)
    gb.eWiseMult(E, None, None, 1, dA, dB, gb.Descriptor())
    assert E.nvals() == 0
    del dA, dB, even, odd, ones
    torch.cuda.empty_cache()
