"""extract on the device (gb.extract / gb200_extract_matrix, _column, _vector) against
the host restatement of tests/extract_reference.py, bit for bit: row offsets, column
indices and values compared as uint32 bit patterns.

Matrices: FP32 and INT32 with stored zeros, the golden graphs, a directed random CSR
with its CSC, a star (one hub row wider than a tile of selected entries) and an
R-MAT-16 with its hubs.  Lists: GrB_ALL, sorted, shuffled, repeated, a single index;
GrB_INP0 = GrB_TRAN; C aliasing A; C's CSC through transpose.  Columns and
subvectors of dense and sparse vectors.  Every refusal in the documented order, with
the output unchanged.  And an induced subgraph A(S,S) of a symmetric A, installed
symmetric, gives cc, mis and lgc the results they give on the same host CSR.
"""
import ctypes as C

import numpy as np
import pytest

import extract_reference as X
import oracle_binding as orc
from support import (Csr, csr, device_matrix, gb, make_matrix, mtx_graph, random_csr,
                     star_graph)

pytestmark = pytest.mark.gpu

VALUES = np.array([-3, -1, 0.5, 1, 2, 7], np.float32)
IVALUES = np.array([-5, -1, 1, 2, 9], np.int32)


def bits(v):
    v = np.asarray(v)
    return v.view(np.uint32) if v.dtype == np.float32 else v.astype(np.int64)


def index_sets(rng, n):
    return [
        ("all", None),
        ("sorted", np.sort(rng.choice(n, max(1, n//3), replace=False))),
        ("shuffled", rng.permutation(n)[:max(1, n//2)]),
        ("repeated", rng.randint(0, n, n + 5)),
        ("sorted_repeated", np.sort(rng.randint(0, n, n))),
        ("single", np.array([rng.randint(n)])),
    ]


def tran_desc(gb, tran):
    d = gb.Descriptor()
    if tran:
        d.set(gb.Desc_field.GrB_INP0, gb.Desc_value.GrB_TRAN)
    return d


def check_matrix(gb, A, S, I, J, tran=False, out=None):
    """gb.extract(C, ..., A, I, J) equals the restatement on the host Csr S; returns C."""
    nr, nc = (S.ncols, S.nrows) if tran else (S.nrows, S.ncols)
    nI = nr if I is None else len(I)
    nJ = nc if J is None else len(J)
    C_ = out if out is not None else gb.Matrix(nI, nJ, dtype=A.dtype)
    gb.extract(C_, None, None, A, I, nI, J, nJ, tran_desc(gb, tran))
    want = X.extract_matrix(S.ptr, S.ind, S.val, S.nrows, S.ncols, I, J, tran=tran)
    rp, ci, val = C_.extract_csr()
    assert np.array_equal(rp, want[0]), "row offsets differ"
    assert np.array_equal(ci, want[1]), "column indices differ"
    assert np.array_equal(bits(val), bits(want[2].astype(val.dtype))), "values differ"
    return C_


@pytest.mark.parametrize("integer", [False, True])
@pytest.mark.parametrize("tran", [False, True])
def test_random_directed_with_csc(gb, integer, tran):
    rng = np.random.RandomState(11 + integer)
    S = random_csr(rng, 120, 97, 0.08, IVALUES if integer else VALUES, zeros=0.2)
    A = device_matrix(gb, S, csc=True, integer=integer)
    for _, I in index_sets(rng, S.ncols if tran else S.nrows):
        for _, J in index_sets(rng, S.nrows if tran else S.ncols):
            check_matrix(gb, A, S, I, J, tran=tran)


@pytest.mark.parametrize("name", ["chesapeake", "test_bc", "test_cc"])
def test_golden_graphs(gb, name):
    rp, ci = mtx_graph(name)
    n = len(rp) - 1
    rng = np.random.RandomState(3)
    S = Csr(n, n, rp, ci, rng.choice(VALUES, len(ci)))
    A = device_matrix(gb, S, csc=True)
    for _, I in index_sets(rng, n):
        for _, J in index_sets(rng, n):
            check_matrix(gb, A, S, I, J)
            check_matrix(gb, A, S, I, J, tran=True)


def test_star_hub_wider_than_a_tile(gb):
    rp, ci = star_graph(5000)
    n = len(rp) - 1
    S = Csr(n, n, rp, ci, np.arange(len(ci), dtype=np.float32))
    A = device_matrix(gb, S, csc=True)
    rng = np.random.RandomState(5)
    hub_first = np.concatenate([[0, 0], rng.randint(0, n, 50)])
    for I in (None, hub_first, np.array([0])):
        for _, J in index_sets(rng, n):
            check_matrix(gb, A, S, I, J)


def test_rmat16_hubs(gb):
    rp, ci = orc.rmat_csr(16)
    n = len(rp) - 1
    rng = np.random.RandomState(9)
    S = Csr(n, n, rp, ci, rng.choice(VALUES, len(ci)))
    A = device_matrix(gb, S, csc=True)
    deg = np.diff(rp)
    hubs = np.argsort(deg)[-20:]
    for I in (None, np.sort(rng.choice(n, n//10, replace=False)), hubs,
              rng.permutation(n)[:n//4]):
        for J in (None, np.sort(rng.choice(n, n//2, replace=False)), rng.permutation(n),
                  np.repeat(hubs, 3)):
            check_matrix(gb, A, S, I, J)


def test_permutation_in_place_and_csc(gb):
    """C = A(P,P) with C being A; C's CSC (read back through transpose) is the host
    transpose of C."""
    rng = np.random.RandomState(2)
    S = random_csr(rng, 150, 150, 0.05, VALUES, zeros=0.2)
    A = device_matrix(gb, S, csc=True)
    P = rng.permutation(150)
    check_matrix(gb, A, S, P, P, out=A)
    want = X.extract_matrix(S.ptr, S.ind, S.val, 150, 150, P, P)
    T = gb.Matrix(150, 150)
    gb.transpose(T, None, None, A, gb.Descriptor())
    wt = X.extract_matrix(want[0], want[1], want[2], 150, 150, None, None, tran=True)
    rp, ci, val = T.extract_csr()
    assert np.array_equal(rp, wt[0]) and np.array_equal(ci, wt[1])
    assert np.array_equal(bits(val), bits(wt[2]))


def test_symmetric_induced_subgraph_and_its_csc(gb):
    rp, ci = orc.rmat_csr(12)
    n = len(rp) - 1
    rng = np.random.RandomState(4)
    # symmetric values, so that the CSC a symmetric matrix adopts holds Aᵀ
    rows = np.repeat(np.arange(n), np.diff(rp))
    val = VALUES[(rows + ci) % len(VALUES)]
    A = make_matrix(gb, rp, ci, val=val)
    S = Csr(n, n, rp, ci, val)
    for Sset in (np.sort(rng.choice(n, n//2, replace=False)), rng.permutation(n)[:n//3],
                 np.sort(rng.randint(0, n, n//4))):
        C_ = check_matrix(gb, A, S, Sset, Sset)
        want = X.extract_matrix(S.ptr, S.ind, S.val, n, n, Sset, Sset)
        T = gb.Matrix(len(Sset), len(Sset))
        gb.transpose(T, None, None, C_, gb.Descriptor())
        wt = X.extract_matrix(want[0], want[1], want[2], len(Sset), len(Sset), None, None,
                              tran=True)
        got = T.extract_csr()
        assert np.array_equal(got[0], wt[0]) and np.array_equal(got[1], wt[1])
        assert np.array_equal(bits(got[2]), bits(wt[2]))


def test_symmetric_results_feed_the_graph_algorithms(gb):
    from graphblast_b200 import algorithm
    rp, ci = orc.rmat_csr(13)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    rng = np.random.RandomState(8)
    Sset = np.sort(rng.choice(n, n//2, replace=False))
    m = len(Sset)
    C_ = gb.Matrix(m, m)
    gb.extract(C_, None, None, A, Sset, m, Sset, m, gb.Descriptor())
    s_rp, s_ci, _ = X.extract_matrix(rp, ci, np.ones(len(ci), np.float32), n, n, Sset, Sset)
    B = make_matrix(gb, s_rp, s_ci, symmetric=True)

    def run(M, f):
        v = gb.Vector(m)
        f(v, M)
        return v.extractTuples()
    desc = gb.Descriptor()
    assert np.array_equal(run(C_, lambda v, M: algorithm.cc(v, M, desc)),
                          run(B, lambda v, M: algorithm.cc(v, M, desc)))
    assert np.array_equal(run(C_, lambda v, M: algorithm.mis(v, M, 3, desc)),
                          run(B, lambda v, M: algorithm.mis(v, M, 3, desc)))
    src = int(np.argmax(np.diff(s_rp)))
    got = run(C_, lambda v, M: algorithm.lgc(v, M, src, 0.15, 1e-6, desc))
    want = run(B, lambda v, M: algorithm.lgc(v, M, src, 0.15, 1e-6, desc))
    assert np.array_equal(bits(np.float32(got)), bits(np.float32(want)))


@pytest.mark.parametrize("tran", [False, True])
def test_columns(gb, tran):
    rng = np.random.RandomState(21)
    S = random_csr(rng, 80, 60, 0.1, VALUES, zeros=0.2)
    A = device_matrix(gb, S, csc=True)
    nr, nc = (60, 80) if tran else (80, 60)
    for _, I in index_sets(rng, nr):
        nI = nr if I is None else len(I)
        for j in (0, nc - 1, int(rng.randint(nc))):
            w = gb.Vector(nI)
            gb.extract(w, None, None, A, I, nI, j, 0, tran_desc(gb, tran))
            want_ind, want_val = X.extract_column(S.ptr, S.ind, S.val, 80, 60, I, j, tran=tran)
            assert w.getStorage() == gb.Storage.GrB_SPARSE
            ind, val = w.extractTuples(sparse=True)
            assert np.array_equal(ind, want_ind)
            assert np.array_equal(bits(np.float32(val)), bits(want_val))


def test_subvectors(gb):
    rng = np.random.RandomState(13)
    n = 300
    u = rng.choice(VALUES, n).astype(np.float32)
    u_ind = np.sort(rng.choice(n, 90, replace=False)).astype(np.int32)
    for _, I in index_sets(rng, n):
        nI = n if I is None else len(I)
        U = gb.Vector(n)
        U.build(u)
        w = gb.Vector(nI)
        gb.extract(w, None, None, U, I, nI, None, 0, gb.Descriptor())
        assert w.getStorage() == gb.Storage.GrB_DENSE
        assert np.array_equal(bits(np.float32(w.extractTuples())),
                              bits(X.extract_dense_vector(u, I)))
        U2 = gb.Vector(n)
        U2.build(u_ind, u[u_ind])
        w = gb.Vector(nI)
        gb.extract(w, None, None, U2, I, nI, None, 0, gb.Descriptor())
        assert w.getStorage() == gb.Storage.GrB_SPARSE
        want_ind, want_val = X.extract_sparse_vector(u_ind, u[u_ind], n, I)
        ind, val = w.extractTuples(sparse=True)
        assert np.array_equal(ind, want_ind)
        assert np.array_equal(bits(np.float32(val)), bits(want_val))
    # in place: w is u, a permutation
    P = rng.permutation(n)
    U = gb.Vector(n)
    U.build(u)
    gb.extract(U, None, None, U, P, n, None, 0, gb.Descriptor())
    assert np.array_equal(bits(np.float32(U.extractTuples())), bits(u[P]))


# ---------------------------------------------------------------------------
# refusals, in the order of include/graphblast_b200_extract.h
# ---------------------------------------------------------------------------

def code(gb, name):
    return int(getattr(gb.Info, name))


def refused(gb, expected, call):
    with pytest.raises(gb.GraphBLASError) as e:
        call()
    assert e.value.info == code(gb, expected), (e.value.info, expected)


def test_refusals_in_order_leave_outputs_untouched(gb):
    rng = np.random.RandomState(1)
    S = random_csr(rng, 40, 30, 0.2, VALUES, zeros=0.1)
    A = device_matrix(gb, S, csc=True)
    A_nocsc = device_matrix(gb, S, csc=False)
    Ai = device_matrix(gb, S.astype(np.int32), csc=True, integer=True)
    Ad = gb.Matrix(40, 30)
    Ad.build_dense(np.ones((40, 30), np.float32))
    mask = gb.Matrix(5, 5)
    d = gb.Descriptor()
    dt = tran_desc(gb, True)
    I5 = np.arange(5)
    C_ = device_matrix(gb, random_csr(rng, 5, 5, 0.5, VALUES), csc=True)
    before = C_.extract_csr()

    def same_c():
        after = C_.extract_csr()
        assert all(np.array_equal(x, y) for x, y in zip(before, after)), "C changed"
    lib = C_._lib
    # 2. a count < 1
    assert lib.gb200_extract_matrix(C_._h, None, A._h, None, 0, None, 5, d._h) == \
        code(gb, "GrB_INVALID_VALUE")
    same_c()
    # 3. element types
    refused(gb, "GrB_DOMAIN_MISMATCH", lambda: gb.extract(C_, None, None, Ai, I5, 5, I5, 5, d))
    same_c()
    # 5. a mask, a dense A (also with wrong shapes)
    I6 = np.arange(6)
    refused(gb, "GrB_NOT_IMPLEMENTED", lambda: gb.extract(C_, mask, None, A, I5, 5, I6, 6, d))
    refused(gb, "GrB_NOT_IMPLEMENTED", lambda: gb.extract(C_, None, None, Ad, I5, 5, I6, 6, d))
    same_c()
    # 6. shapes (with an index also out of range)
    refused(gb, "GrB_DIMENSION_MISMATCH",
            lambda: gb.extract(C_, None, None, A, I5, 5, np.arange(6) + 99, 6, d))
    same_c()
    # 7. an index out of range, ALL with a count that is not the extent
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.extract(C_, None, None, A, I5, 5,
                                                        np.array([0, 1, 2, 3, 30]), 5, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.extract(C_, None, None, A, I5 - 1, 5, I5, 5, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.extract(C_, None, None, A, None, 5, I5, 5, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.extract(C_, None, None, A_nocsc, I5 + 26, 5,
                                                        I5, 5, dt))
    same_c()
    # 8. the orientation that is not there
    refused(gb, "GrB_UNINITIALIZED_OBJECT",
            lambda: gb.extract(C_, None, None, A_nocsc, I5, 5, I5, 5, dt))
    same_c()

    # the column and vector entries
    w = gb.Vector(5)
    w.build(np.arange(5, dtype=np.float32))
    w_before = w.extractTuples()

    def same_w():
        assert np.array_equal(w.extractTuples(), w_before), "w changed"
    vmask = gb.Vector(5)
    refused(gb, "GrB_DOMAIN_MISMATCH", lambda: gb.extract(w, None, None, Ai, I5, 5, 0, 0, d))
    refused(gb, "GrB_NOT_IMPLEMENTED", lambda: gb.extract(w, vmask, None, A, I5, 5, 0, 0, d))
    refused(gb, "GrB_NOT_IMPLEMENTED",
            lambda: gb.extract(w, None, None, Ad, np.arange(6), 6, 0, 0, d))
    refused(gb, "GrB_DIMENSION_MISMATCH",
            lambda: gb.extract(w, None, None, A, np.arange(6), 6, 0, 0, d))
    refused(gb, "GrB_DIMENSION_MISMATCH", lambda: gb.extract(w, None, None, A, I5, 5, 30, 0, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.extract(w, None, None, A, I5 + 38, 5, 0, 0, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.extract(w, None, None, A, I5, 5, -1, 0, d))
    refused(gb, "GrB_UNINITIALIZED_OBJECT",
            lambda: gb.extract(w, None, None, A_nocsc, I5, 5, 0, 0, d))
    same_w()
    u = gb.Vector(8)
    u.build(np.arange(8, dtype=np.float32))
    refused(gb, "GrB_NOT_IMPLEMENTED", lambda: gb.extract(w, vmask, None, u, I5, 5, None, 0, d))
    refused(gb, "GrB_DIMENSION_MISMATCH", lambda: gb.extract(w, None, None, u, I5, 4, None, 0, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.extract(w, None, None, u, I5 + 4, 5, None, 0, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.extract(w, None, None, u, None, 5, None, 0, d))
    same_w()
