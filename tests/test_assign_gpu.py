"""assign into a matrix on the device (gb.assign with a Matrix output /
gb200_assign_matrix, _matrix_scalar, _column, _row) against the host restatement of
tests/assign_reference.py, bit for bit: row offsets, column indices and values
compared as uint32 bit patterns.

Matrices: FP32 and INT32 with stored zeros, the golden graphs, a directed random CSR
with its CSC, a star (one hub row wider than a merge tile) and an R-MAT-16 with its
hubs.  Lists: GrB_ALL, sorted, shuffled, a single index; GrB_INP0 = GrB_TRAN; no
accum, every FP32 monoid and INT32 PLUS; C aliasing A; a fresh C assembled from
blocks; C's CSC read back through transpose.  Row, column (dense, sparse and empty u)
and constant forms.  The round trip through extract.  A symmetric C edited by
C(S,S) = B with a symmetric B stays symmetric, with the right CSC values, and cc and
mis give on it what they give on the same host CSR.  Every refusal in the documented
order, with C unchanged.
"""
import numpy as np
import pytest

import assign_reference as R
import extract_reference as X
import oracle_binding as orc
from support import Csr, csr, device_matrix, gb, mtx_graph, random_csr, star_graph  # noqa: F401

pytestmark = pytest.mark.gpu

VALUES = np.array([-3, -1, 0.5, 1, 2, 7], np.float32)
IVALUES = np.array([-5, -1, 1, 2, 9], np.int32)
# the restatement's accum of each gb.Monoid, in order
MONOID_OPS = ["plus", "mul", "min", "max", "or", "and", "gt", "lt", "ne"]


def bits(v):
    v = np.asarray(v)
    return v.view(np.uint32) if v.dtype == np.float32 else v.astype(np.int64)


def index_sets(rng, n):
    return [
        ("all", None),
        ("sorted", np.sort(rng.choice(n, max(1, n//3), replace=False))),
        ("shuffled", rng.permutation(n)[:max(1, n//2)]),
        ("single", np.array([rng.randint(n)])),
    ]


def tran_desc(gb, tran):
    d = gb.Descriptor()
    if tran:
        d.set(gb.Desc_field.GrB_INP0, gb.Desc_value.GrB_TRAN)
    return d


def accum_name(accum):
    return None if accum is None else MONOID_OPS[int(accum)]


def host(S):
    return (S.ptr, S.ind, S.val)


def check(C_, want, what=""):
    rp, ci, val = C_.extract_csr()
    assert np.array_equal(rp, want[0]), "row offsets differ " + what
    assert np.array_equal(ci, want[1]), "column indices differ " + what
    assert np.array_equal(bits(val), bits(np.asarray(want[2]).astype(val.dtype))), \
        "values differ " + what


def check_csc(gb, C_, want, m, n):
    """C's CSC, read back through transpose, is the host transpose of want."""
    T = gb.Matrix(n, m, dtype=C_.dtype)
    gb.transpose(T, None, None, C_, gb.Descriptor())
    check(T, X.extract_matrix(want[0], want[1], want[2], m, n, None, None, tran=True),
          "(CSC)")


def run_matrix(gb, Cs, A, As, I, J, accum=None, tran=False, integer=False, csc=False):
    """A fresh device copy of the host Csr Cs takes C(I, J) = accum(.., op(A))."""
    C_ = device_matrix(gb, Cs, csc=True, integer=integer)
    m, n = Cs.nrows, Cs.ncols
    nI = m if I is None else len(I)
    nJ = n if J is None else len(J)
    gb.assign(C_, None, accum, A, I, nI, J, nJ, tran_desc(gb, tran))
    want = R.assign_matrix(host(Cs), m, n, (As.ptr, As.ind, As.val, As.nrows, As.ncols),
                           I, J, accum=accum_name(accum), tran=tran)
    check(C_, want)
    if csc:
        check_csc(gb, C_, want, m, n)
    return C_, want


@pytest.mark.parametrize("integer", [False, True])
@pytest.mark.parametrize("tran", [False, True])
def test_random_directed_with_csc(gb, integer, tran):
    rng = np.random.RandomState(11 + integer + 2*tran)
    vals = IVALUES if integer else VALUES
    Cs = random_csr(rng, 90, 70, 0.08, vals, zeros=0.2)
    for _, I in index_sets(rng, 90):
        for _, J in index_sets(rng, 70):
            nI = 90 if I is None else len(I)
            nJ = 70 if J is None else len(J)
            As = random_csr(rng, nJ if tran else nI, nI if tran else nJ, 0.2, vals, zeros=0.2)
            A = device_matrix(gb, As, csc=True, integer=integer)
            for accum in (None, gb.Monoid.Plus):
                run_matrix(gb, Cs, A, As, I, J, accum, tran, integer, csc=accum is None)


def test_every_fp32_monoid(gb):
    rng = np.random.RandomState(3)
    Cs = random_csr(rng, 64, 80, 0.15, VALUES, zeros=0.2)
    I = rng.permutation(64)[:30]
    J = np.sort(rng.choice(80, 50, replace=False))
    As = random_csr(rng, 30, 50, 0.3, VALUES, zeros=0.2)
    A = device_matrix(gb, As, csc=True)
    for accum in gb.Monoid:
        run_matrix(gb, Cs, A, As, I, J, accum)
    As2 = random_csr(rng, 64, 80, 0.1, VALUES, zeros=0.2)
    A2 = device_matrix(gb, As2, csc=True)
    for accum in gb.Monoid:
        run_matrix(gb, Cs, A2, As2, None, None, accum)


@pytest.mark.parametrize("name", ["chesapeake", "test_bc", "test_cc"])
def test_golden_graphs(gb, name):
    rp, ci = mtx_graph(name)
    n = len(rp) - 1
    rng = np.random.RandomState(5)
    Cs = Csr(n, n, rp, ci, rng.choice(VALUES, len(ci)))
    for _, I in index_sets(rng, n):
        for _, J in index_sets(rng, n):
            nI = n if I is None else len(I)
            nJ = n if J is None else len(J)
            As = random_csr(rng, nI, nJ, 0.3, VALUES, zeros=0.2)
            A = device_matrix(gb, As, csc=True)
            run_matrix(gb, Cs, A, As, I, J)
            run_matrix(gb, Cs, A, As, I, J, gb.Monoid.Minimum)
            At = device_matrix(gb, As.T, csc=True)
            run_matrix(gb, Cs, At, As.T, I, J, tran=True)


def test_star_hub_wider_than_a_tile(gb):
    rp, ci = star_graph(5000)
    n = len(rp) - 1
    Cs = Csr(n, n, rp, ci, np.arange(len(ci), dtype=np.float32))
    rng = np.random.RandomState(6)
    hub_first = np.concatenate([[0], rng.choice(np.arange(1, n), 40, replace=False)])
    for I in (np.array([0]), hub_first):
        for J in (None, rng.permutation(n)[:3000], np.sort(rng.choice(n, 4000, replace=False))):
            nJ = n if J is None else len(J)
            As = random_csr(rng, len(I), nJ, 0.4, VALUES, zeros=0.1)
            A = device_matrix(gb, As, csc=True)
            run_matrix(gb, Cs, A, As, I, J)
            run_matrix(gb, Cs, A, As, I, J, gb.Monoid.Plus)
    # the hub row replaced by a dense row, and deleted by an empty one
    for u_ind in (np.arange(n), np.array([], np.int64)):
        u_val = rng.choice(VALUES, len(u_ind)).astype(np.float32)
        C_ = device_matrix(gb, Cs, csc=True)
        u = gb.Vector(n)
        if len(u_ind) == n:
            u.build(u_val)
        else:
            u.build(u_ind.astype(np.int32), u_val)
        gb.assign(C_, None, None, u, 0, None, n, gb.Descriptor())
        check(C_, R.assign_row(host(Cs), n, n, u_ind, u_val, 0, None))


def sparse_random(rng, nrows, ncols, nnz):
    """About nnz uniformly placed entries with VALUES and some stored zeros."""
    key = np.unique(rng.randint(0, nrows*ncols, nnz).astype(np.int64))
    vals = rng.choice(VALUES, len(key))
    vals[rng.rand(len(key)) < 0.1] = 0
    return csr(nrows, ncols, key//ncols, key % ncols, vals, np.float32)


def test_rmat16_hubs(gb):
    rp, ci = orc.rmat_csr(16)
    n = len(rp) - 1
    rng = np.random.RandomState(9)
    Cs = Csr(n, n, rp, ci, rng.choice(VALUES, len(ci)))
    hubs = np.argsort(np.diff(rp))[-20:]
    for I in (hubs, np.sort(rng.choice(n, n//10, replace=False)), rng.permutation(n)[:n//4]):
        for J in (None, np.sort(rng.choice(n, n//2, replace=False)), rng.permutation(n)):
            nJ = n if J is None else len(J)
            As = sparse_random(rng, len(I), nJ, 8*len(I))
            A = device_matrix(gb, As, csc=True)
            run_matrix(gb, Cs, A, As, I, J)
            run_matrix(gb, Cs, A, As, I, J, gb.Monoid.Plus)


def test_c_aliasing_a_and_csc(gb):
    rng = np.random.RandomState(2)
    Cs = random_csr(rng, 120, 120, 0.05, VALUES, zeros=0.2)
    for P in (rng.permutation(120), np.sort(rng.choice(120, 120, replace=False))):
        for accum in (None, gb.Monoid.Plus):
            C_ = device_matrix(gb, Cs, csc=True)
            gb.assign(C_, None, accum, C_, P, 120, P, 120, gb.Descriptor())
            want = R.assign_matrix(host(Cs), 120, 120, (Cs.ptr, Cs.ind, Cs.val, 120, 120),
                                   P, P, accum=accum_name(accum))
            check(C_, want)
            check_csc(gb, C_, want, 120, 120)
    # a block of C assigned from C itself, transposed
    C_ = device_matrix(gb, Cs, csc=True)
    I = rng.permutation(120)
    gb.assign(C_, None, None, C_, I, 120, I, 120, tran_desc(gb, True))
    check(C_, R.assign_matrix(host(Cs), 120, 120, (Cs.ptr, Cs.ind, Cs.val, 120, 120), I, I,
                              tran=True))


def test_fresh_c_from_blocks(gb):
    rng = np.random.RandomState(8)
    m, n = 70, 90
    C_ = gb.Matrix(m, n)
    want = (np.zeros(m + 1, np.int32), np.zeros(0, np.int32), np.zeros(0, np.float32))
    for r0, r1, c0, c1 in ((0, 30, 0, 40), (30, 70, 0, 40), (0, 30, 40, 90), (30, 70, 40, 90)):
        As = random_csr(rng, r1 - r0, c1 - c0, 0.2, VALUES, zeros=0.2)
        A = device_matrix(gb, As, csc=True)
        I, J = np.arange(r0, r1), np.arange(c0, c1)
        gb.assign(C_, None, None, A, I, len(I), J, len(J), gb.Descriptor())
        want = R.assign_matrix(want, m, n, (As.ptr, As.ind, As.val, As.nrows, As.ncols), I, J)
        check(C_, want)
    check_csc(gb, C_, want, m, n)
    # a fresh INT32 C takes a constant block
    Ci = gb.Matrix(m, n, dtype=gb.api.INT32)
    I, J = rng.permutation(m)[:9], rng.permutation(n)[:11]
    gb.assign(Ci, None, None, 5, I, 9, J, 11, gb.Descriptor())
    empty = (np.zeros(m + 1, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int32))
    check(Ci, R.assign_constant(empty, m, n, 5, I, J))


def test_columns_rows_and_constants(gb):
    rng = np.random.RandomState(21)
    m, n = 80, 60
    Cs = random_csr(rng, m, n, 0.1, VALUES, zeros=0.2)
    d = gb.Descriptor()
    for _, I in index_sets(rng, m):
        nI = m if I is None else len(I)
        for u_ind in (np.arange(nI), np.sort(rng.choice(nI, (nI + 1)//2, replace=False)),
                      np.array([], np.int64)):
            u_val = rng.choice(VALUES, len(u_ind)).astype(np.float32)
            u = gb.Vector(nI)
            if len(u_ind) == nI:
                u.build(u_val)
            else:
                u.build(u_ind.astype(np.int32), u_val)
            for accum in (None, gb.Monoid.Plus, gb.Monoid.Maximum):
                j = int(rng.randint(n))
                C_ = device_matrix(gb, Cs, csc=True)
                gb.assign(C_, None, accum, u, I, nI, j, d)
                want = R.assign_column(host(Cs), m, n, u_ind, u_val, I, j, accum_name(accum))
                check(C_, want, "(column)")
                check_csc(gb, C_, want, m, n)
    for _, J in index_sets(rng, n):
        nJ = n if J is None else len(J)
        for u_ind in (np.arange(nJ), np.sort(rng.choice(nJ, (nJ + 1)//2, replace=False)),
                      np.array([], np.int64)):
            u_val = rng.choice(VALUES, len(u_ind)).astype(np.float32)
            u = gb.Vector(nJ)
            if len(u_ind) == nJ:
                u.build(u_val)
            else:
                u.build(u_ind.astype(np.int32), u_val)
            for accum in (None, gb.Monoid.Minimum):
                i = int(rng.randint(m))
                C_ = device_matrix(gb, Cs, csc=True)
                gb.assign(C_, None, accum, u, i, J, nJ, d)
                check(C_, R.assign_row(host(Cs), m, n, u_ind, u_val, i, J, accum_name(accum)),
                      "(row)")
    for _, I in index_sets(rng, m):
        for _, J in index_sets(rng, n):
            nI = m if I is None else len(I)
            nJ = n if J is None else len(J)
            for accum in (None, gb.Monoid.Plus):
                C_ = device_matrix(gb, Cs, csc=True)
                gb.assign(C_, None, accum, 0.5, I, nI, J, nJ, d)
                want = R.assign_constant(host(Cs), m, n, np.float32(0.5), I, J,
                                         accum_name(accum))
                check(C_, want, "(constant)")
    Ci = Cs.with_values(rng.choice(IVALUES, Cs.nnz))
    I, J = rng.permutation(m)[:20], np.sort(rng.choice(n, 25, replace=False))
    for accum in (None, gb.Monoid.Plus):
        C_ = device_matrix(gb, Ci, csc=True, integer=True)
        gb.assign(C_, None, accum, 0, I, 20, J, 25, d)
        check(C_, R.assign_constant(host(Ci), m, n, 0, I, J, accum_name(accum)),
              "(INT32 constant)")


def test_round_trip_through_extract(gb):
    rng = np.random.RandomState(17)
    m, n = 150, 130
    Cs = random_csr(rng, m, n, 0.06, VALUES, zeros=0.2)
    for _, I in index_sets(rng, m):
        for _, J in index_sets(rng, n):
            nI = m if I is None else len(I)
            nJ = n if J is None else len(J)
            As = random_csr(rng, nI, nJ, 0.1, VALUES, zeros=0.2)
            A = device_matrix(gb, As, csc=True)
            C_, _ = run_matrix(gb, Cs, A, As, I, J)
            back = gb.Matrix(nI, nJ)
            gb.extract(back, None, None, C_, I, nI, J, nJ, gb.Descriptor())
            check(back, host(As), "(round trip)")
            if I is not None:
                rest = np.setdiff1d(np.arange(m), I)
                out = gb.Matrix(len(rest), n)
                gb.extract(out, None, None, C_, rest, len(rest), None, n, gb.Descriptor())
                check(out, X.extract_matrix(Cs.ptr, Cs.ind, Cs.val, m, n, rest, None),
                      "(rows outside)")
            if J is not None:
                rest = np.setdiff1d(np.arange(n), J)
                out = gb.Matrix(m, len(rest))
                gb.extract(out, None, None, C_, None, m, rest, len(rest), gb.Descriptor())
                check(out, X.extract_matrix(Cs.ptr, Cs.ind, Cs.val, m, n, None, rest),
                      "(columns outside)")


def symmetric_matrix(gb, rp, ci, val):
    """A Matrix marked symmetric over the pattern (rp, ci) with CSR values val and
    the CSC values of its transpose."""
    import torch
    from graphblast_b200 import graphs
    n = len(rp) - 1
    d_rp, d_ci = torch.from_numpy(rp).cuda(), torch.from_numpy(ci).cuda()
    d_val = torch.from_numpy(np.asarray(val, np.float32)).cuda()
    return graphs.matrix_from_csr(n, d_rp, d_ci, d_val,
                                  cscval=graphs.transpose_values(n, d_rp, d_ci, d_val))


def test_symmetric_edit_stays_symmetric(gb):
    from graphblast_b200 import algorithm
    rp, ci = orc.rmat_csr(12)
    n = len(rp) - 1
    rng = np.random.RandomState(4)
    rows = np.repeat(np.arange(n), np.diff(rp))
    val = VALUES[(3*rows + ci) % len(VALUES)]          # not symmetric: CSC values differ
    Cs = Csr(n, n, rp, ci, val)
    S = np.sort(rng.choice(n, n//3, replace=False))
    # B: a symmetric pattern on S x S from a second R-MAT
    b_rp, b_ci = orc.rmat_csr(11, seed=7)
    keep = np.repeat(np.arange(len(b_rp) - 1), np.diff(b_rp)) < len(S)
    b_rows = np.repeat(np.arange(len(b_rp) - 1), np.diff(b_rp))[keep]
    b_cols = b_ci[keep]
    inside = b_cols < len(S)
    Bs = Csr(len(S), len(S), np.concatenate([[0], np.cumsum(
        np.bincount(b_rows[inside], minlength=len(S)))]).astype(np.int32),
        b_cols[inside], VALUES[(b_rows[inside] + 2*b_cols[inside]) % len(VALUES)])
    for Sset in (S, rng.permutation(S)):
        for accum, tran in ((None, False), (gb.Monoid.Plus, False), (None, True)):
            C_ = symmetric_matrix(gb, rp, ci, val)
            B = symmetric_matrix(gb, Bs.ptr, Bs.ind, Bs.val)
            gb.assign(C_, None, accum, B, Sset, len(S), Sset, len(S), tran_desc(gb, tran))
            want = R.assign_matrix(host(Cs), n, n, (Bs.ptr, Bs.ind, Bs.val, len(S), len(S)),
                                   Sset, Sset, accum=accum_name(accum), tran=tran)
            check(C_, want, "(symmetric)")
            check_csc(gb, C_, want, n, n)
        # a constant block keeps the symmetry too
        C_ = symmetric_matrix(gb, rp, ci, val)
        gb.assign(C_, None, None, 2.0, Sset[:40], 40, Sset[:40], 40, gb.Descriptor())
        want = R.assign_constant(host(Cs), n, n, np.float32(2.0), Sset[:40], Sset[:40])
        check(C_, want, "(symmetric constant)")
        check_csc(gb, C_, want, n, n)
    # the graph algorithms on the edited graph, against the same host CSR
    C_ = symmetric_matrix(gb, rp, ci, np.ones(len(ci), np.float32))
    B = symmetric_matrix(gb, Bs.ptr, Bs.ind, np.ones(Bs.nnz, np.float32))
    gb.assign(C_, None, None, B, S, len(S), S, len(S), gb.Descriptor())
    e_rp, e_ci, _ = R.assign_matrix((rp, ci, np.ones(len(ci), np.float32)), n, n,
                                    (Bs.ptr, Bs.ind, np.ones(Bs.nnz, np.float32), len(S),
                                     len(S)), S, S)
    H = symmetric_matrix(gb, e_rp, e_ci, np.ones(len(e_ci), np.float32))

    def run(M, f):
        v = gb.Vector(n)
        f(v, M)
        return v.extractTuples()
    desc = gb.Descriptor()
    assert np.array_equal(run(C_, lambda v, M: algorithm.cc(v, M, desc)),
                          run(H, lambda v, M: algorithm.cc(v, M, desc)))
    assert np.array_equal(run(C_, lambda v, M: algorithm.mis(v, M, 3, desc)),
                          run(H, lambda v, M: algorithm.mis(v, M, 3, desc)))


# ---------------------------------------------------------------------------
# refusals, in the order of include/graphblast_b200_assign.h
# ---------------------------------------------------------------------------

def code(gb, name):
    return int(getattr(gb.Info, name))


def refused(gb, expected, call):
    with pytest.raises(gb.GraphBLASError) as e:
        call()
    assert e.value.info == code(gb, expected), (e.value.info, expected)


def test_refusals_in_order_leave_c_untouched(gb):
    rng = np.random.RandomState(1)
    Cs = random_csr(rng, 40, 30, 0.2, VALUES, zeros=0.1)
    C_ = device_matrix(gb, Cs, csc=True)
    Ci = device_matrix(gb, Cs.astype(np.int32), csc=True, integer=True)
    As = random_csr(rng, 5, 6, 0.5, VALUES)
    A = device_matrix(gb, As, csc=True)
    A_nocsc = device_matrix(gb, As.T, csc=False)       # 6 x 5, no CSC
    Ai = device_matrix(gb, As.astype(np.int32), csc=True, integer=True)
    Ad = gb.Matrix(5, 6)
    Ad.build_dense(np.ones((5, 6), np.float32))
    Cd = gb.Matrix(40, 30)
    Cd.build_dense(np.ones((40, 30), np.float32))
    mask = gb.Matrix(40, 30)
    vmask = gb.Vector(40)
    u5 = gb.Vector(5)
    u5.build(np.arange(5, dtype=np.float32))
    d = gb.Descriptor()
    dt = tran_desc(gb, True)
    I5, J6 = np.arange(5), np.arange(6)
    before = C_.extract_csr()
    before_i = Ci.extract_csr()

    def same_c():
        for X_, b in ((C_, before), (Ci, before_i)):
            after = X_.extract_csr()
            assert all(np.array_equal(x, y) for x, y in zip(b, after)), "C changed"
    lib = C_._lib
    # 2. a count < 1, an unknown accum
    assert lib.gb200_assign_matrix(C_._h, None, -1, A._h, None, 0, None, 6, d._h) == \
        code(gb, "GrB_INVALID_VALUE")
    assert lib.gb200_assign_matrix(C_._h, None, 9, Ai._h, None, 40, None, 30, d._h) == \
        code(gb, "GrB_INVALID_VALUE")
    assert lib.gb200_assign_row(C_._h, None, -3, u5._h, 0, None, 0, d._h) == \
        code(gb, "GrB_INVALID_VALUE")
    same_c()
    # 3. element types (before a mask or a dense operand)
    refused(gb, "GrB_DOMAIN_MISMATCH", lambda: gb.assign(C_, mask, None, Ai, I5, 5, J6, 6, d))
    refused(gb, "GrB_DOMAIN_MISMATCH", lambda: gb.assign(Ci, vmask, None, u5, I5, 5, 0, d))
    refused(gb, "GrB_DOMAIN_MISMATCH", lambda: gb.assign(Ci, None, None, u5, 0, I5, 5, d))
    same_c()
    # 5. a mask, a dense C or A, INT32 with an accum other than PLUS (also with wrong
    #    shapes)
    I4 = np.arange(4)
    refused(gb, "GrB_NOT_IMPLEMENTED", lambda: gb.assign(C_, mask, None, A, I4, 4, J6, 6, d))
    refused(gb, "GrB_NOT_IMPLEMENTED", lambda: gb.assign(C_, None, None, Ad, I4, 4, J6, 6, d))
    refused(gb, "GrB_NOT_IMPLEMENTED", lambda: gb.assign(Cd, None, None, A, I4, 4, J6, 6, d))
    refused(gb, "GrB_NOT_IMPLEMENTED", lambda: gb.assign(Cd, None, None, 1.0, I4, 4, J6, 6, d))
    refused(gb, "GrB_NOT_IMPLEMENTED",
            lambda: gb.assign(Ci, None, gb.Monoid.Minimum, Ai, I4, 4, J6, 6, d))
    refused(gb, "GrB_NOT_IMPLEMENTED",
            lambda: gb.assign(Ci, None, gb.Monoid.Maximum, 1, I4, 4, J6, 6, d))
    refused(gb, "GrB_NOT_IMPLEMENTED", lambda: gb.assign(C_, vmask, None, u5, I4, 4, 0, d))
    refused(gb, "GrB_NOT_IMPLEMENTED", lambda: gb.assign(C_, vmask, None, u5, 0, I4, 4, d))
    same_c()
    # 6. shapes (with an index also out of range)
    refused(gb, "GrB_DIMENSION_MISMATCH",
            lambda: gb.assign(C_, None, None, A, I4 + 99, 4, J6, 6, d))
    refused(gb, "GrB_DIMENSION_MISMATCH",
            lambda: gb.assign(C_, None, None, A, I5, 5, J6, 6, dt))
    refused(gb, "GrB_DIMENSION_MISMATCH",
            lambda: gb.assign(C_, None, None, u5, I4 + 99, 4, 0, d))
    refused(gb, "GrB_DIMENSION_MISMATCH", lambda: gb.assign(C_, None, None, u5, I5, 5, 30, d))
    refused(gb, "GrB_DIMENSION_MISMATCH", lambda: gb.assign(C_, None, None, u5, 40, I5, 5, d))
    same_c()
    # 7. an index out of range, a negative row or column, ALL with the wrong count
    refused(gb, "GrB_INVALID_INDEX",
            lambda: gb.assign(C_, None, None, A, I5, 5, np.array([0, 1, 2, 3, 4, 30]), 6, d))
    refused(gb, "GrB_INVALID_INDEX",
            lambda: gb.assign(C_, None, None, A, np.array([0, 0, 1, 2, -1]), 5, J6, 6, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.assign(C_, None, None, A, None, 5, J6, 6, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.assign(C_, None, None, 1.0, I5, 5, None, 6, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.assign(C_, None, None, u5, I5, 5, -1, d))
    refused(gb, "GrB_INVALID_INDEX", lambda: gb.assign(C_, None, None, u5, -1, I5, 5, d))
    refused(gb, "GrB_INVALID_INDEX",
            lambda: gb.assign(C_, None, None, u5, np.array([0, 1, 2, 3, 40]), 5, 0, d))
    same_c()
    # 8. a repeated index
    refused(gb, "GrB_INVALID_VALUE",
            lambda: gb.assign(C_, None, None, A, np.array([0, 1, 2, 3, 1]), 5, J6, 6, d))
    refused(gb, "GrB_INVALID_VALUE",
            lambda: gb.assign(C_, None, None, 1.0, I5, 5, np.array([7, 7]), 2, d))
    refused(gb, "GrB_INVALID_VALUE",
            lambda: gb.assign(C_, None, None, u5, 3, np.array([0, 4, 2, 4, 9]), 5, d))
    same_c()
    # 9. the orientation that GrB_TRAN reads is not stored
    refused(gb, "GrB_UNINITIALIZED_OBJECT",
            lambda: gb.assign(C_, None, None, A_nocsc, I5, 5, J6, 6, dt))
    same_c()
    # 10. more than 2^31 - 1 entries: a constant region, refused before it is built
    Big = gb.Matrix(50000, 50000)
    refused(gb, "GrB_OUT_OF_MEMORY",
            lambda: gb.assign(Big, None, None, 1.0, None, 50000, None, 50000, d))
    assert Big.nvals() == 0
    same_c()
