"""k-truss and truss decomposition on the device (algorithm.ktruss / gb200_ktruss,
algorithm.trussness / gb200_trussness) against the CPU bucket peel of
tests/truss_oracle.c, entry for entry: the row offsets, the column indices and every
value.

Covered: the golden graphs; R-MAT 10-18; the closed forms (cliques, a star, a tree,
disjoint cliques, a wheel); a 2-D grid with no triangle; a clique hung off a hub, whose
intersections are split over several warps; FP32 and INT32 A and output; CSR + CSC
against a matrix marked symmetric; a directed A, symmetrised; self-loops; k = 2
against the masked mxm B<A> = A·A; a matrix with no entries and one with self-loops
only (test_sgm.mtx); ktruss(k) against {tau >= k} for every k up to
kmax + 1; cc on a truss against scipy on the oracle's truss; the output aliased to A;
two calls giving identical bytes; and every refusal, with the output untouched.
"""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_binding as orc
import truss_reference as R
from support import (Csr, components, csr, device_matrix, directed_csr, gb, make_matrix,
                     mtx_graph, symmetric_csr)

HERE = os.path.dirname(os.path.abspath(__file__))
CHUNK = 1024                           # GB_KT_CHUNK: longer shorter-lists are split


def expected(rp, ci, k=None):
    """((ptr, ind, val), count) of the oracle on the undirected pattern of (rp, ci)."""
    ptr, ind = R.undirected(rp, ci)
    vals, count = R.trussness(ptr, ind) if k is None else R.ktruss(ptr, ind, k)
    return R.kept_csr(ptr, ind, vals), count


def check_csr(M, want):
    rp, ci, val = M.extract_csr()
    assert np.array_equal(rp, want[0]), "row offsets differ"
    assert np.array_equal(ci, want[1]), "column indices differ"
    assert np.array_equal(val.astype(np.int64), want[2].astype(np.int64)), "values differ"


def out(gb, n, integer):
    return gb.Matrix(n, n, dtype=gb.api.INT32 if integer else gb.api.FP32)


def run_ktruss(gb, A, n, k, integer=True, C_=None):
    from graphblast_b200 import algorithm
    C_ = out(gb, n, integer) if C_ is None else C_
    nedges, ms = algorithm.ktruss(C_, A, k, gb.Descriptor())
    assert ms >= 0
    return C_, nedges


def run_trussness(gb, A, n, integer=True, T=None):
    from graphblast_b200 import algorithm
    T = out(gb, n, integer) if T is None else T
    kmax, ms = algorithm.trussness(T, A, gb.Descriptor())
    assert ms >= 0
    return T, kmax


def check_all(gb, A, rp, ci, ks, integer=True):
    n = len(rp) - 1
    T, kmax = run_trussness(gb, A, n, integer)
    want, want_kmax = expected(rp, ci)
    check_csr(T, want)
    assert kmax == want_kmax
    for k in ks:
        Ck, nedges = run_ktruss(gb, A, n, k, integer)
        want, want_edges = expected(rp, ci, k)
        check_csr(Ck, want)
        assert nedges == want_edges
    return kmax


def clique_edges(vertices):
    v = np.asarray(vertices)
    i, j = np.triu_indices(len(v), 1)
    return v[i], v[j]


def disjoint_cliques(sizes):
    src, dst, base = [], [], 0
    for s in sizes:
        a, b = clique_edges(np.arange(base, base + s))
        src.append(a)
        dst.append(b)
        base += s
    return symmetric_csr(base + 3, np.concatenate(src), np.concatenate(dst))


def wheel(rim):
    cyc = np.arange(1, rim + 1)
    return symmetric_csr(rim + 1, np.concatenate([np.zeros(rim, int), cyc]),
                         np.concatenate([cyc, np.roll(cyc, -1)]))


def grid2d(w, h):
    idx = np.arange(w*h).reshape(h, w)
    src = np.concatenate([idx[:, :-1].ravel(), idx[:-1, :].ravel()])
    dst = np.concatenate([idx[:, 1:].ravel(), idx[1:, :].ravel()])
    return symmetric_csr(w*h, src, dst)


def hub_clique(size=CHUNK + 100, leaves=3000):
    """A clique of `size` vertices 1..size, all joined to hub 0, which also has `leaves`
    leaves: every clique edge and every hub-clique edge has a shorter list past one
    chunk."""
    a, b = clique_edges(np.arange(1, size + 1))
    src = np.concatenate([a, np.zeros(size + leaves, int)])
    dst = np.concatenate([b, np.arange(1, size + leaves + 1)])
    return symmetric_csr(size + leaves + 1, src, dst)


def random_graph(n, m, seed, symmetric=True):
    rng = np.random.RandomState(seed)
    return (symmetric_csr if symmetric else directed_csr)(n, rng.randint(0, n, m),
                                                          rng.randint(0, n, m))


GRAPHS = {
    "chesapeake": lambda: mtx_graph("chesapeake"),
    "test_cc": lambda: mtx_graph("test_cc"),
    "test_bc": lambda: mtx_graph("test_bc"),
    "clique12": lambda: symmetric_csr(12, *clique_edges(np.arange(12))),
    "star": lambda: symmetric_csr(3001, np.zeros(3000, int), np.arange(1, 3001)),
    "tree": lambda: symmetric_csr(2000, np.random.RandomState(1).randint(0, np.arange(1, 2000)),
                                  np.arange(1, 2000)),
    "disjoint_cliques": lambda: disjoint_cliques([3, 5, 9, 4, 30]),
    "wheel": lambda: wheel(50),
    "grid": lambda: grid2d(70, 60),
    "hub_clique": hub_clique,
    "random": lambda: random_graph(3000, 40000, 2),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_graphs(gb, name):
    rp, ci = GRAPHS[name]()
    A = make_matrix(gb, rp, ci)
    _, kmax = R.trussness(rp, ci)
    assert check_all(gb, A, rp, ci, sorted({2, 3, 4, kmax, (kmax + 4)//2})) == kmax
    if name == "grid":
        assert kmax == 2
    if name == "hub_clique":
        assert kmax == CHUNK + 101


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [10, 12, 14, 16, 18])
def test_rmat(gb, scale):
    rp, ci = orc.rmat_csr(scale)
    A = make_matrix(gb, rp, ci)
    kmax = check_all(gb, A, rp, ci, [])
    for k in ([kmax] if scale == 18 else [3, max(3, kmax//2), kmax]):
        Ck, nedges = run_ktruss(gb, A, len(rp) - 1, k)
        want, want_edges = expected(rp, ci, k)
        check_csr(Ck, want)
        assert nedges == want_edges


@pytest.mark.gpu
@pytest.mark.parametrize("a_int,c_int", [(False, False), (False, True), (True, False),
                                         (True, True)])
def test_element_types(gb, a_int, c_int):
    rp, ci = orc.rmat_csr(11)
    A = make_matrix(gb, rp, ci, integer=a_int)
    check_all(gb, A, rp, ci, [4], integer=c_int)


@pytest.mark.gpu
def test_csr_and_csc_equal_the_symmetric_form(gb):
    rp, ci = orc.rmat_csr(12)
    n = len(rp) - 1
    forms = [make_matrix(gb, rp, ci), make_matrix(gb, rp, ci, symmetric=False, csc=True)]
    got = []
    for A in forms:
        T, _ = run_trussness(gb, A, n)
        Ck, _ = run_ktruss(gb, A, n, 5)
        got.append([x.tobytes() for x in T.extract_csr() + Ck.extract_csr()])
    assert got[0] == got[1]


@pytest.mark.gpu
def test_directed_a_is_symmetrised(gb):
    for rp, ci in (random_graph(2000, 30000, 3, symmetric=False), mtx_graph("chesapeake")):
        n = len(rp) - 1
        rows = np.repeat(np.arange(n), np.diff(rp))
        upper = rows < ci                      # each edge one way only
        D = csr(n, n, rows[upper], ci[upper], np.ones(int(upper.sum())), np.float32)
        A = device_matrix(gb, D, csc=True)
        check_all(gb, A, D.ptr, D.ind, [3, 4])


@pytest.mark.gpu
def test_self_loops_are_ignored(gb):
    rp, ci = orc.rmat_csr(11)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    loops = np.arange(0, n, 5)
    S = csr(n, n, np.concatenate([rows, loops]), np.concatenate([ci, loops]),
            np.ones(len(ci) + len(loops)), np.float32)
    for A in (device_matrix(gb, S, csc=True), device_matrix(gb, S, symmetric=True)):
        check_all(gb, A, S.ptr, S.ind, [3, 6])
        T, _ = run_trussness(gb, A, n)
        want, _ = expected(rp, ci)
        check_csr(T, want)


@pytest.mark.gpu
def test_k2_equals_the_masked_mxm(gb):
    import scipy.sparse as sp
    rp, ci = orc.rmat_csr(12)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, integer=True)
    B = gb.Matrix(n, n, dtype=gb.api.INT32)
    gb.mxm(B, A, None, gb.Semiring.PlusMultiplies, A, A, gb.Descriptor())
    Ck, nedges = run_ktruss(gb, A, n, 2)
    assert nedges == len(ci)//2
    c_rp, c_ci, c_v = Ck.extract_csr()
    assert np.array_equal(c_rp, rp) and np.array_equal(c_ci, ci)
    b_rp, b_ci, b_v = B.extract_csr()
    Cs = sp.csr_matrix((c_v.astype(np.int64), c_ci, c_rp), shape=(n, n))
    Bs = sp.csr_matrix((b_v.astype(np.int64), b_ci, b_rp), shape=(n, n))
    assert (Cs - Bs).count_nonzero() == 0
    Bp = sp.csr_matrix((np.ones(len(b_ci)), b_ci, b_rp), shape=(n, n))
    Cp = sp.csr_matrix((np.ones(len(c_ci)), c_ci, c_rp), shape=(n, n))
    assert (Bp - Bp.multiply(Cp)).count_nonzero() == 0     # B inside C's pattern
    assert c_v.sum() > 0


@pytest.mark.gpu
def test_ktruss_is_the_tau_level_set(gb):
    rp, ci = orc.rmat_csr(13)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    T, kmax = run_trussness(gb, A, n)
    t_rp, t_ci, tau = T.extract_csr()
    assert np.array_equal(t_rp, rp) and np.array_equal(t_ci, ci) and tau.max() == kmax
    rows = np.repeat(np.arange(n), np.diff(rp))
    for k in range(2, kmax + 2):
        Ck, nedges = run_ktruss(gb, A, n, k)
        c_rp, c_ci, c_v = Ck.extract_csr()
        keep = tau >= k
        want_rp = np.concatenate([[0], np.cumsum(np.bincount(rows[keep], minlength=n))])
        assert np.array_equal(c_rp, want_rp) and np.array_equal(c_ci, ci[keep]), "k = %d" % k
        assert nedges == keep.sum()//2 and (len(c_v) == 0 or c_v.min() >= k - 2)


@pytest.mark.gpu
def test_cc_on_a_truss(gb):
    from graphblast_b200 import algorithm
    rp, ci = orc.rmat_csr(12)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    Ck, _ = run_ktruss(gb, A, n, 8, integer=False)
    v = gb.Vector(n)
    ncomp, _ = algorithm.cc(v, Ck, gb.Descriptor())
    (w_rp, w_ci, _), _ = expected(rp, ci, 8)
    label, count = components(n, w_rp, w_ci)
    assert ncomp == count
    assert np.array_equal(v.extractTuples().astype(np.int64), label)


@pytest.mark.gpu
def test_output_aliased_to_a(gb):
    from graphblast_b200 import algorithm
    rp, ci = orc.rmat_csr(11)
    n = len(rp) - 1
    for integer in (False, True):
        A = make_matrix(gb, rp, ci, integer=integer)
        algorithm.ktruss(A, A, 5, gb.Descriptor())
        check_csr(A, expected(rp, ci, 5)[0])
        A = make_matrix(gb, rp, ci, symmetric=False, csc=True, integer=integer)
        algorithm.trussness(A, A, gb.Descriptor())
        check_csr(A, expected(rp, ci)[0])


@pytest.mark.gpu
def test_two_calls_give_identical_bytes(gb):
    rp, ci = orc.rmat_csr(14)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    T = out(gb, n, True)
    first = [x.tobytes() for x in run_trussness(gb, A, n, T=T)[0].extract_csr()]
    assert [x.tobytes() for x in run_trussness(gb, A, n, T=T)[0].extract_csr()] == first
    a = [x.tobytes() for x in run_ktruss(gb, A, n, 6)[0].extract_csr()]
    assert [x.tobytes() for x in run_ktruss(gb, A, n, 6)[0].extract_csr()] == a


@pytest.mark.gpu
def test_no_entries(gb):
    E = gb.Matrix(100, 100)
    T, kmax = run_trussness(gb, E, 100)
    assert kmax == 0 and T.nvals() == 0
    Ck, nedges = run_ktruss(gb, E, 100, 3)
    assert nedges == 0 and Ck.nvals() == 0
    # test_sgm.mtx stores self-loops only: no edge
    n, src, dst, _ = orc.read_mtx_edges(os.path.join(HERE, "golden", "test_sgm.mtx"))
    L = device_matrix(gb, csr(n, n, src, dst, np.ones(len(src)), np.float32), csc=True)
    assert L.nvals() == n
    T, kmax = run_trussness(gb, L, n)
    assert kmax == 0 and T.nvals() == 0
    Ck, nedges = run_ktruss(gb, L, n, 2)
    assert nedges == 0 and Ck.nvals() == 0


@pytest.mark.gpu
def test_refusals_in_order_leave_the_output_untouched(gb):
    import graphblast_b200 as g
    UNINIT = int(g.Info.GrB_UNINITIALIZED_OBJECT)
    DIM = int(g.Info.GrB_DIMENSION_MISMATCH)
    NOTIMPL = int(g.Info.GrB_NOT_IMPLEMENTED)
    INVAL = int(g.Info.GrB_INVALID_VALUE)
    lib = g.api._lib.load()
    rp, ci = mtx_graph("chesapeake")
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    rows = np.repeat(np.arange(n), np.diff(rp))
    upper = rows < ci                  # each edge one way: a non-symmetric A, no CSC
    D = device_matrix(gb, csr(n, n, rows[upper], ci[upper], np.ones(int(upper.sum())),
                              np.float32), csc=False)
    Rm = device_matrix(gb, Csr(n, n + 1, rp, ci, np.ones(len(ci), np.float32)))
    Dense = gb.Matrix(n, n)
    Dense.build_dense(np.ones((n, n), np.float32))
    desc = gb.Descriptor()
    Cm = make_matrix(gb, rp, ci)               # an output that holds entries already
    before = [x.copy() for x in Cm.extract_csr()]
    small = gb.Matrix(n - 1, n - 1)

    def kt(O, M, k):
        return lib.gb200_ktruss(O._h, M._h, k, desc._h, None, C.byref(C.c_float()))

    def tr(O, M):
        return lib.gb200_trussness(O._h, M._h, desc._h, None, C.byref(C.c_float()))

    cases = [
        (kt(Cm, A, 1), INVAL),
        (kt(Cm, Dense, 1), INVAL),                 # k before the matrix
        (kt(Cm, Dense, 3), NOTIMPL),
        (tr(Cm, Dense), NOTIMPL),
        (kt(small, Dense, 3), NOTIMPL),            # before the sizes
        (kt(Cm, Rm, 3), DIM),
        (tr(small, A), DIM),
        (kt(small, D, 3), DIM),                    # before the CSC
        (kt(Cm, D, 3), UNINIT),
        (tr(Cm, D), UNINIT),
    ]
    for i, (got, want) in enumerate(cases):
        assert got == want, "case %d: %d, expected %d" % (i, got, want)
    for got_, want_ in zip(Cm.extract_csr(), before):
        assert np.array_equal(got_, want_)
    # an FP32 output past 2^24 vertices; an INT32 one is fine
    big = (1 << 24) + 1
    E = gb.Matrix(big, big)
    assert tr(gb.Matrix(big, big), E) == INVAL
    assert tr(gb.Matrix(big, big, dtype=gb.api.INT32), E) == 0
    with pytest.raises(gb.api.GraphBLASError) as err:
        from graphblast_b200 import algorithm
        algorithm.ktruss(Cm, A, 0, desc)
    assert err.value.info == INVAL
