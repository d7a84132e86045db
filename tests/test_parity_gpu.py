"""GPU parity tests: the CUDA path (through the C ABI) against the oracle on the
same seeded inputs, the committed golden vectors, and size-independent
properties at larger sizes.  Integer/level/count results are compared
bit-exactly; PageRank within 1e-5 relative (BASELINE.json north_star).

Modelled on the reference's own tests: test/gvxm.cu (six vxm cases),
test/greduce.cu (row sums), and the CORRECT/INCORRECT self-checks of
example/g{bfs,sssp,pr,tc}.cu.
"""
import json
import os

import numpy as np
import pytest

import oracle_binding as orc
from support import gb, make_matrix, path_graph, ragged_graph, star_graph, transpose

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden.json")))
FLT_MAX = np.finfo(np.float32).max


def chesapeake():
    g = GOLDEN["chesapeake"]
    return (np.array(g["rowptr"], dtype=np.int32),
            np.array(g["colind"], dtype=np.int32))


def cc_graph():
    g = GOLDEN["test_cc"]
    return (np.array(g["rowptr"], dtype=np.int32),
            np.array(g["colind"], dtype=np.int32))


# ---------------------------------------------------------------------------
# vxm / mxv at operation level
# ---------------------------------------------------------------------------

def run_vxm(gb, A, n, semiring, u_dense=None, u_sparse=None, mask=None,
            scmp=False, mode=1, struconly=False, transpose_mxv=False):
    """Returns (storage, dense_values, (ind, val) or None)."""
    desc = gb.Descriptor(mxvmode=mode, struconly=1 if struconly else 0)
    u = gb.Vector(n)
    if u_sparse is not None:
        u.build(u_sparse[0], u_sparse[1])
    else:
        u.build(u_dense)
    w = gb.Vector(n)
    m = None
    if mask is not None:
        m = gb.Vector(n)
        m.build(mask)
        if scmp:
            desc.toggle(gb.Desc_field.GrB_MASK)
    if transpose_mxv:
        gb.mxv(w, m, None, semiring, A, u, desc)
    else:
        gb.vxm(w, m, None, semiring, u, A, desc)
    storage = w.getStorage()
    sparse = w.extractTuples(sparse=True) if storage == gb.Storage.GrB_SPARSE else None
    return storage, w.extractTuples(), sparse, desc.lastmxv


@pytest.mark.parametrize("mode", [1, 2])
def test_gvxm_dense_times_sparse_matrix(gb, mode):
    """test/gvxm.cu dup1: vec = 2 everywhere on test_cc, PlusMultiplies."""
    rp, ci = cc_graph()
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, symmetric=False)
    u = np.full(n, 2.0, dtype=np.float32)
    _, got, _, _ = run_vxm(gb, A, n, gb.PlusMultipliesSemiring, u_dense=u,
                           mode=mode)
    want, _ = orc.vxm(1, rp, ci, np.ones(len(ci), np.float32), u)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("mode", [1, 2])
def test_gvxm_sparse_times_sparse_matrix(gb, mode):
    """test/gvxm.cu dup3: sparse u on test_cc, PlusMultiplies."""
    rp, ci = cc_graph()
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, symmetric=False)
    ind = np.array([0, 1, 4, 6, 8, 10], dtype=np.int32)
    val = np.array([1., 2., 3., 4., 3., 10.], dtype=np.float32)
    storage, got, sparse, last = run_vxm(gb, A, n, gb.PlusMultipliesSemiring,
                                         u_sparse=(ind, val), mode=mode)
    u = np.zeros(n, np.float32)
    up = np.zeros(n, np.uint8)
    u[ind] = val
    up[ind] = 1
    want, wp = orc.vxm(1, rp, ci, np.ones(len(ci), np.float32), u, u_present=up)
    assert np.array_equal(got, want)
    if mode == 1:
        assert storage == gb.Storage.GrB_SPARSE
        assert last == gb.Desc_value.GrB_PUSHONLY
        assert np.array_equal(sparse[0], np.nonzero(wp)[0])     # sorted, unique
        assert np.array_equal(sparse[1], want[wp != 0])
    else:
        assert storage == gb.Storage.GrB_DENSE
        assert last == gb.Desc_value.GrB_PULLONLY


@pytest.mark.parametrize("scmp", [False, True])
@pytest.mark.parametrize("mode", [1, 2])
def test_gvxm_sparse_vector_dense_mask(gb, mode, scmp):
    """test/gvxm.cu dup5: sparse u + dense mask, normal and GrB_SCMP."""
    rp, ci = cc_graph()
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, symmetric=False)
    ind = np.array([0, 1, 4, 6, 8, 10], dtype=np.int32)
    val = np.array([1., 2., 3., 4., 3., 10.], dtype=np.float32)
    mask = np.array([1., 0., 0., 1., 0., 1., 1., 1., 1., 1., 0.], np.float32)
    _, got, _, _ = run_vxm(gb, A, n, gb.PlusMultipliesSemiring,
                           u_sparse=(ind, val), mask=mask, scmp=scmp, mode=mode)
    u = np.zeros(n, np.float32)
    up = np.zeros(n, np.uint8)
    u[ind] = val
    up[ind] = 1
    want, _ = orc.vxm(1, rp, ci, np.ones(len(ci), np.float32), u, u_present=up,
                      mask=mask, scmp=scmp)
    assert np.array_equal(got, want)


WELL_DEFINED = ["LogicalOrAnd", "PlusMultiplies", "MinimumPlus",
                "MaximumMultiplies", "PlusDivides", "PlusGreater", "PlusMinus",
                "PlusLess", "MinimumMultiplies", "MinimumSelectSecond",
                "PlusNotEqualTo", "MinimumNotEqualTo"]


@pytest.mark.parametrize("name", WELL_DEFINED)
@pytest.mark.parametrize("graph", ["rmat10", "star", "ragged"])
def test_semiring_sweep_push_and_pull(gb, name, graph):
    """Every semiring whose additive op is a commutative, associative monoid:
    push (sparse u) and pull (dense u) against the oracle, bit-exact (values are
    small integers / powers of two so float sums are order-independent)."""
    if graph == "rmat10":
        rp, ci = orc.rmat_csr(10)
    elif graph == "star":
        rp, ci = star_graph(5000)
    else:
        rp, ci = ragged_graph()
    n = len(rp) - 1
    rng = np.random.RandomState(11)
    val = (2.0 ** rng.randint(0, 3, len(ci))).astype(np.float32)     # 1,2,4
    A = make_matrix(gb, rp, ci, val, symmetric=False)
    sem = getattr(gb.Semiring, name)
    ident = orc.identity(int(sem))

    # pull: dense u, every entry participates
    u = (2.0 ** rng.randint(0, 2, n)).astype(np.float32)             # 1,2
    _, got, _, last = run_vxm(gb, A, n, sem, u_dense=u, mode=2)
    want, wp = orc.vxm(int(sem), rp, ci, val, u)
    assert last == gb.Desc_value.GrB_PULLONLY
    assert np.array_equal(got, want), name

    # push: sparse frontier of ~5% of the vertices (plus vertex 0 for the star)
    f_ind = np.unique(np.concatenate([[0], rng.randint(0, n, n // 20)])).astype(np.int32)
    f_val = (2.0 ** rng.randint(0, 2, len(f_ind))).astype(np.float32)
    storage, _, sparse, last = run_vxm(gb, A, n, sem, u_sparse=(f_ind, f_val),
                                       mode=1)
    up = np.zeros(n, np.uint8)
    uu = np.full(n, ident, np.float32)
    up[f_ind] = 1
    uu[f_ind] = f_val
    want, wp = orc.vxm(int(sem), rp, ci, val, uu, u_present=up)
    assert storage == gb.Storage.GrB_SPARSE and last == gb.Desc_value.GrB_PUSHONLY
    assert np.array_equal(sparse[0], np.nonzero(wp)[0]), name
    assert np.array_equal(sparse[1], want[wp != 0]), name


def test_mxv_matches_vxm_on_transpose(gb):
    """mxv(A, u) = vxm(u, A^T): directed graph, both directions."""
    rng = np.random.RandomState(3)
    n = 700
    src = rng.randint(0, n, 6000).astype(np.int32)
    dst = rng.randint(0, n, 6000).astype(np.int32)
    rp, ci = orc.build_csr(n, src, dst, undirected=False)
    val = rng.randint(1, 5, len(ci)).astype(np.float32)
    A = make_matrix(gb, rp, ci, val, symmetric=False)
    t_rp, t_ci, order = transpose(rp, ci)
    t_val = val[order]
    u = rng.randint(1, 4, n).astype(np.float32)
    for mode in (1, 2):
        _, got, _, _ = run_vxm(gb, A, n, gb.PlusMultipliesSemiring, u_dense=u,
                               mode=mode, transpose_mxv=True)
        want, _ = orc.vxm(1, t_rp, t_ci, t_val, u)        # u^T A^T
        assert np.array_equal(got, want)


def test_vxm_empty_frontier_is_uninitialized_object(gb):
    """reference graphblas/operations.hpp:71-74: u.nvals()==0 ->
    GrB_UNINITIALIZED_OBJECT."""
    rp, ci = cc_graph()
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, symmetric=False)
    u = gb.Vector(n)
    u.build(np.zeros(0, np.int32), np.zeros(0, np.float32))
    w = gb.Vector(n)
    with pytest.raises(gb.GraphBLASError) as e:
        gb.vxm(w, None, None, gb.LogicalOrAndSemiring, u, A, gb.Descriptor())
    assert e.value.info == gb.Info.GrB_UNINITIALIZED_OBJECT


def test_vxm_dimension_mismatch(gb):
    rp, ci = cc_graph()
    A = make_matrix(gb, rp, ci, symmetric=False)
    u = gb.Vector(7)
    u.fill(1.0)
    w = gb.Vector(len(rp) - 1)
    with pytest.raises(gb.GraphBLASError) as e:
        gb.vxm(w, None, None, gb.PlusMultipliesSemiring, u, A, gb.Descriptor())
    assert e.value.info == gb.Info.GrB_DIMENSION_MISMATCH


def test_reduce_rows_and_scalars(gb):
    """test/greduce.cu:63-75 row sums of test_cc, plus scalar reductions."""
    rp, ci = cc_graph()
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, symmetric=False)
    desc = gb.Descriptor()
    w = gb.Vector(n)
    gb.reduce(None, gb.PlusMonoid, A, desc, out=w)
    assert w.extractTuples().tolist() == [1, 1, 3, 2, 2, 3, 3, 0, 1, 2, 2]
    assert gb.reduce(None, gb.PlusMonoid, A, desc) == len(ci)
    v = gb.Vector(n)
    v.build(np.arange(1, n + 1, dtype=np.float32))
    assert gb.reduce(None, gb.PlusMonoid, v, desc) == n * (n + 1) / 2
    assert gb.reduce(None, gb.MinimumMonoid, v, desc) == 1
    assert gb.reduce(None, gb.MaximumMonoid, v, desc) == n


def test_vector_storage_rules_and_conversions(gb):
    """SURVEY.md §8a storage rules: fill -> dense, build(ind,val) -> sparse, swap
    needs equal storage, extractTuples(values) densifies with 0."""
    n = 100
    desc = gb.Descriptor()
    a = gb.Vector(n)
    a.fill(0.0)
    assert a.getStorage() == gb.Storage.GrB_DENSE and a.nvals() == n
    b = gb.Vector(n)
    b.build(np.array([3, 50, 99], np.int32), np.array([7, 8, 9], np.float32))
    assert b.getStorage() == gb.Storage.GrB_SPARSE and b.nvals() == 3
    with pytest.raises(gb.GraphBLASError) as e:
        a.swap(b)
    assert e.value.info == gb.Info.GrB_INVALID_OBJECT
    dense = b.extractTuples()
    assert dense[3] == 7 and dense[50] == 8 and dense[99] == 9 and dense.sum() == 24
    c = gb.Vector(n)
    vals = np.zeros(n, np.float32)
    vals[[5, 64, 65, 97]] = [1, 2, 3, 4]
    c.build(vals)
    c.dense2sparse(0.0, desc)
    ind, val = c.extractTuples(sparse=True)
    assert ind.tolist() == [5, 64, 65, 97] and val.tolist() == [1, 2, 3, 4]
    c.sparse2dense(0.0, desc)
    assert np.array_equal(c.extractTuples(), vals)
    with pytest.raises(gb.GraphBLASError) as e:
        b.build(np.array([1], np.int32), np.array([1], np.float32))
    assert e.value.info == gb.Info.GrB_OUTPUT_NOT_EMPTY


def test_elementwise_and_assign_semantics(gb):
    """The variants the SSSP / PageRank loops use (SURVEY.md §8a quirks)."""
    n = 64
    desc = gb.Descriptor()
    rng = np.random.RandomState(2)
    x = rng.randint(0, 5, n).astype(np.float32)
    y = rng.randint(0, 5, n).astype(np.float32)
    vx, vy, w = gb.Vector(n), gb.Vector(n), gb.Vector(n)
    vx.build(x)
    vy.build(y)
    gb.eWiseAdd(w, None, None, gb.PlusMultipliesSemiring, vx, vy, desc)
    assert np.array_equal(w.extractTuples(), x + y)
    gb.eWiseAdd(w, None, None, gb.CustomLessPlusSemiring, vx, vy, desc)
    assert np.array_equal(w.extractTuples(), (x < y).astype(np.float32))
    gb.eWiseAdd(w, None, None, gb.MultipliesMultipliesSemiring, vx, vx, desc)
    assert np.array_equal(w.extractTuples(), x * x)
    gb.eWiseAdd(w, None, None, gb.PlusMultipliesSemiring, vx, 0.25, desc)
    assert np.array_equal(w.extractTuples(), x + np.float32(0.25))
    # dense-dense eWiseMult short-circuits on the identity (kernels/ewisemult.hpp:22-25)
    gb.eWiseMult(w, None, None, gb.PlusMinusSemiring, vx, vy, desc)
    want = np.where((x == 0) | (y == 0), 0, x - y).astype(np.float32)
    assert np.array_equal(w.extractTuples(), want)
    # sparse (+) dense: every element first becomes op(v, identity)
    s = gb.Vector(n)
    s_ind = np.array([1, 9, 33], np.int32)
    s_val = np.array([0.5, 7.0, 1.0], np.float32)
    s.build(s_ind, s_val)
    dist = np.full(n, FLT_MAX, np.float32)
    dist[[1, 2, 9]] = [3.0, 4.0, 6.0]
    vd = gb.Vector(n)
    vd.build(dist)
    m = gb.Vector(n)
    gb.eWiseAdd(m, None, None, gb.CustomLessPlusSemiring, s, vd, desc)
    want = (dist < FLT_MAX).astype(np.float32)
    want[s_ind] = (s_val < dist[s_ind]).astype(np.float32)
    assert np.array_equal(m.extractTuples(), want)
    # in-place min with a sparse operand
    gb.eWiseAdd(vd, None, None, gb.MinimumPlusSemiring, vd, s, desc)
    want = dist.copy()
    want[s_ind] = np.minimum(s_val, dist[s_ind])
    assert np.array_equal(vd.extractTuples(), want)
    # masked constant assign on a sparse vector == masked delete under GrB_SCMP
    keep = np.zeros(n, np.float32)
    keep[[1, 33]] = 1
    mk = gb.Vector(n)
    mk.build(keep)
    desc.toggle(gb.Desc_field.GrB_MASK)
    gb.assign(s, mk, None, FLT_MAX, None, n, desc)
    desc.toggle(gb.Desc_field.GrB_MASK)
    ind, val = s.extractTuples(sparse=True)
    assert ind.tolist() == [1, 33] and val.tolist() == [0.5, 1.0]
    # dense target, sparse mask
    t = gb.Vector(n)
    t.fill(0.0)
    f = gb.Vector(n)
    f.build(np.array([2, 40], np.int32), np.array([1, 1], np.float32))
    gb.assign(t, f, None, 5.0, None, n, desc)
    want = np.zeros(n, np.float32)
    want[[2, 40]] = 5
    assert np.array_equal(t.extractTuples(), want)


# ---------------------------------------------------------------------------
# Algorithms
# ---------------------------------------------------------------------------

BFS_FLAGS = [dict(), dict(struconly=1, opreuse=1, earlyexit=1),
             dict(struconly=1), dict(earlyexit=0, fusedmask=0)]


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("flags", BFS_FLAGS)
def test_bfs_chesapeake_golden(gb, mode, flags):
    from graphblast_b200 import algorithm
    rp, ci = chesapeake()
    A = make_matrix(gb, rp, ci)
    desc = gb.Descriptor(mxvmode=mode, **flags)
    v = gb.Vector(len(rp) - 1)
    algorithm.bfs(v, A, 0, desc)
    assert v.extractTuples().astype(np.int32).tolist() == \
        GOLDEN["chesapeake"]["bfs_levels_src0"]


def test_bfs_through_reference_loader(gb):
    """readMtx -> Matrix::build -> bfs, the path example/gbfs.cu takes."""
    from graphblast_b200 import algorithm
    A = gb.Matrix.from_mtx(os.path.join(HERE, "golden", "chesapeake.mtx"),
                           directed=2)
    rp, ci, _ = A.extract_csr()
    g = GOLDEN["chesapeake"]
    assert rp.tolist() == g["rowptr"] and ci.tolist() == g["colind"]
    v = gb.Vector(A.nrows())
    algorithm.bfs(v, A, 0, gb.Descriptor(mxvmode=0, struconly=1, opreuse=1))
    assert v.extractTuples().astype(np.int32).tolist() == g["bfs_levels_src0"]


GRAPHS = {
    "rmat10": lambda: orc.rmat_csr(10),
    "rmat14": lambda: orc.rmat_csr(14),
    "star": lambda: star_graph(20000),
    "path": lambda: path_graph(300),
    "ragged": ragged_graph,
}


@pytest.mark.parametrize("graph", sorted(GRAPHS))
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_bfs_matches_oracle(gb, graph, mode):
    from graphblast_b200 import algorithm
    rp, ci = GRAPHS[graph]()
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    deg = np.diff(rp)
    sources = {0, int(np.argmax(deg)), int(np.argmin(deg))}
    for flags in (dict(struconly=1, opreuse=1, earlyexit=1), dict()):
        desc = gb.Descriptor(mxvmode=mode, **flags)
        for s in sources:
            v = gb.Vector(n)
            algorithm.bfs(v, A, s, desc)
            got = v.extractTuples().astype(np.int32)
            assert np.array_equal(got, orc.bfs(rp, ci, s)), (graph, mode, s)


def test_bfs_rmat10_golden_histogram(gb):
    from graphblast_b200 import algorithm
    rp, ci = orc.rmat_csr(10)
    A = make_matrix(gb, rp, ci)
    v = gb.Vector(len(rp) - 1)
    algorithm.bfs(v, A, 0, gb.Descriptor(mxvmode=0, struconly=1, opreuse=1))
    hist = np.bincount(v.extractTuples().astype(np.int64)).tolist()
    assert hist == GOLDEN["rmat10"]["bfs_level_hist_src0"]


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_sssp_chesapeake_golden(gb, mode):
    from graphblast_b200 import algorithm
    g = GOLDEN["chesapeake"]
    rp, ci = chesapeake()
    w = np.array(g["sssp_weights_seed1"], dtype=np.float32)
    A = make_matrix(gb, rp, ci, w, symmetric=False)
    d = gb.Vector(len(rp) - 1)
    algorithm.sssp(d, A, 0, gb.Descriptor(mxvmode=mode))
    assert d.extractTuples().tolist() == g["sssp_dist_src0"]


def test_sssp_reference_weight_path(gb):
    """apply(set_uniform_random) in CSR order, as example/gsssp.cu:75-84."""
    from graphblast_b200 import algorithm
    A = gb.Matrix.from_mtx(os.path.join(HERE, "golden", "chesapeake.mtx"),
                           directed=2)
    desc = gb.Descriptor(mxvmode=0)
    A.apply_uniform_random(desc, seed=1, lo=1, hi=64)
    rp, ci, w = A.extract_csr()
    g = GOLDEN["chesapeake"]
    assert w.tolist() == g["sssp_weights_seed1"]
    d = gb.Vector(A.nrows())
    algorithm.sssp(d, A, 0, desc)
    assert d.extractTuples().tolist() == g["sssp_dist_src0"]


@pytest.mark.parametrize("graph", ["rmat10", "rmat14", "star", "path", "ragged"])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_sssp_matches_oracle(gb, graph, mode):
    from graphblast_b200 import algorithm
    import graphblast_b200 as g
    rp, ci = GRAPHS[graph]()
    n = len(rp) - 1
    w = g.api.host_uniform_weights(1, 1, 64, len(ci))
    A = make_matrix(gb, rp, ci, w, symmetric=False)
    s = int(np.argmax(np.diff(rp)))
    d = gb.Vector(n)
    desc = gb.Descriptor(mxvmode=mode, switchpoint=0.025)
    algorithm.sssp(d, A, s, desc)
    assert np.array_equal(d.extractTuples(), orc.sssp(rp, ci, w, s)), (graph, mode)


def test_sssp_rmat10_golden_checksum(gb):
    from graphblast_b200 import algorithm
    import graphblast_b200 as g
    rp, ci = orc.rmat_csr(10)
    w = g.api.host_uniform_weights(1, 1, 64, len(ci))
    A = make_matrix(gb, rp, ci, w, symmetric=False)
    d = gb.Vector(len(rp) - 1)
    algorithm.sssp(d, A, 0, gb.Descriptor(mxvmode=0))
    got = d.extractTuples()
    finite = got[got < FLT_MAX]
    assert len(finite) == GOLDEN["rmat10"]["sssp_reached_src0"]
    assert float(finite.astype(np.float64).sum()) == GOLDEN["rmat10"]["sssp_sum_finite_src0"]


@pytest.mark.parametrize("graph", ["chesapeake", "rmat10", "rmat14"])
def test_pagerank_within_tolerance(gb, graph):
    """10 power iterations, alpha 0.85 (run_pr.sh recipe); 1e-5 relative."""
    from graphblast_b200 import algorithm
    rp, ci = chesapeake() if graph == "chesapeake" else GRAPHS[graph]()
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, np.ones(len(ci), np.float32), symmetric=False)
    desc = gb.Descriptor(mxvmode=0, max_niter=10)
    A.pr_normalize(0.85, desc)
    p = gb.Vector(n)
    # eps = 0 on both sides: exactly 10 iterations.  (With eps > 0 the two stop
    # rules differ — the reference CPU code tests sum(diff^2) < eps, the GraphBLAS
    # loop sqrt(sum) <= eps, test_pr.hpp:66 vs pr.hpp:79-80 — and small graphs
    # would stop after different iteration counts.)
    algorithm.pr(p, A, 0.85, 0.0, desc)
    got = p.extractTuples().astype(np.float64)
    want = orc.pr(rp, ci, 0.85, 0.0, 10).astype(np.float64)
    # isolated vertices: the oracle divides by a zero out-degree but never uses
    # the quotient; both sides keep the teleport term only
    rel = np.abs(got - want) / np.maximum(np.abs(want), 1e-30)
    assert rel.max() < 1e-5, rel.max()
    if graph == "chesapeake":
        # golden vector: reference CPU code with eps 1e-8 also runs all 10 here
        gold = np.array(GOLDEN["chesapeake"]["pagerank_a085_it10"])
        assert (np.abs(got - gold) / gold).max() < 1e-5


@pytest.mark.parametrize("graph", ["chesapeake", "rmat10", "rmat14", "star"])
def test_triangle_count_exact(gb, graph):
    from graphblast_b200 import algorithm
    rp, ci = chesapeake() if graph == "chesapeake" else GRAPHS[graph]()
    n = len(rp) - 1
    lr, lc = orc.tril(rp, ci)
    L = make_matrix(gb, lr, lc, np.ones(len(lc), np.int32), symmetric=False,
                    integer=True)
    B = gb.Matrix(n, n, dtype=gb.api.INT32)
    desc = gb.Descriptor(mxvmode=0)
    ntris, _ = algorithm.tc(L, B, desc)
    assert ntris == orc.tc(lr, lc)
    # B = (L * L^T) .* L entry by entry, not only its sum
    ones = np.ones(len(lc), np.int32)
    want = orc.mxm_masked(lr, lc, ones, lr, lc, ones, lr, lc, ones)
    assert int(want.sum()) == ntris
    b_rp, b_ci, b_val = B.extract_csr()
    assert np.array_equal(b_rp, lr) and np.array_equal(b_ci, lc)
    assert np.array_equal(b_val.astype(np.int64), want)
    ntris2, _ = algorithm.tc(L, B, desc)          # second call reuses B
    assert ntris2 == ntris
    assert np.array_equal(B.extract_csr()[2].astype(np.int64), want)
    if graph == "chesapeake":
        assert ntris == 194
    if graph == "rmat10":
        assert ntris == GOLDEN["rmat10"]["triangles_tril"]


def test_triangle_count_through_reference_loader_and_tril(gb):
    from graphblast_b200 import algorithm
    L = gb.Matrix.from_mtx(os.path.join(HERE, "golden", "chesapeake.mtx"),
                           directed=2, dtype=gb.api.INT32)
    desc = gb.Descriptor(mxvmode=0)
    L.tril(desc)
    assert L.nvals() == 170
    B = gb.Matrix(L.nrows(), L.nrows(), dtype=gb.api.INT32)
    assert algorithm.tc(L, B, desc)[0] == 194


# ---------------------------------------------------------------------------
# Larger sizes: device ingest + size-independent properties
# ---------------------------------------------------------------------------

def test_device_rmat_and_csr_build_match_oracle(gb):
    from graphblast_b200 import graphs
    scale = 12
    src, dst = graphs.rmat_edges(scale, 16, seed=1)
    osrc, odst = orc.rmat_edges(scale, 16, 1)
    assert np.array_equal(src.cpu().numpy(), osrc)
    assert np.array_equal(dst.cpu().numpy(), odst)
    rp, ci = graphs.build_csr(1 << scale, src, dst, undirected=True)
    orp, oci = orc.build_csr(1 << scale, osrc, odst, True)
    assert np.array_equal(rp.cpu().numpy(), orp)
    assert np.array_equal(ci.cpu().numpy(), oci)


def test_scale20_direction_modes_agree_and_match_oracle(gb):
    """RMAT-20 (1M vertices, ~31M stored entries): push-only, pull-only and
    direction-optimised BFS give identical levels, equal to the oracle's; SSSP
    push-pull equals pull-only (idempotent min) and the oracle."""
    from graphblast_b200 import algorithm, graphs
    import torch
    scale = 20
    n = 1 << scale
    src, dst = graphs.rmat_edges(scale, 16, seed=1)
    rp, ci = graphs.build_csr(n, src, dst, undirected=True)
    del src, dst
    A = graphs.matrix_from_csr(n, rp, ci)
    h_rp, h_ci = rp.cpu().numpy(), ci.cpu().numpy()
    s = int(np.argmax(np.diff(h_rp)))
    want = orc.bfs(h_rp, h_ci, s)
    for mode in (0, 1, 2):
        v = gb.Vector(n)
        algorithm.bfs(v, A, s, gb.Descriptor(mxvmode=mode, struconly=1,
                                             opreuse=1, earlyexit=1))
        got = v.extractTuples().astype(np.int32)
        assert np.array_equal(got, want), mode
    # level structure property: levels of adjacent vertices differ by at most 1
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(h_rp))
    lv = want.astype(np.int64)
    reached = lv[rows] > 0
    assert np.all(np.abs(lv[rows][reached] - lv[h_ci][reached]) <= 1)

    import graphblast_b200 as g
    w = g.api.host_uniform_weights(1, 1, 64, len(h_ci))
    d_w = torch.from_numpy(w).cuda()
    d_wt = graphs.transpose_values(n, rp, ci, d_w)
    Aw = graphs.matrix_from_csr(n, rp, ci, d_w, cscval=d_wt)
    want_d = orc.sssp(h_rp, h_ci, w, s)
    for mode in (0, 2):
        d = gb.Vector(n)
        algorithm.sssp(d, Aw, s, gb.Descriptor(mxvmode=mode, switchpoint=0.025))
        assert np.array_equal(d.extractTuples(), want_d), mode
