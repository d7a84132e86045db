"""Connected components on the device (algorithm::cc, gb200_cc) against a checker
written here, entry for entry.

The result depends only on A's pattern: v[i] is the smallest vertex id in the weakly
connected component of i, and the count is the number of components.  So every entry
and the count are compared exactly.  The checker is scipy's weak components, each
label mapped to its component's minimum id; a second check, without scipy, asks that
every stored entry joins equal labels and that label[label[i]] == label[i] <= i.

The graphs cover the kernel's phases and classes: the two neighbour rounds and the
finish, lists a lane, a warp and the grid pass take, the sampled component that a
symmetric matrix skips and the non-symmetric matrix that must not skip it, long chains
for link and compress, a hub that 150 000 CASs contend on, many small components,
stored zeros, self-loops, and the refusals.
"""
import os
import subprocess

import numpy as np
import pytest

import oracle_binding as orc
from support import (check_structure, components, directed_csr, gb, launches_per_call,
                     make_matrix, mtx_graph, symmetric_csr)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")


# ---------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------

def run_cc(gb, A, n, v=None):
    from graphblast_b200 import algorithm
    v = gb.Vector(n) if v is None else v
    k, ms = algorithm.cc(v, A, gb.Descriptor())
    assert ms >= 0
    assert v.getStorage() == gb.Storage.GrB_DENSE
    got = v.extractTuples()
    assert np.array_equal(got, np.round(got)), "a label that is not an id"
    return got.astype(np.int64), k


def check(gb, A, rp, ci):
    """The device labels and count of A (whose pattern is rp, ci) equal the checker's."""
    n = len(rp) - 1
    got, k = run_cc(gb, A, n)
    want, want_k = components(n, rp, ci)
    assert np.array_equal(got, want)
    assert k == want_k == int(np.count_nonzero(want == np.arange(n)))
    check_structure(rp, ci, got)
    return got, k


# ---------------------------------------------------------------------------
# golden graphs and small cases
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["chesapeake", "test_cc", "test_bc", "test_sgm"])
def test_golden_graphs(gb, name):
    rp, ci = mtx_graph(name)
    if len(ci) == 0:              # test_sgm holds only self-loops: keep them
        n = len(rp) - 1
        rp, ci = np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32)
        got, k = check(gb, make_matrix(gb, rp, ci), rp, ci)
        assert k == n and np.array_equal(got, np.arange(n))
        return
    check(gb, make_matrix(gb, rp, ci), rp, ci)
    check(gb, make_matrix(gb, rp, ci, symmetric=False, csc=False), rp, ci)


@pytest.mark.parametrize("directed", [0, 1, 2])
def test_cc_mtx_known_answer(gb, directed):
    """test_cc.mtx has two components: vertices 0-6 and 7-10."""
    A = gb.Matrix.from_mtx(os.path.join(GOLDEN, "test_cc.mtx"), directed=directed)
    got, k = run_cc(gb, A, A.nrows())
    assert got.tolist() == [0]*7 + [7]*4 and k == 2


def test_chesapeake_is_one_component(gb):
    A = gb.Matrix.from_mtx(os.path.join(GOLDEN, "chesapeake.mtx"), directed=2)
    got, k = run_cc(gb, A, A.nrows())
    assert k == 1 and not got.any()


def test_no_stored_entries_and_one_vertex(gb):
    for n in (1, 5, 1000, 100003):
        got, k = run_cc(gb, gb.Matrix(n, n), n)
        assert np.array_equal(got, np.arange(n)) and k == n
    B = make_matrix(gb, np.array([0, 1], np.int32), np.array([0], np.int32))   # a loop
    got, k = run_cc(gb, B, 1)
    assert got.tolist() == [0] and k == 1


def test_self_loops_are_ignored(gb):
    rp, ci = orc.rmat_csr(10)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    loops = np.arange(0, n, 3)
    r = np.concatenate([rows, loops])
    c = np.concatenate([ci, loops])
    order = np.lexsort((c, r))
    r, c = r[order], c[order]
    lrp = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=n))]).astype(np.int32)
    got, _ = check(gb, make_matrix(gb, lrp, c.astype(np.int32)), lrp, c)
    assert np.array_equal(got, components(n, rp, ci)[0])


def test_no_rows_and_no_device_csr_through_the_backend(tmp_path):
    """Two cases the C ABI cannot build, run through the headers.  n = 0 (the C ABI
    makes no vector of size 0): success and count 0, on Vector<int> through
    backend::ccRun and Vector<float> through algorithm::cc.  An A with stored entries
    but no device CSR (the C ABI uploads every CSR it builds):
    GrB_UNINITIALIZED_OBJECT, with v's storage untouched and nothing allocated."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    src = tmp_path / "cc_n0.cu"
    src.write_text(
        "#define GRB_USE_CUDA\n"
        "#include <cstdio>\n"
        "#include \"graphblas/graphblas.hpp\"\n"
        "#include \"graphblas/algorithm/cc.hpp\"\n"
        "bool debug_;\nbool memory_;\n"
        "int main() {\n"
        "  graphblas::Matrix<float> A(0, 0);\n"
        "  graphblas::Matrix<int> B(0, 0);\n"
        "  graphblas::Vector<int> v(0);\n"
        "  graphblas::Vector<float> w(0);\n"
        "  graphblas::Descriptor desc;\n"
        "  int k = -1, m = -1;\n"
        "  float ms = -1.f;\n"
        "  const graphblas::Info info =\n"
        "      graphblas::backend::ccRun(&v.vector_, &A.matrix_, &k, &ms);\n"
        "  const float t = graphblas::algorithm::cc(&w, &B, &desc, &m);\n"
        "  graphblas::Matrix<float> U(4, 4);\n"
        "  U.matrix_.sparse_.setNvals(5);\n"
        "  graphblas::Vector<int> u(4);\n"
        "  int ku = -1;\n"
        "  const graphblas::Info refused =\n"
        "      graphblas::backend::ccRun(&u.vector_, &U.matrix_, &ku);\n"
        "  std::printf(\"%d %d %d %d %d %d %d %d %d\\n\", static_cast<int>(info), k,\n"
        "              ms >= 0.f, m, t >= 0.f,\n"
        "              refused == graphblas::GrB_UNINITIALIZED_OBJECT, ku,\n"
        "              u.vector_.vec_type_ == graphblas::GrB_UNKNOWN,\n"
        "              u.vector_.dense_.d_val_ == NULL);\n"
        "  return 0;\n}\n")
    exe = tmp_path / "cc_n0"
    out = subprocess.run(
        [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-w",
         "-I", os.path.join(ROOT, "include"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc", "shim"),
         str(src), "-o", str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0, run.stderr[-2000:]
    assert run.stdout.split() == ["0", "0", "1", "0", "1", "1", "-1", "1", "1"], run.stdout


# ---------------------------------------------------------------------------
# long chains, contention, many components
# ---------------------------------------------------------------------------

def path_order(kind, n):
    if kind == "increasing":
        return np.arange(n, dtype=np.int32)
    if kind == "decreasing":
        return np.arange(n - 1, -1, -1, dtype=np.int32)
    return np.random.RandomState(7).permutation(n).astype(np.int32)


@pytest.mark.parametrize("kind", ["increasing", "decreasing", "permuted"])
def test_long_path(gb, kind):
    """10^6 vertices in one path, stored both ways (symmetric) and one way only."""
    n = 1000000
    p = path_order(kind, n)
    rp, ci = symmetric_csr(n, p[:-1], p[1:])
    got, k = check(gb, make_matrix(gb, rp, ci), rp, ci)
    assert k == 1 and not got.any()
    drp, dci = directed_csr(n, p[:-1], p[1:])
    got, k = check(gb, make_matrix(gb, drp, dci, symmetric=False, csc=False), drp, dci)
    assert k == 1 and not got.any()


def test_star_with_the_hub_last(gb):
    """150 000 leaves whose only neighbour is the hub, id n - 1: every leaf's first
    link contends on the hub's word."""
    leaves = 150000
    n = leaves + 1
    hub = np.full(leaves, n - 1, np.int32)
    leaf = np.arange(leaves, dtype=np.int32)
    rp, ci = symmetric_csr(n, hub, leaf)
    got, k = check(gb, make_matrix(gb, rp, ci), rp, ci)
    assert k == 1 and not got.any()
    drp, dci = directed_csr(n, leaf, hub)              # one way, leaf -> hub
    got, k = check(gb, make_matrix(gb, drp, dci, symmetric=False, csc=False), drp, dci)
    assert k == 1 and not got.any()
    drp, dci = directed_csr(n, hub, leaf)              # one way, hub -> leaf: one warp list
    check(gb, make_matrix(gb, drp, dci, symmetric=False, csc=False), drp, dci)


def test_disjoint_edges_and_triangles(gb):
    """50 000 edges and 50 000 triangles, ids interleaved across the range: 100 000
    components, and one sample finds no large one."""
    ne, nt = 50000, 50000
    n = 2*ne + 3*nt
    perm = np.random.RandomState(3).permutation(n).astype(np.int32)
    e = perm[:2*ne].reshape(ne, 2)
    t = perm[2*ne:].reshape(nt, 3)
    src = np.concatenate([e[:, 0], t[:, 0], t[:, 1], t[:, 2]])
    dst = np.concatenate([e[:, 1], t[:, 1], t[:, 2], t[:, 0]])
    rp, ci = symmetric_csr(n, src, dst)
    _, k = check(gb, make_matrix(gb, rp, ci), rp, ci)
    assert k == ne + nt
    drp, dci = directed_csr(n, src, dst)
    check(gb, make_matrix(gb, drp, dci, symmetric=False, csc=False), drp, dci)


def random_component(rng, ids, extra):
    """A random spanning tree over ids plus `extra` random edges inside them."""
    ids = rng.permutation(ids)
    parents = ids[rng.randint(0, np.arange(1, len(ids)))]
    src = np.concatenate([ids[1:], rng.choice(ids, extra)])
    dst = np.concatenate([parents, rng.choice(ids, extra)])
    return src, dst


def test_two_equal_components(gb):
    """Even and odd ids form two components of 100 000 vertices each, so the sample
    ties; neither may be lost whichever root it picks."""
    n = 200000
    rng = np.random.RandomState(12)
    s0, d0 = random_component(rng, np.arange(0, n, 2), 300000)
    s1, d1 = random_component(rng, np.arange(1, n, 2), 300000)
    src, dst = np.concatenate([s0, s1]), np.concatenate([d0, d1])
    rp, ci = symmetric_csr(n, src, dst)
    got, k = check(gb, make_matrix(gb, rp, ci), rp, ci)
    assert k == 2 and np.array_equal(got, np.arange(n) % 2)


def test_largest_component_without_vertex_zero(gb):
    """Vertices 0..999 are small components (pairs); the rest is one large component,
    the one the sample picks, whose minimum is 1000."""
    n = 300000
    rng = np.random.RandomState(13)
    s0 = np.arange(0, 1000, 2)
    s1, d1 = random_component(rng, np.arange(1000, n), 600000)
    src, dst = np.concatenate([s0, s1]), np.concatenate([s0 + 1, d1])
    rp, ci = symmetric_csr(n, src, dst)
    got, k = check(gb, make_matrix(gb, rp, ci), rp, ci)
    assert k == 501 and np.all(got[1000:] == 1000)


@pytest.mark.parametrize("scale", [16, 18])
def test_rmat(gb, scale):
    """A giant component, lists far longer than a warp, and isolated vertices."""
    rp, ci = orc.rmat_csr(scale)
    n = len(rp) - 1
    assert np.diff(rp).max() > 5000 and np.count_nonzero(np.diff(rp) == 0) > 0
    got, k = check(gb, make_matrix(gb, rp, ci), rp, ci)
    assert k > 1 and np.count_nonzero(got == 0) > n//2
    got2, k2 = check(gb, make_matrix(gb, rp, ci, symmetric=False, csc=False),
                     rp, ci)                                    # the same graph, no skip
    assert np.array_equal(got, got2) and k == k2


def test_non_symmetric_matrix_never_skips(gb):
    """The skip is sound only for a symmetric A.  Here the large component is a path
    0..N-1 stored both ways, which the neighbour rounds join into one tree, so the
    sample picks its root and every path vertex reads it.  Rows 0, 7 and 5 also hold
    one-way entries, at positions 2 and later, to vertices whose own rows are empty:
    row 0 a list for the grid pass (1 999 entries), row 7 a warp's (100), row 5 a
    lane's (10).  Only the finish of those rows can join these vertices, so a
    non-symmetric A that took the skip would leave them as singletons."""
    N = 100000
    path = np.arange(N - 1, dtype=np.int32)
    sizes = ((0, 2000), (7, 100), (5, 10))             # row, one-way targets
    src, dst = [path, path + 1], [path + 1, path]
    first = N
    for row, m in sizes:
        src.append(np.full(m, row, np.int32))
        dst.append(np.arange(first, first + m, dtype=np.int32))
        first += m
    n = first + 5                                      # and 5 isolated vertices
    src, dst = np.concatenate(src), np.concatenate(dst)
    drp, dci = directed_csr(n, src, dst)
    first = N
    for row, m in sizes:
        r = dci[drp[row]:drp[row + 1]]
        assert r[0] == row - 1 if row else r[0] == 1
        assert r[2:].tolist() == list(range(first + (1 if row == 0 else 0), first + m))
        first += m
    assert drp[N + 1] - drp[N] == 0
    want = np.concatenate([np.zeros(first, np.int64), np.arange(first, n)])
    for A in (make_matrix(gb, drp, dci, symmetric=False),
              make_matrix(gb, drp, dci, symmetric=False, csc=False)):
        got, k = check(gb, A, drp, dci)
        assert np.array_equal(got, want) and k == 6
    # the same pattern made symmetric may skip, and gives the same components
    srp, sci = symmetric_csr(n, src, dst)
    got, k = check(gb, make_matrix(gb, srp, sci), srp, sci)
    assert np.array_equal(got, want) and k == 6


def test_directed_one_way_matrix(gb):
    """i -> i + 1 stored one way only: one component, with a CSC and with the CSR alone."""
    n = 5000
    src = np.arange(n - 1, dtype=np.int32)
    drp, dci = directed_csr(n, src, src + 1)
    for A in (make_matrix(gb, drp, dci, symmetric=False),
              make_matrix(gb, drp, dci, symmetric=False, csc=False)):
        got, k = check(gb, A, drp, dci)
        assert k == 1 and not got.any()
    # 50..99 join the path 100..4999 only through 100 -> 50, an entry of row 100 alone
    src2 = np.concatenate([np.arange(100, 4999), [100]]).astype(np.int32)
    dst2 = np.concatenate([np.arange(101, 5000), [50]]).astype(np.int32)
    src2 = np.concatenate([src2, np.arange(50, 99)]).astype(np.int32)
    dst2 = np.concatenate([dst2, np.arange(51, 100)]).astype(np.int32)
    drp, dci = directed_csr(n, src2, dst2)
    got, k = check(gb, make_matrix(gb, drp, dci, symmetric=False, csc=False), drp, dci)
    assert k == 51 and np.all(got[50:] == 50)


def test_int32_matrix_and_stored_zeros(gb):
    rp, ci = orc.rmat_csr(12)
    check(gb, make_matrix(gb, rp, ci, integer=True), rp, ci)
    check(gb, make_matrix(gb, rp, ci, symmetric=False, csc=False, integer=True), rp, ci)
    zeros = np.zeros(len(ci), np.float32)
    got, _ = check(gb, make_matrix(gb, rp, ci, zeros, symmetric=False), rp, ci)
    got_i, _ = check(gb, make_matrix(gb, rp, ci, zeros.astype(np.int32),
                                     symmetric=False, integer=True), rp, ci)
    assert np.array_equal(got, got_i)


def test_reused_vector_and_repeated_calls(gb):
    """v is overwritten completely whatever it held, and calls repeat exactly."""
    from graphblast_b200 import algorithm
    rp, ci = orc.rmat_csr(16)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    want, want_k = components(n, rp, ci)
    rng = np.random.RandomState(1)
    v = gb.Vector(n)
    ind = np.sort(rng.choice(n, n//4, replace=False)).astype(np.int32)
    v.build(ind, rng.rand(len(ind)).astype(np.float32)*1e6)        # sparse junk
    got, k = run_cc(gb, A, n, v)
    assert np.array_equal(got, want) and k == want_k
    v.build((rng.rand(n)*-1e6).astype(np.float32))                # dense junk
    got, k = run_cc(gb, A, n, v)
    assert np.array_equal(got, want) and k == want_k
    for _ in range(3):
        k, _ = algorithm.cc(v, A, gb.Descriptor())
        assert np.array_equal(v.extractTuples().astype(np.int64), want) and k == want_k


@pytest.mark.parametrize("graph", ["rmat", "no_entries"])
def test_launches_per_call(gb, graph):
    """One cooperative launch per call."""
    from graphblast_b200 import algorithm
    if graph == "rmat":
        rp, ci = orc.rmat_csr(14)
        A, n = make_matrix(gb, rp, ci), len(rp) - 1
    else:
        A, n = gb.Matrix(1000, 1000), 1000
    v = gb.Vector(n)
    assert launches_per_call(gb, lambda: algorithm.cc(v, A, gb.Descriptor())) == 1


def test_largest_float_size(gb):
    """nrows = 2^24 + 1 is the largest a float vector takes: every id is exact."""
    n = (1 << 24) + 1
    got, k = run_cc(gb, gb.Matrix(n, n), n)
    assert k == n and np.array_equal(got, np.arange(n))


# ---------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------

def expect_refusal(gb, v, A, info, sparse=False):
    """cc(v, A) raises `info`, and v keeps its storage and values (read as a sparse
    list when sparse, since a dense read of a sparse vector converts it)."""
    from graphblast_b200 import algorithm
    storage = v.getStorage()
    before = v.extractTuples(sparse=sparse)
    with pytest.raises(gb.GraphBLASError) as e:
        algorithm.cc(v, A, gb.Descriptor())
    assert e.value.info == info
    assert v.getStorage() == storage
    after = v.extractTuples(sparse=sparse)
    if sparse:
        assert all(np.array_equal(x, y) for x, y in zip(after, before))
    else:
        assert np.array_equal(after, before)


def test_refusals_leave_v_unchanged(gb):
    rp, ci = mtx_graph("test_cc")
    n = len(rp) - 1
    junk = np.arange(n + 1, dtype=np.float32) + 0.5
    A = make_matrix(gb, rp, ci)

    v = gb.Vector(n + 1)                                          # wrong size
    v.build(junk)
    expect_refusal(gb, v, A, gb.Info.GrB_DIMENSION_MISMATCH)

    w = gb.Vector(n)
    w.build(junk[:n])
    R = gb.Matrix(n, n + 1)                                       # not square
    rows = np.repeat(np.arange(n), np.diff(rp))
    R.build(rows, ci, np.ones(len(ci), np.float32))
    expect_refusal(gb, w, R, gb.Info.GrB_DIMENSION_MISMATCH)

    D = gb.Matrix(n, n)                                           # dense
    D.build_dense(np.ones((n, n), np.float32))
    expect_refusal(gb, w, D, gb.Info.GrB_NOT_IMPLEMENTED)

    s = gb.Vector(n)                                             # sparse v, refused too
    s.build(np.array([1, 4], np.int32), np.array([7.5, -2], np.float32))
    assert s.getStorage() == gb.Storage.GrB_SPARSE
    expect_refusal(gb, s, R, gb.Info.GrB_DIMENSION_MISMATCH, sparse=True)
    expect_refusal(gb, s, D, gb.Info.GrB_NOT_IMPLEMENTED, sparse=True)
    assert s.nvals() == 2


def test_float_vector_too_large_for_exact_ids(gb):
    """nrows = 2^24 + 2: a float cannot hold id 2^24 + 1.  The matrix has no stored
    entries, so the refusal comes before anything is allocated."""
    n = (1 << 24) + 2
    v = gb.Vector(n)
    v.build(np.full(n, 3.25, np.float32))
    expect_refusal(gb, v, gb.Matrix(n, n), gb.Info.GrB_INVALID_VALUE)
