"""Community detection by label propagation on the device (algorithm::cdlp, gb200_cdlp)
against the checker (tests/cdlp_reference.py: the C restatement of the semantics),
entry for entry, with the same community and iteration counts.

The graphs reach every class of the kernel: R-MAT lists of every length, a star whose
hub holds 150 000 distinct labels in iteration 1 (the partitioned long path, as
cdlp_stats() shows), and lists of exactly each class bound and one more.  Then planted
communities, a path and a cycle of 2^16, the input forms (stored zeros, self-loops,
element types, symmetric and CSR + CSC forms, library-built and adopted CSCs), reused
and repeated calls, empty cases, the launch count and every refusal.
"""
import os
import subprocess

import numpy as np
import pytest

import cdlp_reference as R
import oracle_binding as orc
from support import Csr, csr, device_matrix, directed_csr, gb, graphs, launches_per_call, \
    make_matrix, symmetric_csr

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ---------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------

def run_cdlp(gb, A, n, max_iter, v=None):
    from graphblast_b200 import algorithm
    v = gb.Vector(n) if v is None else v
    k, it, ms = algorithm.cdlp(v, A, max_iter, gb.Descriptor())
    assert ms >= 0
    assert v.getStorage() == gb.Storage.GrB_DENSE
    got = v.extractTuples()
    assert np.array_equal(got, np.round(got)), "a label that is not an id"
    return got.astype(np.int64), k, it


def check(gb, A, rp, ci, max_iter=10, v=None):
    """The device labels, community and iteration counts of A (pattern rp, ci) equal the
    checker's; returns them with cdlp_stats()."""
    from graphblast_b200 import algorithm
    n = len(rp) - 1
    got, k, it = run_cdlp(gb, A, n, max_iter, v)
    want, want_k, want_it = R.cdlp(rp, ci, max_iter)
    if not np.array_equal(got, want):
        bad = np.flatnonzero(got != want)
        pytest.fail("%d of %d labels differ, first at %d: got %d want %d" % (
            len(bad), n, bad[0], got[bad[0]], want[bad[0]]))
    assert (k, it) == (want_k, want_it)
    stats = algorithm.cdlp_stats()
    assert sum(stats[:3]) == n
    assert stats[4] == 2*it + 2
    return got, k, it, stats


def directed(gb, rp, ci, integer=False, val=None):
    """A with CSR and CSC adopted, not marked symmetric."""
    return make_matrix(gb, rp, ci, val, symmetric=False, integer=integer)


def rmat_directed(scale, seed=1):
    src, dst = orc.rmat_edges(scale, seed=seed)
    return directed_csr(1 << scale, src, dst)


def star(nleaves, centre=0):
    leaves = np.array([x for x in range(nleaves + 1) if x != centre], np.int32)
    return symmetric_csr(nleaves + 1, np.full(nleaves, centre, np.int32), leaves)


# ---------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["chesapeake", "test_cc", "test_bc", "test_sgm"])
def test_golden_graphs(gb, name):
    _, rp, ci = [g for g in graphs() if g[0] == name][0]
    n = len(rp) - 1
    # a pattern without entries cannot be adopted marked symmetric: the library builds it
    check(gb, make_matrix(gb, rp, ci) if len(ci) else gb.Matrix(n, n), rp, ci)
    check(gb, directed(gb, rp, ci), rp, ci)


@pytest.mark.parametrize("scale", [10, 12, 14, 16, 18])
def test_rmat_symmetrised(gb, scale):
    rp, ci = orc.rmat_csr(scale)
    _, _, _, stats = check(gb, make_matrix(gb, rp, ci), rp, ci)
    assert stats[0] > 0 and stats[1] > 0 and stats[2] > 0


@pytest.mark.parametrize("scale", [10, 12, 14, 16, 18])
def test_rmat_directed(gb, scale):
    rp, ci = rmat_directed(scale)
    check(gb, directed(gb, rp, ci), rp, ci)


@pytest.mark.parametrize("max_iter", [0, 1, 2, 10, 1000])
def test_iteration_counts(gb, max_iter):
    rp, ci = orc.rmat_csr(12)
    got, k, it, _ = check(gb, make_matrix(gb, rp, ci), rp, ci, max_iter)
    if max_iter == 0:
        assert it == 0 and np.array_equal(got, np.arange(len(rp) - 1))
    drp, dci = rmat_directed(12)
    check(gb, directed(gb, drp, dci), drp, dci, max_iter)


def test_fixpoint_is_reached_and_reported(gb):
    """Planted cliques joined by single edges reach a fixpoint well before 1000."""
    rp, ci = planted(64, 16, 0)
    _, _, it, _ = check(gb, make_matrix(gb, rp, ci), rp, ci, 1000)
    assert it < 1000


def test_star_with_150000_leaves_takes_the_partitioned_path(gb):
    """The hub sees 150 000 distinct labels in iteration 1; its list is cut into
    ceil(150000 / 2048) = 74 partitions.  The star oscillates, so every iteration runs."""
    m = 150000
    rp, ci = star(m, centre=7)
    for max_iter in (1, 2, 3):
        got, k, it, stats = check(gb, make_matrix(gb, rp, ci), rp, ci, max_iter)
        assert it == max_iter and k == 2
        assert stats[2] == 1 and stats[3] == (m + 2047)//2048
        assert got[7] == (0 if max_iter % 2 else 7)
    # the same star with CSR and CSC: the hub's list is twice as long
    got, _, _, stats = check(gb, directed(gb, rp, ci), rp, ci, 3)
    assert stats[3] == (2*m + 2047)//2048


@pytest.mark.parametrize("d", [32, 33, 128, 129, 2048, 2049, 4097])
def test_class_bounds(gb, d):
    """A hub of exactly d entries (symmetric: d leaves) and of d entries out + in
    (directed: d/2 each way), with leaves grouped so the hub's labels repeat."""
    from graphblast_b200 import algorithm
    rp, ci = star(d, centre=3)
    _, _, _, stats = check(gb, make_matrix(gb, rp, ci), rp, ci, 4)
    cls = 0 if d <= 32 else 1 if d <= 128 else 2
    assert stats[cls] == (d + 1 if cls == 0 else 1)
    # leaves in cliques of 4, so labels repeat in the hub's list
    rng = np.random.RandomState(d)
    leaves = rng.permutation(np.arange(1, d + 1))
    groups = [leaves[i:i + 4] for i in range(0, d, 4)]
    src = [np.zeros(d, np.int32)] + [np.repeat(g, len(g)) for g in groups]
    dst = [np.arange(1, d + 1, dtype=np.int32)] + [np.tile(g, len(g)) for g in groups]
    rp2, ci2 = symmetric_csr(d + 1, np.concatenate(src), np.concatenate(dst))
    check(gb, make_matrix(gb, rp2, ci2), rp2, ci2, 5)
    if d % 2 == 0:                     # d/2 out-arcs and d/2 in-arcs at the hub
        h = d // 2
        rp3, ci3 = directed_csr(d + 1, np.concatenate([np.zeros(h, int), np.arange(h + 1, d + 1)]),
                                np.concatenate([np.arange(1, h + 1), np.zeros(h, int)]))
        _, _, _, stats = check(gb, directed(gb, rp3, ci3), rp3, ci3, 3)
        assert algorithm.cdlp_stats()[cls] >= 1


def planted(count, size, seed, bridges=2):
    """count dense blocks of size vertices (each pair joined with probability 0.7), ids
    permuted, joined by `bridges` random edges per block."""
    rng = np.random.RandomState(seed)
    src, dst = [], []
    for b in range(count):
        a, c = np.triu_indices(size, 1)
        keep = rng.rand(len(a)) < 0.7
        src.append(a[keep] + b*size)
        dst.append(c[keep] + b*size)
    src.append(rng.randint(0, count*size, bridges*count))
    dst.append(rng.randint(0, count*size, bridges*count))
    perm = rng.permutation(count*size)
    return symmetric_csr(count*size, perm[np.concatenate(src)], perm[np.concatenate(dst)])


def test_planted_communities(gb):
    rp, ci = planted(256, 24, 3)
    got, k, _, _ = check(gb, make_matrix(gb, rp, ci), rp, ci, 10)
    assert k <= 2*256


@pytest.mark.parametrize("shape", ["path", "cycle"])
def test_long_path_and_cycle(gb, shape):
    n = 1 << 16
    perm = np.random.RandomState(4).permutation(n).astype(np.int32)
    src, dst = perm, np.roll(perm, -1)
    if shape == "path":
        src, dst = src[:-1], dst[:-1]
    rp, ci = symmetric_csr(n, src, dst)
    for max_iter in (10, 1000):
        check(gb, make_matrix(gb, rp, ci), rp, ci, max_iter)
    drp, dci = directed_csr(n, src, dst)
    check(gb, directed(gb, drp, dci), drp, dci, 10)


# ---------------------------------------------------------------------------
# input forms
# ---------------------------------------------------------------------------

def with_loops(n, src, dst, loops):
    S = csr(n, n, np.concatenate([src, loops]), np.concatenate([dst, loops]),
            np.ones(len(src) + len(loops)), np.float32)
    return S.ptr.astype(np.int32), S.ind.astype(np.int32)


def test_stored_zeros_and_self_loops(gb):
    # 0: only a self-loop; 1 <-> 2 with loops on both; 3 -> 4 with a loop on 4
    rp, ci = with_loops(6, np.array([1, 2, 3]), np.array([2, 1, 4]), np.array([0, 1, 2, 4]))
    got, _, _, _ = check(gb, directed(gb, rp, ci), rp, ci, 3)
    assert got[0] == 0 and got[5] == 5
    rp, ci = rmat_directed(12)
    n = len(rp) - 1
    lrp, lci = with_loops(n, np.repeat(np.arange(n), np.diff(rp)), ci, np.arange(0, n, 3))
    got, k, it, _ = check(gb, directed(gb, lrp, lci), lrp, lci)
    want, want_k, want_it = R.cdlp(rp, ci, 10)
    assert np.array_equal(got, want) and (k, it) == (want_k, want_it)
    zeros = np.zeros(len(lci), np.float32)
    got_z, _, _, _ = check(gb, directed(gb, lrp, lci, val=zeros), lrp, lci)
    assert np.array_equal(got_z, got)


def test_fp32_and_int32_agree(gb):
    rp, ci = rmat_directed(13)
    got_f, k_f, it_f, _ = check(gb, directed(gb, rp, ci), rp, ci)
    got_i, k_i, it_i, _ = check(gb, directed(gb, rp, ci, integer=True), rp, ci)
    assert np.array_equal(got_f, got_i) and (k_f, it_f) == (k_i, it_i)


def test_symmetric_marked_and_csr_csc_forms_agree(gb):
    rp, ci = orc.rmat_csr(14)
    got_m, k_m, it_m, stats_m = check(gb, make_matrix(gb, rp, ci), rp, ci)
    got_u, k_u, it_u, stats_u = check(gb, directed(gb, rp, ci), rp, ci)
    assert np.array_equal(got_m, got_u) and (k_m, it_m) == (k_u, it_u)
    assert stats_u[3] >= stats_m[3]    # the CSR + CSC lists are twice as long


def test_library_built_and_adopted_csc(gb):
    rp, ci = rmat_directed(13)
    n = len(rp) - 1
    B = gb.Matrix(n, n)
    B.build(np.repeat(np.arange(n), np.diff(rp)), ci, np.ones(len(ci), np.float32))
    got_b, k_b, _, _ = check(gb, B, rp, ci)
    got_a, k_a, _, _ = check(gb, directed(gb, rp, ci), rp, ci)
    assert np.array_equal(got_b, got_a) and k_b == k_a
    # the transpose adopted with CSR and CSC swapped: in- and out-lists trade places
    T = Csr(n, n, rp, ci, np.ones(len(ci), np.float32)).T
    check(gb, device_matrix(gb, T), T.ptr, T.ind)


# ---------------------------------------------------------------------------
# calls and edge cases
# ---------------------------------------------------------------------------

def test_reused_vector_and_identical_bytes(gb):
    from graphblast_b200 import algorithm
    rp, ci = orc.rmat_csr(16)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    rng = np.random.RandomState(1)
    v = gb.Vector(n)
    ind = np.sort(rng.choice(n, n//4, replace=False)).astype(np.int32)
    v.build(ind, rng.rand(len(ind)).astype(np.float32)*1e6)        # sparse junk
    check(gb, A, rp, ci, 10, v)
    v.build((rng.rand(n)*-1e6).astype(np.float32))                # dense junk
    check(gb, A, rp, ci, 10, v)
    first = v.extractTuples().tobytes()
    stats = algorithm.cdlp_stats()
    for _ in range(3):
        algorithm.cdlp(v, A, 10, gb.Descriptor())
        assert v.extractTuples().tobytes() == first
        assert algorithm.cdlp_stats() == stats


def test_no_stored_entries_and_one_vertex(gb):
    for n in (1, 5, 1000, 100003):
        for max_iter in (0, 3):
            got, k, it = run_cdlp(gb, gb.Matrix(n, n), n, max_iter)
            assert np.array_equal(got, np.arange(n)) and k == n and it == min(max_iter, 1)
    rp, ci = np.array([0, 1], np.int32), np.array([0], np.int32)     # one self-loop
    got, k, it = run_cdlp(gb, directed(gb, rp, ci), 1, 10)
    assert got.tolist() == [0] and k == 1 and it == 1


def test_no_rows_through_the_backend(tmp_path):
    """n = 0, which the C ABI cannot build: success, 0 communities and one iteration
    that changes nothing, on Vector<int> through backend::cdlpRun and Vector<float>
    through algorithm::cdlp."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    src = tmp_path / "cdlp_n0.cu"
    src.write_text(
        "#define GRB_USE_CUDA\n"
        "#include <cstdio>\n"
        "#include \"graphblas/graphblas.hpp\"\n"
        "#include \"graphblas/algorithm/cdlp.hpp\"\n"
        "bool debug_;\nbool memory_;\n"
        "int main() {\n"
        "  graphblas::Matrix<float> A(0, 0);\n"
        "  graphblas::Matrix<int> B(0, 0);\n"
        "  graphblas::Vector<int> v(0);\n"
        "  graphblas::Vector<float> w(0);\n"
        "  graphblas::Descriptor desc;\n"
        "  int k = -1, m = -1, i = -1, j = -1;\n"
        "  float ms = -1.f;\n"
        "  const graphblas::Info info =\n"
        "      graphblas::backend::cdlpRun(&v.vector_, &A.matrix_, 10, &k, &i, &ms);\n"
        "  const float t = graphblas::algorithm::cdlp(&w, &B, 0, &desc, &m, &j);\n"
        "  std::printf(\"%d %d %d %d %d %d %d\\n\", static_cast<int>(info), k, i, ms >= 0.f,\n"
        "              m, j, t >= 0.f);\n"
        "  return 0;\n}\n")
    exe = tmp_path / "cdlp_n0"
    out = subprocess.run(
        [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-w",
         "-I", os.path.join(ROOT, "include"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc", "shim"),
         str(src), "-o", str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0, run.stderr[-2000:]
    assert run.stdout.split() == ["0", "0", "1", "1", "0", "0", "1"], run.stdout


def test_launches_per_call_do_not_depend_on_max_iter_or_the_graph(gb):
    from graphblast_b200 import algorithm
    counts = []
    for rp, ci in (orc.rmat_csr(14), star(20000), planted(64, 16, 1)):
        n = len(rp) - 1
        A = make_matrix(gb, rp, ci)
        v = gb.Vector(n)
        for max_iter in (0, 1, 10, 1000):
            counts.append(launches_per_call(
                gb, lambda: algorithm.cdlp(v, A, max_iter, gb.Descriptor())))
    assert len(set(counts)) == 1 and counts[0] >= 1


def test_largest_float_size(gb):
    """nrows = 2^24 + 1 is the largest a float vector takes: every id is exact."""
    n = (1 << 24) + 1
    got, k, it = run_cdlp(gb, gb.Matrix(n, n), n, 2)
    assert k == n and it == 1 and np.array_equal(got, np.arange(n))


# ---------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------

def expect_refusal(gb, v, A, info, max_iter=10, sparse=False):
    """cdlp(v, A) raises `info`, and v keeps its storage and bytes."""
    from graphblast_b200 import algorithm
    storage = v.getStorage()
    before = v.extractTuples(sparse=sparse)
    with pytest.raises(gb.GraphBLASError) as e:
        algorithm.cdlp(v, A, max_iter, gb.Descriptor())
    assert e.value.info == info
    assert v.getStorage() == storage
    after = v.extractTuples(sparse=sparse)
    if sparse:
        assert all(x.tobytes() == y.tobytes() for x, y in zip(after, before))
    else:
        assert after.tobytes() == before.tobytes()


def test_refusals_leave_v_unchanged(gb):
    import ctypes as C
    rp, ci = rmat_directed(10)
    n = len(rp) - 1
    junk = np.arange(n + 1, dtype=np.float32) + 0.5
    A = directed(gb, rp, ci)
    lib = gb.api._lib.load()
    w = gb.Vector(n)
    w.build(junk[:n])
    ms = C.byref(C.c_float())
    UNINIT = int(gb.Info.GrB_UNINITIALIZED_OBJECT)
    assert lib.gb200_cdlp(None, A._h, 10, gb.Descriptor()._h, None, None, ms) == UNINIT
    assert lib.gb200_cdlp(w._h, None, 10, gb.Descriptor()._h, None, None, ms) == UNINIT
    assert lib.gb200_cdlp(w._h, A._h, 10, None, None, None, ms) == UNINIT
    assert w.extractTuples().tobytes() == junk[:n].tobytes()

    v = gb.Vector(n + 1)                                          # wrong size
    v.build(junk)
    expect_refusal(gb, v, A, gb.Info.GrB_DIMENSION_MISMATCH)
    expect_refusal(gb, v, A, gb.Info.GrB_DIMENSION_MISMATCH, max_iter=-1)   # before max_iter

    R_ = gb.Matrix(n, n + 1)                                      # not square
    R_.build(np.repeat(np.arange(n), np.diff(rp)), ci, np.ones(len(ci), np.float32))
    expect_refusal(gb, w, R_, gb.Info.GrB_DIMENSION_MISMATCH)

    D = gb.Matrix(n, n)                                           # dense
    D.build_dense(np.ones((n, n), np.float32))
    expect_refusal(gb, w, D, gb.Info.GrB_NOT_IMPLEMENTED)
    expect_refusal(gb, v, D, gb.Info.GrB_NOT_IMPLEMENTED)          # before the sizes

    N = make_matrix(gb, rp, ci, symmetric=False, csc=False)       # no CSC
    expect_refusal(gb, w, N, gb.Info.GrB_UNINITIALIZED_OBJECT)
    expect_refusal(gb, w, N, gb.Info.GrB_UNINITIALIZED_OBJECT, max_iter=-1)

    expect_refusal(gb, w, A, gb.Info.GrB_INVALID_VALUE, max_iter=-1)

    s = gb.Vector(n)                                              # a sparse v, too
    s.build(np.array([1, 4], np.int32), np.array([7.5, -2], np.float32))
    expect_refusal(gb, s, N, gb.Info.GrB_UNINITIALIZED_OBJECT, sparse=True)
    expect_refusal(gb, s, A, gb.Info.GrB_INVALID_VALUE, max_iter=-3, sparse=True)
    assert s.nvals() == 2


def test_float_vector_too_large_for_exact_ids(gb):
    """nrows = 2^24 + 2 with no entries: a float cannot hold id 2^24 + 1."""
    n = (1 << 24) + 2
    v = gb.Vector(n)
    v.build(np.full(n, 3.25, np.float32))
    expect_refusal(gb, v, gb.Matrix(n, n), gb.Info.GrB_INVALID_VALUE)
