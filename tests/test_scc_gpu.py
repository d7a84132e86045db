"""Strongly connected components on the device (algorithm::scc, gb200_scc) against the
checker (tests/scc_reference.py: scipy's strong components, each label mapped to its
component's minimum id), entry for entry and count for count.

The graphs are chosen so that each phase of the kernel settles work: DAGs and paths
that the trim settles whole, R-MAT and a bowtie whose giant component the pivot's
forward-backward reach settles, and pieces joined one way and tendrils holding cycles
that only the colouring settles.  scc_stats() checks which phase ran.  A hub with
150 000 arcs each way exercises the grid pass of long lists; a directed cycle and a
path of 2^16 vertices exercise deep reaches and long trims.  Then the input forms
(element types, stored zeros, self-loops, symmetric and CSR + CSC forms, library-built
and adopted CSCs, the transpose), repeated and reused calls, empty cases, the launch
count and every refusal.
"""
import os
import subprocess

import numpy as np
import pytest

import oracle_binding as orc
import scc_reference as R
from support import Csr, csr, device_matrix, directed_csr, gb, launches_per_call, make_matrix

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")


# ---------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------

def run_scc(gb, A, n, v=None):
    from graphblast_b200 import algorithm
    v = gb.Vector(n) if v is None else v
    k, ms = algorithm.scc(v, A, gb.Descriptor())
    assert ms >= 0
    assert v.getStorage() == gb.Storage.GrB_DENSE
    got = v.extractTuples()
    assert np.array_equal(got, np.round(got)), "a label that is not an id"
    return got.astype(np.int64), k


def directed(gb, rp, ci, integer=False, val=None):
    """A with CSR and CSC adopted, not marked symmetric: the kernel's path."""
    return make_matrix(gb, rp, ci, val, symmetric=False, integer=integer)


def check(gb, A, rp, ci):
    """The device labels and count of A (pattern rp, ci) equal the checker's; returns
    them with scc_stats()."""
    from graphblast_b200 import algorithm
    n = len(rp) - 1
    got, k = run_scc(gb, A, n)
    want, want_k = R.scc(rp, ci)
    assert np.array_equal(got, want)
    assert k == want_k == int(np.count_nonzero(want == np.arange(n)))
    return got, k, algorithm.scc_stats()


def largest(rp, ci):
    return int(np.bincount(R.scc(rp, ci)[0]).max())


def rmat_directed(scale, seed=1):
    """R-MAT edges one way, self-loops and duplicates removed."""
    src, dst = orc.rmat_edges(scale, seed=seed)
    return directed_csr(1 << scale, src, dst)


def cycle_arcs(ids):
    ids = np.asarray(ids)
    return ids, np.roll(ids, -1)


# ---------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["chesapeake", "test_cc", "test_bc", "test_sgm"])
def test_golden_graphs_directed(gb, name):
    n, src, dst, _ = orc.read_mtx_edges(os.path.join(GOLDEN, name + ".mtx"))
    rp, ci = directed_csr(n, src, dst)
    check(gb, directed(gb, rp, ci), rp, ci)


@pytest.mark.parametrize("scale", [10, 12, 14, 16, 18])
def test_rmat_directed(gb, scale):
    rp, ci = rmat_directed(scale)
    _, k, (trimmed, pivot, colours, barriers) = check(gb, directed(gb, rp, ci), rp, ci)
    assert 1 < k < len(rp) - 1 and trimmed > 0 and barriers > 0
    if scale == 16:
        assert pivot == largest(rp, ci) > (len(rp) - 1)//10


def test_permuted_dag(gb):
    n = 100000
    rng = np.random.RandomState(4)
    a, b = rng.randint(0, n, 8*n), rng.randint(0, n, 8*n)
    keep = a != b
    perm = rng.permutation(n)
    rp, ci = directed_csr(n, perm[np.minimum(a, b)[keep]], perm[np.maximum(a, b)[keep]])
    got, k, (trimmed, pivot, colours, _) = check(gb, directed(gb, rp, ci), rp, ci)
    assert k == n and trimmed == n and pivot == 0 and colours == 0


def test_long_cycle(gb):
    n = 1 << 16
    ids = np.random.RandomState(5).permutation(n)
    rp, ci = directed_csr(n, *cycle_arcs(ids))
    got, k, (trimmed, pivot, colours, _) = check(gb, directed(gb, rp, ci), rp, ci)
    assert k == 1 and not got.any() and trimmed == 0 and pivot == n and colours == 0


def test_long_path(gb):
    n = 1 << 16
    ids = np.random.RandomState(6).permutation(n)
    rp, ci = directed_csr(n, ids[:-1], ids[1:])
    got, k, (trimmed, _, _, _) = check(gb, directed(gb, rp, ci), rp, ci)
    assert k == n and trimmed == n


# ---------------------------------------------------------------------------
# components and phases
# ---------------------------------------------------------------------------

def bowtie(rng, core=20000, tendril_cycles=3000):
    """A core (a Hamiltonian cycle plus random arcs, with a hub at core vertex 0), 3-cycles
    feeding into it (the in-tendril) and 3-cycles fed from it (the out-tendril), some
    of them chained, plus isolated vertices; ids permuted."""
    src, dst = [], []
    cs, cd = cycle_arcs(np.arange(core))
    src += [cs, rng.randint(0, core, 3*core), np.zeros(2000, int), rng.randint(0, core, 2000)]
    dst += [cd, rng.randint(0, core, 3*core), rng.randint(0, core, 2000), np.zeros(2000, int)]
    base = core
    for into in (True, False):
        for t in range(tendril_cycles):
            tri = np.arange(base, base + 3)
            s, d = cycle_arcs(tri)
            src.append(s)
            dst.append(d)
            c = rng.randint(0, core)
            src.append([tri[0] if into else c])
            dst.append([c if into else tri[0]])
            if t > 0 and t % 3:                         # chain to the previous triangle
                src.append([tri[1] if into else base - 1])
                dst.append([base - 1 if into else tri[1]])
            base += 3
    n = base + 100
    perm = rng.permutation(n)
    src = perm[np.concatenate([np.asarray(x) for x in src])]
    dst = perm[np.concatenate([np.asarray(x) for x in dst])]
    return directed_csr(n, src, dst)


def test_bowtie(gb):
    rp, ci = bowtie(np.random.RandomState(7))
    _, k, (_, pivot, colours, _) = check(gb, directed(gb, rp, ci), rp, ci)
    assert pivot == largest(rp, ci) >= 20000 and colours >= 1
    assert k == (len(rp) - 1) - 20000 - 2*3000*2 + 1   # every triangle its own component


def pieces(count=512, size=64, seed=8):
    """count pieces of size vertices, each a directed Hamiltonian cycle plus random
    arcs inside it, arcs only from lower to higher piece index, ids interleaved by a
    permutation."""
    rng = np.random.RandomState(seed)
    n = count*size
    base = (np.arange(count)*size)[:, None]
    local = np.arange(size)
    src = [(base + local).ravel(), (base + rng.randint(0, size, (count, size))).ravel()]
    dst = [(base + (local + 1) % size).ravel(), (base + rng.randint(0, size, (count, size))).ravel()]
    a, b = rng.randint(0, count, 4*count), rng.randint(0, count, 4*count)
    keep = a != b
    lo, hi = np.minimum(a, b)[keep], np.maximum(a, b)[keep]
    src.append(lo*size + rng.randint(0, size, len(lo)))
    dst.append(hi*size + rng.randint(0, size, len(hi)))
    perm = rng.permutation(n)
    return directed_csr(n, perm[np.concatenate(src)], perm[np.concatenate(dst)])


def test_pieces_joined_one_way(gb):
    rp, ci = pieces()
    _, k, (_, pivot, colours, _) = check(gb, directed(gb, rp, ci), rp, ci)
    assert k == 512 and pivot == 64 and colours >= 1


def test_hub_onto_one_cycle(gb):
    """A hub with 150 000 out-arcs and 150 000 in-arcs onto a cycle of 150 000: lists
    for the grid pass in both directions."""
    m = 150000
    cyc = np.random.RandomState(9).permutation(np.arange(1, m + 1))
    cs, cd = cycle_arcs(cyc)
    src = np.concatenate([cs, np.zeros(m, int), cyc])
    dst = np.concatenate([cd, cyc, np.zeros(m, int)])
    rp, ci = directed_csr(m + 3, src, dst)                 # and two isolated vertices
    got, k, (_, pivot, _, _) = check(gb, directed(gb, rp, ci), rp, ci)
    assert k == 3 and pivot == m + 1
    # the hub reaching the cycle one way only: the cycle and the hub apart
    rp, ci = directed_csr(m + 1, np.concatenate([cs, np.zeros(m, int)]),
                          np.concatenate([cd, cyc]))
    _, k, _ = check(gb, directed(gb, rp, ci), rp, ci)
    assert k == 2


# ---------------------------------------------------------------------------
# input forms
# ---------------------------------------------------------------------------

def test_int32_and_stored_zeros(gb):
    rp, ci = rmat_directed(12)
    got_f, k_f, _ = check(gb, directed(gb, rp, ci), rp, ci)
    got_i, k_i, _ = check(gb, directed(gb, rp, ci, integer=True), rp, ci)
    zeros = np.zeros(len(ci), np.float32)
    got_z, _, _ = check(gb, directed(gb, rp, ci, val=zeros), rp, ci)
    got_zi, _, _ = check(gb, directed(gb, rp, ci, integer=True, val=zeros.astype(np.int32)),
                         rp, ci)
    assert all(np.array_equal(got_f, g) for g in (got_i, got_z, got_zi)) and k_f == k_i


def with_loops(n, src, dst, loops):
    S = csr(n, n, np.concatenate([src, loops]), np.concatenate([dst, loops]),
            np.ones(len(src) + len(loops)), np.float32)
    return S.ptr.astype(np.int32), S.ind.astype(np.int32)


def test_self_loops(gb):
    # 0: only a self-loop; 1 <-> 2 with loops on both; 3 -> 4 with a loop on 4; 5 alone
    rp, ci = with_loops(6, np.array([1, 2, 3]), np.array([2, 1, 4]), np.array([0, 1, 2, 4]))
    got, k, (trimmed, pivot, _, _) = check(gb, directed(gb, rp, ci), rp, ci)
    assert got.tolist() == [0, 1, 1, 3, 4, 5] and k == 5
    assert trimmed == 4 and pivot == 2                     # loops do not stop the trim
    # an R-MAT with loops on every third vertex: the same as without
    rp, ci = rmat_directed(12)
    n = len(rp) - 1
    lrp, lci = with_loops(n, np.repeat(np.arange(n), np.diff(rp)), ci, np.arange(0, n, 3))
    got, _, _ = check(gb, directed(gb, lrp, lci), lrp, lci)
    assert np.array_equal(got, R.scc(rp, ci)[0])


def test_symmetric_marked_and_unmarked(gb):
    """A symmetric pattern marked symmetric takes cc; adopted as CSR + CSC unmarked it
    takes the kernel.  Both give the checker's answer."""
    rp, ci = orc.rmat_csr(14)
    got_m, k_m, stats_m = check(gb, make_matrix(gb, rp, ci), rp, ci)
    assert stats_m == (0, 0, 0, -1)
    got_u, k_u, stats_u = check(gb, directed(gb, rp, ci), rp, ci)
    assert stats_u[3] > 0 and stats_u[1] == largest(rp, ci)
    assert np.array_equal(got_m, got_u) and k_m == k_u


def test_library_built_csc(gb):
    """A built from host triples, CSR and CSC by the library, against the same pattern
    with both adopted."""
    rp, ci = rmat_directed(13)
    n = len(rp) - 1
    B = gb.Matrix(n, n)
    B.build(np.repeat(np.arange(n), np.diff(rp)), ci, np.ones(len(ci), np.float32))
    got_b, k_b, _ = check(gb, B, rp, ci)
    got_a, k_a, _ = check(gb, directed(gb, rp, ci), rp, ci)
    assert np.array_equal(got_b, got_a) and k_b == k_a


def test_transpose_has_the_same_components(gb):
    """scc(A') with A's CSR and CSC swapped on adoption equals scc(A)."""
    rp, ci = rmat_directed(14)
    n = len(rp) - 1
    S = Csr(n, n, rp, ci, np.ones(len(ci), np.float32))
    T = S.T
    At = device_matrix(gb, T)
    got, k, _ = check(gb, At, T.ptr, T.ind)
    want, want_k = R.scc(rp, ci)
    assert np.array_equal(got, want) and k == want_k


# ---------------------------------------------------------------------------
# calls and edge cases
# ---------------------------------------------------------------------------

def test_repeated_calls_and_reused_vector(gb):
    from graphblast_b200 import algorithm
    rp, ci = rmat_directed(16)
    n = len(rp) - 1
    A = directed(gb, rp, ci)
    want, want_k = R.scc(rp, ci)
    rng = np.random.RandomState(1)
    v = gb.Vector(n)
    ind = np.sort(rng.choice(n, n//4, replace=False)).astype(np.int32)
    v.build(ind, rng.rand(len(ind)).astype(np.float32)*1e6)        # sparse junk
    got, k = run_scc(gb, A, n, v)
    assert np.array_equal(got, want) and k == want_k
    v.build((rng.rand(n)*-1e6).astype(np.float32))                # dense junk
    got, k = run_scc(gb, A, n, v)
    assert np.array_equal(got, want) and k == want_k
    first = v.extractTuples().tobytes()
    stats = algorithm.scc_stats()
    for _ in range(3):
        k, _ = algorithm.scc(v, A, gb.Descriptor())
        assert v.extractTuples().tobytes() == first and k == want_k
        assert algorithm.scc_stats()[:3] == stats[:3]


def test_no_stored_entries_and_one_vertex(gb):
    for n in (1, 5, 1000, 100003):
        got, k = run_scc(gb, gb.Matrix(n, n), n)
        assert np.array_equal(got, np.arange(n)) and k == n
    for loop in (False, True):
        rp = np.array([0, 1 if loop else 0], np.int32)
        ci = np.array([0] if loop else [], np.int32)
        A = directed(gb, rp, ci) if loop else gb.Matrix(1, 1)
        got, k = run_scc(gb, A, 1)
        assert got.tolist() == [0] and k == 1


def test_no_rows_through_the_backend(tmp_path):
    """n = 0, which the C ABI cannot build: success and count 0, on Vector<int> through
    backend::sccRun and Vector<float> through algorithm::scc."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    src = tmp_path / "scc_n0.cu"
    src.write_text(
        "#define GRB_USE_CUDA\n"
        "#include <cstdio>\n"
        "#include \"graphblas/graphblas.hpp\"\n"
        "#include \"graphblas/algorithm/scc.hpp\"\n"
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
        "      graphblas::backend::sccRun(&v.vector_, &A.matrix_, &k, &ms);\n"
        "  const float t = graphblas::algorithm::scc(&w, &B, &desc, &m);\n"
        "  std::printf(\"%d %d %d %d %d\\n\", static_cast<int>(info), k, ms >= 0.f, m,\n"
        "              t >= 0.f);\n"
        "  return 0;\n}\n")
    exe = tmp_path / "scc_n0"
    out = subprocess.run(
        [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-w",
         "-I", os.path.join(ROOT, "include"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc", "shim"),
         str(src), "-o", str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert run.returncode == 0, run.stderr[-2000:]
    assert run.stdout.split() == ["0", "0", "1", "0", "1"], run.stdout


def test_launches_per_call_do_not_depend_on_the_graph(gb):
    from graphblast_b200 import algorithm
    counts = []
    n = 1 << 14
    ids = np.arange(n)
    for rp, ci in (rmat_directed(14), pieces(64, 32), directed_csr(n, *cycle_arcs(ids)),
                   directed_csr(n, ids[:-1], ids[1:])):
        n = len(rp) - 1
        A = directed(gb, rp, ci)
        v = gb.Vector(n)
        counts.append(launches_per_call(gb, lambda: algorithm.scc(v, A, gb.Descriptor())))
    assert len(set(counts)) == 1 and counts[0] >= 1


def test_largest_float_size(gb):
    """nrows = 2^24 + 1 is the largest a float vector takes: every id is exact."""
    n = (1 << 24) + 1
    got, k = run_scc(gb, gb.Matrix(n, n), n)
    assert k == n and np.array_equal(got, np.arange(n))


# ---------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------

def expect_refusal(gb, v, A, info, sparse=False):
    """scc(v, A) raises `info`, and v keeps its storage and bytes."""
    from graphblast_b200 import algorithm
    storage = v.getStorage()
    before = v.extractTuples(sparse=sparse)
    with pytest.raises(gb.GraphBLASError) as e:
        algorithm.scc(v, A, gb.Descriptor())
    assert e.value.info == info
    assert v.getStorage() == storage
    after = v.extractTuples(sparse=sparse)
    if sparse:
        assert all(x.tobytes() == y.tobytes() for x, y in zip(after, before))
    else:
        assert after.tobytes() == before.tobytes()


def test_refusals_leave_v_unchanged(gb):
    rp, ci = rmat_directed(10)
    n = len(rp) - 1
    junk = np.arange(n + 1, dtype=np.float32) + 0.5
    A = directed(gb, rp, ci)

    v = gb.Vector(n + 1)                                          # wrong size
    v.build(junk)
    expect_refusal(gb, v, A, gb.Info.GrB_DIMENSION_MISMATCH)

    w = gb.Vector(n)
    w.build(junk[:n])
    R_ = gb.Matrix(n, n + 1)                                      # not square
    R_.build(np.repeat(np.arange(n), np.diff(rp)), ci, np.ones(len(ci), np.float32))
    expect_refusal(gb, w, R_, gb.Info.GrB_DIMENSION_MISMATCH)

    D = gb.Matrix(n, n)                                           # dense
    D.build_dense(np.ones((n, n), np.float32))
    expect_refusal(gb, w, D, gb.Info.GrB_NOT_IMPLEMENTED)

    N = make_matrix(gb, rp, ci, symmetric=False, csc=False)       # no CSC
    expect_refusal(gb, w, N, gb.Info.GrB_UNINITIALIZED_OBJECT)

    s = gb.Vector(n)                                              # a sparse v, too
    s.build(np.array([1, 4], np.int32), np.array([7.5, -2], np.float32))
    expect_refusal(gb, s, N, gb.Info.GrB_UNINITIALIZED_OBJECT, sparse=True)
    expect_refusal(gb, s, D, gb.Info.GrB_NOT_IMPLEMENTED, sparse=True)
    assert s.nvals() == 2


def test_float_vector_too_large_for_exact_ids(gb):
    """nrows = 2^24 + 2: a float cannot hold id 2^24 + 1."""
    n = (1 << 24) + 2
    v = gb.Vector(n)
    v.build(np.full(n, 3.25, np.float32))
    expect_refusal(gb, v, gb.Matrix(n, n), gb.Info.GrB_INVALID_VALUE)
