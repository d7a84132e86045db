"""CPU tests of the graph-colouring oracle (tests/gc_oracle.c orc_gc) and a
compile-only check of graphblas::graphColor.

orc_gc is ours: the reference's SimpleReferenceGc orders vertices with
std::mt19937, so it cannot pin a hashed order.  The oracle is pinned by properties
instead: its colouring is proper, uses at most max degree + 1 colours, and is the
greedy colouring in decreasing priority order, which these tests check through a
characterisation that determines it uniquely and through a short pure-Python
restatement that also fixes the priority hash.
"""
import os
import shutil
import subprocess

import numpy as np
import pytest

import greedy_oracle
import oracle_binding as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
M32 = 0xFFFFFFFF


def py_hash(seed, v):
    """fmix32(v ^ (seed * 0x9E3779B9)), the priority hash of kernels/greedy_schedule.cuh."""
    x = (v ^ (seed*0x9E3779B9)) & M32
    x ^= x >> 16
    x = (x*0x85EBCA6B) & M32
    x ^= x >> 13
    x = (x*0xC2B2AE35) & M32
    return x ^ (x >> 16)


def py_gc(n, rowptr, colind, seed):
    """Sequential greedy first-fit in decreasing (hash, v) order."""
    colors = [0]*n
    for v in sorted(range(n), key=lambda v: (py_hash(seed & M32, v), v), reverse=True):
        used = {colors[u] for u in colind[rowptr[v]:rowptr[v + 1]] if u != v}
        c = 1
        while c in used:
            c += 1
        colors[v] = c
    return colors


def mtx_graph(name):
    n, src, dst, _ = orc.read_mtx_edges(os.path.join(GOLDEN, name + ".mtx"))
    return orc.build_csr(n, src, dst, True)


def check_greedy(rowptr, colind, colors, seed):
    """Proper, at most max degree + 1 colours, and greedy in priority order: a vertex
    coloured c has, for every c' < c, a higher-priority neighbour coloured c', and no
    higher-priority neighbour coloured c.  With properness this is the greedy
    colouring and nothing else."""
    n = len(rowptr) - 1
    deg = np.diff(rowptr)
    assert colors.min(initial=1) >= 1
    assert colors.max(initial=0) <= (deg.max(initial=0) + 1)
    rows = np.repeat(np.arange(n), deg)
    off_diag = rows != colind
    assert not np.any(colors[rows[off_diag]] == colors[colind[off_diag]]), "not proper"
    prio = np.array([py_hash(seed & M32, v) for v in range(n)], dtype=np.uint64)
    key = (prio << np.uint64(32)) | np.arange(n, dtype=np.uint64)
    for v in range(n):
        nb = colind[rowptr[v]:rowptr[v + 1]]
        higher = nb[key[nb] > key[v]]
        held = set(colors[higher].tolist())
        c = int(colors[v])
        assert c not in held
        assert held >= set(range(1, c)), "vertex %d could take a smaller colour" % v


def graphs():
    out = [("chesapeake",) + mtx_graph("chesapeake"), ("test_cc",) + mtx_graph("test_cc"),
           ("test_bc",) + mtx_graph("test_bc"), ("test_sgm",) + mtx_graph("test_sgm")]
    for scale in (10, 11, 12):
        out.append(("rmat%d" % scale,) + orc.rmat_csr(scale))
    return out


@pytest.mark.parametrize("seed", [0, 1, 12345])
def test_oracle_is_the_greedy_colouring(seed):
    for name, rp, ci in graphs():
        colors, ncolors, depth = greedy_oracle.gc(rp, ci, seed)
        assert ncolors == colors.max(initial=0), name
        assert 1 <= ncolors <= depth, name         # a colour c needs a chain of c
        check_greedy(rp, ci, colors, seed)


def test_oracle_equals_the_python_restatement():
    rng = np.random.RandomState(3)
    for trial in range(40):
        n = int(rng.randint(1, 60))
        m = int(rng.randint(0, 4*n))
        src = rng.randint(0, n, m).astype(np.int32)
        dst = rng.randint(0, n, m).astype(np.int32)
        rp, ci = orc.build_csr(n, src, dst, True)
        seed = int(rng.randint(0, 1 << 31)) if trial % 3 else trial
        colors, ncolors, _ = greedy_oracle.gc(rp, ci, seed)
        want = py_gc(n, rp.tolist(), ci.tolist(), seed)
        assert colors.tolist() == want, (trial, seed)
        assert ncolors == max(want)


def test_oracle_ignores_self_loops_and_handles_tiny_graphs():
    # a triangle with a loop on every vertex: colours 1..3, the loops change nothing
    rp = np.array([0, 3, 6, 9], np.int32)
    ci = np.array([0, 1, 2, 0, 1, 2, 0, 1, 2], np.int32)
    colors, ncolors, depth = greedy_oracle.gc(rp, ci, 0)
    assert sorted(colors.tolist()) == [1, 2, 3] and ncolors == 3 and depth == 3
    colors, ncolors, depth = greedy_oracle.gc(np.zeros(1, np.int32), np.zeros(0, np.int32), 0)
    assert len(colors) == 0 and ncolors == 0 and depth == 0
    colors, ncolors, depth = greedy_oracle.gc(np.zeros(2, np.int32), np.zeros(0, np.int32), 0)
    assert colors.tolist() == [1] and ncolors == 1 and depth == 1


def test_oracle_depth_is_the_longest_priority_chain():
    # on a path every vertex's round is 1 + the round of its higher-priority neighbours
    n = 200
    src = np.arange(n - 1, dtype=np.int32)
    rp, ci = orc.build_csr(n, src, src + 1, True)
    _, ncolors, depth = greedy_oracle.gc(rp, ci, 7)
    key = [(py_hash(7, v), v) for v in range(n)]
    rounds = [0]*n
    for v in sorted(range(n), key=lambda v: key[v], reverse=True):
        rounds[v] = 1 + max([rounds[u] for u in ci[rp[v]:rp[v + 1]] if key[u] > key[v]],
                            default=0)
    assert depth == max(rounds) and ncolors <= 3


def test_graph_color_compiles_for_int_and_float_vectors(tmp_path):
    """graphblas::graphColor on Vector<int> and Vector<float>, compiled for sm_90a."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not present")
    src = tmp_path / "gc_tu.cu"
    src.write_text(
        "#define GRB_USE_CUDA\n"
        "#include \"graphblas/graphblas.hpp\"\n"
        "bool debug_;\nbool memory_;\n"
        "graphblas::Info colour_int(graphblas::Vector<int>* w,\n"
        "    const graphblas::Matrix<float>* A, graphblas::Descriptor* d) {\n"
        "  return graphblas::graphColor(w, A, d);\n}\n"
        "graphblas::Info colour_float(graphblas::Vector<float>* w,\n"
        "    const graphblas::Matrix<int>* A, graphblas::Descriptor* d) {\n"
        "  return graphblas::graphColor(w, A, d);\n}\n")
    out = subprocess.run(
        [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-w",
         "-I", os.path.join(ROOT, "include"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc"),
         "-I", os.path.join(ROOT, "graphblast_b200", "csrc", "shim"),
         "-c", str(src), "-o", str(tmp_path / "gc_tu.o")],
        capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
