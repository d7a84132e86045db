"""CPU tests of the connected-components checker (support.components) and a
compile-only check of backend::ccRun.

The checker is pinned against a pure-Python union-find on small random directed
graphs, with self-loops, repeated entries and one-way entries: the labels must be the
components' minimum ids, the count the number of components.
"""
import os
import shutil
import subprocess

import numpy as np
import pytest

from support import check_structure, components


def py_components(n, edges):
    """Union-find over (i, j) pairs, each component labelled with its minimum id."""
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for i, j in edges:
        a, b = find(i), find(j)
        if a != b:
            parent[max(a, b)] = min(a, b)
    label = [find(x) for x in range(n)]
    return label, sum(1 for x in range(n) if label[x] == x)


def random_directed_csr(rng, nmax=80):
    """A CSR of random one-way entries, self-loops and repeats included."""
    n = int(rng.randint(1, nmax))
    m = int(rng.randint(0, 2*n))
    src = rng.randint(0, n, m)
    dst = rng.randint(0, n, m)
    order = np.lexsort((dst, src))
    src, dst = src[order], dst[order]
    rp = np.concatenate([[0], np.cumsum(np.bincount(src, minlength=n))]).astype(np.int32)
    return n, rp, dst.astype(np.int32), list(zip(src.tolist(), dst.tolist()))


def test_checker_equals_python_union_find():
    rng = np.random.RandomState(21)
    for trial in range(200):
        n, rp, ci, edges = random_directed_csr(rng)
        label, k = components(n, rp, ci)
        want, want_k = py_components(n, edges)
        assert label.tolist() == want and k == want_k, trial
        check_structure(rp, ci, label)


def test_checker_small_cases():
    assert components(0, np.zeros(1, np.int32), np.zeros(0, np.int32))[1] == 0
    label, k = components(4, np.zeros(5, np.int32), np.zeros(0, np.int32))
    assert label.tolist() == [0, 1, 2, 3] and k == 4
    # 3 -> 1 and 2 -> 0 only one way: {0, 2}, {1, 3}
    rp = np.array([0, 0, 0, 1, 2], np.int32)
    ci = np.array([0, 1], np.int32)
    label, k = components(4, rp, ci)
    assert label.tolist() == [0, 1, 0, 1] and k == 2
    # the structural check catches an edge across labels and a label above its vertex
    with pytest.raises(AssertionError):
        check_structure(rp, ci, np.array([0, 1, 2, 1]))
    with pytest.raises(AssertionError):
        check_structure(np.zeros(3, np.int32), np.zeros(0, np.int32), np.array([1, 1]))


def test_cc_compiles_for_int_and_float_vectors(tmp_path):
    """backend::ccRun on Vector<int> and Vector<float> with FP32 and INT32 matrices,
    and algorithm::cc, compiled for sm_90a."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not present")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "cc_tu.cu"
    src.write_text(
        "#define GRB_USE_CUDA\n"
        "#include \"graphblas/graphblas.hpp\"\n"
        "#include \"graphblas/algorithm/cc.hpp\"\n"
        "bool debug_;\nbool memory_;\n"
        "template <typename W, typename a>\n"
        "graphblas::Info run(graphblas::Vector<W>* w, const graphblas::Matrix<a>* A,\n"
        "    int* k) {\n"
        "  return graphblas::backend::ccRun(&w->vector_, &A->matrix_, k);\n}\n"
        "template graphblas::Info run(graphblas::Vector<int>*,\n"
        "    const graphblas::Matrix<float>*, int*);\n"
        "template graphblas::Info run(graphblas::Vector<int>*,\n"
        "    const graphblas::Matrix<int>*, int*);\n"
        "template graphblas::Info run(graphblas::Vector<float>*,\n"
        "    const graphblas::Matrix<float>*, int*);\n"
        "template graphblas::Info run(graphblas::Vector<float>*,\n"
        "    const graphblas::Matrix<int>*, int*);\n"
        "template float graphblas::algorithm::cc(graphblas::Vector<float>*,\n"
        "    const graphblas::Matrix<float>*, graphblas::Descriptor*, int*);\n"
        "template float graphblas::algorithm::cc(graphblas::Vector<float>*,\n"
        "    const graphblas::Matrix<int>*, graphblas::Descriptor*, int*);\n")
    out = subprocess.run(
        [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-w",
         "-I", os.path.join(root, "include"),
         "-I", os.path.join(root, "graphblast_b200", "csrc"),
         "-I", os.path.join(root, "graphblast_b200", "csrc", "shim"),
         "-c", str(src), "-o", str(tmp_path / "cc_tu.o")],
        capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
