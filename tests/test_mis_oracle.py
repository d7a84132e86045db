"""CPU tests of the maximal-independent-set oracle (tests/mis_oracle.c orc_mis) and a
compile-only check of backend::misRun.

orc_mis is pinned three ways: its set is colour class 1 of the greedy colouring
(orc_gc) in the same priority order, it equals a short pure-Python restatement of
the sequential greedy MIS with and without candidates, and it is independent and
maximal within the candidates.  Its depth is checked against a simulation of
synchronous Luby rounds with the same fixed priorities.
"""
import os
import shutil
import subprocess

import numpy as np
import pytest

import greedy_oracle
import oracle_binding as orc
from test_gc_oracle import M32, graphs, py_hash


def py_mis(n, rowptr, colind, seed, cand=None):
    """Sequential greedy MIS in decreasing (hash, v) order over the candidates."""
    member = [0]*n
    for v in sorted(range(n), key=lambda v: (py_hash(seed & M32, v), v), reverse=True):
        if cand is not None and not cand[v]:
            continue
        if not any(member[u] for u in colind[rowptr[v]:rowptr[v + 1]] if u != v):
            member[v] = 1
    return member


def py_luby_rounds(n, rowptr, colind, seed, cand=None):
    """Synchronous Luby rounds with fixed priorities: each round, every undecided
    vertex above all its undecided neighbours joins, and it and its neighbours leave.
    Returns (member, rounds)."""
    key = [(py_hash(seed & M32, v), v) for v in range(n)]
    nbrs = [set(colind[rowptr[v]:rowptr[v + 1]]) - {v} for v in range(n)]
    undecided = {v for v in range(n) if cand is None or cand[v]}
    member = [0]*n
    rounds = 0
    while undecided:
        rounds += 1
        join = [v for v in undecided
                if all(key[u] < key[v] for u in nbrs[v] if u in undecided)]
        assert join
        for v in join:
            member[v] = 1
        for v in join:
            undecided.discard(v)
            undecided -= nbrs[v]
    return member, rounds


def check_independent_and_maximal(rp, ci, member, cand=None):
    n = len(rp) - 1
    cand = np.ones(n, bool) if cand is None else np.asarray(cand) != 0
    rows = np.repeat(np.arange(n), np.diff(rp))
    off = rows != ci
    assert not np.any(member[rows[off]] & member[ci[off]]), "not independent"
    assert not np.any(member[~cand]), "a non-candidate is a member"
    covered = member.astype(bool).copy()
    covered[rows[off][member[ci[off]] == 1]] = True
    assert np.all(covered[cand]), "not maximal"


def random_graph(rng, nmax=60):
    n = int(rng.randint(1, nmax))
    m = int(rng.randint(0, 4*n))
    src = rng.randint(0, n, m).astype(np.int32)
    dst = rng.randint(0, n, m).astype(np.int32)
    rp, ci = orc.build_csr(n, src, dst, True)
    return n, rp, ci


@pytest.mark.parametrize("seed", [0, 1, 12345])
def test_oracle_is_colour_class_one(seed):
    for name, rp, ci in graphs():
        member, size, depth = greedy_oracle.mis(rp, ci, seed)
        colors, _, jp_depth = greedy_oracle.gc(rp, ci, seed)
        assert np.array_equal(member, (colors == 1).astype(np.int32)), name
        assert size == int(member.sum()), name
        assert 1 <= depth <= jp_depth, name
        check_independent_and_maximal(rp, ci, member)
    rng = np.random.RandomState(seed & 0xFFFF)
    for _ in range(20):
        _, rp, ci = random_graph(rng)
        assert np.array_equal(greedy_oracle.mis(rp, ci, seed)[0],
                              (greedy_oracle.gc(rp, ci, seed)[0] == 1).astype(np.int32))


def test_oracle_equals_the_python_restatement():
    rng = np.random.RandomState(5)
    for trial in range(60):
        n, rp, ci = random_graph(rng)
        seed = int(rng.randint(0, 1 << 31)) if trial % 3 else trial
        cand = None if trial % 2 == 0 else (rng.rand(n) < 0.6).astype(np.int32)
        member, size, depth = greedy_oracle.mis(rp, ci, seed, cand)
        want = py_mis(n, rp.tolist(), ci.tolist(), seed,
                      None if cand is None else cand.tolist())
        assert member.tolist() == want, (trial, seed)
        assert size == sum(want)
        check_independent_and_maximal(rp, ci, member, cand)


def test_oracle_depth_is_the_synchronous_luby_round_count():
    rng = np.random.RandomState(9)
    cases = [random_graph(rng, 80)[1:] for _ in range(40)]
    n = 200
    src = np.arange(n - 1, dtype=np.int32)
    cases.append(orc.build_csr(n, src, src + 1, True))         # a path
    cases.append(graphs()[0][1:])                               # chesapeake
    for trial, (rp, ci) in enumerate(cases):
        n = len(rp) - 1
        seed = trial*7 + 1
        cand = None if trial % 3 else (rng.rand(n) < 0.7).astype(np.int32)
        member, _, depth = greedy_oracle.mis(rp, ci, seed, cand)
        want, rounds = py_luby_rounds(n, rp.tolist(), ci.tolist(), seed,
                                      None if cand is None else cand.tolist())
        assert member.tolist() == want, trial
        assert depth == rounds, trial


def test_oracle_candidates_and_tiny_graphs():
    rp, ci = graphs()[0][1:]
    n = len(rp) - 1
    member, size, depth = greedy_oracle.mis(rp, ci, 0, np.zeros(n, np.int32))
    assert size == 0 and depth == 0 and not member.any()
    # every vertex a candidate is the same as no candidate vector
    assert np.array_equal(greedy_oracle.mis(rp, ci, 3, np.full(n, 2.5))[0],
                          greedy_oracle.mis(rp, ci, 3)[0])
    # a triangle with loops: one member; no edges: every candidate
    rp3 = np.array([0, 3, 6, 9], np.int32)
    ci3 = np.array([0, 1, 2, 0, 1, 2, 0, 1, 2], np.int32)
    member, size, depth = greedy_oracle.mis(rp3, ci3, 0)
    assert size == 1 and depth == 1
    member, size, depth = greedy_oracle.mis(np.zeros(6, np.int32), np.zeros(0, np.int32), 0,
                                        np.array([1, 0, 1, 1, 0]))
    assert member.tolist() == [1, 0, 1, 1, 0] and size == 3 and depth == 1
    member, size, depth = greedy_oracle.mis(np.zeros(1, np.int32), np.zeros(0, np.int32), 0)
    assert len(member) == 0 and size == 0 and depth == 0


def test_mis_compiles_for_int_and_float_vectors(tmp_path):
    """backend::misRun on Vector<int> and Vector<float> with FP32 and INT32 matrices,
    compiled for sm_90a."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not present")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "mis_tu.cu"
    src.write_text(
        "#define GRB_USE_CUDA\n"
        "#include \"graphblas/graphblas.hpp\"\n"
        "bool debug_;\nbool memory_;\n"
        "template <typename W, typename a>\n"
        "graphblas::Info run(graphblas::Vector<W>* w, const graphblas::Matrix<a>* A,\n"
        "    const graphblas::Vector<W>* c, int* k) {\n"
        "  return graphblas::backend::misRun(&w->vector_, &A->matrix_, 7u,\n"
        "      c != NULL ? &c->vector_ : NULL, k);\n}\n"
        "template graphblas::Info run(graphblas::Vector<int>*,\n"
        "    const graphblas::Matrix<float>*, const graphblas::Vector<int>*, int*);\n"
        "template graphblas::Info run(graphblas::Vector<int>*,\n"
        "    const graphblas::Matrix<int>*, const graphblas::Vector<int>*, int*);\n"
        "template graphblas::Info run(graphblas::Vector<float>*,\n"
        "    const graphblas::Matrix<float>*, const graphblas::Vector<float>*, int*);\n"
        "template graphblas::Info run(graphblas::Vector<float>*,\n"
        "    const graphblas::Matrix<int>*, const graphblas::Vector<float>*, int*);\n")
    out = subprocess.run(
        [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-w",
         "-I", os.path.join(root, "include"),
         "-I", os.path.join(root, "graphblast_b200", "csrc"),
         "-I", os.path.join(root, "graphblast_b200", "csrc", "shim"),
         "-c", str(src), "-o", str(tmp_path / "mis_tu.o")],
        capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
