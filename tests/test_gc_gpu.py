"""Graph colouring on the device (algorithm::gc, gb200_gc, backend::graphColor)
against the CPU greedy colouring (tests/gc_oracle.c), entry for entry.

The colouring is greedy first-fit in decreasing priority order, so it does not depend
on launch shape or timing and every colour can be compared exactly.  The graphs cover
the kernel's classes: lists a lane takes alone and lists a warp takes, the sweeps and
the tail, several 64-colour windows, empty and isolated rows, self-loops, and a
directed matrix read through its CSR and its CSC.
"""
import numpy as np
import pytest

import greedy_oracle
import oracle_binding as orc
from support import (gb, launches_per_call, make_matrix, mtx_graph, path_graph, ragged_graph,
                     star_graph, symmetric_csr)

pytestmark = pytest.mark.gpu


def colour(gb, A, n, seed=0):
    from graphblast_b200 import algorithm
    v = gb.Vector(n)
    ncolors, ms = algorithm.gc(v, A, seed, gb.Descriptor())
    assert ms >= 0
    return v.extractTuples(), ncolors


def check(gb, rp, ci, seeds=(0,), integer=False):
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, integer=integer)
    for seed in seeds:
        got, ncolors = colour(gb, A, n, seed)
        want, want_n, _ = greedy_oracle.gc(rp, ci, seed)
        assert np.array_equal(got, want.astype(np.float32)), seed
        assert ncolors == want_n, seed
    return A


@pytest.mark.parametrize("name", ["chesapeake", "test_cc", "test_bc", "test_sgm"])
def test_golden_graphs(gb, name):
    rp, ci = mtx_graph(name)
    if len(ci) == 0:              # test_sgm holds only self-loops: keep them
        n = len(rp) - 1
        rp, ci = np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32)
        assert greedy_oracle.gc(rp, ci, 0)[1] == 1
    check(gb, rp, ci, seeds=(0, 1, 99))


def test_star_with_many_leaves(gb):
    rp, ci = star_graph(150000)
    check(gb, rp, ci, seeds=(0, 5))


def test_path(gb):
    rp, ci = path_graph(100003)
    check(gb, rp, ci, seeds=(0, 3))


def test_ragged_rows(gb):
    rp, ci = ragged_graph()
    check(gb, rp, ci, seeds=(0, 17))


def test_clique_with_pendants_needs_several_windows(gb):
    """K300 plus a pendant on every clique vertex: 300 colours, five 64-colour
    windows, and a chain of 300 vertices each waiting on the one before."""
    k = 300
    src, dst = [], []
    for i in range(k):
        for j in range(i + 1, k):
            src.append(i)
            dst.append(j)
        src.append(i)
        dst.append(k + i)
    rp, ci = symmetric_csr(2*k, src, dst)
    check(gb, rp, ci, seeds=(0, 2))
    assert greedy_oracle.gc(rp, ci, 0)[1] == k


def test_complete_bipartite(gb):
    a, b = 70, 130
    src = np.repeat(np.arange(a), b)
    dst = a + np.tile(np.arange(b), a)
    rp, ci = symmetric_csr(a + b, src, dst)
    check(gb, rp, ci, seeds=(0, 4))


def test_self_loops_are_ignored(gb):
    rp, ci = orc.rmat_csr(10)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    # a loop on every third vertex, kept in sorted position
    loops = np.arange(0, n, 3)
    r = np.concatenate([rows, loops])
    c = np.concatenate([ci, loops])
    order = np.lexsort((c, r))
    r, c = r[order], c[order]
    lrp = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=n))]).astype(np.int32)
    A = make_matrix(gb, lrp, c.astype(np.int32))
    got, ncolors = colour(gb, A, n, 0)
    want, want_n, _ = greedy_oracle.gc(rp, ci, 0)
    assert np.array_equal(got, want.astype(np.float32)) and ncolors == want_n
    # the oracle ignores them too
    assert np.array_equal(greedy_oracle.gc(lrp, c, 0)[0], want)


def test_one_vertex(gb):
    A = gb.Matrix(1, 1)
    got, ncolors = colour(gb, A, 1)
    assert got.tolist() == [1.0] and ncolors == 1
    B = make_matrix(gb, np.array([0, 1], np.int32), np.array([0], np.int32))   # a loop
    got, ncolors = colour(gb, B, 1)
    assert got.tolist() == [1.0] and ncolors == 1


def test_empty_graph_is_not_constructible_through_the_c_abi(gb):
    """n = 0 colours with 0 colours in C++ (and the oracle); the C ABI has no
    0 x 0 matrix or 0-vector to hand it."""
    assert greedy_oracle.gc(np.zeros(1, np.int32), np.zeros(0, np.int32), 0)[1] == 0
    with pytest.raises(gb.GraphBLASError) as e:
        gb.Matrix(0, 0)
    assert e.value.info == gb.Info.GrB_INVALID_VALUE


def test_directed_matrix_is_coloured_as_its_symmetrised_pattern(gb):
    """CSR and explicit CSC of a directed pattern: the graph coloured is the
    undirected one."""
    n = 3000
    rng = np.random.RandomState(11)
    src = rng.randint(0, n, 20000).astype(np.int32)
    dst = (src + rng.randint(1, 200, 20000)).astype(np.int32) % n
    drp, dci = orc.build_csr(n, src, dst, False)
    srp, sci = orc.build_csr(n, src, dst, True)
    A = make_matrix(gb, drp, dci, symmetric=False)
    for seed in (0, 8):
        got, ncolors = colour(gb, A, n, seed)
        want, want_n, _ = greedy_oracle.gc(srp, sci, seed)
        assert np.array_equal(got, want.astype(np.float32)) and ncolors == want_n
    # the case tells the two apart: the CSR alone colours differently
    assert not np.array_equal(greedy_oracle.gc(drp, dci, 0)[0], greedy_oracle.gc(srp, sci, 0)[0])


@pytest.mark.parametrize("scale", [16, 18])
def test_rmat(gb, scale):
    rp, ci = orc.rmat_csr(scale)
    assert np.diff(rp).max() > 5000
    check(gb, rp, ci, seeds=(0, 1))


def test_int32_matrix(gb):
    rp, ci = orc.rmat_csr(12)
    check(gb, rp, ci, seeds=(0, 6), integer=True)


def test_same_call_twice_is_identical_and_seeds_differ(gb):
    rp, ci = orc.rmat_csr(14)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    a1, k1 = colour(gb, A, n, 0)
    a2, k2 = colour(gb, A, n, 0)
    assert np.array_equal(a1, a2) and k1 == k2
    b, _ = colour(gb, A, n, 1)
    assert not np.array_equal(a1, b)
    rows = np.repeat(np.arange(n), np.diff(rp))
    for c in (a1, b):
        assert not np.any(c[rows] == c[ci])


@pytest.mark.parametrize("graph", ["rmat", "no_entries"])
def test_launches_per_call(gb, graph):
    """One cooperative launch per call; zeroing the colours is no launch."""
    from graphblast_b200 import algorithm
    if graph == "rmat":
        rp, ci = orc.rmat_csr(14)
        A, n = make_matrix(gb, rp, ci), len(rp) - 1
    else:
        A, n = gb.Matrix(1000, 1000), 1000
    v = gb.Vector(n)
    assert launches_per_call(gb, lambda: algorithm.gc(v, A, 0, gb.Descriptor())) == 1


def test_refusals_leave_v_unchanged(gb):
    from graphblast_b200 import algorithm
    rp, ci = mtx_graph("test_cc")
    n = len(rp) - 1
    desc = gb.Descriptor()
    before = np.arange(n + 1, dtype=np.float32) + 0.5

    v = gb.Vector(n + 1)                                      # wrong size
    v.build(before)
    with pytest.raises(gb.GraphBLASError) as e:
        algorithm.gc(v, make_matrix(gb, rp, ci), 0, desc)
    assert e.value.info == gb.Info.GrB_DIMENSION_MISMATCH
    assert np.array_equal(v.extractTuples(), before)

    R = gb.Matrix(n, n + 1)                                   # not square
    rows = np.repeat(np.arange(n), np.diff(rp))
    R.build(rows, ci, np.ones(len(ci), np.float32))
    v = gb.Vector(n)
    v.build(before[:n])
    with pytest.raises(gb.GraphBLASError) as e:
        algorithm.gc(v, R, 0, desc)
    assert e.value.info == gb.Info.GrB_DIMENSION_MISMATCH
    assert np.array_equal(v.extractTuples(), before[:n])

    import torch                                              # no CSC, not symmetric
    D = gb.Matrix(n, n)
    D.build_device_csr(torch.from_numpy(rp).cuda(), torch.from_numpy(ci).cuda(),
                       torch.ones(len(ci), device="cuda"), len(ci), symmetric=False)
    with pytest.raises(gb.GraphBLASError) as e:
        algorithm.gc(v, D, 0, desc)
    assert e.value.info == gb.Info.GrB_UNINITIALIZED_OBJECT
    assert np.array_equal(v.extractTuples(), before[:n])
