"""Maximal independent set on the device (algorithm::mis, gb200_mis) against the CPU
greedy MIS (tests/mis_oracle.c orc_mis), entry for entry.

The set is the greedy MIS in decreasing priority order over the candidates, so it
does not depend on launch shape or timing and every entry can be compared exactly.
The graphs cover the kernel's classes: lists a lane takes alone and lists a warp
takes, the sweeps (more than 32 undecided vertices per resident warp) and the tail, a
long blocking chain, empty and isolated rows, self-loops, a directed matrix read
through its CSR and its CSC, and dense, sparse and aliased candidate vectors.
"""
import os

import numpy as np
import pytest

import greedy_oracle
import oracle_binding as orc
from test_parity_gpu import make_matrix, path_graph, ragged_graph, star_graph

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
M32 = np.uint64(0xFFFFFFFF)


@pytest.fixture(scope="module")
def gb():
    import graphblast_b200 as g
    g.init(0)
    return g


def np_hash(seed, v):
    """The priority hash of kernels/greedy_schedule.cuh over an array of vertices."""
    x = (np.asarray(v, np.uint64) ^ np.uint64((seed*0x9E3779B9) & 0xFFFFFFFF)) & M32
    x ^= x >> np.uint64(16)
    x = (x*np.uint64(0x85EBCA6B)) & M32
    x ^= x >> np.uint64(13)
    x = (x*np.uint64(0xC2B2AE35)) & M32
    return x ^ (x >> np.uint64(16))


def run_mis(gb, A, n, seed=0, candidates=None, v=None):
    from graphblast_b200 import algorithm
    v = gb.Vector(n) if v is None else v
    nmembers, ms = algorithm.mis(v, A, seed, gb.Descriptor(), candidates)
    assert ms >= 0
    return v.extractTuples(), nmembers


def check(gb, rp, ci, seeds=(0,), dtype=None):
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, dtype=dtype)
    for seed in seeds:
        got, k = run_mis(gb, A, n, seed)
        want, want_k, _ = greedy_oracle.mis(rp, ci, seed)
        assert np.array_equal(got, want.astype(np.float32)), seed
        assert k == want_k, seed
    return A


def mtx_graph(name):
    n, src, dst, _ = orc.read_mtx_edges(os.path.join(GOLDEN, name + ".mtx"))
    return orc.build_csr(n, src, dst, True)


def symmetric_csr(n, src, dst):
    return orc.build_csr(n, np.asarray(src, np.int32), np.asarray(dst, np.int32), True)


@pytest.mark.parametrize("name", ["chesapeake", "test_cc", "test_bc", "test_sgm"])
def test_golden_graphs(gb, name):
    rp, ci = mtx_graph(name)
    if len(ci) == 0:              # test_sgm holds only self-loops: keep them
        n = len(rp) - 1
        rp, ci = np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32)
        assert greedy_oracle.mis(rp, ci, 0)[1] == n
    check(gb, rp, ci, seeds=(0, 1, 99))


def test_star_with_many_leaves(gb):
    """More vertices than the tail takes; the hub is a warp's list.  With seed 0 a
    leaf outranks the hub, so every leaf joins; with seed 845704 the hub outranks all
    150 000 leaves and joins alone."""
    rp, ci = star_graph(150000)
    check(gb, rp, ci, seeds=(0, 5, 845704))
    assert greedy_oracle.mis(rp, ci, 0)[0][0] == 0
    member, size, _ = greedy_oracle.mis(rp, ci, 845704)
    assert member[0] == 1 and size == 1


def test_path(gb):
    rp, ci = path_graph(100003)
    check(gb, rp, ci, seeds=(0, 3))


def test_ragged_rows(gb):
    rp, ci = ragged_graph()
    check(gb, rp, ci, seeds=(0, 17))


def test_clique_with_pendants(gb):
    """K300 plus a pendant on every clique vertex: one clique vertex joins, and every
    other pendant."""
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
    assert greedy_oracle.mis(rp, ci, 0)[1] == k


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
    loops = np.arange(0, n, 3)                      # a loop on every third vertex
    r = np.concatenate([rows, loops])
    c = np.concatenate([ci, loops])
    order = np.lexsort((c, r))
    r, c = r[order], c[order]
    lrp = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=n))]).astype(np.int32)
    A = make_matrix(gb, lrp, c.astype(np.int32))
    got, k = run_mis(gb, A, n, 0)
    want, want_k, _ = greedy_oracle.mis(rp, ci, 0)
    assert np.array_equal(got, want.astype(np.float32)) and k == want_k
    assert np.array_equal(greedy_oracle.mis(lrp, c, 0)[0], want)


def test_one_vertex_and_no_edges(gb):
    A = gb.Matrix(1, 1)
    got, k = run_mis(gb, A, 1)
    assert got.tolist() == [1.0] and k == 1
    B = make_matrix(gb, np.array([0, 1], np.int32), np.array([0], np.int32))   # a loop
    got, k = run_mis(gb, B, 1)
    assert got.tolist() == [1.0] and k == 1
    # no stored entries: every candidate is a member
    n = 1000
    E = gb.Matrix(n, n)
    got, k = run_mis(gb, E, n, 3)
    assert np.all(got == 1) and k == n
    cand = (np.arange(n) % 3 == 0).astype(np.float32)
    c = gb.Vector(n)
    c.build(cand)
    got, k = run_mis(gb, E, n, 3, c)
    assert np.array_equal(got, cand) and k == int(cand.sum())


def test_directed_matrix_uses_its_symmetrised_pattern(gb):
    """CSR and explicit CSC of a directed pattern: the graph is the undirected one."""
    n = 3000
    rng = np.random.RandomState(11)
    src = rng.randint(0, n, 20000).astype(np.int32)
    dst = (src + rng.randint(1, 200, 20000)).astype(np.int32) % n
    drp, dci = orc.build_csr(n, src, dst, False)
    srp, sci = orc.build_csr(n, src, dst, True)
    A = make_matrix(gb, drp, dci, symmetric=False)
    for seed in (0, 8):
        got, k = run_mis(gb, A, n, seed)
        want, want_k, _ = greedy_oracle.mis(srp, sci, seed)
        assert np.array_equal(got, want.astype(np.float32)) and k == want_k
    # the case tells the two apart: the CSR alone gives another set
    assert not np.array_equal(greedy_oracle.mis(drp, dci, 0)[0], greedy_oracle.mis(srp, sci, 0)[0])


@pytest.mark.parametrize("scale", [16, 18])
def test_rmat(gb, scale):
    rp, ci = orc.rmat_csr(scale)
    assert np.diff(rp).max() > 5000
    check(gb, rp, ci, seeds=(0, 1))


def test_int32_matrix(gb):
    rp, ci = orc.rmat_csr(12)
    check(gb, rp, ci, seeds=(0, 6), dtype=gb.api.INT32)


def test_path_in_increasing_priority_order(gb):
    """A 20 000-vertex path whose vertices follow increasing priority: every vertex
    waits on the next one, so the tail resolves a chain of about 10 000 rounds."""
    n, seed = 20000, 21
    order = np.argsort(np.asarray(np_hash(seed, np.arange(n))), kind="stable")
    rp, ci = symmetric_csr(n, order[:-1], order[1:])
    _, _, depth = greedy_oracle.mis(rp, ci, seed)
    assert depth >= 9000
    check(gb, rp, ci, seeds=(seed,))


# ---------------------------------------------------------------------------
# candidate sets
# ---------------------------------------------------------------------------

def test_dense_candidates(gb):
    rp, ci = orc.rmat_csr(16)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    rng = np.random.RandomState(4)
    for seed, frac in ((0, 0.5), (3, 0.9), (7, 0.1)):
        cand = (rng.rand(n) < frac).astype(np.float32)*rng.choice([1, -2, 0.5], n)
        c = gb.Vector(n)
        c.build(cand.astype(np.float32))
        got, k = run_mis(gb, A, n, seed, c)
        want, want_k, _ = greedy_oracle.mis(rp, ci, seed, cand)
        assert np.array_equal(got, want.astype(np.float32)) and k == want_k, seed
        assert not np.array_equal(want, greedy_oracle.mis(rp, ci, seed)[0])
        assert c.getStorage() == gb.Storage.GrB_DENSE
        assert np.array_equal(c.extractTuples(), cand.astype(np.float32))


def test_sparse_candidates(gb):
    """Stored entries with a non-zero value are the candidates; stored zeros and
    absent entries are not."""
    rp, ci = orc.rmat_csr(18)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    rng = np.random.RandomState(8)
    ind = np.sort(rng.choice(n, n//3, replace=False)).astype(np.int32)
    val = rng.choice(np.float32([0, 1, 3.5, -1]), len(ind))
    c = gb.Vector(n)
    c.build(ind, val)
    assert c.getStorage() == gb.Storage.GrB_SPARSE
    cand = np.zeros(n, np.float32)
    cand[ind] = val
    for seed in (0, 2):
        got, k = run_mis(gb, A, n, seed, c)
        want, want_k, _ = greedy_oracle.mis(rp, ci, seed, cand)
        assert np.array_equal(got, want.astype(np.float32)) and k == want_k, seed
    assert c.getStorage() == gb.Storage.GrB_SPARSE and c.nvals() == len(ind)
    got_ind, got_val = c.extractTuples(sparse=True)
    assert np.array_equal(got_ind, ind) and np.array_equal(got_val, val)


def test_no_candidates_gives_an_empty_set(gb):
    rp, ci = orc.rmat_csr(14)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    c = gb.Vector(n)
    c.build(np.zeros(n, np.float32))
    got, k = run_mis(gb, A, n, 0, c)
    assert k == 0 and not got.any()
    s = gb.Vector(n)
    s.build(np.array([5, 9], np.int32), np.zeros(2, np.float32))      # stored zeros only
    got, k = run_mis(gb, A, n, 0, s)
    assert k == 0 and not got.any()
    assert s.nvals() == 2


@pytest.mark.parametrize("storage", ["dense", "sparse"])
def test_candidates_aliased_with_v(gb, storage):
    rp, ci = orc.rmat_csr(15)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    rng = np.random.RandomState(2)
    cand = (rng.rand(n) < 0.6).astype(np.float32)
    v = gb.Vector(n)
    if storage == "dense":
        v.build(cand)
    else:
        ind = np.nonzero(cand)[0].astype(np.int32)
        v.build(ind, cand[ind])
    got, k = run_mis(gb, A, n, 5, v, v=v)
    want, want_k, _ = greedy_oracle.mis(rp, ci, 5, cand)
    assert np.array_equal(got, want.astype(np.float32)) and k == want_k


# ---------------------------------------------------------------------------
# cross-checks and refusals
# ---------------------------------------------------------------------------

def test_equals_colour_class_one_on_the_device(gb):
    """Two independent device kernels agree: mis(seed) == (gc(seed) == 1)."""
    from graphblast_b200 import algorithm
    rp, ci = orc.rmat_csr(16)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    for seed in (0, 13):
        got, k = run_mis(gb, A, n, seed)
        colours = gb.Vector(n)
        algorithm.gc(colours, A, seed, gb.Descriptor())
        class1 = (colours.extractTuples() == 1).astype(np.float32)
        assert np.array_equal(got, class1) and k == int(class1.sum())


def test_same_call_twice_is_identical_and_seeds_differ(gb):
    rp, ci = orc.rmat_csr(14)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    a1, k1 = run_mis(gb, A, n, 0)
    a2, k2 = run_mis(gb, A, n, 0)
    assert np.array_equal(a1, a2) and k1 == k2
    b, _ = run_mis(gb, A, n, 1)
    assert not np.array_equal(a1, b)
    rows = np.repeat(np.arange(n), np.diff(rp))
    for m in (a1, b):
        assert not np.any((m[rows] == 1) & (m[ci] == 1))


def test_refusals_leave_v_unchanged(gb):
    from graphblast_b200 import algorithm
    rp, ci = mtx_graph("test_cc")
    n = len(rp) - 1
    desc = gb.Descriptor()
    before = np.arange(n + 1, dtype=np.float32) + 0.5
    A = make_matrix(gb, rp, ci)

    v = gb.Vector(n + 1)                                      # wrong size
    v.build(before)
    with pytest.raises(gb.GraphBLASError) as e:
        algorithm.mis(v, A, 0, desc)
    assert e.value.info == gb.Info.GrB_DIMENSION_MISMATCH
    assert np.array_equal(v.extractTuples(), before)

    R = gb.Matrix(n, n + 1)                                   # not square
    rows = np.repeat(np.arange(n), np.diff(rp))
    R.build(rows, ci, np.ones(len(ci), np.float32))
    v = gb.Vector(n)
    v.build(before[:n])
    with pytest.raises(gb.GraphBLASError) as e:
        algorithm.mis(v, R, 0, desc)
    assert e.value.info == gb.Info.GrB_DIMENSION_MISMATCH
    assert np.array_equal(v.extractTuples(), before[:n])

    c = gb.Vector(n + 1)                                      # wrong candidate size
    c.build(np.ones(n + 1, np.float32))
    with pytest.raises(gb.GraphBLASError) as e:
        algorithm.mis(v, A, 0, desc, c)
    assert e.value.info == gb.Info.GrB_DIMENSION_MISMATCH
    assert np.array_equal(v.extractTuples(), before[:n])

    import torch                                              # no CSC, not symmetric
    D = gb.Matrix(n, n)
    D.build_device_csr(torch.from_numpy(rp).cuda(), torch.from_numpy(ci).cuda(),
                       torch.ones(len(ci), device="cuda"), len(ci), symmetric=False)
    with pytest.raises(gb.GraphBLASError) as e:
        algorithm.mis(v, D, 0, desc)
    assert e.value.info == gb.Info.GrB_UNINITIALIZED_OBJECT
    assert np.array_equal(v.extractTuples(), before[:n])
