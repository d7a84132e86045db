"""The fused BFS without a host wait: algorithm.bfs only enqueues the traversal
unless timed=True, and the kernel itself adds its algorithmic bytes to the
profiler (one launch per traversal).  Levels are compared bit-exactly with the
oracle's BFS in all three mxvmodes."""
import ctypes as C

import numpy as np
import pytest

import oracle_binding as orc
from support import fused_stats, gb, make_matrix

pytestmark = pytest.mark.gpu

FUSED = dict(struconly=1, opreuse=1, earlyexit=1)


@pytest.fixture(scope="module")
def graphs():
    """(rp, ci, directed): a symmetric R-MAT with n not a multiple of 32 (its top
    rows cut off) and a directed R-MAT."""
    rp, ci = orc.rmat_csr(12)
    n = len(rp) - 1 - 21
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    keep = (rows < n) & (ci < n)
    cut_rp, cut_ci = orc.build_csr(n, rows[keep].astype(np.int32),
                                   ci[keep].astype(np.int32), True)
    src, dst = orc.rmat_edges(11, 8, seed=3)
    d_rp, d_ci = orc.build_csr(1 << 11, src, dst, False)
    return {"rmat12-cut": (cut_rp, cut_ci, False), "directed-rmat11": (d_rp, d_ci, True)}


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("name", ["rmat12-cut", "directed-rmat11"])
def test_two_traversals_queued_on_one_descriptor(gb, graphs, name, mode):
    """Two traversals from different sources into different vectors, issued back to
    back on one descriptor (the second reuses the first's scratch) with nothing
    waiting in between; then both results are read."""
    from graphblast_b200 import algorithm
    rp, ci, directed = graphs[name]
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, symmetric=not directed)
    deg = np.diff(rp)
    s1, s2 = int(np.argmax(deg)), int(np.nonzero(deg)[0][-1])
    desc = gb.Descriptor(mxvmode=mode, **FUSED)
    v1, v2 = gb.Vector(n), gb.Vector(n)
    assert algorithm.bfs(v1, A, s1, desc) is None
    assert algorithm.bfs(v2, A, s2, desc) is None
    assert np.array_equal(v1.extractTuples().astype(np.int32), orc.bfs(rp, ci, s1))
    assert np.array_equal(v2.extractTuples().astype(np.int32), orc.bfs(rp, ci, s2))
    assert fused_stats(desc, n)[0] > 0          # the fused kernel ran


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_timed_returns_the_device_time(gb, graphs, mode):
    from graphblast_b200 import algorithm
    rp, ci, _ = graphs["rmat12-cut"]
    n = len(rp) - 1
    assert n % 32 != 0
    A = make_matrix(gb, rp, ci)
    s = int(np.argmax(np.diff(rp)))
    v = gb.Vector(n)
    ms = algorithm.bfs(v, A, s, gb.Descriptor(mxvmode=mode, **FUSED), timed=True)
    assert isinstance(ms, float) and ms > 0.0
    assert np.array_equal(v.extractTuples().astype(np.int32), orc.bfs(rp, ci, s))


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_profiled_traversal_is_one_launch_and_counts_its_bytes(gb, graphs, mode):
    """With the profiler on, each traversal is one launch, and the bytes the kernel
    adds are those its work counters give (per pull level 12n + 4, 4 per inspected
    entry, 12 per pushed vertex, 8 per pushed edge and per vertex discovered
    pushing)."""
    from graphblast_b200 import _lib, algorithm
    lib = _lib.load()
    rp, ci, directed = graphs["directed-rmat11"]
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, symmetric=not directed)
    s = int(np.argmax(np.diff(rp)))
    desc = gb.Descriptor(mxvmode=mode, **FUSED)
    v = gb.Vector(n)
    algorithm.bfs(v, A, s, desc)                # builds the cached summaries
    gb.sync()
    runs = 3
    before = C.c_ulonglong(0)
    lib.gb200_launch_count(C.byref(before))
    lib.gb200_profile_enable(1)
    lib.gb200_profile_reset()
    try:
        for _ in range(runs):
            algorithm.bfs(v, A, s, desc)
        ms, launches, nbytes = C.c_double(0), C.c_longlong(0), C.c_double(0)
        lib.gb200_profile_read(1, C.byref(ms), C.byref(launches), C.byref(nbytes))
    finally:
        lib.gb200_profile_enable(0)
    after = C.c_ulonglong(0)
    lib.gb200_launch_count(C.byref(after))
    assert after.value - before.value == runs
    assert launches.value == runs and ms.value > 0.0
    st = fused_stats(desc, n)
    per_run = st[2] * (12 * n + 4) + 4 * st[1] + 12 * st[3] + 8 * st[4] + 8 * st[5]
    assert per_run > 0
    assert int(nbytes.value) == runs * per_run
    assert np.array_equal(v.extractTuples().astype(np.int32), orc.bfs(rp, ci, s))
