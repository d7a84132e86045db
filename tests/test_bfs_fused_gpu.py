"""The fused BFS kernel (kernels/bfs_fused.cuh) beyond one traversal of a symmetric
graph: state carried from one traversal to the next, directed graphs (the pushed
CSR and the pulled CSC differ), and the overflow of the push level's heavy-vertex
list.  Levels are compared bit-exactly with the oracle's BFS."""
import numpy as np
import pytest

import oracle_binding as orc
from support import bfs_levels, fused_stats, gb, make_matrix

pytestmark = pytest.mark.gpu

FUSED = dict(struconly=1, opreuse=1, earlyexit=1)


def two_components(scale):
    """Two R-MAT graphs side by side: a traversal from one leaves the other
    unreached, so a vector reused across traversals must be cleared there."""
    rp, ci = orc.rmat_csr(scale)
    m = len(rp) - 1
    rp2 = np.concatenate([rp, rp[1:] + rp[-1]]).astype(np.int32)
    ci2 = np.concatenate([ci, ci + m]).astype(np.int32)
    return rp2, ci2


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_vector_and_descriptor_reused_across_traversals(gb, mode):
    from graphblast_b200 import algorithm
    desc = gb.Descriptor(mxvmode=mode, **FUSED)
    big = two_components(14)
    small = two_components(10)
    for rp, ci in (big, small):
        n = len(rp) - 1
        deg = np.diff(rp)
        hub_a = int(np.argmax(deg[:n // 2]))
        hub_b = n // 2 + int(np.argmax(deg[n // 2:]))
        A = make_matrix(gb, rp, ci)
        v = gb.Vector(n)
        for s in (hub_a, hub_b, hub_a, int(np.argmin(deg))):
            algorithm.bfs(v, A, s, desc)
            assert fused_stats(desc, n)[0] > 0
            got = v.extractTuples().astype(np.int32)
            assert np.array_equal(got, bfs_levels(rp, ci, s)), (mode, n, s)
        # a cut-off traversal after a full one from the same source, checked
        # against the operation-by-operation loop too
        for cut in (3, 2, 1):
            cdesc = gb.Descriptor(mxvmode=mode, max_niter=cut, **FUSED)
            algorithm.bfs(v, A, hub_b, cdesc)
            got = v.extractTuples().astype(np.int32)
            assert np.array_equal(got, bfs_levels(rp, ci, hub_b, cut)), (mode, n, cut)
            w = gb.Vector(n)
            algorithm.bfs(w, A, hub_b, gb.Descriptor(mxvmode=mode, max_niter=cut))
            assert np.array_equal(got, w.extractTuples().astype(np.int32)), (mode, n, cut)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_directed_graph(gb, mode):
    from graphblast_b200 import algorithm
    scale = 14
    n = 1 << scale
    src, dst = orc.rmat_edges(scale, 8, seed=3)
    rp, ci = orc.build_csr(n, src, dst, False)
    assert not np.array_equal(rp, orc.build_csr(n, dst, src, False)[0])
    A = make_matrix(gb, rp, ci, symmetric=False)
    desc = gb.Descriptor(mxvmode=mode, **FUSED)
    deg = np.diff(rp)
    for s in (int(np.argmax(deg)), 0, int(np.argmin(deg))):
        v = gb.Vector(n)
        algorithm.bfs(v, A, s, desc)
        got = v.extractTuples().astype(np.int32)
        assert np.array_equal(got, bfs_levels(rp, ci, s)), (mode, s)
    stats = fused_stats(desc, n)
    assert stats[0] > 0
    if mode == 2:
        assert stats[2] == stats[0]


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_heavy_list_overflow(gb, mode):
    """Source 0 reaches 4100 hubs of degree 2050 in one level: more vertices of
    more than 2048 neighbours than the push level's list holds (4096), so the
    last ones are expanded by the warp that found them."""
    from graphblast_b200 import algorithm
    hubs, leaves = 4100, 2049
    hub_ids = np.arange(1, hubs + 1, dtype=np.int32)
    leaf_ids = np.arange(hubs + 1, hubs + 1 + leaves, dtype=np.int32)
    src = np.concatenate([np.zeros(hubs, np.int32), np.repeat(hub_ids, leaves)])
    dst = np.concatenate([hub_ids, np.tile(leaf_ids, hubs)])
    n = hubs + leaves + 8                       # a few isolated vertices at the end
    rp, ci = orc.build_csr(n, src, dst, True)
    A = make_matrix(gb, rp, ci)
    desc = gb.Descriptor(mxvmode=mode, **FUSED)
    v = gb.Vector(n)
    for s in (0, int(leaf_ids[0])):
        algorithm.bfs(v, A, s, desc)
        got = v.extractTuples().astype(np.int32)
        assert np.array_equal(got, bfs_levels(rp, ci, s)), (mode, s)
    if mode == 1:
        # from source 0: one vertex pushed at level 1, the hubs at level 2
        algorithm.bfs(v, A, 0, desc)
        stats = fused_stats(desc, n)
        assert stats[3] >= 1 + hubs and stats[4] >= hubs * (leaves + 1)
