"""How the fused BFS kernel (kernels/bfs_fused.cuh) writes the levels: one byte per
row while the traversal runs, the float result in one pass of 16-byte stores at the
end.  Covered here: traversals deeper than 254 levels (a row reached at level 255 or
later keeps byte 255 and gets its float when discovered), cut-offs on both sides of
that depth, one vector and descriptor reused between deep and shallow traversals,
sizes that are not a multiple of 4 or 16, and a result array that is not 16-byte
aligned.  Levels are compared bit-exactly with the oracle's BFS."""
import numpy as np
import pytest

import oracle_binding as orc
from support import bfs_levels, gb, make_matrix

pytestmark = pytest.mark.gpu

FUSED = dict(struconly=1, opreuse=1, earlyexit=1)
PATH = 330                      # path vertices: a traversal from vertex 0 is deeper
STAR = 2100                     # leaves of a star: more than GB_BFS_HEAVY (2048)


def csr_edges(rp, ci):
    return np.repeat(np.arange(len(rp) - 1, dtype=np.int32), np.diff(rp)), ci


def deep_graph():
    """A path 0..PATH-1 whose end is tied to the hub of an R-MAT-10 and to the centre
    of a star of STAR leaves, then a second R-MAT-10 on its own.  From 0 the
    traversal is ~PATH levels deep, the star's leaves are found by the grid-wide
    expansion of a vertex with more than 2048 neighbours, and the second R-MAT is
    unreached; from the second R-MAT's hub it is ~6 deep and the rest is unreached."""
    rp, ci = orc.rmat_csr(10)
    m = len(rp) - 1
    hub = int(np.argmax(np.diff(rp)))
    rs, rd = csr_edges(rp, ci)
    path = np.arange(PATH - 1, dtype=np.int32)
    centre = PATH + 2 * m
    leaves = np.arange(centre + 1, centre + 1 + STAR, dtype=np.int32)
    src = np.concatenate([path, [PATH - 1, PATH - 1], rs + PATH, rs + PATH + m,
                          np.full(STAR, centre, np.int32)])
    dst = np.concatenate([path + 1, [PATH + hub, centre], rd + PATH, rd + PATH + m,
                          leaves])
    n = centre + 1 + STAR
    rp2, ci2 = orc.build_csr(n, src.astype(np.int32), dst.astype(np.int32), True)
    return rp2, ci2, PATH + m + hub


def levels(v):
    return v.extractTuples().astype(np.int32)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_deeper_than_a_byte(gb, mode):
    from graphblast_b200 import algorithm
    rp, ci, _ = deep_graph()
    want = bfs_levels(rp, ci, 0)
    assert want.max() > 300 and want[-1] == PATH + 2        # a leaf of the star
    A = make_matrix(gb, rp, ci)
    v = gb.Vector(len(rp) - 1)
    algorithm.bfs(v, A, 0, gb.Descriptor(mxvmode=mode, max_niter=1000, **FUSED))
    assert np.array_equal(levels(v), want)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("cut", [260, 100])
def test_deep_traversal_cut_off(gb, mode, cut):
    from graphblast_b200 import algorithm
    rp, ci, _ = deep_graph()
    A = make_matrix(gb, rp, ci)
    v = gb.Vector(len(rp) - 1)
    algorithm.bfs(v, A, 0, gb.Descriptor(mxvmode=mode, max_niter=cut, **FUSED))
    assert np.array_equal(levels(v), bfs_levels(rp, ci, 0, cut)), (mode, cut)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_deep_and_shallow_share_vector_and_descriptor(gb, mode):
    """Neither the bytes nor the floats written directly for levels >= 255 of one
    traversal may show through in the next."""
    from graphblast_b200 import algorithm
    rp, ci, shallow = deep_graph()
    A = make_matrix(gb, rp, ci)
    v = gb.Vector(len(rp) - 1)
    desc = gb.Descriptor(mxvmode=mode, max_niter=1000, **FUSED)
    for s in (0, shallow, 0, shallow, PATH - 1, 0):
        algorithm.bfs(v, A, s, desc)
        assert np.array_equal(levels(v), bfs_levels(rp, ci, s)), (mode, s)


def small_graph(n, seed):
    """Random edges among the first 3/4 of n vertices, the last quarter isolated;
    n = 1: one vertex with a loop to itself."""
    if n == 1:
        return np.array([0, 1], np.int32), np.array([0], np.int32)
    rng = np.random.default_rng(seed)
    live = max(2, (3 * n) // 4)
    k = 3 * live
    src = rng.integers(0, live, k).astype(np.int32)
    dst = rng.integers(0, live, k).astype(np.int32)
    keep = src != dst
    return orc.build_csr(n, src[keep], dst[keep], True)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n", [1, 17, 33, 1003])
def test_sizes_not_a_multiple_of_16(gb, mode, n):
    from graphblast_b200 import algorithm
    rp, ci = small_graph(n, seed=n)
    A = make_matrix(gb, rp, ci)
    desc = gb.Descriptor(mxvmode=mode, **FUSED)
    deg = np.diff(rp)
    v = gb.Vector(n)
    for s in sorted({int(np.argmax(deg)), n - 1, 0}):
        algorithm.bfs(v, A, s, desc)
        assert np.array_equal(levels(v), bfs_levels(rp, ci, s)), (mode, n, s)


@pytest.mark.parametrize("mode", [0, 2])
def test_result_array_not_16_byte_aligned(gb, mode):
    """A vector that adopts a caller's array one float past an aligned address:
    every row is stored alone, and the floats around the array stay untouched."""
    import torch
    from graphblast_b200 import algorithm
    rp, ci = orc.rmat_csr(12)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    buf = torch.full((n + 8,), -7.0, dtype=torch.float32, device="cuda")
    v = gb.Vector(n)
    v.build_device(buf[1:n + 1])
    s = int(np.argmax(np.diff(rp)))
    algorithm.bfs(v, A, s, gb.Descriptor(mxvmode=mode, **FUSED))
    got = buf.cpu().numpy()
    assert np.array_equal(got[1:n + 1].astype(np.int32), bfs_levels(rp, ci, s))
    assert got[0] == -7.0 and np.all(got[n + 1:] == -7.0)
