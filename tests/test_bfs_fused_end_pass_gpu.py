"""Sizes around the end of a pull chunk, and graphs with more 512-row blocks than the
grid has warps, for the fused BFS (kernels/bfs_fused.cuh).  The end pass of the pull
instantiation requests a warp's next block's reach masks and level bytes before it
stores the current block's floats, so only a graph whose blocks outnumber the warps
hands loaded values from one block to the next; the deep tail puts rows of level 255
and more (stored one by one) into such a later block.  Levels are compared bit-exactly
with the oracle's BFS."""
import numpy as np
import pytest

import oracle_binding as orc
from support import bfs_levels, gb, make_matrix

pytestmark = pytest.mark.gpu

FUSED = dict(struconly=1, opreuse=1, earlyexit=1)
BLOCK = 512                     # rows of an end-pass block
WARPS_PER_SM = 2*512//32        # the pull instantiation's 2 CTAs of 512 threads per SM
TAIL = 300                      # path at the end of the ids: levels past 255


def grid_warps():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count*WARPS_PER_SM


def random_graph(n, seed, tail=0):
    """Random edges among the first n - tail vertices, three per vertex, then a path
    of the last tail vertices hanging off vertex 0."""
    rng = np.random.default_rng(seed)
    m = n - tail
    src = rng.integers(0, m, 3*m).astype(np.int32)
    dst = rng.integers(0, m, 3*m).astype(np.int32)
    keep = src != dst
    path = np.arange(m, n, dtype=np.int32)
    src = np.concatenate([src[keep], [0], path[:-1]]) if tail else src[keep]
    dst = np.concatenate([dst[keep], [m], path[1:]]) if tail else dst[keep]
    return orc.build_csr(n, src.astype(np.int32), dst.astype(np.int32), True)


def check(gb, n, mode, tail=0):
    from graphblast_b200 import algorithm
    rp, ci = random_graph(n, seed=n, tail=tail)
    A = make_matrix(gb, rp, ci)
    desc = gb.Descriptor(mxvmode=mode, max_niter=1000, **FUSED)
    v = gb.Vector(n)
    for s in (int(np.argmax(np.diff(rp))), n - 1):
        algorithm.bfs(v, A, s, desc)
        assert np.array_equal(v.extractTuples().astype(np.int32), bfs_levels(rp, ci, s)), \
            (mode, n, s)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n", [1023, 1025, 2049, 32*1024 + 1])
def test_sizes_around_a_chunk_end(gb, mode, n):
    check(gb, n, mode)


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("extra", [1, 33, BLOCK - 1])
def test_more_end_pass_blocks_than_warps(gb, mode, extra):
    """Two blocks per warp and a partial third for some: the last rows, a path
    reached at levels past 255, lie in blocks whose loads went out a block early."""
    check(gb, 2*grid_warps()*BLOCK + extra, mode, tail=TAIL)
