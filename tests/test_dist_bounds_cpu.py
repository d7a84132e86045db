"""CPU tests of the partition rules of the multi-GPU layer: partition_bounds never
returns an empty slice, and PeerExchange refuses bounds the kernels cannot run
(a bitmap slice that does not start on a multiple of 128 vertices, an empty slice)
before it touches the library or the process group."""
import numpy as np
import pytest

import oracle_binding as orc
import support
from graphblast_b200 import dist as gdist


def _check(b, n, world, align):
    assert len(b) == world + 1 and b[0] == 0 and b[-1] == n
    assert all(x % align == 0 for x in b[:-1]), b
    assert all(b[p] < b[p + 1] for p in range(world)), "an empty slice: %s" % b


@pytest.mark.parametrize("align", [32, 128, 1024])
def test_no_empty_slice(align):
    graphs = [orc.rmat_csr(12), support.star_graph(5000), support.path_graph(3000),
              support.ragged_graph()]
    rng = np.random.RandomState(2)
    # a few rows holding nearly all the entries, the rest empty
    heavy = rng.randint(0, 200, 20000)
    graphs.append(support.symmetric_csr(8192, np.zeros(20000, np.int32) + heavy % 3,
                                        heavy + 300))
    for rp, _ in graphs:
        n = len(rp) - 1
        for world in range(1, 9):
            if n < world * align:
                continue
            for weight in (0.0, 1e9):
                _check(gdist.partition_bounds(rp, world, align=align, row_weight=weight),
                       n, world, align)


def test_exactly_one_block_per_rank():
    """n = world * align: every rank gets one block, whatever the row costs."""
    for world in (2, 3, 4):
        rp, _ = support.star_graph(world * 128 - 1)
        assert gdist.partition_bounds(rp, world, align=128) == [128 * p for p in range(world + 1)]


@pytest.mark.parametrize("world", [2, 3, 4])
def test_too_few_vertices_raise(world):
    for align in (128, 1024):
        rp, _ = support.path_graph(world * align - 1)
        with pytest.raises(ValueError, match="cannot give"):
            gdist.partition_bounds(rp, world, align=align)
    # the scale-10 R-MAT at 2 ranks and the default 1024 alignment
    rp, _ = orc.rmat_csr(10)
    with pytest.raises(ValueError):
        gdist.partition_bounds(rp, world)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_star_hub_row_gets_its_own_block(world):
    """The hub row holds half of the entries, more than 1/world of them: balancing
    entries puts the first bound inside the hub's block, which moves forward to
    the block's end instead of leaving rank 0 empty; the other bounds stay
    balanced on the leaves."""
    rp, _ = support.star_graph(5000)
    n = len(rp) - 1
    for align in (128, 1024):
        b = gdist.partition_bounds(rp, world, align=align)
        _check(b, n, world, align)
        assert b[1] == align
        # every later bound is the balanced one, or one block past the bound before
        # it when the balanced one falls inside the hub's share
        for p in range(2, world):
            balanced = abs(float(rp[b[p]]) - rp[-1] * p / world) <= align
            assert balanced or b[p] == b[p - 1] + align, b


def test_bounds_that_run_past_the_end_move_back():
    """Rows so heavy at the end that every balanced bound falls in the last block:
    the bounds step back so that every rank after them but the last still gets a
    block, and the last its 5 vertices."""
    n = 4 * 128 + 5
    rp, _ = support.symmetric_csr(n, np.full(n - 1, n - 1), np.arange(n - 1))
    for world in (2, 3, 4):
        b = gdist.partition_bounds(rp, world, align=128)
        _check(b, n, world, 128)
        assert b[1:world] == [512 - 128 * (world - 1 - p) for p in range(1, world)], b


def test_peer_exchange_refuses_bounds_before_connecting():
    """Refused before the library is loaded and before any collective: gb is not
    even consulted."""
    with pytest.raises(ValueError, match="multiple of 128 vertices for a bitmap"):
        gdist.PeerExchange(None, [0, 1024, 1056, 2000], None, bits=True)
    with pytest.raises(ValueError, match="multiple of 32"):
        gdist.PeerExchange(None, [0, 1000, 2000], None, bits=False)
    for bits in (True, False):
        with pytest.raises(ValueError, match="at least one vertex"):
            gdist.PeerExchange(None, [0, 1024, 1024, 3000], None, bits=bits)
        with pytest.raises(ValueError, match="at least one vertex"):
            gdist.PeerExchange(None, [0, 0, 4096], None, bits=bits)
        with pytest.raises(ValueError, match="at least one vertex"):
            gdist.PeerExchange(None, [0, 2048, 2048], None, bits=bits)
