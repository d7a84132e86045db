"""CPU checks of the betweenness-centrality restatement (tests/bc_reference.py).

- Against brute force on small graphs: all-pairs BFS distances and path counts, with
  sigma_st(v) = sigma_sv * sigma_vt when d(s, v) + d(v, t) = d(s, t), for all sources and
  for source lists with repeats, directed and symmetric, with self-loops and isolated
  vertices.
- Against networkx (skipped where it is not installed), all sources: on a directed graph
  bc equals betweenness_centrality(DiGraph, normalized=False); on a symmetric pattern it
  equals twice the undirected unnormalised value.  The golden graphs and random directed
  and symmetric graphs, disconnected ones included.
"""
import numpy as np
import pytest

import bc_reference as R
from support import csr, directed_csr, mtx_graph, symmetric_csr


def random_graph(n, m, seed, symmetric):
    rng = np.random.RandomState(seed)
    src = rng.randint(0, n, m).astype(np.int32)
    dst = rng.randint(0, n, m).astype(np.int32)
    return (symmetric_csr if symmetric else directed_csr)(n, src, dst)


def two_pieces(symmetric):
    """Two random pieces with no edge between them, and two isolated vertices."""
    rng = np.random.RandomState(11)
    src = np.concatenate([rng.randint(0, 20, 50), rng.randint(20, 45, 60)]).astype(np.int32)
    dst = np.concatenate([rng.randint(0, 20, 50), rng.randint(20, 45, 60)]).astype(np.int32)
    return (symmetric_csr if symmetric else directed_csr)(47, src, dst)


def close(x, y):
    return np.allclose(x, y, rtol=1e-12, atol=1e-12)


SMALL = {
    "directed": lambda: random_graph(30, 70, 1, False),
    "symmetric": lambda: random_graph(30, 45, 2, True),
    "sparse_directed": lambda: random_graph(40, 45, 3, False),
    "pieces": lambda: two_pieces(True),
    "pieces_directed": lambda: two_pieces(False),
    "path": lambda: symmetric_csr(12, np.arange(11), np.arange(1, 12)),
}


@pytest.mark.parametrize("name", sorted(SMALL))
def test_equals_brute_force(name):
    rp, ci = SMALL[name]()
    n = len(rp) - 1
    assert close(R.brandes(rp, ci), R.brute_force(rp, ci))
    rng = np.random.RandomState(n)
    sources = rng.randint(0, n, 9)
    sources[3] = sources[0]                          # a repeated source counts twice
    assert close(R.brandes(rp, ci, sources), R.brute_force(rp, ci, sources))
    assert close(R.brandes(rp, ci, []), np.zeros(n))


def test_self_loops_are_ignored():
    rp, ci = random_graph(25, 60, 4, False)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    assert not np.any(rows == ci)
    S = csr(n, n, np.concatenate([rows, np.arange(n)]), np.concatenate([ci, np.arange(n)]),
            np.ones(len(ci) + n), np.float32)
    rp2, ci2 = S.ptr, S.ind
    assert np.array_equal(R.brandes(rp2, ci2), R.brandes(rp, ci))


def test_blocks_of_sources_add_up():
    """The sum over a list is the sum over any split of it (the blocks of BLOCK)."""
    rp, ci = mtx_graph("test_cc")
    n = len(rp) - 1
    src = np.random.RandomState(5).randint(0, n, 2*R.BLOCK + 7)
    parts = R.brandes(rp, ci, src[:R.BLOCK]) + R.brandes(rp, ci, src[R.BLOCK:])
    assert close(R.brandes(rp, ci, src), parts)


def networkx_bc(rp, ci, directed):
    nx = pytest.importorskip("networkx")
    n = len(rp) - 1
    G = nx.DiGraph() if directed else nx.Graph()
    G.add_nodes_from(range(n))
    rows = np.repeat(np.arange(n), np.diff(rp))
    G.add_edges_from((int(u), int(v)) for u, v in zip(rows, ci) if u != v)
    got = nx.betweenness_centrality(G, normalized=False)
    return np.array([got[i] for i in range(n)])


NX = {
    "chesapeake": lambda: mtx_graph("chesapeake"),
    "test_bc": lambda: mtx_graph("test_bc"),
    "test_cc": lambda: mtx_graph("test_cc"),
    "random_symmetric": lambda: random_graph(300, 700, 6, True),
    "random_symmetric_sparse": lambda: random_graph(300, 200, 7, True),
    "random_directed": lambda: random_graph(300, 1200, 8, False),
    "random_directed_sparse": lambda: random_graph(300, 350, 9, False),
}


@pytest.mark.parametrize("name", sorted(NX))
def test_equals_networkx(name):
    rp, ci = NX[name]()
    n = len(rp) - 1
    got = R.brandes(rp, ci)
    rows = np.repeat(np.arange(n), np.diff(rp))
    A = np.zeros((n, n), bool)
    A[rows, ci] = True
    if name.startswith("random_directed"):
        assert not np.array_equal(A, A.T)
        want = networkx_bc(rp, ci, directed=True)
    else:
        assert np.array_equal(A, A.T)
        want = 2.0*networkx_bc(rp, ci, directed=False)
        assert np.allclose(got, networkx_bc(rp, ci, directed=True), rtol=1e-9, atol=1e-9)
    assert np.allclose(got, want, rtol=1e-9, atol=1e-9)
