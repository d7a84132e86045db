"""The minimum spanning forest checker (tests/msf_oracle.c through tests/msf_reference.py)
against brute force over every spanning forest of tiny graphs, against networkx on 300
seeded random graphs, and against closed forms; then the companion header
graphblast_b200_msf.h: its exports, bindings, a C99 compile, and the refusals that come
before the device check.  No device needed."""
import ctypes as C
import itertools
import os
import re
import subprocess

import numpy as np
import pytest

import msf_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "graphblast_b200_msf.h")).read()


def csr_of(n, rows, cols, vals):
    """CSR of the entries (rows, cols, vals); no entry twice."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    order = np.lexsort((cols, rows))
    rp = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n))]).astype(np.int32)
    return rp, cols[order].astype(np.int32), np.asarray(vals, np.float64)[order]


def sym_csr(n, edges):
    """CSR of the weighted edges [(u, v, w)] stored both ways with equal values."""
    r = [u for u, v, _ in edges] + [v for u, v, _ in edges]
    c = [v for u, v, _ in edges] + [u for u, v, _ in edges]
    w = [x for _, _, x in edges]*2
    return csr_of(n, r, c, w)


def forest_edges(f):
    """[(u, v, w)], u < v, of a result CSR."""
    rp, ci, val = f
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    keep = rows < ci
    return sorted(zip(rows[keep].tolist(), ci[keep].tolist(), val[keep].tolist()))


def canonical(rp, ci, val):
    """{(u, v): w} of the graph algorithm.msf defines: min of both directions, loops
    dropped, -0.0 as +0.0."""
    out = {}
    for i in range(len(rp) - 1):
        for k in range(rp[i], rp[i + 1]):
            j = int(ci[k])
            if j == i:
                continue
            e = (min(i, j), max(i, j))
            w = float(val[k]) + 0.0
            out[e] = min(out.get(e, w), w)
    return out


def components(n, edges):
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x
    for u, v in edges:
        a, b = find(u), find(v)
        parent[max(a, b)] = min(a, b)
    return [find(x) for x in range(n)]


def brute_force(n, graph):
    """The forest among all spanning forests of graph ({(u, v): w}) whose sorted keys
    (w, u, v) are lexicographically least, and the least total weight."""
    edges = sorted(graph)
    full = len(set(components(n, []))) - len(set(components(n, edges)))
    best, best_weight = None, None
    for sub in itertools.combinations(edges, full):
        if len(set(components(n, sub))) != n - full:
            continue                    # a cycle
        keys = sorted((graph[e],) + e for e in sub)
        if best is None or keys < best:
            best = keys
        w = sum(graph[e] for e in sub)
        best_weight = w if best_weight is None else min(best_weight, w)
    return sorted((u, v, w) for w, u, v in best), best_weight


# ---------------------------------------------------------------------------
# brute force
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("seed", range(40))
def test_brute_force_on_tiny_graphs(seed):
    """At most 12 edges, each stored one way, the other or both (with its own value),
    weights with ties, zeros of both signs and +inf, and self-loops."""
    rng = np.random.RandomState(seed)
    n = rng.randint(2, 8)
    pairs = [(i, j) for i in range(n) for j in range(i + 1, n)]
    rows, cols, vals = [], [], []
    for t in rng.choice(len(pairs), rng.randint(1, min(12, len(pairs)) + 1), replace=False):
        u, v = pairs[t]
        how = rng.randint(3)
        for a, b in ([(u, v)] if how == 0 else [(v, u)] if how == 1 else [(u, v), (v, u)]):
            rows.append(a)
            cols.append(b)
            vals.append(rng.choice([-2.0, 0.0, -0.0, 1.0, 1.0, 3.0, np.inf]))
    for x in set(rng.randint(0, n, 2).tolist()):
        rows.append(x)
        cols.append(x)
        vals.append(-5.0)
    rp, ci, val = csr_of(n, rows, cols, vals)
    graph = canonical(rp, ci, val)
    f, nf, weight = R.msf(rp, ci, val)
    want, want_weight = brute_force(n, graph)
    assert forest_edges(f) == want
    assert nf == len(want) and weight == want_weight


# ---------------------------------------------------------------------------
# networkx
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("seed", range(300))
def test_networkx_minimum_spanning_tree(seed):
    nx = pytest.importorskip("networkx")
    rng = np.random.RandomState(1000 + seed)
    n = rng.randint(1, 60)
    m = rng.randint(0, 3*n + 1)
    src, dst = rng.randint(0, n, m), rng.randint(0, n, m)
    w = rng.randint(1, 5, m).astype(np.float64)          # positive, heavy ties
    graph = {}
    for u, v, x in zip(src.tolist(), dst.tolist(), w.tolist()):
        if u != v:
            e = (min(u, v), max(u, v))
            graph[e] = min(graph.get(e, x), x)
    rp, ci, val = sym_csr(n, [(u, v, x) for (u, v), x in graph.items()])
    f, nf, weight = R.msf(rp, ci, val)
    G = nx.Graph()
    G.add_nodes_from(range(n))
    G.add_weighted_edges_from((u, v, x) for (u, v), x in graph.items())
    T = nx.minimum_spanning_tree(G)
    assert nf == T.number_of_edges()
    assert weight == T.size(weight="weight")
    got = forest_edges(f)
    assert all(graph[(u, v)] == x for u, v, x in got)
    assert components(n, [(u, v) for u, v, _ in got]) == components(n, list(T.edges()))


# ---------------------------------------------------------------------------
# closed forms
# ---------------------------------------------------------------------------

def test_path():
    n = 50
    edges = [(i, i + 1, float(i % 7) - 3) for i in range(n - 1)]
    f, nf, weight = R.msf(*sym_csr(n, edges))
    assert forest_edges(f) == edges and nf == n - 1
    assert weight == sum(e[2] for e in edges)


def test_star():
    n = 40
    edges = [(0, j, float(j)) for j in range(1, n)]
    f, nf, weight = R.msf(*sym_csr(n, edges))
    assert forest_edges(f) == edges and nf == n - 1 and weight == sum(range(1, n))
    rp, ci, val = f
    assert rp.tolist() == [0, n - 1] + list(range(n, 2*n - 1))


def test_cycle_with_one_heavy_edge():
    n = 30
    edges = [(i, i + 1, 1.0) for i in range(n - 1)] + [(0, n - 1, 9.0)]
    f, nf, weight = R.msf(*sym_csr(n, edges))
    assert forest_edges(f) == edges[:-1] and weight == n - 1


def test_equal_weights_are_the_lexicographic_kruskal_forest():
    rng = np.random.RandomState(3)
    n = 40
    pairs = sorted({(min(u, v), max(u, v)) for u, v in rng.randint(0, n, (120, 2)) if u != v})
    f, nf, _ = R.msf(*sym_csr(n, [(u, v, 2.0) for u, v in pairs]))
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x
    want = []
    for u, v in pairs:                                  # Kruskal in (min, max) order
        a, b = find(u), find(v)
        if a != b:
            parent[max(a, b)] = min(a, b)
            want.append((u, v, 2.0))
    assert forest_edges(f) == want and nf == len(want)


def test_disconnected_pieces_and_isolated_vertices():
    edges = [(0, 1, 5.0), (1, 2, 1.0), (0, 2, 2.0), (4, 5, 7.0), (7, 8, -1.0), (7, 9, -1.0)]
    f, nf, weight = R.msf(*sym_csr(11, edges))
    assert forest_edges(f) == [(0, 2, 2.0), (1, 2, 1.0), (4, 5, 7.0), (7, 8, -1.0), (7, 9, -1.0)]
    assert nf == 5 and weight == 8.0


def test_min_of_both_directions_zero_sign_and_loops():
    # A(0,1) = 3, A(1,0) = -0.0, A(1,2) only, loops on 0 and 2
    rp, ci, val = csr_of(3, [0, 0, 1, 1, 2], [0, 1, 0, 2, 2], [1.0, 3.0, -0.0, 4.0, 8.0])
    f, nf, weight = R.msf(rp, ci, val)
    assert forest_edges(f) == [(0, 1, 0.0), (1, 2, 4.0)] and nf == 2 and weight == 4.0
    assert not np.signbit(f[2]).any()


def test_empty_cases_and_nan():
    f, nf, weight = R.msf(np.zeros(1, np.int32), np.zeros(0, np.int32), np.zeros(0))
    assert nf == 0 and weight == 0.0 and f[0].tolist() == [0]
    rp, ci, val = csr_of(3, [0, 1], [0, 1], [np.nan, 1.0])    # a NaN self-loop is fine
    assert R.msf(rp, ci, val)[1] == 0
    with pytest.raises(ValueError):
        R.msf(*csr_of(2, [0], [1], [np.nan]))


# ---------------------------------------------------------------------------
# the companion header's contract
# ---------------------------------------------------------------------------

def test_header_symbols_exported_and_bound():
    from graphblast_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    names = sorted(set(re.findall(r"\b(gb200_[a-z0-9_]+)\s*\(", HEADER)))
    assert names == ["gb200_msf", "gb200_msf_stats"]
    for name in names:
        assert hasattr(lib, name), "missing export: " + name
    assert {s[0] for s in _lib.MSF_SIGNATURES} == set(names)


def test_header_is_plain_c(tmp_path):
    src = str(tmp_path / "msf_header_check.c")
    with open(src, "w") as f:
        f.write('#include "graphblast_b200_msf.h"\nint main(void) { return 0; }\n')
    out = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror",
                          "-I", os.path.join(ROOT, "include"), "-fsyntax-only", src],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


import graphblast_b200 as _gb          # noqa: E402  (the codes; no device needed)

UNINITIALIZED = int(_gb.Info.GrB_UNINITIALIZED_OBJECT)
DOMAIN = int(_gb.Info.GrB_DOMAIN_MISMATCH)
PANIC = int(_gb.Info.GrB_PANIC)

# Host buffers standing in for handles in calls that refuse before reading them: ZERO
# is a matrix handle of neither element type; FAKE one that claims an FP32 matrix, and
# FAKE_INT one that claims an INT32 matrix.
_ZERO = (C.c_ubyte*64)()
ZERO = C.cast(_ZERO, C.c_void_p)
_ONES = (C.c_ubyte*4096)(*([1]*4096))
_FAKE = (C.c_void_p*8)(C.cast(_ONES, C.c_void_p).value)
FAKE = C.cast(_FAKE, C.c_void_p)
_FAKE_INT = (C.c_void_p*8)(None, C.cast(_ONES, C.c_void_p).value)
FAKE_INT = C.cast(_FAKE_INT, C.c_void_p)


def _lib():
    from graphblast_b200 import _lib as lib
    return lib.load()


def test_refusals_before_the_device_check():
    lib = _lib()
    d = ZERO                           # a descriptor that is never read
    ms = C.byref(C.c_float())
    ne = C.byref(C.c_longlong())
    w = C.byref(C.c_double())
    cases = [
        (lib.gb200_msf(None, FAKE, d, ne, w, ms), UNINITIALIZED),
        (lib.gb200_msf(FAKE, None, d, ne, w, ms), UNINITIALIZED),
        (lib.gb200_msf(FAKE, FAKE, None, ne, w, ms), UNINITIALIZED),
        (lib.gb200_msf(None, ZERO, d, ne, w, ms), UNINITIALIZED),
        (lib.gb200_msf(ZERO, FAKE, d, ne, w, ms), DOMAIN),
        (lib.gb200_msf(FAKE, ZERO, d, ne, w, ms), DOMAIN),
        (lib.gb200_msf(FAKE, FAKE_INT, d, ne, w, ms), DOMAIN),
        (lib.gb200_msf(FAKE_INT, FAKE, d, ne, w, ms), DOMAIN),
    ]
    for i, (got, want) in enumerate(cases):
        assert got == want, "case %d: %d, expected %d" % (i, got, want)


def test_compute_entry_panics_without_a_device():
    from conftest import _have_gpu
    if _have_gpu():
        pytest.skip("a device is present")
    ms = C.byref(C.c_float())
    assert _lib().gb200_msf(FAKE, FAKE, ZERO, None, None, ms) == PANIC
    assert _lib().gb200_msf(FAKE_INT, FAKE_INT, ZERO, None, None, ms) == PANIC
