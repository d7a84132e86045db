"""CPU checks of the k-truss and truss decomposition checker (tests/truss_oracle.c
through tests/truss_reference.py).

- Against networkx.k_truss for every k up to kmax + 1, on random graphs, the golden
  graphs and an R-MAT.
- Against a brute-force peel that recomputes every support from scratch (a dense
  A² ∘ A) and deletes all edges below k - 2 at once, for the k-truss supports and tau.
- Against closed forms: every edge of K_n has tau = n; a star or a tree has tau = 2;
  disjoint cliques keep their own sizes; a wheel has tau = 3 (4 for the wheel on 3
  rim vertices, which is K_4).
- The companion header include/graphblast_b200_ktruss.h: every declared symbol is
  exported and bound, it compiles as C99, and the refusals before the device check.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import oracle_binding as orc
import truss_reference as R
from support import csr, mtx_graph, symmetric_csr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HEADER = open(os.path.join(ROOT, "include", "graphblast_b200_ktruss.h")).read()


def random_graph(n, m, seed):
    rng = np.random.RandomState(seed)
    return symmetric_csr(n, rng.randint(0, n, m), rng.randint(0, n, m))


def clique_edges(vertices):
    v = np.asarray(vertices)
    i, j = np.triu_indices(len(v), 1)
    return v[i], v[j]


def clique(n):
    return symmetric_csr(n, *clique_edges(np.arange(n)))


def wheel(rim):
    """Hub 0 joined to a cycle of rim vertices 1..rim."""
    cyc = np.arange(1, rim + 1)
    src = np.concatenate([np.zeros(rim, int), cyc])
    dst = np.concatenate([cyc, np.roll(cyc, -1)])
    return symmetric_csr(rim + 1, src, dst)


def dense(rp, ci):
    n = len(rp) - 1
    A = np.zeros((n, n), np.int64)
    A[np.repeat(np.arange(n), np.diff(rp)), ci] = 1
    np.fill_diagonal(A, 0)
    return A


def brute_ktruss(A, k):
    """Dense support matrix of the k-truss: all edges below k - 2 deleted at once, the
    supports recomputed from scratch, until nothing changes."""
    A = A.copy()
    while True:
        S = (A @ A)*A
        drop = (A == 1) & (S < k - 2)
        if not drop.any():
            return A, S
        A[drop] = 0


def entry_values(rp, ci, M, keep):
    """M at each entry of (rp, ci), -1 where keep is 0 or on the diagonal."""
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    return np.where((keep[rows, ci] == 1) & (rows != ci), M[rows, ci], -1).astype(np.int32)


def brute_tau(A):
    tau = np.where(A == 1, 2, 0)
    k = 3
    while True:
        K, _ = brute_ktruss(A, k)
        if not K.any():
            return tau
        tau[K == 1] = k
        k += 1


SMALL = {
    "random_sparse": lambda: random_graph(60, 150, 1),
    "random_dense": lambda: random_graph(40, 400, 2),
    "random_mid": lambda: random_graph(80, 500, 3),
    "test_cc": lambda: mtx_graph("test_cc"),
    "chesapeake": lambda: mtx_graph("chesapeake"),
}


@pytest.mark.parametrize("name", sorted(SMALL))
def test_equals_brute_force(name):
    rp, ci = SMALL[name]()
    A = dense(rp, ci)
    tau, kmax = R.trussness(rp, ci)
    want_tau = brute_tau(A)
    assert np.array_equal(tau, entry_values(rp, ci, want_tau, A))
    assert kmax == (want_tau.max() if A.any() else 0)
    for k in range(2, kmax + 2):
        sup, kept = R.ktruss(rp, ci, k)
        K, S = brute_ktruss(A, k)
        assert np.array_equal(sup, entry_values(rp, ci, S, K)), "k = %d" % k
        assert kept == K.sum()//2


def test_self_loops_are_ignored():
    rp, ci = random_graph(50, 300, 4)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    assert not np.any(rows == ci)
    loops = np.arange(0, n, 3)
    S = csr(n, n, np.concatenate([rows, loops]), np.concatenate([ci, loops]),
            np.ones(len(ci) + len(loops)), np.float32)
    lp, lc = S.ptr, S.ind
    loops = np.repeat(np.arange(n), np.diff(lp)) == lc
    tau, kmax = R.trussness(lp, lc)
    want, want_kmax = R.trussness(rp, ci)
    assert kmax == want_kmax and np.all(tau[loops] == -1)
    assert np.array_equal(tau[~loops], want)
    sup, kept = R.ktruss(lp, lc, 4)
    want_sup, want_kept = R.ktruss(rp, ci, 4)
    assert kept == want_kept and np.array_equal(sup[~loops], want_sup)


def networkx_edges(rp, ci, k):
    nx = pytest.importorskip("networkx")
    n = len(rp) - 1
    G = nx.Graph()
    rows = np.repeat(np.arange(n), np.diff(rp))
    G.add_edges_from((int(u), int(v)) for u, v in zip(rows, ci) if u < v)
    return {(min(u, v), max(u, v)) for u, v in nx.k_truss(G, k).edges()}


NX = {
    "random_a": lambda: random_graph(200, 1500, 5),
    "random_b": lambda: random_graph(300, 1200, 6),
    "chesapeake": lambda: mtx_graph("chesapeake"),
    "test_bc": lambda: mtx_graph("test_bc"),
    "rmat10": lambda: orc.rmat_csr(10),
}


@pytest.mark.parametrize("name", sorted(NX))
def test_equals_networkx(name):
    rp, ci = NX[name]()
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    tau, kmax = R.trussness(rp, ci)
    assert kmax >= 3
    for k in range(2, kmax + 2):
        sup, kept = R.ktruss(rp, ci, k)
        mine = {(int(u), int(v)) for u, v, s in zip(rows, ci, sup) if u < v and s >= 0}
        assert mine == networkx_edges(rp, ci, k), "k = %d" % k
        assert kept == len(mine)
        assert mine == {(int(u), int(v)) for u, v, t in zip(rows, ci, tau) if u < v and t >= k}


@pytest.mark.parametrize("n", [2, 3, 4, 7, 12])
def test_clique(n):
    rp, ci = clique(n)
    tau, kmax = R.trussness(rp, ci)
    assert kmax == n and np.all(tau == n)
    sup, kept = R.ktruss(rp, ci, n)
    assert kept == n*(n - 1)//2 and np.all(sup == n - 2)
    sup, kept = R.ktruss(rp, ci, n + 1)
    assert kept == 0 and np.all(sup == -1)


def test_star_and_tree():
    rng = np.random.RandomState(7)
    for rp, ci in (symmetric_csr(101, np.zeros(100, int), np.arange(1, 101)),
                   symmetric_csr(500, rng.randint(0, np.arange(1, 500)), np.arange(1, 500))):
        tau, kmax = R.trussness(rp, ci)
        assert kmax == 2 and np.all(tau == 2)
        assert R.ktruss(rp, ci, 3)[1] == 0


def test_disjoint_cliques():
    sizes = [3, 5, 8, 4]
    src, dst, base = [], [], 0
    for s in sizes:
        a, b = clique_edges(np.arange(base, base + s))
        src.append(a)
        dst.append(b)
        base += s
    rp, ci = symmetric_csr(base + 2, np.concatenate(src), np.concatenate(dst))
    tau, kmax = R.trussness(rp, ci)
    assert kmax == 8
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    owner = np.repeat(np.arange(len(sizes)), sizes)
    assert np.array_equal(tau, np.asarray(sizes)[owner[rows]])


@pytest.mark.parametrize("rim", [3, 4, 5, 9])
def test_wheel(rim):
    rp, ci = wheel(rim)
    tau, kmax = R.trussness(rp, ci)
    want = 4 if rim == 3 else 3
    assert kmax == want and np.all(tau == want)


def test_empty_and_edgeless():
    tau, kmax = R.trussness(np.zeros(6, np.int32), np.zeros(0, np.int32))
    assert kmax == 0 and len(tau) == 0
    rp, ci = symmetric_csr(4, [1, 2], [1, 2])          # self-loops only
    tau, kmax = R.trussness(rp, ci)
    assert kmax == 0 and np.all(tau == -1)


def test_undirected_pattern():
    rp = np.array([0, 2, 2, 3], np.int32)
    ci = np.array([1, 2, 0], np.int32)                 # 0->1, 0->2, 2->0
    ptr, ind = R.undirected(rp, ci)
    assert ptr.tolist() == [0, 2, 3, 4] and ind.tolist() == [1, 2, 0, 0]


# ---------------------------------------------------------------------------
# the companion header's contract
# ---------------------------------------------------------------------------

def test_header_symbols_exported_and_bound():
    from graphblast_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    names = sorted(set(re.findall(r"\b(gb200_[a-z0-9_]+)\s*\(", HEADER)))
    assert names == ["gb200_ktruss", "gb200_ktruss_stats", "gb200_trussness"]
    for name in names:
        assert hasattr(lib, name), "missing export: " + name
    assert {s[0] for s in _lib.KTRUSS_SIGNATURES} == set(names)


def test_header_is_plain_c(tmp_path):
    src = str(tmp_path / "ktruss_header_check.c")
    with open(src, "w") as f:
        f.write('#include "graphblast_b200_ktruss.h"\nint main(void) { return 0; }\n')
    out = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror",
                          "-I", os.path.join(ROOT, "include"), "-fsyntax-only", src],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


import graphblast_b200 as _gb          # noqa: E402  (the codes; no device needed)

UNINITIALIZED = int(_gb.Info.GrB_UNINITIALIZED_OBJECT)
DOMAIN = int(_gb.Info.GrB_DOMAIN_MISMATCH)
INVALID_VALUE = int(_gb.Info.GrB_INVALID_VALUE)
PANIC = int(_gb.Info.GrB_PANIC)

# Host buffers standing in for handles in calls that refuse before reading them: ZERO
# is a matrix handle of neither element type; FAKE one that claims an FP32 matrix.
_ZERO = (C.c_ubyte*64)()
ZERO = C.cast(_ZERO, C.c_void_p)
_ONES = (C.c_ubyte*4096)(*([1]*4096))
_FAKE = (C.c_void_p*8)(C.cast(_ONES, C.c_void_p).value)
FAKE = C.cast(_FAKE, C.c_void_p)


def _lib():
    from graphblast_b200 import _lib as lib
    return lib.load()


def test_refusals_before_the_device_check():
    lib = _lib()
    d = ZERO                           # a descriptor that is never read
    ms = C.byref(C.c_float())
    ne = C.byref(C.c_longlong())
    km = C.byref(C.c_int())
    cases = [
        (lib.gb200_ktruss(None, FAKE, 3, d, ne, ms), UNINITIALIZED),
        (lib.gb200_ktruss(FAKE, None, 3, d, ne, ms), UNINITIALIZED),
        (lib.gb200_ktruss(FAKE, FAKE, 3, None, ne, ms), UNINITIALIZED),
        (lib.gb200_ktruss(None, ZERO, 1, d, ne, ms), UNINITIALIZED),
        (lib.gb200_ktruss(ZERO, FAKE, 3, d, ne, ms), DOMAIN),
        (lib.gb200_ktruss(FAKE, ZERO, 1, d, ne, ms), DOMAIN),       # before k
        (lib.gb200_ktruss(FAKE, FAKE, 1, d, ne, ms), INVALID_VALUE),
        (lib.gb200_ktruss(FAKE, FAKE, -5, d, ne, ms), INVALID_VALUE),
        (lib.gb200_trussness(None, FAKE, d, km, ms), UNINITIALIZED),
        (lib.gb200_trussness(FAKE, None, d, km, ms), UNINITIALIZED),
        (lib.gb200_trussness(FAKE, FAKE, None, km, ms), UNINITIALIZED),
        (lib.gb200_trussness(ZERO, FAKE, d, km, ms), DOMAIN),
        (lib.gb200_trussness(FAKE, ZERO, d, km, ms), DOMAIN),
    ]
    for i, (got, want) in enumerate(cases):
        assert got == want, "case %d: %d, expected %d" % (i, got, want)


def test_compute_entries_panic_without_a_device():
    from conftest import _have_gpu
    if _have_gpu():
        pytest.skip("a device is present")
    ms = C.byref(C.c_float())
    assert _lib().gb200_ktruss(FAKE, FAKE, 2, ZERO, None, ms) == PANIC
    assert _lib().gb200_trussness(FAKE, FAKE, ZERO, None, ms) == PANIC
