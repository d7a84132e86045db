"""CPU checks of the strongly connected components checker (tests/scc_reference.py)
and of the companion header include/graphblast_b200_scc.h.

- Against networkx's strongly_connected_components, mapped to minimum ids, on a few
  hundred seeded random digraphs across densities, with self-loops and isolated
  vertices.
- Against closed forms: a directed cycle is one component, a DAG has n, two cycles
  joined one way have two, and a bowtie has its core plus one per tendril vertex.
- The header: every declared symbol is exported and bound, it compiles as C99, and
  the refusals before the device check.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import scc_reference as R
from support import directed_csr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HEADER = open(os.path.join(ROOT, "include", "graphblast_b200_scc.h")).read()


def networkx_labels(n, src, dst):
    nx = pytest.importorskip("networkx")
    G = nx.DiGraph()
    G.add_nodes_from(range(n))
    G.add_edges_from(zip(src.tolist(), dst.tolist()))
    label = np.empty(n, np.int64)
    comps = list(nx.strongly_connected_components(G))
    for comp in comps:
        c = list(comp)
        label[c] = min(c)
    return label, len(comps)


@pytest.mark.parametrize("density", [0.5, 1.0, 1.5, 2.5, 4.0])
def test_equals_networkx_on_random_digraphs(density):
    for seed in range(60):
        rng = np.random.RandomState(1000*int(density*10) + seed)
        n = int(rng.randint(1, 80))
        m = int(density*n)
        src = rng.randint(0, n, m)
        dst = rng.randint(0, n, m)
        loops = rng.choice(n, min(n, 3), replace=False)   # self-loops, kept in the CSR
        src = np.concatenate([src, loops])
        dst = np.concatenate([dst, loops])
        pairs = np.unique(np.stack([src, dst], 1), axis=0)
        rp = np.concatenate([[0], np.cumsum(np.bincount(pairs[:, 0], minlength=n))])
        got, k = R.scc(rp, pairs[:, 1])
        want, want_k = networkx_labels(n, pairs[:, 0], pairs[:, 1])
        assert np.array_equal(got, want) and k == want_k, (density, seed)


def test_directed_cycle():
    n = 1000
    rp, ci = directed_csr(n, np.arange(n), (np.arange(n) + 1) % n)
    got, k = R.scc(rp, ci)
    assert k == 1 and not got.any()


def test_dag():
    n = 500
    rng = np.random.RandomState(3)
    a, b = rng.randint(0, n, 3000), rng.randint(0, n, 3000)
    keep = a != b
    src, dst = np.minimum(a, b)[keep], np.maximum(a, b)[keep]
    perm = rng.permutation(n)
    rp, ci = directed_csr(n, perm[src], perm[dst])
    got, k = R.scc(rp, ci)
    assert k == n and np.array_equal(got, np.arange(n))


def test_two_cycles_joined_one_way():
    cyc = np.arange(10)
    src = np.concatenate([cyc, cyc + 10, [3]])
    dst = np.concatenate([(cyc + 1) % 10, (cyc + 1) % 10 + 10, [15]])
    rp, ci = directed_csr(20, src, dst)
    got, k = R.scc(rp, ci)
    assert k == 2 and got.tolist() == [0]*10 + [10]*10


def test_bowtie():
    """Core 5..9 a cycle; in-tendril 0..4 a path into 5; out-tendril 10..14 a path out
    of 9; 15 isolated."""
    src = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 10, 11, 12, 13]
    dst = [1, 2, 3, 4, 5, 6, 7, 8, 9, 5, 10, 11, 12, 13, 14]
    rp, ci = directed_csr(16, src, dst)
    got, k = R.scc(rp, ci)
    assert k == 12
    assert got.tolist() == [0, 1, 2, 3, 4] + [5]*5 + list(range(10, 16))


def test_empty_and_loops_only():
    got, k = R.scc(np.zeros(1, np.int64), np.zeros(0, np.int64))
    assert k == 0 and len(got) == 0
    rp, ci = np.arange(5), np.arange(4)                 # four self-loops
    got, k = R.scc(rp, ci)
    assert k == 4 and np.array_equal(got, np.arange(4))


# ---------------------------------------------------------------------------
# the companion header's contract
# ---------------------------------------------------------------------------

def test_header_symbols_exported_and_bound():
    from graphblast_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    names = sorted(set(re.findall(r"\b(gb200_[a-z0-9_]+)\s*\(", HEADER)))
    assert names == ["gb200_scc", "gb200_scc_stats"]
    for name in names:
        assert hasattr(lib, name), "missing export: " + name
    assert {s[0] for s in _lib.SCC_SIGNATURES} == set(names)


def test_header_is_plain_c(tmp_path):
    src = str(tmp_path / "scc_header_check.c")
    with open(src, "w") as f:
        f.write('#include "graphblast_b200_scc.h"\nint main(void) { return 0; }\n')
    out = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror",
                          "-I", os.path.join(ROOT, "include"), "-fsyntax-only", src],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


import graphblast_b200 as _gb          # noqa: E402  (the codes; no device needed)

UNINITIALIZED = int(_gb.Info.GrB_UNINITIALIZED_OBJECT)
DOMAIN = int(_gb.Info.GrB_DOMAIN_MISMATCH)
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
    k = C.byref(C.c_int())
    cases = [
        (lib.gb200_scc(None, FAKE, d, k, ms), UNINITIALIZED),
        (lib.gb200_scc(FAKE, None, d, k, ms), UNINITIALIZED),
        (lib.gb200_scc(FAKE, FAKE, None, k, ms), UNINITIALIZED),
        (lib.gb200_scc(None, ZERO, d, k, ms), UNINITIALIZED),     # before the type
        (lib.gb200_scc(FAKE, ZERO, d, k, ms), DOMAIN),
    ]
    for i, (got, want) in enumerate(cases):
        assert got == want, "case %d: %d, expected %d" % (i, got, want)


def test_stats_take_null_pointers():
    assert _lib().gb200_scc_stats(None, None, None, None) == 0


def test_compute_entry_panics_without_a_device():
    from conftest import _have_gpu
    if _have_gpu():
        pytest.skip("a device is present")
    ms = C.byref(C.c_float())
    assert _lib().gb200_scc(FAKE, FAKE, ZERO, None, ms) == PANIC
