"""The label propagation checker (tests/cdlp_oracle.c through tests/cdlp_reference.py)
against the numpy restatement of the same semantics on a few hundred seeded random
graphs, and against closed forms; then the companion header graphblast_b200_cdlp.h: its
exports, bindings, a C99 compile, and the refusals that come before the device check.
No device needed."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import cdlp_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "graphblast_b200_cdlp.h")).read()


def csr_of(n, src, dst):
    """CSR of the arcs (src, dst), duplicates removed, rows sorted."""
    src, dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
    key = np.unique(src*max(n, 1) + dst)
    rows, cols = key // max(n, 1), key % max(n, 1)
    rp = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n))]).astype(np.int32)
    return rp, cols.astype(np.int32)


def sym_csr(n, src, dst):
    return csr_of(n, np.concatenate([src, dst]), np.concatenate([dst, src]))


# ---------------------------------------------------------------------------
# the numpy restatement
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("seed", range(300))
def test_numpy_restatement(seed):
    """Directed and undirected random graphs with self-loops, sparse to dense, at a
    random iteration count."""
    rng = np.random.RandomState(seed)
    n = rng.randint(1, 80)
    m = rng.randint(0, 4*n + 1)
    src, dst = rng.randint(0, n, m), rng.randint(0, n, m)
    rp, ci = sym_csr(n, src, dst) if seed % 2 else csr_of(n, src, dst)
    max_iter = int(rng.choice([0, 1, 2, 3, 5, 10, 100]))
    got, k, it = R.cdlp(rp, ci, max_iter)
    want, want_k, want_it = R.numpy_cdlp(rp, ci, max_iter)
    assert np.array_equal(got, want)
    assert (k, it) == (want_k, want_it)
    assert k == len(np.unique(got))


# ---------------------------------------------------------------------------
# closed forms
# ---------------------------------------------------------------------------

def test_isolated_vertices_keep_their_ids():
    rp, ci = csr_of(7, [], [])
    for max_iter in (0, 1, 10):
        labels, k, it = R.cdlp(rp, ci, max_iter)
        assert labels.tolist() == list(range(7)) and k == 7
        assert it == min(max_iter, 1)


def test_max_iter_zero_is_the_identity():
    rp, ci = sym_csr(20, np.arange(19), np.arange(1, 20))
    labels, k, it = R.cdlp(rp, ci, 0)
    assert labels.tolist() == list(range(20)) and k == 20 and it == 0


@pytest.mark.parametrize("sizes", [[3], [3, 4, 5], [10, 3, 7, 3]])
def test_disjoint_cliques(sizes):
    """Each clique of size >= 3 ends labelled by its smallest id; iteration 2 reaches
    it, so iteration 3 is the first that changes nothing."""
    perm = np.random.RandomState(len(sizes)).permutation(sum(sizes))
    src, dst, groups, at = [], [], [], 0
    for s in sizes:
        ids = perm[at:at + s]
        at += s
        groups.append(ids)
        for a in ids:
            for b in ids:
                if a != b:
                    src.append(a)
                    dst.append(b)
    rp, ci = csr_of(sum(sizes), src, dst)
    labels, k, it = R.cdlp(rp, ci, 100)
    for ids in groups:
        assert (labels[ids] == ids.min()).all()
    assert k == len(sizes) and it == 3


@pytest.mark.parametrize("m", [2, 3, 10, 50])
def test_star_oscillates(m):
    """Centre c and leaves: after odd k the centre holds the smallest leaf id and the
    leaves the centre's id, after even k the reverse; never a fixpoint."""
    c = m // 2                                   # the centre is not the smallest id
    leaves = np.array([x for x in range(m + 1) if x != c])
    rp, ci = sym_csr(m + 1, np.full(m, c), leaves)
    for k in range(1, 8):
        labels, ncomm, it = R.cdlp(rp, ci, k)
        assert it == k
        if k % 2:
            assert labels[c] == leaves.min() and (labels[leaves] == c).all()
        else:
            assert labels[c] == c and (labels[leaves] == leaves.min()).all()
        assert ncomm == 2


def test_an_arc_both_ways_counts_twice():
    """0 -> 5, 5 -> 0, 0 -> 1, 0 -> 2: vertex 0 sees label 5 twice and 1 and 2 once each,
    so it takes 5; counting each neighbour once would give 1."""
    rp, ci = csr_of(6, [0, 5, 0, 0], [5, 0, 1, 2])
    labels, _, _ = R.cdlp(rp, ci, 1)
    assert labels[0] == 5
    assert labels.tolist() == [5, 0, 0, 3, 4, 0]
    assert R.numpy_cdlp(rp, ci, 1)[0].tolist() == labels.tolist()


def test_self_loops_are_ignored():
    # 0 only a loop; 1 - 2 with loops on both
    rp, ci = csr_of(3, [0, 1, 1, 2, 2], [0, 1, 2, 1, 2])
    labels, k, it = R.cdlp(rp, ci, 5)
    assert labels.tolist()[0] == 0 and it == 5       # 1 and 2 swap forever
    assert labels.tolist() == R.numpy_cdlp(rp, ci, 5)[0].tolist()


def test_empty_graph():
    labels, k, it = R.cdlp(np.zeros(1, np.int32), np.zeros(0, np.int32), 10)
    assert len(labels) == 0 and k == 0 and it == 1


# ---------------------------------------------------------------------------
# the companion header's contract
# ---------------------------------------------------------------------------

def test_header_symbols_exported_and_bound():
    from graphblast_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    names = sorted(set(re.findall(r"\b(gb200_[a-z0-9_]+)\s*\(", HEADER)))
    assert names == ["gb200_cdlp", "gb200_cdlp_stats"]
    for name in names:
        assert hasattr(lib, name), "missing export: " + name
    assert {s[0] for s in _lib.CDLP_SIGNATURES} == set(names)


def test_header_is_plain_c(tmp_path):
    src = str(tmp_path / "cdlp_header_check.c")
    with open(src, "w") as f:
        f.write('#include "graphblast_b200_cdlp.h"\nint main(void) { return 0; }\n')
    out = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror",
                          "-I", os.path.join(ROOT, "include"), "-fsyntax-only", src],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


import graphblast_b200 as _gb          # noqa: E402  (the codes; no device needed)

UNINITIALIZED = int(_gb.Info.GrB_UNINITIALIZED_OBJECT)
DOMAIN = int(_gb.Info.GrB_DOMAIN_MISMATCH)
PANIC = int(_gb.Info.GrB_PANIC)

# Host buffers standing in for handles in calls that refuse before reading them: ZERO
# is a handle of neither element type; FAKE one that claims an FP32 matrix or vector,
# and FAKE_INT one that claims an INT32 matrix.
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
    k = C.byref(C.c_int())
    it = C.byref(C.c_int())
    cases = [
        (lib.gb200_cdlp(None, FAKE, 10, d, k, it, ms), UNINITIALIZED),
        (lib.gb200_cdlp(FAKE, None, 10, d, k, it, ms), UNINITIALIZED),
        (lib.gb200_cdlp(FAKE, FAKE, 10, None, k, it, ms), UNINITIALIZED),
        (lib.gb200_cdlp(None, ZERO, -1, d, k, it, ms), UNINITIALIZED),
        (lib.gb200_cdlp(FAKE, ZERO, 10, d, k, it, ms), DOMAIN),
        (lib.gb200_cdlp(FAKE, ZERO, -1, d, k, it, ms), DOMAIN),
    ]
    for i, (got, want) in enumerate(cases):
        assert got == want, "case %d: %d, expected %d" % (i, got, want)


def test_compute_entry_panics_without_a_device():
    from conftest import _have_gpu
    if _have_gpu():
        pytest.skip("a device is present")
    ms = C.byref(C.c_float())
    assert _lib().gb200_cdlp(FAKE, FAKE, 10, ZERO, None, None, ms) == PANIC
    assert _lib().gb200_cdlp(FAKE, FAKE_INT, -1, ZERO, None, None, ms) == PANIC


def test_stats_take_null_pointers():
    assert _lib().gb200_cdlp_stats(None, None, None, None, None) == 0
