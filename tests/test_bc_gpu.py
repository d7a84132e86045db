"""Betweenness centrality on the device (algorithm.bc / gb200_bc) against the float64
restatement of tests/bc_reference.py.

Every entry equals float32(reference) or lies one float step from it, and an entry whose
reference is 0 is exactly 0.  All terms are positive, so fp64 sums in any order round to
within one step.  Covered: the golden graphs, a star whose hub list is split over
several warps, a long path (many levels), a ragged graph, random directed and symmetric
graphs, an R-MAT with a seeded sample of sources, batch boundaries, repeated sources, a
source with no out-edges, empty source lists and a matrix with no stored entries.  INT32
and FP32 A, and a symmetric pattern read through its CSR and CSC or marked symmetric,
give identical bytes; so do two calls.  The launches per call are the batches plus one.
The companion header is checked the way tests/test_capi_abi.py and
test_capi_refusals.py check the main header: every declared symbol is exported and
bound, the header compiles as C99, and the refusals come in order and leave v untouched.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import bc_reference as R
import oracle_binding as orc
from support import (Csr, csr, device_matrix, directed_csr, gb, launches_per_call,
                     make_matrix, mtx_graph, path_graph, ragged_graph, star_graph,
                     symmetric_csr)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HEADER = open(os.path.join(ROOT, "include", "graphblast_b200_bc.h")).read()
CHUNK = 1024                           # GB_BC_CHUNK: longer lists are split over warps


def run(gb, A, n, sources=None, v=None):
    from graphblast_b200 import algorithm
    v = gb.Vector(n) if v is None else v
    ms = algorithm.bc(v, A, gb.Descriptor(), sources=sources)
    assert ms >= 0
    assert v.getStorage() == gb.Storage.GrB_DENSE
    return np.asarray(v.extractTuples(), np.float32)


def check_close(got, want64):
    """got equals float32(want64) or is one float step from it; zeros are exact."""
    want = np.asarray(want64, np.float64).astype(np.float32)
    got = np.asarray(got, np.float32)
    assert got.shape == want.shape
    assert np.all(got[want == 0] == 0), "an entry off every counted path is not 0"
    steps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    bad = np.nonzero(steps > 1)[0]
    assert len(bad) == 0, "%d of %d entries differ, first %d: %r, want %r" % (
        len(bad), len(got), bad[0], got[bad[0]], want[bad[0]])


def check(gb, A, rp, ci, sources=None):
    got = run(gb, A, len(rp) - 1, sources)
    check_close(got, R.brandes(rp, ci, sources))
    return got


def random_graph(n, m, seed, symmetric):
    rng = np.random.RandomState(seed)
    src = rng.randint(0, n, m).astype(np.int32)
    dst = rng.randint(0, n, m).astype(np.int32)
    return (symmetric_csr if symmetric else directed_csr)(n, src, dst)


# name -> (rp, ci, symmetric pattern, sources: None for all, else a count drawn with a seed)
GRAPHS = {
    "chesapeake": lambda: mtx_graph("chesapeake") + (True, None),
    "test_bc": lambda: mtx_graph("test_bc") + (True, None),
    "test_cc": lambda: mtx_graph("test_cc") + (True, None),
    "star": lambda: star_graph(2*CHUNK + 500) + (True, None),
    "path": lambda: path_graph(3000) + (True, 40),
    "ragged": lambda: ragged_graph() + (True, None),
    "random_directed": lambda: random_graph(2000, 9000, 1, False) + (False, None),
    "random_directed_sparse": lambda: random_graph(3000, 3500, 2, False) + (False, 100),
    "random_symmetric": lambda: random_graph(2000, 5000, 3, True) + (True, None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_graphs(gb, name):
    rp, ci, symmetric, count = GRAPHS[name]()
    n = len(rp) - 1
    sources = None if count is None else np.random.RandomState(count).randint(0, n, count)
    A = make_matrix(gb, rp, ci, symmetric=symmetric, csc=True)
    got = check(gb, A, rp, ci, sources)
    assert got.max() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("scale,directed", [(13, False), (12, True)])
def test_rmat(gb, scale, directed):
    src, dst = orc.rmat_edges(scale, 16, 1)
    n = 1 << scale
    rp, ci = (directed_csr if directed else symmetric_csr)(n, src, dst)
    A = make_matrix(gb, rp, ci, symmetric=not directed, csc=True)
    deg = np.diff(rp)
    assert deg.max() > CHUNK or directed       # the hub's lists are split
    sources = np.random.RandomState(scale).choice(np.nonzero(deg > 0)[0], 100, replace=False)
    check(gb, A, rp, ci, sources)


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 31, 32, 33, 65])
def test_batch_boundaries(gb, count):
    rp, ci = orc.rmat_csr(11)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    sources = np.random.RandomState(count).randint(0, n, count)
    check(gb, A, rp, ci, sources)
    check(gb, A, rp, ci, list(range(n - count, n)))


@pytest.mark.gpu
def test_repeated_sources_and_a_dead_end(gb):
    """A repeated id counts once per entry, within a batch and across batches; a source
    with no out-edges contributes nothing."""
    rp, ci = random_graph(500, 1500, 4, False)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, symmetric=False, csc=True)
    deg = np.diff(rp)
    dead = int(np.nonzero(deg == 0)[0][0])
    hub = int(np.argmax(deg))
    sources = [hub, hub, 7, dead, hub] + [7]*30 + [hub]
    got = check(gb, A, rp, ci, sources)
    check_close(got, R.brandes(rp, ci, [hub]*4 + [7]*31))
    assert np.array_equal(run(gb, A, n, [dead]), np.zeros(n, np.float32))


@pytest.mark.gpu
def test_split_in_and_out_lists(gb):
    """x -> hub -> L leaves -> sink, directed, L > 2 chunks: the sink's in-list is split in
    the path-count pull and the hub's out-list in the dependency gather."""
    leaves = 3*CHUNK + 17
    hub, sink, x = 0, leaves + 1, leaves + 2
    n = leaves + 3
    ids = np.arange(1, leaves + 1)
    src = np.concatenate([[x], np.zeros(leaves, int), ids])
    dst = np.concatenate([[hub], ids, np.full(leaves, sink)])
    rp, ci = directed_csr(n, src.astype(np.int32), dst.astype(np.int32))
    A = make_matrix(gb, rp, ci, symmetric=False, csc=True)
    got = check(gb, A, rp, ci, [x, hub, x])
    assert np.isclose(got[hub], 2*(leaves + 1))         # on every path from x
    check(gb, A, rp, ci)


@pytest.mark.gpu
def test_no_sources_and_no_entries(gb):
    rp, ci = mtx_graph("chesapeake")
    n = len(rp) - 1
    v = gb.Vector(n)
    v.fill(3.0)
    assert np.array_equal(run(gb, make_matrix(gb, rp, ci), n, [], v=v), np.zeros(n, np.float32))
    E = gb.Matrix(100, 100)
    assert np.array_equal(run(gb, E, 100), np.zeros(100, np.float32))
    assert np.array_equal(run(gb, E, 100, [5, 5, 99]), np.zeros(100, np.float32))


@pytest.mark.gpu
def test_int32_and_symmetric_forms_give_the_same_bytes(gb):
    rp, ci = mtx_graph("test_bc")
    n = len(rp) - 1
    want = run(gb, make_matrix(gb, rp, ci), n)
    for A in (make_matrix(gb, rp, ci, integer=True),
              make_matrix(gb, rp, ci, symmetric=False, csc=True),
              make_matrix(gb, rp, ci, symmetric=False, csc=True, integer=True)):
        assert np.array_equal(run(gb, A, n).view(np.uint32), want.view(np.uint32))


@pytest.mark.gpu
def test_two_calls_give_identical_bytes(gb):
    rp, ci = orc.rmat_csr(12)
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    sources = np.random.RandomState(3).randint(0, n, 70)
    v = gb.Vector(n)
    first = run(gb, A, n, sources, v=v)
    assert np.array_equal(run(gb, A, n, sources, v=v).view(np.uint32), first.view(np.uint32))
    assert np.array_equal(run(gb, A, n, sources).view(np.uint32), first.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("count", [0, 1, 32, 33, 65])
def test_launches_per_call(gb, count):
    """One cooperative launch per batch of 32 sources, and the finish."""
    from graphblast_b200 import algorithm
    rp, ci = mtx_graph("chesapeake")
    n = len(rp) - 1
    A, v = make_matrix(gb, rp, ci), gb.Vector(n)
    sources = np.arange(count) % n
    batches = (count + 31)//32
    assert launches_per_call(gb, lambda: algorithm.bc(v, A, gb.Descriptor(), sources)) == \
        batches + 1


# ---------------------------------------------------------------------------
# the companion header's contract
# ---------------------------------------------------------------------------

def test_header_symbols_exported_and_bound():
    from graphblast_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    names = sorted(set(re.findall(r"\b(gb200_[a-z0-9_]+)\s*\(", HEADER)))
    assert names == ["gb200_bc"]
    for name in names:
        assert hasattr(lib, name), "missing export: " + name
    assert {s[0] for s in _lib.BC_SIGNATURES} == set(names)


def test_header_is_plain_c(tmp_path):
    src = str(tmp_path / "bc_header_check.c")
    with open(src, "w") as f:
        f.write('#include "graphblast_b200_bc.h"\nint main(void) { return 0; }\n')
    out = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror",
                          "-I", os.path.join(ROOT, "include"), "-fsyntax-only", src],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


import graphblast_b200 as _gb          # noqa: E402  (the codes; no device needed)

UNINITIALIZED = int(_gb.Info.GrB_UNINITIALIZED_OBJECT)
DOMAIN = int(_gb.Info.GrB_DOMAIN_MISMATCH)
INVALID_VALUE = int(_gb.Info.GrB_INVALID_VALUE)
INVALID_INDEX = int(_gb.Info.GrB_INVALID_INDEX)
DIMENSION = int(_gb.Info.GrB_DIMENSION_MISMATCH)
NOT_IMPLEMENTED = int(_gb.Info.GrB_NOT_IMPLEMENTED)
PANIC = int(_gb.Info.GrB_PANIC)

# Host buffers standing in for handles in calls that refuse before reading them: ZERO
# is a matrix handle of neither element type; FAKE one that claims an FP32 matrix whose
# every byte is 1, so that it reports 0x01010101 rows (nrows reads no pointer), which
# lets gb200_bc reach its device check.
_ZERO = (C.c_ubyte*64)()
ZERO = C.cast(_ZERO, C.c_void_p)
_ONES = (C.c_ubyte*4096)(*([1]*4096))
_FAKE = (C.c_void_p*8)(C.cast(_ONES, C.c_void_p).value)
FAKE = C.cast(_FAKE, C.c_void_p)
FAKE_ROWS = 0x01010101


def _lib():
    from graphblast_b200 import _lib as lib
    return lib.load()


def _ids(*ids):
    return (C.c_int*max(len(ids), 1))(*ids)


def test_refusals_before_the_device_check():
    lib = _lib()
    d = ZERO                           # a descriptor that is never read
    ms = C.byref(C.c_float())
    cases = [
        ([None, ZERO, _ids(0), 1, d, ms], UNINITIALIZED),
        ([ZERO, None, _ids(0), 1, d, ms], UNINITIALIZED),
        ([ZERO, ZERO, _ids(0), 1, None, ms], UNINITIALIZED),
        ([ZERO, ZERO, _ids(0), 1, d, ms], DOMAIN),
        ([ZERO, ZERO, None, -1, d, ms], DOMAIN),
        ([ZERO, FAKE, _ids(0), -1, d, ms], INVALID_VALUE),
        ([ZERO, FAKE, None, -1, d, ms], INVALID_VALUE),
        ([ZERO, FAKE, None, FAKE_ROWS - 1, d, ms], INVALID_INDEX),
        ([ZERO, FAKE, _ids(0, FAKE_ROWS), 2, d, ms], INVALID_INDEX),
        ([ZERO, FAKE, _ids(-1), 1, d, ms], INVALID_INDEX),
    ]
    for args, want in cases:
        got = lib.gb200_bc(*args)
        assert got == want, "gb200_bc%r: %d, expected %d" % (tuple(args), got, want)


def test_compute_entry_panics_without_a_device():
    from conftest import _have_gpu
    if _have_gpu():
        pytest.skip("a device is present")
    ms = C.byref(C.c_float())
    assert _lib().gb200_bc(ZERO, FAKE, None, FAKE_ROWS, ZERO, ms) == PANIC
    assert _lib().gb200_bc(ZERO, FAKE, _ids(0, FAKE_ROWS - 1), 2, ZERO, ms) == PANIC
    assert _lib().gb200_bc(ZERO, FAKE, _ids(), 0, ZERO, ms) == PANIC


@pytest.mark.gpu
def test_refusals_in_order_leave_v_untouched(gb):
    """Each refusal in the documented order, with later checks also failing where the
    arguments allow, and v (dense or sparse) unchanged after each."""
    from graphblast_b200 import algorithm
    rp, ci = mtx_graph("chesapeake")
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    rows = np.repeat(np.arange(n), np.diff(rp))
    upper = rows < ci                  # each edge one way: a non-symmetric A, no CSC
    D = device_matrix(gb, csr(n, n, rows[upper], ci[upper], np.ones(int(upper.sum())),
                              np.float32), csc=False)
    Rm = device_matrix(gb, Csr(n, n + 1, rp, ci, np.ones(len(ci), np.float32)))
    Dense = gb.Matrix(n, n)
    Dense.build_dense(np.ones((n, n), np.float32))
    desc = gb.Descriptor()
    v, s = gb.Vector(n), gb.Vector(n)
    v.fill(3.0)
    s.build(np.array([2], np.int32), np.float32([5.0]))
    small = gb.Vector(n - 1)
    small.fill(1.0)

    def code(V, M, ids, count):
        return _lib().gb200_bc(V._h, M._h, None if ids is None else _ids(*ids), count,
                               desc._h, C.byref(C.c_float()))

    cases = []
    for V in (v, s):
        cases += [
            (code(V, A, [0], -1), INVALID_VALUE),
            (code(V, Dense, [n], -1), INVALID_VALUE),            # before the ids
            (code(V, A, None, n - 1), INVALID_INDEX),
            (code(V, A, [0, n], 2), INVALID_INDEX),
            (code(V, A, [-1], 1), INVALID_INDEX),
            (code(V, Dense, [n], 1), INVALID_INDEX),              # before the matrix
            (code(V, Dense, [0], 1), NOT_IMPLEMENTED),
            (code(small, Dense, [0], 1), NOT_IMPLEMENTED),        # before sizes
            (code(V, Rm, [0], 1), DIMENSION),
            (code(small, A, [0], 1), DIMENSION),
            (code(small, D, [0], 1), DIMENSION),                  # before the CSC
            (code(V, D, [0], 1), UNINITIALIZED),
            (code(V, D, [], 0), UNINITIALIZED),
        ]
    for i, (got, want) in enumerate(cases):
        assert got == want, "case %d: %d, expected %d" % (i, got, want)
    assert np.all(v.extractTuples() == 3.0)
    assert v.getStorage() == gb.Storage.GrB_DENSE
    assert s.getStorage() == gb.Storage.GrB_SPARSE
    want_s = np.zeros(n, np.float32)
    want_s[2] = 5.0
    assert np.array_equal(s.extractTuples(), want_s)
    assert np.all(small.extractTuples() == 1.0)
    for bad in ([n], [-1], [2**40]):
        with pytest.raises(gb.api.GraphBLASError) as err:
            algorithm.bc(v, A, desc, bad)
        assert err.value.info == INVALID_INDEX
    assert np.all(v.extractTuples() == 3.0)
