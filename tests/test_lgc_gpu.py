"""Local graph clustering on the device (algorithm.lgc / gb200_lgc and the sweep cut
algorithm.lgc_sweep / gb200_lgc_sweep) against the host restatements of
tests/lgc_reference.py, bit for bit.

p, the residual r and the round count equal the restatement of the reference's CPU
checker exactly (compared as uint32 bit patterns) on every route: mxvmode 1 (sparse
rounds only), 2 (dense rounds only) and 0 (chosen per round, also with a lower
switchpoint).  The sweep's cluster, size and
conductance equal the host sweep run on the device's own p.  The companion header's
contract is checked the way tests/test_capi_abi.py and test_capi_refusals.py check the
main header's: every declared symbol is exported and bound, the header compiles as C99,
and the refusals come in order and leave their vectors untouched.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import lgc_reference as L
import oracle_binding as orc
from support import (Csr, csr, device_matrix, directed_csr, gb, launches_per_call,
                     make_matrix, mtx_graph, path_graph, star_graph)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HEADER = open(os.path.join(ROOT, "include", "graphblast_b200_lgc.h")).read()

MODES = [1, 2, 0]


def _run(gb, A, n, s, alpha, eps, mode=0, max_niter=None, switchpoint=None, p=None,
         r=None, residual=True):
    from graphblast_b200 import algorithm
    knobs = dict(mxvmode=mode)
    if max_niter is not None:
        knobs["max_niter"] = max_niter
    if switchpoint is not None:
        knobs["switchpoint"] = switchpoint
    p = gb.Vector(n) if p is None else p
    if residual:
        r = gb.Vector(n) if r is None else r
    rounds, ms = algorithm.lgc(p, A, s, alpha, eps, gb.Descriptor(**knobs),
                               residual=r if residual else None)
    assert ms >= 0
    assert p.getStorage() == gb.Storage.GrB_DENSE
    return p.extractTuples(), (r.extractTuples() if residual else None), rounds


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def check(gb, A, rp, ci, s, alpha, eps, modes=MODES, max_niter=10000, **kw):
    """The device's p, r and rounds equal the restatement's under each mode; on graphs
    of up to 20 000 vertices the restatement's p is also checked against the
    reference's own checker when it is built."""
    want_p, want_r, want_k, _ = L.push(rp, ci, s, alpha, eps, max_niter)
    n = len(rp) - 1
    if L.ref_lgc_available() and n <= 20000 and max_niter > 0:
        ref = L.ref_lgc(rp, ci, s, alpha, eps, want_k if want_k == max_niter else want_k + 1)
        assert np.array_equal(_bits(ref), _bits(want_p)), "restatement differs from ref_lgc"
    for mode in modes:
        p, r, k = _run(gb, A, n, s, alpha, eps, mode=mode, max_niter=max_niter, **kw)
        assert k == want_k, "mode %d: %d rounds, want %d" % (mode, k, want_k)
        bad = np.nonzero(_bits(p) != _bits(want_p))[0]
        assert len(bad) == 0, "mode %d: %d of p differ, first %d: %r vs %r" % (
            mode, len(bad), bad[0], p[bad[0]], want_p[bad[0]])
        assert np.array_equal(_bits(r), _bits(want_r)), "mode %d: r differs" % mode
    return want_p, want_k


def golden(name):
    rp, ci = mtx_graph(name)
    return rp, ci


# ---------------------------------------------------------------------------
# bit-exact runs
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["chesapeake", "test_bc", "test_cc"])
@pytest.mark.parametrize("params", ["driver", "0.01", "0.15"])
def test_golden_graphs(gb, name, params):
    rp, ci = golden(name)
    A = make_matrix(gb, rp, ci)
    alpha, eps = {"driver": (L.driver_alpha(len(ci)), 1e-7), "0.01": (0.01, 1e-6),
                  "0.15": (0.15, 1e-6)}[params]
    deg = np.diff(rp)
    for s in (int(np.argmax(deg)), int(np.nonzero(deg > 0)[0][-1])):
        check(gb, A, rp, ci, s, alpha, eps, max_niter=3000)


@pytest.mark.gpu
def test_sgm_self_loops_and_isolated_sources(gb):
    """test_sgm.mtx holds only self-loops; loaded as they are, every source has d = 1
    and pushes into itself; with them removed every source is isolated."""
    n = 10
    rp, ci = np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32)
    check(gb, make_matrix(gb, rp, ci), rp, ci, 3, 0.15, 1e-6)
    A = gb.Matrix.from_mtx(os.path.join(HERE, "golden", "test_sgm.mtx"), directed=2)
    rp2, ci2, _ = A.extract_csr()
    check(gb, A, rp2, ci2, 0, 0.15, 1e-6)


@pytest.mark.gpu
def test_isolated_source(gb):
    """d[s] = 0: s keeps pushing into nothing until its residual underflows to 0."""
    rp, ci = path_graph(50)
    rp = np.concatenate([rp, [rp[-1]]]).astype(np.int32)      # vertex 50, no entries
    A = make_matrix(gb, rp, ci)
    _, k = check(gb, A, rp, ci, 50, 0.01, 1e-6)
    assert k > 100


@pytest.mark.gpu
@pytest.mark.parametrize("hub", [True, False])
def test_star(gb, hub):
    rp, ci = star_graph(5000)
    A = make_matrix(gb, rp, ci)
    check(gb, A, rp, ci, 0 if hub else 4321, 0.15, 1e-6)
    check(gb, A, rp, ci, 0 if hub else 4321, 0.01, 1e-7, max_niter=400)


@pytest.mark.gpu
def test_long_path(gb):
    rp, ci = path_graph(20000)
    A = make_matrix(gb, rp, ci)
    check(gb, A, rp, ci, 10000, 0.01, 1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [14, 16])
def test_rmat(gb, scale):
    rp, ci = orc.rmat_csr(scale)
    A = make_matrix(gb, rp, ci)
    deg = np.diff(rp)
    rng = np.random.RandomState(scale)
    for s in (int(np.argmax(deg)), int(rng.choice(np.nonzero(deg > 0)[0]))):
        check(gb, A, rp, ci, s, 0.15, 1e-6)
        check(gb, A, rp, ci, s, 0.01, 1e-6)
    # the driver's alpha over a few hundred rounds, and the default route with a lower
    # switchpoint
    s = int(np.argmax(deg))
    check(gb, A, rp, ci, s, L.driver_alpha(len(ci)), 1e-7, modes=[0, 1, 2], max_niter=300)
    check(gb, A, rp, ci, s, 0.01, 1e-6, modes=[0], switchpoint=0.002)


def _directed():
    rng = np.random.RandomState(7)
    n = 3000
    src = rng.randint(0, n, 30000).astype(np.int32)
    dst = (rng.zipf(1.5, 30000) % n).astype(np.int32)
    return directed_csr(n, src, dst)


@pytest.mark.gpu
def test_directed_with_csc(gb):
    rp, ci = _directed()
    A = make_matrix(gb, rp, ci, symmetric=False, csc=True)
    deg = np.diff(rp)
    for s in (int(np.argmax(deg)), int(np.nonzero(deg > 0)[0][0])):
        check(gb, A, rp, ci, s, 0.15, 1e-6)
        check(gb, A, rp, ci, s, 0.01, 1e-6)


@pytest.mark.gpu
def test_directed_without_csc_is_refused(gb):
    from graphblast_b200 import algorithm
    rp, ci = _directed()
    A = make_matrix(gb, rp, ci, symmetric=False, csc=False)
    n = len(rp) - 1
    p = gb.Vector(n)
    p.fill(3.0)
    with pytest.raises(gb.api.GraphBLASError) as e:
        algorithm.lgc(p, A, 0, 0.15, 1e-6, gb.Descriptor())
    assert e.value.info == gb.Info.GrB_UNINITIALIZED_OBJECT
    assert np.all(p.extractTuples() == 3.0)


@pytest.mark.gpu
def test_int32_equals_fp32(gb):
    rp, ci = orc.rmat_csr(12)
    s = int(np.argmax(np.diff(rp)))
    want_p, _ = check(gb, make_matrix(gb, rp, ci, integer=True), rp, ci, s, 0.01, 1e-6)
    p, _, _ = _run(gb, make_matrix(gb, rp, ci), len(rp) - 1, s, 0.01, 1e-6)
    assert np.array_equal(_bits(p), _bits(want_p))


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [0, 1, 2, 7, 40])
def test_max_niter_cap(gb, cap):
    rp, ci = golden("chesapeake")
    A = make_matrix(gb, rp, ci)
    _, k = check(gb, A, rp, ci, 5, 0.01, 1e-7, max_niter=cap)
    assert k == max(cap, 0)
    if cap == 0:
        p, r, _ = _run(gb, A, len(rp) - 1, 5, 0.01, 1e-7, max_niter=0)
        assert not p.any() and r[5] == 1.0 and np.count_nonzero(r) == 1


@pytest.mark.gpu
def test_repeated_calls_and_reused_vectors(gb):
    """Repeated calls give the same bits, into fresh vectors and into vectors that hold
    sparse or dense contents of another size of support."""
    rp, ci = orc.rmat_csr(13)
    A = make_matrix(gb, rp, ci)
    n = len(rp) - 1
    s = int(np.argmax(np.diff(rp)))
    want_p, want_r, _, _ = L.push(rp, ci, s, 0.15, 1e-6)
    p, r = gb.Vector(n), gb.Vector(n)
    p.build(np.array([1, 5], np.int32), np.array([7.0, 9.0], np.float32))
    r.fill(2.0)
    for _ in range(3):
        got_p, got_r, _ = _run(gb, A, n, s, 0.15, 1e-6, p=p, r=r)
        assert np.array_equal(_bits(got_p), _bits(want_p))
        assert np.array_equal(_bits(got_r), _bits(want_r))
    r.build(np.array([0], np.int32), np.array([4.0], np.float32))
    got_p, got_r, _ = _run(gb, A, n, s, 0.15, 1e-6, p=p, r=r, mode=2)
    assert np.array_equal(_bits(got_p), _bits(want_p))
    assert np.array_equal(_bits(got_r), _bits(want_r))


@pytest.mark.gpu
def test_without_residual(gb):
    rp, ci = golden("chesapeake")
    A = make_matrix(gb, rp, ci)
    want_p, _, want_k, _ = L.push(rp, ci, 0, 0.15, 1e-6)
    for mode in MODES:
        p, _, k = _run(gb, A, len(rp) - 1, 0, 0.15, 1e-6, mode=mode, residual=False)
        assert k == want_k and np.array_equal(_bits(p), _bits(want_p))


@pytest.mark.gpu
@pytest.mark.parametrize("graph", ["rmat", "no_entries"])
def test_launches_per_call(gb, graph):
    """The push is one cooperative launch.  The sweep of a support of more than one
    vertex runs the keys, the radix sort's eight 8-bit passes, the ranks, the deltas,
    the two passes of the minimum and the out pass; with no support, the keys and the
    out pass."""
    from graphblast_b200 import algorithm
    if graph == "rmat":
        rp, ci = orc.rmat_csr(14)
        A, n, s, sweep = make_matrix(gb, rp, ci), len(rp) - 1, int(np.argmax(np.diff(rp))), 38
    else:
        A, n, s, sweep = gb.Matrix(1000, 1000), 1000, 0, 2
    p, r, cluster = gb.Vector(n), gb.Vector(n), gb.Vector(n)
    assert launches_per_call(gb, lambda: algorithm.lgc(
        p, A, s, 0.15, 1e-6, gb.Descriptor(), residual=r)) == 1
    assert launches_per_call(
        gb, lambda: algorithm.lgc_sweep(cluster, p, A, gb.Descriptor())) == sweep


# ---------------------------------------------------------------------------
# sweep
# ---------------------------------------------------------------------------

def sweep_check(gb, A, rp, ci, p_host, p_vec=None):
    from graphblast_b200 import algorithm
    n = len(rp) - 1
    if p_vec is None:
        p_vec = gb.Vector(n)
        p_vec.build(np.asarray(p_host, np.float32))
    cl = gb.Vector(n)
    size, phi, ms = algorithm.lgc_sweep(cl, p_vec, A, gb.Descriptor())
    want_c, want_size, want_phi = L.sweep(rp, ci, p_host)
    assert ms >= 0
    assert size == want_size
    assert (np.isnan(phi) and np.isnan(want_phi)) or phi == want_phi, (phi, want_phi)
    assert np.array_equal(cl.extractTuples(), want_c)
    return size, phi


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["chesapeake", "test_bc", "rmat12", "directed"])
def test_sweep_of_lgc(gb, name):
    from graphblast_b200 import algorithm
    if name == "directed":
        rp, ci = _directed()
        A = make_matrix(gb, rp, ci, symmetric=False, csc=True)
    elif name == "rmat12":
        rp, ci = orc.rmat_csr(12)
        A = make_matrix(gb, rp, ci)
    else:
        rp, ci = golden(name)
        A = make_matrix(gb, rp, ci)
    n = len(rp) - 1
    s = int(np.argmax(np.diff(rp)))
    p = gb.Vector(n)
    algorithm.lgc(p, A, s, 0.15, 1e-5, gb.Descriptor())
    size, phi = sweep_check(gb, A, rp, ci, p.extractTuples(), p_vec=p)
    assert size >= 1 and 0.0 <= phi <= 1.0


@pytest.mark.gpu
def test_sweep_ties_empty_and_zero_denominator(gb):
    rp, ci = golden("chesapeake")
    A = make_matrix(gb, rp, ci)
    n = len(rp) - 1
    deg = np.diff(rp)
    # ties: p proportional to d gives one key for every vertex, ordered by id
    sweep_check(gb, A, rp, ci, deg.astype(np.float32)*0.25)
    # an empty support
    size, phi = sweep_check(gb, A, rp, ci, np.zeros(n, np.float32))
    assert size == 0 and np.isnan(phi)
    # the whole vertex set: the last prefix has denominator 0 and does not qualify
    sweep_check(gb, A, rp, ci, np.linspace(1, 2, n).astype(np.float32))
    # one isolated vertex with p > 0 (d = 0) is not in the support
    rp2 = np.concatenate([rp, [rp[-1]]]).astype(np.int32)
    A2 = make_matrix(gb, rp2, ci)
    p2 = np.zeros(n + 1, np.float32)
    p2[n] = 1.0
    size, phi = sweep_check(gb, A2, rp2, ci, p2)
    assert size == 0 and np.isnan(phi)
    # a two-vertex graph: every prefix of the support has min(vol, nnz - vol) = 0 or
    # qualifies once
    rp3, ci3 = np.array([0, 1, 2], np.int32), np.array([1, 0], np.int32)
    sweep_check(gb, make_matrix(gb, rp3, ci3), rp3, ci3, np.float32([0.5, 0.25]))


@pytest.mark.gpu
def test_sweep_of_a_sparse_p(gb):
    rp, ci = golden("chesapeake")
    A = make_matrix(gb, rp, ci)
    n = len(rp) - 1
    p = gb.Vector(n)
    p.build(np.array([3, 7, 11], np.int32), np.float32([0.5, 0.25, 0.125]))
    host = np.zeros(n, np.float32)
    host[[3, 7, 11]] = [0.5, 0.25, 0.125]
    sweep_check(gb, A, rp, ci, host, p_vec=p)


# ---------------------------------------------------------------------------
# the companion header's contract
# ---------------------------------------------------------------------------

def declared_symbols():
    return sorted(set(re.findall(r"\b(gb200_[a-z0-9_]+)\s*\(", HEADER)))


def test_header_symbols_exported_and_bound():
    from graphblast_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    names = declared_symbols()
    assert names == ["gb200_lgc", "gb200_lgc_sweep"]
    for name in names:
        assert hasattr(lib, name), "missing export: " + name
    assert {s[0] for s in _lib.LGC_SIGNATURES} == set(names)


def test_header_is_plain_c(tmp_path):
    src = str(tmp_path / "lgc_header_check.c")
    with open(src, "w") as f:
        f.write('#include "graphblast_b200_lgc.h"\nint main(void) { return 0; }\n')
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
# every byte is 1, so that it reports neither sparse nor dense storage and 0x01010101
# rows (nrows reads no pointer), which lets gb200_lgc reach its device check.
_ZERO = (C.c_ubyte*64)()
ZERO = C.cast(_ZERO, C.c_void_p)
_ONES = (C.c_ubyte*4096)(*([1]*4096))
_FAKE = (C.c_void_p*8)(C.cast(_ONES, C.c_void_p).value)
FAKE = C.cast(_FAKE, C.c_void_p)


def _lib():
    from graphblast_b200 import _lib as lib
    return lib.load()


def _outs():
    return C.byref(C.c_int()), C.byref(C.c_float())


def test_refusals_before_the_device_check():
    lib = _lib()
    d = ZERO                           # a descriptor that is never read
    k, ms = _outs()
    phi = C.byref(C.c_double())
    cases = [
        ("gb200_lgc", [None, None, ZERO, 0, 0.1, 1e-6, d, k, ms], UNINITIALIZED),
        ("gb200_lgc", [ZERO, None, None, 0, 0.1, 1e-6, d, k, ms], UNINITIALIZED),
        ("gb200_lgc", [ZERO, None, ZERO, 0, 0.1, 1e-6, None, k, ms], UNINITIALIZED),
        ("gb200_lgc", [ZERO, None, ZERO, 0, 0.1, 1e-6, d, k, ms], DOMAIN),
        ("gb200_lgc", [ZERO, ZERO, ZERO, -1, 2.0, 0.0, d, k, ms], DOMAIN),
        ("gb200_lgc_sweep", [None, ZERO, ZERO, d, k, phi, ms], UNINITIALIZED),
        ("gb200_lgc_sweep", [ZERO, None, ZERO, d, k, phi, ms], UNINITIALIZED),
        ("gb200_lgc_sweep", [ZERO, ZERO, None, d, k, phi, ms], UNINITIALIZED),
        ("gb200_lgc_sweep", [ZERO, ZERO, ZERO, None, k, phi, ms], UNINITIALIZED),
        ("gb200_lgc_sweep", [ZERO, ZERO, ZERO, d, k, phi, ms], DOMAIN),
    ]
    for name, args, want in cases:
        got = getattr(lib, name)(*args)
        assert got == want, "%s%r: %d, expected %d" % (name, tuple(args), got, want)


def test_compute_entries_panic_without_a_device():
    from conftest import _have_gpu
    if _have_gpu():
        pytest.skip("a device is present")
    k, ms = _outs()
    got = _lib().gb200_lgc_sweep(ZERO, ZERO, FAKE, ZERO, k, C.byref(C.c_double()), ms)
    assert got == PANIC
    got = _lib().gb200_lgc(ZERO, ZERO, FAKE, 0, 0.1, 1e-6, ZERO, k, ms)
    assert got == PANIC
    # the checks before the device check still come first with that handle
    assert _lib().gb200_lgc(ZERO, ZERO, FAKE, -1, 0.1, 1e-6, ZERO, k, ms) == INVALID_INDEX
    assert _lib().gb200_lgc(ZERO, ZERO, FAKE, 0, 0.0, 1e-6, ZERO, k, ms) == INVALID_VALUE


@pytest.mark.gpu
def test_refusals_in_order_leave_vectors_untouched(gb):
    """Each refusal in the documented order, with every later check also failing where the
    arguments allow, and p, r and cluster unchanged after each."""
    from graphblast_b200 import algorithm
    rp, ci = golden("chesapeake")
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci)
    rows = np.repeat(np.arange(n), np.diff(rp))
    upper = rows < ci                  # each edge one way: a non-symmetric A, no CSC
    D = device_matrix(gb, csr(n, n, rows[upper], ci[upper], np.ones(int(upper.sum())),
                              np.float32), csc=False)
    R = device_matrix(gb, Csr(n, n + 1, rp, ci, np.ones(len(ci), np.float32)))
    Dense = gb.Matrix(n, n)
    Dense.build_dense(np.ones((n, n), np.float32))
    desc = gb.Descriptor()
    p, r, cl = gb.Vector(n), gb.Vector(n), gb.Vector(n)
    p.fill(3.0)
    r.build(np.array([2], np.int32), np.float32([5.0]))
    cl.fill(7.0)
    small = gb.Vector(n - 1)
    small.fill(1.0)

    def lgc_code(P, Rv, M, s, alpha, eps):
        k, ms = _outs()
        return _lib().gb200_lgc(P._h, Rv._h if Rv is not None else None, M._h, s, alpha,
                                eps, desc._h, k, ms)

    def sweep_code(Cv, P, M):
        k, ms = _outs()
        return _lib().gb200_lgc_sweep(Cv._h, P._h, M._h, desc._h, k, C.byref(C.c_double()),
                                      ms)

    cases = [
        (lgc_code(p, r, A, n, 0.1, 1e-6), INVALID_INDEX),
        (lgc_code(p, r, A, -1, 0.0, 0.0), INVALID_INDEX),
        (lgc_code(p, r, A, 0, 0.0, 1e-6), INVALID_VALUE),
        (lgc_code(p, r, A, 0, 1.5, 1e-6), INVALID_VALUE),
        (lgc_code(p, r, A, 0, float("nan"), 1e-6), INVALID_VALUE),
        (lgc_code(p, r, A, 0, 0.1, 0.0), INVALID_VALUE),
        (lgc_code(p, r, A, 0, 0.1, float("nan")), INVALID_VALUE),
        (lgc_code(p, r, R, 0, 0.1, 1e-6), DIMENSION),
        (lgc_code(small, r, A, 0, 0.1, 1e-6), DIMENSION),
        (lgc_code(p, small, A, 0, 0.1, 1e-6), DIMENSION),
        (lgc_code(p, r, Dense, 0, 0.1, 1e-6), NOT_IMPLEMENTED),
        (lgc_code(small, small, Dense, 0, 0.1, 1e-6), NOT_IMPLEMENTED),   # before sizes
        (lgc_code(p, r, D, 0, 0.1, 1e-6), UNINITIALIZED),
        (lgc_code(p, p, A, 0, 0.1, 1e-6), INVALID_VALUE),
        (sweep_code(cl, p, R), DIMENSION),
        (sweep_code(small, p, A), DIMENSION),
        (sweep_code(cl, small, A), DIMENSION),
        (sweep_code(cl, p, Dense), NOT_IMPLEMENTED),
        (sweep_code(small, small, Dense), NOT_IMPLEMENTED),
        (sweep_code(cl, p, D), UNINITIALIZED),
        (sweep_code(p, p, A), INVALID_VALUE),
    ]
    for i, (got, want) in enumerate(cases):
        assert got == want, "case %d: %d, expected %d" % (i, got, want)
    assert np.all(p.extractTuples() == 3.0)
    assert p.getStorage() == gb.Storage.GrB_DENSE
    assert r.getStorage() == gb.Storage.GrB_SPARSE
    want_r = np.zeros(n, np.float32)
    want_r[2] = 5.0
    assert np.array_equal(r.extractTuples(), want_r)
    assert np.all(cl.extractTuples() == 7.0)
    assert np.all(small.extractTuples() == 1.0)
    with pytest.raises(gb.api.GraphBLASError):
        algorithm.lgc(p, A, 0, 0.1, 1e-6, desc, residual=p)
