"""Return codes of the C ABI's refusals, entry by entry, and the order of its checks.

Every entry point checks its arguments in a fixed order and answers the first
failed check with one graphblas::Info code.  A binding that maps codes to errors
relies on both the code and the order: a NULL handle must be reported as such with
or without a device, and an unknown semiring or monoid id or a wrong element type
must not turn into a different code.

The CPU part calls every declared entry whose argument checks come before the
device check with NULL handles, NULL out-pointers or out-of-range scalars; it means
the same with or without a device.  Without a device, the entries that reach the
device check must answer GrB_PANIC.  The GPU part uses real FP32 and INT32 handles
for the checks that come after it, or that need a handle to reach.
"""
import ctypes as C
import os

import numpy as np
import pytest

import graphblast_b200 as gb
from graphblast_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
CHESAPEAKE = os.path.join(HERE, "golden", "chesapeake.mtx")

SUCCESS = 0
UNINITIALIZED = int(gb.Info.GrB_UNINITIALIZED_OBJECT)
NULL_POINTER = int(gb.Info.GrB_NULL_POINTER)
INVALID_VALUE = int(gb.Info.GrB_INVALID_VALUE)
INVALID_INDEX = int(gb.Info.GrB_INVALID_INDEX)
DOMAIN = int(gb.Info.GrB_DOMAIN_MISMATCH)
DIMENSION = int(gb.Info.GrB_DIMENSION_MISMATCH)
NO_VALUE = int(gb.Info.GrB_NO_VALUE)
NOT_IMPLEMENTED = int(gb.Info.GrB_NOT_IMPLEMENTED)
PANIC = int(gb.Info.GrB_PANIC)

PLUS_TIMES = int(gb.Semiring.PlusMultiplies)
MIN_PLUS = int(gb.Semiring.MinimumPlus)
BAD_SEMIRINGS = (int(gb.Semiring.MinimumNotEqualTo) + 1, -1)      # 17, -1
BAD_MONOIDS = (int(gb.Monoid.NotEqualTo) + 1, -1)                 # 9, -1


def _have_gpu():
    import torch
    return torch.cuda.is_available()


def _out(ctype):
    return C.byref(ctype())


# ---------------------------------------------------------------------------
# CPU part: checks that come before the device check
# ---------------------------------------------------------------------------

# A host buffer standing in for a non-NULL device pointer in calls that refuse
# before reading it.
_BUF = (C.c_ubyte*64)()
P = C.cast(_BUF, C.c_void_p)


def before_device_cases(desc):
    """(entry, args, code) for refusals that come before the device check."""
    d = desc
    return [
        # descriptor (host only)
        ("gb200_desc_new", [None], NULL_POINTER),
        ("gb200_desc_free", [None], SUCCESS),
        ("gb200_desc_set", [None, 0, 0], NULL_POINTER),
        ("gb200_desc_set", [d, -1, 0], INVALID_VALUE),
        ("gb200_desc_set", [d, 11, 0], INVALID_VALUE),
        ("gb200_desc_get", [None, 0, _out(C.c_int)], NULL_POINTER),
        ("gb200_desc_get", [d, 0, None], NULL_POINTER),
        ("gb200_desc_get", [d, 11, _out(C.c_int)], INVALID_VALUE),
        ("gb200_desc_toggle", [None, 0], NULL_POINTER),
        ("gb200_desc_toggle", [d, 11], INVALID_VALUE),
        ("gb200_desc_set_knob", [None, b"niter", 1.0], NULL_POINTER),
        ("gb200_desc_set_knob", [d, None, 1.0], NULL_POINTER),
        ("gb200_desc_get_knob", [None, b"niter", _out(C.c_double)], NULL_POINTER),
        ("gb200_desc_get_knob", [d, None, _out(C.c_double)], NULL_POINTER),
        ("gb200_desc_get_knob", [d, b"niter", None], NULL_POINTER),
        # matrix
        ("gb200_matrix_new", [None, gb.api.FP32, 4, 4], NULL_POINTER),
        ("gb200_matrix_new", [None, gb.api.FP32, 0, 0], NULL_POINTER),
        ("gb200_matrix_new", [_out(C.c_void_p), gb.api.FP32, 0, 4], INVALID_VALUE),
        ("gb200_matrix_new", [_out(C.c_void_p), gb.api.FP32, 4, -1], INVALID_VALUE),
        ("gb200_matrix_new", [_out(C.c_void_p), 7, 0, 4], INVALID_VALUE),
        ("gb200_matrix_free", [None], SUCCESS),
        ("gb200_matrix_build_coo", [None, P, P, None, 1, 0], NULL_POINTER),
        ("gb200_matrix_build_coo", [None, P, P, None, 0, 0], NULL_POINTER),
        ("gb200_matrix_load_mtx", [None, gb.api.FP32, b"x.mtx", 0], NULL_POINTER),
        ("gb200_matrix_load_mtx", [_out(C.c_void_p), gb.api.FP32, None, 0], NULL_POINTER),
        ("gb200_matrix_build_coo_device", [None, None, None, None, 0, 0], NULL_POINTER),
        ("gb200_matrix_build_coo_device", [None, P, P, None, -1, 0], NULL_POINTER),
        ("gb200_matrix_adopt_csr", [None, P, P, P, 1], NULL_POINTER),
        ("gb200_matrix_adopt_csc", [None, P, P, P, 0], NULL_POINTER),
        ("gb200_matrix_nrows", [None, _out(C.c_int)], NULL_POINTER),
        ("gb200_matrix_nrows", [None, None], NULL_POINTER),
        ("gb200_matrix_ncols", [None, _out(C.c_int)], NULL_POINTER),
        ("gb200_matrix_nvals", [None, _out(C.c_int)], NULL_POINTER),
        ("gb200_matrix_extract_csr", [None, P, P, None], NULL_POINTER),
        ("gb200_matrix_build_dense", [None, P, 1], NULL_POINTER),
        ("gb200_matrix_adopt_dense", [None, P], NULL_POINTER),
        ("gb200_matrix_extract_dense", [None, P, 1], NULL_POINTER),
        ("gb200_matrix_dense_ptr", [None, _out(C.c_void_p)], NULL_POINTER),
        ("gb200_matrix_storage", [None, _out(C.c_int)], NULL_POINTER),
        ("gb200_matrix_tril", [None, d], NULL_POINTER),
        ("gb200_matrix_tril", [None, None], NULL_POINTER),
        ("gb200_matrix_apply_uniform_random", [None, d, 1, 1, 64], NULL_POINTER),
        ("gb200_host_uniform_weights", [1, 1, 64, 4, None], NULL_POINTER),
        ("gb200_pr_normalize", [None, 0.85, d], NULL_POINTER),
        # ingest and sorting
        ("gb200_ingest_coo", [4, 4, None, None, None, 0, 0, None, _out(C.c_longlong)],
         NULL_POINTER),
        ("gb200_ingest_coo", [4, 4, None, None, None, 1, 0, _out(C.c_void_p),
                              _out(C.c_longlong)], NULL_POINTER),
        ("gb200_ingest_coo", [0, 4, None, None, None, 0, 0, _out(C.c_void_p),
                              _out(C.c_longlong)], INVALID_VALUE),
        ("gb200_ingest_coo", [4, 4, None, None, None, -1, 0, _out(C.c_void_p),
                              _out(C.c_longlong)], INVALID_VALUE),
        ("gb200_ingest_export", [None, P, P, P], NULL_POINTER),
        ("gb200_ingest_free", [None], SUCCESS),
        ("gb200_csr_transpose_values", [4, 4, 0, None, P, P, P, P, P], NULL_POINTER),
        ("gb200_csr_transpose_values", [4, 4, 0, P, P, None, P, P, P], NULL_POINTER),
        ("gb200_sort_pairs_u64", [None, None, 0, 8], NULL_POINTER),
        ("gb200_sort_pairs_u64", [None, None, -1, 0], NULL_POINTER),
        ("gb200_sort_pairs_u64", [P, None, -1, 8], INVALID_VALUE),
        ("gb200_sort_pairs_u64", [P, None, 0, 0], INVALID_VALUE),
        ("gb200_sort_pairs_u64", [P, None, 0, 65], INVALID_VALUE),
        # vector
        ("gb200_vector_new", [None, gb.api.FP32, 8], NULL_POINTER),
        ("gb200_vector_new", [_out(C.c_void_p), gb.api.INT32, 8], DOMAIN),
        ("gb200_vector_new", [_out(C.c_void_p), 7, 0], DOMAIN),
        ("gb200_vector_new", [_out(C.c_void_p), gb.api.FP32, 0], INVALID_VALUE),
        ("gb200_vector_free", [None], SUCCESS),
        ("gb200_vector_fill", [None, 0.0], NULL_POINTER),
        ("gb200_vector_build_sparse", [None, P, P, 1], NULL_POINTER),
        ("gb200_vector_build_dense", [None, P, 1], NULL_POINTER),
        ("gb200_vector_adopt_dense", [None, P, 1], NULL_POINTER),
        ("gb200_vector_adopt_sparse", [None, P, P, 1], NULL_POINTER),
        ("gb200_vector_set_element", [None, 0.0, 0], NULL_POINTER),
        ("gb200_vector_size", [None, _out(C.c_int)], NULL_POINTER),
        ("gb200_vector_nvals", [None, _out(C.c_int)], NULL_POINTER),
        ("gb200_vector_storage", [None, _out(C.c_int)], NULL_POINTER),
        ("gb200_vector_extract_dense", [None, P, 1], NULL_POINTER),
        ("gb200_vector_extract_sparse", [None, P, P, _out(C.c_int)], NULL_POINTER),
        ("gb200_vector_swap", [None, None], NULL_POINTER),
        ("gb200_vector_dup", [None, None], NULL_POINTER),
        ("gb200_vector_clear", [None], NULL_POINTER),
        ("gb200_vector_sparse2dense", [None, 0.0, None], NULL_POINTER),
        ("gb200_vector_dense2sparse", [None, 0.0, d], NULL_POINTER),
        ("gb200_vector_device_ptr", [None, _out(C.c_void_p)], NULL_POINTER),
        ("gb200_vector_export_bits", [None, P, None], NULL_POINTER),
        # operations: a NULL operand is an uninitialised object
        ("gb200_vxm", [None, None, 0, PLUS_TIMES, None, None, d], UNINITIALIZED),
        ("gb200_mxv", [None, None, 0, PLUS_TIMES, None, None, d], UNINITIALIZED),
        ("gb200_mxm", [None, None, PLUS_TIMES, None, None, d], UNINITIALIZED),
        ("gb200_mxm", [None, None, BAD_SEMIRINGS[0], None, None, None], UNINITIALIZED),
        ("gb200_ewise_add", [None, None, PLUS_TIMES, None, None, d], UNINITIALIZED),
        ("gb200_ewise_add_scalar", [None, None, PLUS_TIMES, None, 1.0, d], UNINITIALIZED),
        ("gb200_ewise_mult", [None, None, PLUS_TIMES, None, None, d], UNINITIALIZED),
        ("gb200_ewise_add_matrix", [None, None, PLUS_TIMES, None, None, d], UNINITIALIZED),
        ("gb200_ewise_mult_matrix", [None, None, PLUS_TIMES, None, None, d], UNINITIALIZED),
        ("gb200_transpose", [None, None, None, d], UNINITIALIZED),
        ("gb200_assign_scalar", [None, None, 1.0, d], UNINITIALIZED),
        ("gb200_reduce_vector", [None, 0, None, d], UNINITIALIZED),
        ("gb200_reduce_vector", [_out(C.c_double), BAD_MONOIDS[0], None, d], UNINITIALIZED),
        ("gb200_reduce_matrix", [None, 0, None, d], UNINITIALIZED),
        ("gb200_reduce_matrix_rows", [None, 0, None, d], UNINITIALIZED),
        ("gb200_scatter", [None, None, 1.0, d], NULL_POINTER),
        ("gb200_assign_scatter", [None, None, None, d], NULL_POINTER),
        ("gb200_extract_gather", [None, None, None, d], NULL_POINTER),
        # algorithms
        ("gb200_bfs", [None, None, 0, d, None], UNINITIALIZED),
        ("gb200_bfs_stats", [None, 0, P], NULL_POINTER),
        ("gb200_bfs_stats", [d, 0, None], NULL_POINTER),
        ("gb200_sssp", [None, None, 0, d, None], UNINITIALIZED),
        ("gb200_pr", [None, None, 0.85, 1e-8, d, None], UNINITIALIZED),
        ("gb200_tc", [None, None, None, d, None], UNINITIALIZED),
        ("gb200_gc", [None, None, 0, d, None, None], UNINITIALIZED),
        ("gb200_mis", [None, None, 0, None, d, None, None], UNINITIALIZED),
        ("gb200_cc", [None, None, d, None, None], UNINITIALIZED),
        # measurement hooks and graph generation
        ("gb200_profile_read", [0, None, _out(C.c_longlong), _out(C.c_double)], NULL_POINTER),
        ("gb200_profile_read", [-1, _out(C.c_double), _out(C.c_longlong), _out(C.c_double)],
         INVALID_VALUE),
        ("gb200_profile_read", [5, _out(C.c_double), _out(C.c_longlong), _out(C.c_double)],
         INVALID_VALUE),
        ("gb200_launch_count", [None], NULL_POINTER),
        ("gb200_rmat_edges", [10, 16, 1, 0, None, P], NULL_POINTER),
        ("gb200_rmat_edges", [0, 16, 1, 0, P, P], INVALID_VALUE),
        ("gb200_rmat_edges", [31, 16, 1, 0, P, P], INVALID_VALUE),
        ("gb200_rmat_edges", [10, -1, 1, 0, P, P], INVALID_VALUE),
        # multi-GPU exchange
        ("gb200_xchg_create", [None, 1, 0, (C.c_longlong*2)(0, 1)], INVALID_VALUE),
        ("gb200_xchg_create", [_out(C.c_void_p), 1, 0, None], INVALID_VALUE),
        ("gb200_xchg_create", [_out(C.c_void_p), 0, 0, (C.c_longlong*2)(0, 1)], INVALID_VALUE),
        ("gb200_xchg_create", [_out(C.c_void_p), 33, 0, (C.c_longlong*34)()], INVALID_VALUE),
        ("gb200_xchg_create", [_out(C.c_void_p), 2, 2, (C.c_longlong*3)(0, 1, 2)], INVALID_VALUE),
        # a rank that owns nothing: every rank refuses, none waits on its publishes
        ("gb200_xchg_create", [_out(C.c_void_p), 2, 0, (C.c_longlong*3)(0, 0, 4)], INVALID_VALUE),
        ("gb200_xchg_create", [_out(C.c_void_p), 2, 1, (C.c_longlong*3)(0, 0, 4)], INVALID_VALUE),
        ("gb200_xchg_create", [_out(C.c_void_p), 2, 0, (C.c_longlong*3)(0, 4, 4)], INVALID_VALUE),
        ("gb200_xchg_create", [_out(C.c_void_p), 3, 2, (C.c_longlong*4)(0, 8, 4, 12)],
         INVALID_VALUE),
        ("gb200_xchg_create", [_out(C.c_void_p), 1, 0, (C.c_longlong*2)(0, 0)], INVALID_VALUE),
        # the slices start at word 0: words before the first would belong to no rank
        ("gb200_xchg_create", [_out(C.c_void_p), 1, 0, (C.c_longlong*2)(-4, 4)], INVALID_VALUE),
        ("gb200_xchg_create", [_out(C.c_void_p), 1, 0, (C.c_longlong*2)(4, 8)], INVALID_VALUE),
        ("gb200_xchg_create", [_out(C.c_void_p), 2, 1, (C.c_longlong*3)(4, 8, 12)], INVALID_VALUE),
        ("gb200_xchg_handle", [None, P], NULL_POINTER),
        ("gb200_xchg_connect", [None, P], NULL_POINTER),
        ("gb200_xchg_free", [None], SUCCESS),
        ("gb200_xchg_allgather_words", [None, P, 0.0, _out(C.c_double)], NULL_POINTER),
        ("gb200_dist_bfs_fused", [None, None, None, 1, 0, d, None], NULL_POINTER),
        ("gb200_dist_pr", [None, None, None, 1, 0.85, 1e-8, d, None], NULL_POINTER),
        ("gb200_dist_sssp", [None, None, None, 1, 0, d, None], NULL_POINTER),
    ]


# Entries that reach the device check with these arguments: without a device they
# must refuse with GrB_PANIC (no CPU fallback).
DEVICE_CHECK_CASES = [
    ("gb200_init", [0]),
    ("gb200_set_stream", [None]),
    ("gb200_sync", []),
    ("gb200_sm_count", [_out(C.c_int)]),
    ("gb200_matrix_new", [_out(C.c_void_p), gb.api.FP32, 4, 4]),
    ("gb200_matrix_new", [_out(C.c_void_p), 7, 4, 4]),
    ("gb200_matrix_load_mtx", [_out(C.c_void_p), gb.api.FP32, CHESAPEAKE.encode(), 0]),
    ("gb200_matrix_load_mtx", [_out(C.c_void_p), gb.api.FP32, b"/no/such/file.mtx", 0]),
    ("gb200_matrix_load_mtx", [_out(C.c_void_p), 7, CHESAPEAKE.encode(), 0]),
    ("gb200_ingest_coo", [4, 4, None, None, None, 0, 0, _out(C.c_void_p),
                          _out(C.c_longlong)]),
    ("gb200_csr_transpose_values", [4, 4, 0, P, P, P, None, None, None]),
    ("gb200_sort_pairs_u64", [P, None, 0, 8]),
    ("gb200_vector_new", [_out(C.c_void_p), gb.api.FP32, 8]),
    ("gb200_profile_enable", [1]),
    ("gb200_profile_reset", []),
    ("gb200_profile_read", [0, _out(C.c_double), _out(C.c_longlong), _out(C.c_double)]),
    ("gb200_rmat_edges", [10, 0, 1, 0, P, P]),
    ("gb200_xchg_create", [_out(C.c_void_p), 1, 0, (C.c_longlong*2)(0, 1)]),
]


def test_every_declared_entry_is_covered():
    """Each declared entry that returns a code appears in one of the two tables."""
    from test_capi_abi import declared_symbols
    named = {c[0] for c in before_device_cases(None)} | {c[0] for c in DEVICE_CHECK_CASES}
    assert set(declared_symbols()) - named == {"gb200_version"}


def test_refusals_before_the_device_check():
    lib = _lib.load()
    desc = gb.Descriptor()
    for name, args, want in before_device_cases(desc._h):
        got = getattr(lib, name)(*args)
        assert got == want, "%s%r: %d, expected %d" % (name, tuple(args), got, want)


def test_host_only_entries_run_without_a_device():
    lib = _lib.load()
    w = np.zeros(4, np.float32)
    assert lib.gb200_host_uniform_weights(1, 1, 64, 4, w.ctypes.data_as(C.c_void_p)) == 0
    assert np.all((w >= 1) & (w <= 64))
    n = C.c_ulonglong(0)
    assert lib.gb200_launch_count(C.byref(n)) == 0


def test_compute_entries_panic_without_a_device():
    if _have_gpu():
        pytest.skip("a device is present")
    lib = _lib.load()
    for name, args in DEVICE_CHECK_CASES:
        got = getattr(lib, name)(*args)
        assert got == PANIC, "%s%r: %d, expected GrB_PANIC" % (name, tuple(args), got)


# ---------------------------------------------------------------------------
# GPU part: checks that need real handles or come after the device check
# ---------------------------------------------------------------------------

@pytest.fixture(scope="module")
def g():
    """FP32 and INT32 handles on the chesapeake graph (39 vertices)."""
    gb.init(0)

    class G:
        pass
    g = G()
    g.lib = _lib.load()
    g.F = gb.Matrix.from_mtx(CHESAPEAKE, directed=2)
    g.I = gb.Matrix.from_mtx(CHESAPEAKE, directed=2, dtype=gb.api.INT32)
    g.n = g.F.nrows()
    g.Cf = gb.Matrix(g.n, g.n)
    g.Ci = gb.Matrix(g.n, g.n, dtype=gb.api.INT32)
    g.u = gb.Vector(g.n)
    g.u.fill(1.0)
    g.w = gb.Vector(g.n)
    g.desc = gb.Descriptor()
    return g


def expect(g, want, name, *args):
    h = [a._h if isinstance(a, (gb.Matrix, gb.Vector, gb.Descriptor)) else a for a in args]
    got = getattr(g.lib, name)(*h)
    assert got == want, "%s: %d, expected %d" % (name, got, want)


@pytest.mark.gpu
def test_mixed_element_types_are_a_domain_mismatch(g):
    F, I, Cf, Ci, d = g.F, g.I, g.Cf, g.Ci, g.desc
    for entry in ("gb200_mxm", "gb200_ewise_add_matrix", "gb200_ewise_mult_matrix"):
        expect(g, DOMAIN, entry, Cf, None, PLUS_TIMES, F, I, d)
        expect(g, DOMAIN, entry, Cf, None, PLUS_TIMES, I, F, d)
        expect(g, DOMAIN, entry, Cf, None, PLUS_TIMES, I, I, d)
        expect(g, DOMAIN, entry, Ci, None, PLUS_TIMES, I, F, d)
        expect(g, DOMAIN, entry, Ci, F, PLUS_TIMES, I, I, d)
        expect(g, DOMAIN, entry, Cf, I, PLUS_TIMES, F, F, d)
    expect(g, DOMAIN, "gb200_transpose", Cf, None, I, d)
    expect(g, DOMAIN, "gb200_transpose", Ci, None, F, d)
    expect(g, DOMAIN, "gb200_transpose", Ci, F, I, d)
    expect(g, DOMAIN, "gb200_transpose", Cf, I, F, d)
    expect(g, DOMAIN, "gb200_tc", _out(C.c_longlong), F, Ci, d, None)
    expect(g, DOMAIN, "gb200_tc", _out(C.c_longlong), I, Cf, d, None)


@pytest.mark.gpu
def test_int32_operations_other_than_plus_times_are_not_implemented(g):
    for entry in ("gb200_mxm", "gb200_ewise_add_matrix", "gb200_ewise_mult_matrix"):
        for s in (MIN_PLUS,) + BAD_SEMIRINGS:
            expect(g, NOT_IMPLEMENTED, entry, g.Ci, None, s, g.I, g.I, g.desc)


@pytest.mark.gpu
def test_fp32_only_entries_refuse_int32(g):
    I, u, w, d = g.I, g.u, g.w, g.desc
    expect(g, DOMAIN, "gb200_bfs", w, I, 0, d, None)
    expect(g, DOMAIN, "gb200_sssp", w, I, 0, d, None)
    expect(g, DOMAIN, "gb200_pr", w, I, 0.85, 1e-8, d, None)
    expect(g, DOMAIN, "gb200_vxm", w, None, 0, PLUS_TIMES, u, I, d)
    expect(g, DOMAIN, "gb200_mxv", w, None, 0, PLUS_TIMES, I, u, d)
    expect(g, DOMAIN, "gb200_reduce_matrix_rows", w, 0, I, d)
    expect(g, DOMAIN, "gb200_matrix_apply_uniform_random", I, d, 1, 1, 64)
    expect(g, DOMAIN, "gb200_pr_normalize", I, 0.85, d)
    expect(g, NOT_IMPLEMENTED, "gb200_matrix_build_dense", I, P, 1)
    expect(g, NOT_IMPLEMENTED, "gb200_matrix_adopt_dense", I, P)
    expect(g, UNINITIALIZED, "gb200_matrix_extract_dense", I, P, 1)
    expect(g, UNINITIALIZED, "gb200_matrix_dense_ptr", I, _out(C.c_void_p))


@pytest.mark.gpu
def test_int32_reduce_matrix_takes_the_plus_monoid_only(g):
    for m in (int(gb.Monoid.Multiplies), int(gb.Monoid.Maximum)) + BAD_MONOIDS:
        expect(g, NOT_IMPLEMENTED, "gb200_reduce_matrix", _out(C.c_double), m, g.I, g.desc)
    total = C.c_double(0)
    expect(g, SUCCESS, "gb200_reduce_matrix", C.byref(total), 0, g.I, g.desc)
    assert total.value == g.I.extract_csr()[2].sum()


@pytest.mark.gpu
def test_unknown_semiring_ids_are_invalid_values(g):
    F, Cf, u, w, d = g.F, g.Cf, g.u, g.w, g.desc
    for s in BAD_SEMIRINGS:
        for accum in (0, 1):
            expect(g, INVALID_VALUE, "gb200_vxm", w, None, accum, s, u, F, d)
            expect(g, INVALID_VALUE, "gb200_mxv", w, None, accum, s, F, u, d)
        expect(g, INVALID_VALUE, "gb200_mxm", Cf, None, s, F, F, d)
        expect(g, INVALID_VALUE, "gb200_ewise_add", w, None, s, u, u, d)
        expect(g, INVALID_VALUE, "gb200_ewise_add_scalar", w, None, s, u, 1.0, d)
        expect(g, INVALID_VALUE, "gb200_ewise_mult", w, None, s, u, u, d)
        expect(g, INVALID_VALUE, "gb200_ewise_add_matrix", Cf, None, s, F, F, d)
        expect(g, INVALID_VALUE, "gb200_ewise_mult_matrix", Cf, None, s, F, F, d)


@pytest.mark.gpu
def test_unknown_monoid_ids_are_invalid_values(g):
    for m in BAD_MONOIDS:
        expect(g, INVALID_VALUE, "gb200_reduce_vector", _out(C.c_double), m, g.u, g.desc)
        expect(g, INVALID_VALUE, "gb200_reduce_matrix", _out(C.c_double), m, g.F, g.desc)
        expect(g, INVALID_VALUE, "gb200_reduce_matrix_rows", g.w, m, g.F, g.desc)


@pytest.mark.gpu
def test_fp32_mxm_masks(g):
    # a sparse x sparse product takes no FP32 mask
    expect(g, DOMAIN, "gb200_mxm", g.Cf, g.F, PLUS_TIMES, g.F, g.F, g.desc)
    # beside a dense operand the mask reaches the backend, which refuses it
    B = gb.Matrix(g.n, 8)
    B.build_dense(np.ones((g.n, 8), np.float32))
    CB = gb.Matrix(g.n, 8)
    expect(g, NOT_IMPLEMENTED, "gb200_mxm", CB, B, PLUS_TIMES, g.F, B, g.desc)
    # ... after the semiring id is checked
    expect(g, INVALID_VALUE, "gb200_mxm", CB, B, BAD_SEMIRINGS[0], g.F, B, g.desc)


@pytest.mark.gpu
def test_source_out_of_range(g):
    for s in (-1, g.n):
        expect(g, INVALID_INDEX, "gb200_bfs", g.w, g.F, s, g.desc, None)
        expect(g, INVALID_INDEX, "gb200_sssp", g.w, g.F, s, g.desc, None)


@pytest.mark.gpu
def test_dist_entries_refuse_slices_the_kernels_cannot_run(g):
    """Nothing is launched: the bitmap BFS refuses an owned slice that does not
    start on a multiple of 4 words (128 vertices) before it looks at the peers,
    and every traversal refuses a vector that is not the owned slice."""
    lib, n, d = g.lib, g.n, g.desc

    def xchg(world, rank, offsets):
        h = C.c_void_p()
        assert lib.gb200_xchg_create(C.byref(h), world, rank,
                                     (C.c_longlong*len(offsets))(*offsets)) == SUCCESS
        return h

    # rank 1 of 2 owns words [1, 4): not connected, refused for the offset first
    x = xchg(2, 1, [0, 1, 4])
    try:
        expect(g, INVALID_VALUE, "gb200_dist_bfs_fused", x, gb.Vector(96), g.F, 128, 0, d,
               None)
        expect(g, UNINITIALIZED, "gb200_dist_pr", x, gb.Vector(96), g.F, 128, 0.85, 0.0, d,
               None)
    finally:
        lib.gb200_xchg_free(x)
    # one rank over the chesapeake graph: 39 vertices, 2 bitmap words / 39 floats
    for words, entry, args in (
            (2, "gb200_dist_bfs_fused", (0, d, None)),
            (n, "gb200_dist_sssp", (0, d, None)),
            (n, "gb200_dist_pr", (0.85, 0.0, d, None))):
        x = xchg(1, 0, [0, words])
        try:
            for size, nn in ((n - 1, n), (n + 1, n), (n, n + 33)):
                expect(g, DIMENSION, entry, x, gb.Vector(size), g.F, nn, *args)
        finally:
            lib.gb200_xchg_free(x)


@pytest.mark.gpu
def test_checks_after_the_device_check(g):
    expect(g, DOMAIN, "gb200_matrix_new", _out(C.c_void_p), 7, 4, 4)
    expect(g, INVALID_VALUE, "gb200_matrix_load_mtx", _out(C.c_void_p), gb.api.FP32,
           b"/no/such/file.mtx", 0)
    expect(g, DOMAIN, "gb200_matrix_load_mtx", _out(C.c_void_p), 7, CHESAPEAKE.encode(), 0)
    expect(g, NO_VALUE, "gb200_matrix_build_coo", gb.Matrix(4, 4), P, P, None, 0, 0)


@pytest.mark.gpu
def test_gc_mis_cc_on_int32_match_fp32(g):
    d = g.desc
    for name, args in (("gb200_gc", (3,)), ("gb200_mis", (3, None)), ("gb200_cc", ())):
        got = []
        for A in (g.F, g.I):
            v = gb.Vector(g.n)
            k, ms = C.c_int(-1), C.c_float(-1)
            expect(g, SUCCESS, name, v, A, *args, d, C.byref(k), C.byref(ms))
            assert k.value > 0 and ms.value >= 0
            got.append((k.value, v.extractTuples()))
            # the count and time outputs are optional
            expect(g, SUCCESS, name, gb.Vector(g.n), A, *args, d, None, None)
        assert got[0][0] == got[1][0], name
        assert np.array_equal(got[0][1], got[1][1]), name
