"""ctypes binding of the CPU greedy graph colouring (tests/gc_oracle.c orc_gc) and the
CPU greedy maximal independent set (tests/mis_oracle.c orc_mis), the checkers of the
device colouring and MIS.  mis_oracle.c includes gc_oracle.c for its priority order,
so one library built from it exports both.  priority_hash restates their priority
order in numpy.  Test infrastructure only: tests/, smoke() and tools/bench_gc.py /
bench_mis.py import it.

build() compiles the library into build/libgreedyoracle.so; where that file is missing
or older than either source, it is compiled into a temporary directory instead, so
nothing is written into the tree at run time.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, "tests", "mis_oracle.c")
SOURCES = [SOURCE, os.path.join(ROOT, "tests", "gc_oracle.c")]
LIB_PATH = os.path.join(ROOT, "build", "libgreedyoracle.so")
M32 = 0xFFFFFFFF

_lib = None


def priority_hash(seed, v):
    """fmix32(v ^ (seed * 0x9E3779B9)), the priority hash of
    kernels/greedy_schedule.cuh, of one vertex or an array of vertices (uint64)."""
    m32 = np.uint64(M32)
    x = (np.asarray(v, np.uint64) ^ np.uint64((seed*0x9E3779B9) & M32)) & m32
    x ^= x >> np.uint64(16)
    x = (x*np.uint64(0x85EBCA6B)) & m32
    x ^= x >> np.uint64(13)
    x = (x*np.uint64(0xC2B2AE35)) & m32
    return x ^ (x >> np.uint64(16))


def compile_to(path):
    """gcc -O3 shared library of mis_oracle.c (and the gc_oracle.c it includes) at path."""
    subprocess.check_call(["gcc", "-O3", "-std=c11", "-fPIC", "-shared", "-o", path,
                           SOURCE])


def lib():
    global _lib
    if _lib is None:
        path = LIB_PATH
        if not os.path.exists(path) or any(os.path.getmtime(path) < os.path.getmtime(s)
                                           for s in SOURCES):
            path = os.path.join(tempfile.mkdtemp(prefix="greedy_oracle_"),
                                "libgreedyoracle.so")
            compile_to(path)
        _lib = C.CDLL(path)
        _lib.orc_gc.restype = C.c_int
        _lib.orc_gc.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p,
                                C.POINTER(C.c_int)]
        _lib.orc_mis.restype = C.c_int
        _lib.orc_mis.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p,
                                 C.c_void_p, C.POINTER(C.c_int)]
    return _lib


def _csr(rowptr, colind):
    """int32 copies (colind at least one entry long, for a valid pointer) and n."""
    rowptr = np.ascontiguousarray(rowptr, dtype=np.int32)
    colind = np.ascontiguousarray(colind, dtype=np.int32)
    if len(colind) == 0:
        colind = np.zeros(1, dtype=np.int32)
    return rowptr, colind, len(rowptr) - 1


def gc(rowptr, colind, seed=0):
    """Greedy first-fit colouring in decreasing (hash(seed, v), v) order of a CSR
    with a symmetric pattern.  Returns (colors int32[n], ncolors, jp_depth)."""
    rowptr, colind, n = _csr(rowptr, colind)
    colors = np.zeros(max(n, 1), dtype=np.int32)
    depth = C.c_int(0)
    ncolors = lib().orc_gc(n, rowptr.ctypes.data, colind.ctypes.data, seed & 0xFFFFFFFF,
                           colors.ctypes.data, C.byref(depth))
    return colors[:n], int(ncolors), depth.value


def mis(rowptr, colind, seed=0, candidates=None):
    """Greedy maximal independent set in decreasing (hash(seed, v), v) order of a CSR
    with a symmetric pattern, over the vertices where candidates (length n, or None
    for all) is non-zero.  Returns (member int32[n], size, luby_depth)."""
    rowptr, colind, n = _csr(rowptr, colind)
    member = np.zeros(max(n, 1), dtype=np.int32)
    cand = None
    if candidates is not None:
        cand = np.ascontiguousarray(np.asarray(candidates) != 0, dtype=np.int32)
        assert len(cand) == n
        if n == 0:
            cand = np.zeros(1, dtype=np.int32)
    depth = C.c_int(0)
    size = lib().orc_mis(n, rowptr.ctypes.data, colind.ctypes.data, seed & 0xFFFFFFFF,
                         cand.ctypes.data if cand is not None else None,
                         member.ctypes.data, C.byref(depth))
    return member[:n], int(size), depth.value
