"""ctypes binding of the CPU greedy graph colouring (tests/gc_oracle.c), the checker
of the device colouring.  Test infrastructure only: tests/, smoke() and
tools/bench_gc.py import it.

build() compiles the library into build/libgcoracle.so; where that file is missing
or older than the source, it is compiled into a temporary directory instead, so
nothing is written into the tree at run time.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, "tests", "gc_oracle.c")
LIB_PATH = os.path.join(ROOT, "build", "libgcoracle.so")

_lib = None


def compile_to(path):
    """gcc -O3 shared library of gc_oracle.c at path."""
    subprocess.check_call(["gcc", "-O3", "-std=c11", "-fPIC", "-shared", "-o", path,
                           SOURCE])


def lib():
    global _lib
    if _lib is None:
        path = LIB_PATH
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(SOURCE):
            path = os.path.join(tempfile.mkdtemp(prefix="gc_oracle_"), "libgcoracle.so")
            compile_to(path)
        _lib = C.CDLL(path)
        _lib.orc_gc.restype = C.c_int
        _lib.orc_gc.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p,
                                C.POINTER(C.c_int)]
    return _lib


def gc(rowptr, colind, seed=0):
    """Greedy first-fit colouring in decreasing (hash(seed, v), v) order of a CSR
    with a symmetric pattern.  Returns (colors int32[n], ncolors, jp_depth)."""
    rowptr = np.ascontiguousarray(rowptr, dtype=np.int32)
    colind = np.ascontiguousarray(colind, dtype=np.int32)
    n = len(rowptr) - 1
    colors = np.zeros(max(n, 1), dtype=np.int32)
    if len(colind) == 0:
        colind = np.zeros(1, dtype=np.int32)
    depth = C.c_int(0)
    ncolors = lib().orc_gc(n, rowptr.ctypes.data, colind.ctypes.data, seed & 0xFFFFFFFF,
                           colors.ctypes.data, C.byref(depth))
    return colors[:n], int(ncolors), depth.value
