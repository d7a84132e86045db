"""ctypes binding of the CPU minimum spanning forest (tests/msf_oracle.c orc_msf), the
checker of the device msf, which the MSF tests, tools/bench_msf.py and smoke() compare
against.  Test infrastructure only.

build() compiles the library into build/libmsforacle.so; where that file is missing or
older than the source, it is compiled into a temporary directory instead, so nothing is
written into the tree at run time.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, "tests", "msf_oracle.c")
SOURCES = [SOURCE]
LIB_PATH = os.path.join(ROOT, "build", "libmsforacle.so")

_lib = None


def compile_to(path):
    """gcc -O3 shared library of msf_oracle.c at path."""
    subprocess.check_call(["gcc", "-O3", "-std=c11", "-fPIC", "-shared", "-o", path, SOURCE])


def lib():
    global _lib
    if _lib is None:
        path = LIB_PATH
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(SOURCE):
            path = os.path.join(tempfile.mkdtemp(prefix="msf_oracle_"), "libmsforacle.so")
            compile_to(path)
        _lib = C.CDLL(path)
        _lib.orc_msf.restype = C.c_longlong
        _lib.orc_msf.argtypes = [C.c_int] + [C.c_void_p]*6
    return _lib


def msf(rp, ci, val):
    """The minimum spanning forest of the square CSR (rp, ci, val), as algorithm.msf
    defines it: ((ptr, ind, val) of F, both directions of every forest edge, rows sorted
    by column, values float64; nedges; weight, the fp64 sum of the forest's weights in
    (min, max) order).  Raises ValueError on a NaN off the diagonal."""
    rp = np.ascontiguousarray(rp, np.int32)
    n = len(rp) - 1
    ci = np.ascontiguousarray(ci, np.int32)
    val = np.ascontiguousarray(val, np.float64)
    cap = max(2*n, 1)
    out_rp = np.zeros(n + 1, np.int32)
    out_ci = np.zeros(cap, np.int32)
    out_val = np.zeros(cap, np.float64)
    weight = C.c_double(0)
    nf = lib().orc_msf(n, rp.ctypes.data, (ci if len(ci) else np.zeros(1, np.int32)).ctypes.data,
                       (val if len(val) else np.zeros(1)).ctypes.data, out_rp.ctypes.data,
                       out_ci.ctypes.data, out_val.ctypes.data, C.byref(weight))
    if nf == -1:
        raise ValueError("NaN weight off the diagonal")
    assert nf >= 0, "out of memory"
    nz = int(out_rp[-1]) if n > 0 else 0
    return (out_rp, out_ci[:nz], out_val[:nz]), int(nf), weight.value
