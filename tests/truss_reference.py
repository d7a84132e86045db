"""ctypes binding of the CPU k-truss and truss decomposition (tests/truss_oracle.c
orc_ktruss, orc_trussness), the checker of the device ktruss and trussness, and the
host helpers the tests and tools/bench_ktruss.py share: the undirected simple pattern
of a CSR and the expected result as a CSR.  Test infrastructure only.

build() compiles the library into build/libtrussoracle.so; where that file is missing
or older than the source, it is compiled into a temporary directory instead, so nothing
is written into the tree at run time.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, "tests", "truss_oracle.c")
SOURCES = [SOURCE]
LIB_PATH = os.path.join(ROOT, "build", "libtrussoracle.so")

_lib = None


def compile_to(path):
    """gcc -O3 shared library of truss_oracle.c at path."""
    subprocess.check_call(["gcc", "-O3", "-std=c11", "-fPIC", "-shared", "-o", path, SOURCE])


def lib():
    global _lib
    if _lib is None:
        path = LIB_PATH
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(SOURCE):
            path = os.path.join(tempfile.mkdtemp(prefix="truss_oracle_"), "libtrussoracle.so")
            compile_to(path)
        _lib = C.CDLL(path)
        _lib.orc_trussness.restype = C.c_int
        _lib.orc_trussness.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.orc_ktruss.restype = C.c_longlong
        _lib.orc_ktruss.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    return _lib


def _csr(rp, ci):
    rp = np.ascontiguousarray(rp, dtype=np.int32)
    ci = np.ascontiguousarray(ci, dtype=np.int32)
    return rp, (ci if len(ci) else np.zeros(1, np.int32)), len(rp) - 1


def undirected(rp, ci):
    """(ptr, ind) of the pattern of A ∪ Aᵀ of a square CSR, sorted, self-loops kept."""
    n = len(rp) - 1
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(rp))
    ci = np.asarray(ci, np.int64)
    key = np.unique(np.concatenate([rows*n + ci, ci*n + rows]))
    ptr = np.concatenate([[0], np.cumsum(np.bincount(key // n, minlength=n))]).astype(np.int32)
    return ptr, (key % n).astype(np.int32)


def trussness(rp, ci):
    """tau of every entry of a symmetric sorted CSR (-1 on self-loops), and kmax."""
    rp, ci, n = _csr(rp, ci)
    tau = np.zeros(max(len(ci), 1), np.int32)
    kmax = lib().orc_trussness(n, rp.ctypes.data, ci.ctypes.data, tau.ctypes.data)
    assert kmax >= 0
    return tau[:rp[-1]], int(kmax)


def ktruss(rp, ci, k):
    """The k-truss support of every entry of a symmetric sorted CSR (-1 where the edge
    is removed, or on a self-loop), and the undirected edges kept."""
    rp, ci, n = _csr(rp, ci)
    sup = np.zeros(max(len(ci), 1), np.int32)
    kept = lib().orc_ktruss(n, rp.ctypes.data, ci.ctypes.data, int(k), sup.ctypes.data)
    assert kept >= 0
    return sup[:rp[-1]], int(kept)


def kept_csr(rp, ci, val):
    """(ptr, ind, val) of the entries of (rp, ci) whose val is >= 0."""
    n = len(rp) - 1
    keep = np.asarray(val) >= 0
    rows = np.repeat(np.arange(n), np.diff(rp))[keep]
    ptr = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n))]).astype(np.int32)
    return ptr, np.asarray(ci)[keep].astype(np.int32), np.asarray(val)[keep]
