"""ctypes binding of the CPU label propagation (tests/cdlp_oracle.c orc_cdlp), the checker of
the device cdlp, which the CDLP tests, tools/bench_cdlp.py and smoke() compare against,
and an independent numpy restatement of the same semantics (numpy_cdlp) that the
checker is pinned to.  Test infrastructure only.

build() compiles the library into build/libcdlporacle.so; where that file is missing or
older than the source, it is compiled into a temporary directory instead, so nothing is
written into the tree at run time.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, "tests", "cdlp_oracle.c")
SOURCES = [SOURCE]
LIB_PATH = os.path.join(ROOT, "build", "libcdlporacle.so")

_lib = None


def compile_to(path):
    """gcc -O3 shared library of cdlp_oracle.c at path."""
    subprocess.check_call(["gcc", "-O3", "-std=c11", "-fPIC", "-shared", "-o", path, SOURCE])


def lib():
    global _lib
    if _lib is None:
        path = LIB_PATH
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(SOURCE):
            path = os.path.join(tempfile.mkdtemp(prefix="cdlp_oracle_"), "libcdlporacle.so")
            compile_to(path)
        _lib = C.CDLL(path)
        _lib.orc_cdlp.restype = C.c_longlong
        _lib.orc_cdlp.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                  C.POINTER(C.c_int)]
    return _lib


def cdlp(rp, ci, max_iter):
    """The labels of the square pattern (rp, ci) after max_iter iterations (or the first
    that changes nothing), as algorithm.cdlp defines them: (labels int64, ncommunities,
    iterations)."""
    rp = np.ascontiguousarray(rp, np.int32)
    n = len(rp) - 1
    ci = np.ascontiguousarray(ci, np.int32)
    labels = np.zeros(max(n, 1), np.int32)
    iters = C.c_int(0)
    k = lib().orc_cdlp(n, rp.ctypes.data, (ci if len(ci) else np.zeros(1, np.int32)).ctypes.data,
                       int(max_iter), labels.ctypes.data, C.byref(iters))
    assert k >= 0, "out of memory"
    return labels[:n].astype(np.int64), int(k), iters.value


def numpy_cdlp(rp, ci, max_iter):
    """The same semantics restated with numpy: each iteration lists the (vertex, label)
    pairs of every arc end, sorts them with a lexsort, counts each run and keeps per
    vertex the longest run of the smallest label.  Same return as cdlp()."""
    rp = np.asarray(rp, np.int64)
    ci = np.asarray(ci, np.int64)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(rp))
    keep = rows != ci
    src, dst = rows[keep], ci[keep]
    who = np.concatenate([src, dst])          # v, for out-neighbour u = dst and in-neighbour u = src
    nbr = np.concatenate([dst, src])
    labels = np.arange(n, dtype=np.int64)
    t = 0
    while t < max_iter:
        t += 1
        lab = labels[nbr]
        order = np.lexsort((lab, who))
        w, x = who[order], lab[order]
        new = labels.copy()
        if len(w):
            first = np.ones(len(w), bool)
            first[1:] = (w[1:] != w[:-1]) | (x[1:] != x[:-1])
            starts = np.flatnonzero(first)
            runs = np.diff(np.append(starts, len(w)))
            rv, rx = w[starts], x[starts]
            # per vertex: highest count, then smallest label
            pick = np.lexsort((rx, -runs, rv))
            rv, rx = rv[pick], rx[pick]
            head = np.ones(len(rv), bool)
            head[1:] = rv[1:] != rv[:-1]
            new[rv[head]] = rx[head]
        changed = bool(np.any(new != labels))
        labels = new
        if not changed:
            break
    return labels, int(len(np.unique(labels))), t
