"""graphblas::algorithm — the GraphBLAS algorithm drivers of the reference
(graphblas/algorithm/{bfs,sssp,pr,tc}.hpp), executed inside the native library as
loops of backend operations (include/graphblas/algorithm/*.hpp), and the graph
colouring gc, the maximal independent set mis and the connected components cc, one
kernel each on the device.

sssp, pr, tc, gc, mis and cc return the device time of the operation loop in milliseconds
("tight" in the reference drivers, example/gbfs.cu:110-115).  bfs returns it only
when called with timed=True; otherwise it returns None and, when the traversal runs
as the fused kernel, only enqueues it, so that back-to-back traversals keep the GPU
busy.  Reading the result (extractTuples, extract_into) waits for it.
"""
import ctypes as C

from . import _lib
from .api import _check


def bfs(v, A, s, desc, timed=False):
    """v[i] = BFS level of i from source s (source = 1, unreached = 0).  Returns
    the device time in milliseconds when timed, else None.
    reference algorithm/bfs.hpp:14-89"""
    ms = C.c_float(0) if timed else None
    _check(_lib.load().gb200_bfs(v._h, A._h, int(s), desc._h,
                                 C.byref(ms) if timed else None),
           "algorithm::bfs")
    return ms.value if timed else None


def sssp(v, A, s, desc):
    """v[i] = shortest distance from s (unreached = FLT_MAX).
    reference algorithm/sssp.hpp:15-103"""
    ms = C.c_float(0)
    _check(_lib.load().gb200_sssp(v._h, A._h, int(s), desc._h, C.byref(ms)),
           "algorithm::sssp")
    return ms.value


def pr(p, A, alpha, eps, desc):
    """PageRank power iteration on a pre-normalised A (Matrix.pr_normalize).
    reference algorithm/pr.hpp:15-94"""
    ms = C.c_float(0)
    _check(_lib.load().gb200_pr(p._h, A._h, float(alpha), float(eps), desc._h,
                                C.byref(ms)), "algorithm::pr")
    return ms.value


def tc(A, B, desc):
    """Triangle count of a lower-triangular INT32 matrix A; B receives
    (A*A^T).*A.  Returns (ntris, tight_ms).  reference algorithm/tc.hpp:15-54"""
    ms = C.c_float(0)
    n = C.c_longlong(0)
    _check(_lib.load().gb200_tc(C.byref(n), A._h, B._h, desc._h, C.byref(ms)),
           "algorithm::tc")
    return n.value, ms.value


def gc(v, A, seed, desc):
    """v[i] = colour of vertex i (1-based) in the undirected graph of A's pattern:
    greedy first-fit colouring in decreasing priority (hash(seed, i), i) order, one
    cooperative kernel (include/graphblas/algorithm/gc.hpp).  A is FP32 or INT32; a
    non-symmetric A needs its CSC.  Returns (ncolors, tight_ms)."""
    ms = C.c_float(0)
    k = C.c_int(0)
    _check(_lib.load().gb200_gc(v._h, A._h, int(seed), desc._h, C.byref(k), C.byref(ms)),
           "algorithm::gc")
    return k.value, ms.value


def mis(v, A, seed, desc, candidates=None):
    """v[i] = 1 when vertex i is in the maximal independent set of the undirected graph
    of A's pattern, else 0: the greedy set in decreasing priority (hash(seed, i), i)
    order over the candidates, the priority of gc (include/graphblas/algorithm/mis.hpp).
    candidates: None (every vertex) or a Vector whose non-zero entries name the
    candidates; it is not converted and may be v itself.  A is FP32 or INT32; a
    non-symmetric A needs its CSC.  Returns (nmembers, tight_ms)."""
    ms = C.c_float(0)
    k = C.c_int(0)
    _check(_lib.load().gb200_mis(v._h, A._h, int(seed),
                                 candidates._h if candidates is not None else None,
                                 desc._h, C.byref(k), C.byref(ms)),
           "algorithm::mis")
    return k.value, ms.value


def cc(v, A, desc):
    """v[i] = the smallest vertex id in the connected component of i in the undirected
    graph of A's pattern (i and j joined when A(i,j) or A(j,i) is stored; self-loops
    ignored), one cooperative union-find kernel (include/graphblas/algorithm/cc.hpp).
    The result depends only on A's pattern, so there is no seed.  A is FP32 or INT32;
    only its CSR is read.  v becomes dense and is overwritten.  A float v holds ids
    exactly only up to 2^24, so nrows(A) > 2^24 + 1 raises GrB_INVALID_VALUE.
    Returns (ncomponents, tight_ms)."""
    ms = C.c_float(0)
    k = C.c_int(0)
    _check(_lib.load().gb200_cc(v._h, A._h, desc._h, C.byref(k), C.byref(ms)),
           "algorithm::cc")
    return k.value, ms.value
