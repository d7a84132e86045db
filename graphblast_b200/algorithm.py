"""graphblas::algorithm — the GraphBLAS algorithm drivers of the reference
(graphblas/algorithm/{bfs,sssp,pr,tc}.hpp), executed inside the native library as
loops of backend operations (include/graphblas/algorithm/*.hpp), and the graph
colouring gc, the maximal independent set mis, the connected components cc and the
local graph clustering lgc, one kernel each on the device, with lgc_sweep, the
conductance sweep cut of lgc's result.

sssp, pr, tc, gc, mis, cc, lgc and lgc_sweep return the device time of the operation loop in milliseconds
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


def lgc(p, A, s, alpha, eps, desc, residual=None):
    """p = the approximate personalised PageRank of source s on the lazy walk of A's
    pattern (Andersen-Chung-Lang push, synchronous rounds), bit for bit the floats of
    the reference's CPU checker SimpleReferenceLgc<float> (algorithm/test_lgc.hpp) for
    sorted column lists; one cooperative kernel (include/graphblas/algorithm/lgc.hpp).
    residual: None or a Vector that receives the final residual r.  At most desc's
    max_niter rounds; desc's mxvmode picks each round's route (1 sparse, 2 dense, 0 by
    the frontier's volume against switchpoint * nnz) and never changes the result.  A
    is FP32 or INT32 (same result); a non-symmetric A needs its CSC.  alpha in (0, 1],
    eps > 0.  p and residual become dense.  Returns (rounds, tight_ms)."""
    ms = C.c_float(0)
    k = C.c_int(0)
    _check(_lib.load().gb200_lgc(p._h, residual._h if residual is not None else None, A._h,
                                 int(s), float(alpha), float(eps), desc._h, C.byref(k),
                                 C.byref(ms)),
           "algorithm::lgc")
    return k.value, ms.value


def lgc_sweep(cluster, p, A, desc):
    """cluster[i] = 1 for the members of the sweep cut of p, else 0: of the prefixes of
    {v : p[v] > 0, row v not empty} ordered by p[v]/d[v] descending (fp32, ties by
    ascending id), the smallest one of least conductance cut/min(vol, nnz - vol), with
    exact integer cut and volume (include/graphblas/algorithm/lgc.hpp).  A is FP32 or
    INT32; a non-symmetric A needs its CSC.  A p held sparse is converted to dense
    storage (its values unchanged).  Returns (size, conductance, tight_ms);
    (0, nan, ...) and an empty cluster when no prefix qualifies."""
    ms = C.c_float(0)
    k = C.c_int(0)
    phi = C.c_double(0)
    _check(_lib.load().gb200_lgc_sweep(cluster._h, p._h, A._h, desc._h, C.byref(k),
                                       C.byref(phi), C.byref(ms)),
           "algorithm::lgc_sweep")
    return k.value, phi.value, ms.value
