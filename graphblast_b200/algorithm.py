"""graphblas::algorithm — the GraphBLAS algorithm drivers of the reference
(graphblas/algorithm/{bfs,sssp,pr,tc}.hpp), executed inside the native library as
loops of backend operations (include/graphblas/algorithm/*.hpp), and the graph
colouring gc, the maximal independent set mis, the connected components cc and the
local graph clustering lgc, one kernel each on the device, with lgc_sweep, the
conductance sweep cut of lgc's result, the betweenness centrality bc, one kernel
per batch of 32 sources, the k-truss ktruss and truss decomposition trussness, one
cooperative edge-peeling kernel each, the strongly connected components scc, one
cooperative trim, forward-backward and colouring kernel, the minimum spanning
forest msf, one cooperative Boruvka kernel, and the community detection by label
propagation cdlp, one cooperative kernel for every iteration.

sssp, pr, tc, gc, mis, cc, lgc, lgc_sweep, bc, ktruss, trussness, scc, msf and cdlp return the device time of the operation
loop in milliseconds ("tight" in the reference drivers, example/gbfs.cu:110-115).  bfs returns it only
when called with timed=True; otherwise it returns None and, when the traversal runs
as the fused kernel, only enqueues it, so that back-to-back traversals keep the GPU
busy.  Reading the result (extractTuples, extract_into) waits for it.
"""
import ctypes as C

import numpy as np

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


def bc(v, A, desc, sources=None):
    """v[x] = the betweenness centrality of x: over the sources s (any int sequence or
    ndarray; a repeated id counts once per entry; None: every vertex, exact BC) and the
    targets t not in {s, x} reachable from s, the sum of sigma_st(x) / sigma_st, the
    share of the shortest s -> t paths that pass through x.  Each stored A(i,j), i != j,
    is an edge i -> j; values and self-loops are ignored.  No normalisation and no
    halving: for a symmetric A and all sources, twice networkx's undirected unnormalised
    value (include/graphblas/algorithm/bc.hpp).  fp64 on the device, rounded to float
    once; two calls give identical bytes.  A is FP32 or INT32; a non-symmetric A needs
    its CSC.  v becomes dense.  An id outside [0, n) raises GrB_INVALID_INDEX.
    Returns tight_ms."""
    ms = C.c_float(0)
    lib = _lib.load()
    if sources is None:
        code = lib.gb200_bc(v._h, A._h, None, A.nrows(), desc._h, C.byref(ms))
    else:
        ids = np.asarray(sources, dtype=np.int64).ravel()
        # ids that do not fit an int become -1, which the library refuses
        ids = np.where((ids < 0) | (ids > np.iinfo(np.int32).max), -1, ids).astype(np.int32)
        buf = ids if len(ids) else np.zeros(1, np.int32)   # an empty list is not NULL
        code = lib.gb200_bc(v._h, A._h, buf.ctypes.data_as(C.c_void_p), len(ids), desc._h,
                            C.byref(ms))
    _check(code, "algorithm::bc")
    return ms.value




def ktruss(out, A, k, desc):
    """out = the k-truss (k >= 2) of the undirected simple graph G of A's pattern ({i, j},
    i != j, when A(i,j) or A(j,i) is stored; values and self-loops ignored): starting
    from G, every edge in fewer than k - 2 triangles of the remaining graph is deleted
    until none is left to delete.  out(i,j) = out(j,i) = the number of triangles of the
    k-truss that contain {i, j}; with k = 2, every edge with its triangle count in G.
    out is n x n, sorted, installed as symmetric, FP32 or INT32 independently of A, and
    may be A.  A is FP32 or INT32; a non-symmetric A needs its CSC.  Integers only, so
    two calls give identical bytes (include/graphblas/algorithm/ktruss.hpp).
    Returns (nedges, tight_ms), nedges the undirected edges kept."""
    ms = C.c_float(0)
    count = C.c_longlong(0)
    _check(_lib.load().gb200_ktruss(out._h, A._h, int(k), desc._h, C.byref(count),
                                    C.byref(ms)),
           "algorithm::ktruss")
    return count.value, ms.value


def trussness(out, A, desc):
    """out = the truss decomposition of the undirected simple graph G of A's pattern (as
    in ktruss): G's pattern in both directions, out(i,j) = out(j,i) = the largest k
    whose k-truss contains {i, j}, 2 for an edge in no triangle.  out is n x n, sorted,
    installed as symmetric, FP32 or INT32 independently of A, and may be A.  Returns
    (kmax, tight_ms), kmax the largest value, 0 when G has no edge."""
    ms = C.c_float(0)
    kmax = C.c_int(0)
    _check(_lib.load().gb200_trussness(out._h, A._h, desc._h, C.byref(kmax), C.byref(ms)),
           "algorithm::trussness")
    return kmax.value, ms.value


def ktruss_stats():
    """(rounds, levels, support_ms) of the last ktruss or trussness call of this process:
    the peel rounds that removed edges, the levels that did, and the device time of the
    support pass alone in milliseconds."""
    rounds, levels, support = C.c_int(0), C.c_int(0), C.c_float(0)
    _lib.load().gb200_ktruss_stats(C.byref(rounds), C.byref(levels), C.byref(support))
    return rounds.value, levels.value, support.value


def scc(v, A, desc):
    """v[i] = the smallest vertex id in the strongly connected component of i, over the
    arcs i -> j with A(i,j) stored and i != j (values and self-loops ignored), one
    cooperative trim, forward-backward and colouring kernel
    (include/graphblas/algorithm/scc.hpp).  The result depends only on A's pattern, so
    there is no seed.  A is FP32 or INT32; out-lists come from its CSR and in-lists from
    its CSC, so a non-symmetric A needs its CSC.  An A marked symmetric (or whose CSC
    aliases its CSR) takes cc, whose components are then the strong ones.  v becomes
    dense and is overwritten.  A float v holds ids exactly only up to 2^24, so
    nrows(A) > 2^24 + 1 raises GrB_INVALID_VALUE.  Returns (ncomponents, tight_ms)."""
    ms = C.c_float(0)
    k = C.c_int(0)
    _check(_lib.load().gb200_scc(v._h, A._h, desc._h, C.byref(k), C.byref(ms)),
           "algorithm::scc")
    return k.value, ms.value


def scc_stats():
    """(trimmed, pivot_size, colour_iterations, barriers) of the last scc call of this
    process: the vertices settled by the trim, the size of the pivot's component, the
    colouring iterations and the grid barriers of the kernel.  After an A marked
    symmetric (cc's kernel) all are 0 except barriers, which is -1."""
    t, p, c, b = C.c_longlong(0), C.c_longlong(0), C.c_int(0), C.c_int(0)
    _lib.load().gb200_scc_stats(C.byref(t), C.byref(p), C.byref(c), C.byref(b))
    return t.value, p.value, c.value, b.value


def msf(F, A, desc):
    """F = the minimum spanning forest of the undirected graph G with the edge {i, j},
    i != j, when A(i,j) or A(j,i) is stored, weighted by the smaller of the stored
    values among A(i,j) and A(j,i).  Self-loops are ignored; stored zeros are edges of
    weight 0 (scipy treats explicit zeros as missing).  Only A's CSR is read.  Edges are
    ranked by (w, min(i,j), max(i,j)): numbers compare as numbers, -0.0 equal to +0.0,
    +-inf allowed, INT32 as signed integers.  The order is strict and total, so the
    forest is unique: Kruskal's forest under it.  F is n x n, replaced, a sorted CSR
    installed as symmetric with F(i,j) = F(j,i) = w({i,j}) (-0.0 written as +0.0), of
    A's element type, and may be A; two calls give identical bytes.  An FP32 A with a
    NaN on a stored off-diagonal entry raises GrB_INVALID_VALUE
    (include/graphblas/algorithm/msf.hpp).  Returns (nedges, weight, tight_ms): the
    undirected forest edges (n minus the number of trees) and their fp64 sum, taken in
    an order that depends only on the forest (exact while every partial sum is an
    integer below 2^53)."""
    ms = C.c_float(0)
    count = C.c_longlong(0)
    weight = C.c_double(0)
    _check(_lib.load().gb200_msf(F._h, A._h, desc._h, C.byref(count), C.byref(weight),
                                 C.byref(ms)),
           "algorithm::msf")
    return count.value, weight.value, ms.value


def msf_stats():
    """(rounds, barriers, canon_ms) of the last msf call of this process: the Boruvka
    rounds, at most ceil(log2 n) + 1, the grid barriers of the kernel, and the device
    time of building the canonical edge list in milliseconds."""
    rounds, barriers, canon = C.c_int(0), C.c_int(0), C.c_float(0)
    _lib.load().gb200_msf_stats(C.byref(rounds), C.byref(barriers), C.byref(canon))
    return rounds.value, barriers.value, canon.value


def cdlp(v, A, max_iter, desc):
    """v[i] = the label of i after synchronous label propagation (LDBC Graphalytics CDLP,
    include/graphblas/algorithm/cdlp.hpp).  The arc i -> j when A(i,j) is stored and
    i != j (values and self-loops ignored; FP32 and INT32 A give the same result).
    L_0(v) = v; iteration k gives v the smallest label of highest multiplicity among the
    labels of its out-neighbours (A's CSR) and in-neighbours (A's CSC), an arc stored
    both ways counted twice; a vertex without neighbours keeps its label.  An A marked
    symmetric (or whose CSC aliases its CSR) is read through its CSR alone, with the same
    answer; a non-symmetric A needs its CSC.  max_iter >= 0 iterations, stopping early
    after the first iteration that changes no label (a fixpoint, so the result is the
    same).  v becomes dense and is overwritten; two calls give identical bytes.  A float
    v holds ids exactly only up to 2^24, so nrows(A) > 2^24 + 1 raises
    GrB_INVALID_VALUE, as does max_iter < 0.  Returns (ncommunities, iterations,
    tight_ms): the distinct labels and the iterations run, including the one that changed
    nothing."""
    ms = C.c_float(0)
    k = C.c_int(0)
    it = C.c_int(0)
    _check(_lib.load().gb200_cdlp(v._h, A._h, int(max_iter), desc._h, C.byref(k), C.byref(it),
                                  C.byref(ms)),
           "algorithm::cdlp")
    return k.value, it.value, ms.value


def cdlp_stats():
    """(short_vertices, warp_vertices, long_vertices, long_items, barriers) of the last cdlp
    call of this process: the vertices whose list (out- plus in-list, self-loops
    included) has at most 32 entries, at most 128, and more; the (vertex, partition)
    items of the long lists, one per 2048 entries or part of it; and the grid barriers of
    the kernel, 2 per iteration and 2 more."""
    s, w, lv, li, b = (C.c_longlong(0), C.c_longlong(0), C.c_longlong(0), C.c_longlong(0),
                       C.c_int(0))
    _lib.load().gb200_cdlp_stats(C.byref(s), C.byref(w), C.byref(lv), C.byref(li), C.byref(b))
    return s.value, w.value, lv.value, li.value, b.value
