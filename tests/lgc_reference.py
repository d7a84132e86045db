"""Host restatements of local graph clustering (algorithm::lgc, gb200_lgc and its sweep
cut), the checkers of tests/test_lgc_*.py and tools/bench_lgc.py.

push() restates the reference's CPU checker SimpleReferenceLgc<float>
(graphblas/algorithm/test_lgc.hpp) with the arithmetic its C++ evaluates: alpha and eps
are double, the vectors float32, no fused multiply-add:

    d[v]  = float32(row length of v)
    p = 0, r = 0, r[s] = 1, F = {s}
    while F is not empty and fewer than max_niter rounds have run:
      for v in F:  p[v]  = float32(double(p[v]) + alpha*double(r[v]))
                   nr[v] = float32((1 - alpha)*double(r[v])/2)
      r2 = r;  r2[v] = nr[v] for v in F
      for every w, in ascending order of v over the v in F with A(v,w) stored:
                   r2[w] = r2[w] + float32(nr[v]/d[v])           (float32 add and divide)
      r = r2
      F = {v : double(r[v]) >= double(d[v])*eps}, less the no-op vertices d[v] = 0, r[v] = 0

The per-target order comes from np.add.at, which adds its terms one at a time in the
order given; the terms are laid out by ascending v.  Only the touched set F + N(F) can
change, and the reference's rescan of every vertex finds no frontier vertex outside it
(an untouched vertex failed the test the round before), so each round costs the
frontier's volume, not n.

sweep() restates the sweep cut: the support {v : p[v] > 0, d[v] > 0} ordered by
float32(p[v]/d[v]) descending, ties by ascending id; of its prefixes, the smallest one of
least conductance cut/min(vol, nnz - vol) (integer cut and volume, the quotient in
float64; prefixes with a zero denominator do not qualify).  sweep_brute() recomputes
every prefix's cut and volume from scratch, for small graphs.

ref_lgc() calls the reference's own SimpleReferenceLgc<float>, compiled from the
reference sources into oracle/_ref/libgbref_lgc.so (oracle/ref_lgc.cpp, ref_lgc.mk);
ref_lgc_available() is False where that library was not built.
"""
import ctypes as C
import os

import numpy as np

REF_LGC_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                          "oracle", "_ref", "libgbref_lgc.so")
_ref_lgc = None


def ref_lgc_available():
    return os.path.exists(REF_LGC_SO)


def ref_lgc(rp, ci, s, alpha, eps, max_niter):
    """p of the reference's SimpleReferenceLgc<float>, which runs exactly max_niter
    rounds (those after its frontier empties change nothing)."""
    global _ref_lgc
    if _ref_lgc is None:
        _ref_lgc = C.CDLL(REF_LGC_SO)
        _ref_lgc.ref_lgc.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                     C.c_double, C.c_double, C.c_int]
        _ref_lgc.ref_lgc.restype = None
    rp = np.ascontiguousarray(rp, np.int32)
    ci = np.ascontiguousarray(ci if len(ci) else np.zeros(1), np.int32)
    p = np.zeros(len(rp) - 1, np.float32)
    _ref_lgc.ref_lgc(len(rp) - 1, rp.ctypes.data, ci.ctypes.data, p.ctypes.data, int(s),
                     float(alpha), float(eps), int(max_niter))
    return p


def driver_alpha(nnz, phi=0.5):
    """The reference driver's alpha (example/glgc.cu): phi^2 / (225 ln(100 sqrt(nnz)))."""
    return phi*phi/(225.0*np.log(100.0*np.sqrt(float(nnz))))


def degrees(rp):
    return np.diff(np.asarray(rp, np.int64))


def _gather(rp, ci, rows):
    """(sources, targets) of the entries of the given rows, rows in the order given and
    each row's entries in stored order."""
    rp = np.asarray(rp, np.int64)
    lens = rp[rows + 1] - rp[rows]
    total = int(lens.sum())
    if total == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    starts = np.repeat(rp[rows] - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
    pos = starts + np.arange(total)
    return np.repeat(rows, lens), np.asarray(ci, np.int64)[pos]


def push(rp, ci, s, alpha, eps, max_niter=10000):
    """(p, r, rounds, pushed): the restatement above on the CSR (rp, ci); pushed = the
    sum over the rounds of the frontier's volume."""
    n = len(rp) - 1
    deg = degrees(rp)
    d32 = deg.astype(np.float32)
    p = np.zeros(n, np.float32)
    r = np.zeros(n, np.float32)
    r[s] = 1.0
    front = np.array([s], np.int64)
    rounds, pushed = 0, 0
    alpha, eps = float(alpha), float(eps)
    while len(front) > 0 and rounds < max_niter:
        pushed += int(deg[front].sum())
        rv = r[front].astype(np.float64)
        p[front] = (p[front].astype(np.float64) + alpha*rv).astype(np.float32)
        nr = ((1.0 - alpha)*rv/2.0).astype(np.float32)
        r[front] = nr
        c = np.zeros(len(front), np.float32)
        has = deg[front] > 0
        c[has] = nr[has]/d32[front][has]
        src, dst = _gather(rp, ci, front)            # front is ascending
        term = np.repeat(c, deg[front])
        np.add.at(r, dst, term)
        rounds += 1
        touched = np.unique(np.concatenate([front, dst]))
        rt = r[touched]
        dt = deg[touched]
        ok = (rt.astype(np.float64) >= dt.astype(np.float32).astype(np.float64)*eps) & \
            ~((dt == 0) & (rt == 0))
        front = touched[ok]
    return p, r, rounds, pushed


def _order(p, deg):
    """The support in sweep order."""
    p = np.asarray(p, np.float32)
    u = np.nonzero((p > 0) & (deg > 0))[0]
    key = p[u]/deg[u].astype(np.float32)
    return u[np.lexsort((u, -key))]


def _best(cut, vol, nnz):
    den = np.minimum(vol, nnz - vol)
    ok = den > 0
    if not ok.any():
        return 0, float("nan")
    phi = np.full(len(cut), np.inf)
    phi[ok] = cut[ok].astype(np.float64)/den[ok].astype(np.float64)
    k = int(np.argmin(phi))                          # the first of the least
    return k + 1, float(phi[k])


def sweep(rp, ci, p):
    """(cluster, size, conductance): cluster a float32 0/1 vector over n."""
    n = len(rp) - 1
    deg = degrees(rp)
    order = _order(p, deg)
    m = len(order)
    rank = np.full(n, np.iinfo(np.int64).max, np.int64)
    rank[order] = np.arange(m)
    rows = np.repeat(np.arange(n, dtype=np.int64), deg)
    cols = np.asarray(ci, np.int64)
    ri, rj = rank[rows], rank[cols]
    # entry (i, j), i != j, is cut by the prefixes of sizes ri + 1 .. rj (j outside)
    live = (rows != cols) & (ri < m) & (ri < rj)
    diff = np.zeros(m + 2, np.int64)
    np.add.at(diff, ri[live] + 1, 1)
    np.add.at(diff, np.minimum(rj[live], m) + 1, -1)
    cut = np.cumsum(diff)[1:m + 1]
    vol = np.cumsum(deg[order])
    size, phi = _best(cut, vol, len(cols)) if m > 0 else (0, float("nan"))
    cluster = np.zeros(n, np.float32)
    cluster[order[:size]] = 1.0
    return cluster, size, phi


def sweep_brute(rp, ci, p):
    """(size, conductance) with every prefix's cut and volume counted from scratch."""
    n = len(rp) - 1
    deg = degrees(rp)
    order = _order(p, deg)
    rows = np.repeat(np.arange(n, dtype=np.int64), deg)
    cols = np.asarray(ci, np.int64)
    cut, vol = [], []
    member = np.zeros(n, bool)
    for v in order:
        member[v] = True
        cut.append(int(np.count_nonzero(member[rows] & ~member[cols] & (rows != cols))))
        vol.append(int(deg[member].sum()))
    if not cut:
        return 0, float("nan")
    return _best(np.array(cut, np.int64), np.array(vol, np.int64), len(cols))


def lazy_pagerank(rp, ci, alpha, x):
    """pr_alpha(x) in float64: the solution y of y = alpha x + (1 - alpha) y W with
    W = (I + D^-1 A)/2, the lazy walk (rows with d = 0 keep their mass: W = I there)."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as sla
    n = len(rp) - 1
    deg = degrees(rp).astype(np.float64)
    A = sp.csr_matrix((np.ones(len(ci)), np.asarray(ci, np.int64), np.asarray(rp, np.int64)),
                      shape=(n, n))
    inv = np.where(deg > 0, 1.0/np.maximum(deg, 1.0), 0.0)
    W = 0.5*(sp.identity(n) + sp.diags(inv) @ A)
    W = W + 0.5*sp.diags((deg == 0).astype(np.float64))
    M = (sp.identity(n) - (1.0 - alpha)*W).T.tocsc()
    return sla.spsolve(M, alpha*np.asarray(x, np.float64))
