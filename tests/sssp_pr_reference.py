"""Host references of the single-GPU SSSP and PageRank drivers
(include/graphblas/algorithm/sssp.hpp, pr.hpp); test infrastructure only.

  sssp_rounds     the SSSP loop round by round in float32.  Every candidate distance
                  is a left-to-right float32 sum along a path and min is exact, so
                  with non-negative weights (fl(a + w) is monotone in a) every push /
                  pull route and order must reproduce it bit for bit.  MinimumPlus has
                  no multiply, so a fused multiply-add cannot change a rounding.
  pagerank64      the PageRank power iteration in float64 on the device's own
                  normalised values, with the device's float32 jump and start value:
                  only the iteration's summation order is left to differ.
  pagerank_bound  a per-vertex bound on |float32 device result - pagerank64| that
                  holds for any summation order (merge tiles, hub partials, push
                  atomics).
"""
import numpy as np

FLT_MAX = np.float32(np.finfo(np.float32).max)
U = 2.0**-24
# slack on top of the first-order bound: the float64 reference's own rounding and
# the bound's use of the float64 iterate where the device's float32 one belongs
SAFETY = 1.05
TINY = 1e-30


def sssp_rounds(rp, ci, w, s, k=None):
    """(distances, rounds) of the frontier Bellman-Ford of algorithm::sssp from s:
    per round, relaxed[j] = min over the frontier's entries (u, d_u) and edges
    u -> j of fl(d_u + w), the distances take min(d, relaxed) and the next frontier
    is the vertices whose distance went down.  The loop stops after the round that
    improves nothing, or after k rounds.  Unreached vertices hold FLT_MAX; a path
    sum that overflows to inf never improves FLT_MAX, so it leaves FLT_MAX too."""
    rp = np.asarray(rp, np.int64)
    ci = np.asarray(ci, np.int64)
    w = np.asarray(w, np.float32)
    n = len(rp) - 1
    d = np.full(n, FLT_MAX, np.float32)
    d[s] = 0
    front, fval = np.array([s], np.int64), np.zeros(1, np.float32)
    rounds = 0
    while len(front) and (k is None or rounds < k):
        rounds += 1
        lens = rp[front + 1] - rp[front]
        edge = np.repeat(rp[front] - np.cumsum(lens) + lens, lens) + np.arange(lens.sum())
        with np.errstate(over="ignore"):
            cand = np.repeat(fval, lens) + w[edge]
        relaxed = np.full(n, FLT_MAX, np.float32)
        np.minimum.at(relaxed, ci[edge], cand)
        improved = relaxed < d
        d = np.minimum(d, relaxed)
        front = np.nonzero(improved)[0]
        fval = relaxed[front]
    return d, rounds


def sssp_weights(kind, nnz, seed=5):
    """Edge weights of the SSSP cases: int 1..64, real [0.5, 2), zero10 real with
    about 10% exact zeros, spread 2^-12..2^12, overflow [1e37, 3e38] (path sums of
    two edges can overflow)."""
    rng = np.random.RandomState(seed)
    if kind == "int":
        return rng.randint(1, 65, nnz).astype(np.float32)
    if kind == "real":
        return rng.uniform(0.5, 2.0, nnz).astype(np.float32)
    if kind == "zero10":
        w = rng.uniform(0.5, 2.0, nnz).astype(np.float32)
        w[rng.rand(nnz) < 0.1] = 0
        return w
    if kind == "spread":
        return np.exp2(rng.uniform(-12, 12, nnz)).astype(np.float32)
    if kind == "overflow":
        return rng.uniform(1e37, 3e38, nnz).astype(np.float32)
    raise KeyError(kind)


def jump_and_start(alpha, n):
    """The float32 (1 - alpha)/n and 1/n of algorithm::pr."""
    f = np.float32
    return f(f(1) - f(alpha)) / f(n), f(1) / f(n)


def _transpose64(ptr, ind, val):
    import scipy.sparse as sp
    n = len(ptr) - 1
    A = sp.csr_matrix((np.asarray(val, np.float64), np.asarray(ind, np.int64),
                       np.asarray(ptr, np.int64)), shape=(n, n))
    return A.T.tocsr()


def pagerank64(ptr, ind, val, jump, p0, iters):
    """[p_0, ..., p_iters] in float64: p_0 = p0 everywhere, p_t = A' p_{t-1} + jump,
    where A is the CSR (ptr, ind, val) of the normalised matrix as the device holds
    it (A(i, j) = alpha * w(i, j) / rowsum(i), rounded to float32)."""
    At = _transpose64(ptr, ind, val)
    ps = [np.full(len(ptr) - 1, float(p0))]
    for _ in range(iters):
        ps.append(At @ ps[-1] + float(jump))
    return ps


def _gamma(k):
    return k*U / (1 - k*U)


def pagerank_bound(ptr, ind, val, ps, jump, order="device"):
    """[b_0, ..., b_T] for the iterates ps of pagerank64, b_0 = 0 (1/n is the same
    float32 on both sides).  order "device" (p = fl(sum of fl(p_i A_ij), any order)
    + jump):
        b_t[j] = g(k_j + 1) sum_i |A_ij| p_{t-1}[i] + u |p_t[j]| + sum_i |A_ij| b_{t-1}[i]
    order "oracle" (oracle_binding.pr: next = jump, next += alpha * (p / outdeg) in
    source order; each product rounded twice against a normalised value rounded
    once, the jump summed first):
        b_t[j] = g(k_j + 3) (sum_i |A_ij| p_{t-1}[i] + jump) + sum_i |A_ij| b_{t-1}[i]
    with u = 2^-24, g(k) = k u / (1 - k u) and k_j the in-degree of j.  Compare
    with within()."""
    At = _transpose64(ptr, ind, np.abs(np.asarray(val, np.float64)))
    indeg = np.diff(At.indptr)
    bs = [np.zeros(len(ptr) - 1)]
    for t in range(1, len(ps)):
        mag = At @ ps[t - 1]
        carried = At @ bs[-1]
        if order == "device":
            b = _gamma(indeg + 1)*mag + U*np.abs(ps[t]) + carried
        else:
            b = _gamma(indeg + 3)*(mag + abs(float(jump))) + carried
        bs.append(b)
    return bs


def outside(got, want, bound):
    """Mask of the vertices where |got - want| exceeds SAFETY * bound + TINY."""
    return np.abs(np.asarray(got, np.float64) - want) > SAFETY*bound + TINY


def within(got, want, bound):
    return not outside(got, want, bound).any()
