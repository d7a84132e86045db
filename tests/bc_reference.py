"""Betweenness centrality restated in float64 on a host CSR (numpy / scipy), with the
semantics of include/graphblas/algorithm/bc.hpp: each stored A(i,j), i != j, is an edge
i -> j (self-loops and values ignored); for the source list S (a repeated id counts once
per entry; None = every vertex)

    bc[v] = sum over s in S, over t not in {s, v} reachable from s, of sigma_st(v)/sigma_st

with no normalisation and no halving.  Brandes' two passes, run for a block of sources at
once as products of the pattern with an n x k matrix: forward, level by level,
sigma[v, s] = the sum of sigma[u, s] over in-neighbours u at depth d(s, v) - 1; backward,
delta[u, s] = the sum over out-neighbours v at depth d(s, u) + 1 of
sigma[u, s]/sigma[v, s]*(1 + delta[v, s]); bc adds delta[u, s] for every u at depth >= 1.
"""
import numpy as np
import scipy.sparse as sp

BLOCK = 64                           # sources per block of the dense n x k arrays


def pattern(rp, ci):
    """The n x n float64 pattern of (rp, ci) without its diagonal, and its transpose."""
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    ci = np.asarray(ci, np.int64)
    keep = rows != ci
    A = sp.csr_matrix((np.ones(int(keep.sum())), (rows[keep], ci[keep])), shape=(n, n))
    return A, A.T.tocsr()


def brandes(rp, ci, sources=None):
    """bc as float64 (length n) for the sources (None: all vertices)."""
    n = len(rp) - 1
    src = np.arange(n) if sources is None else np.asarray(sources, np.int64).ravel()
    A, AT = pattern(rp, ci)
    bc = np.zeros(n)
    for b in range(0, len(src), BLOCK):
        S = src[b:b + BLOCK]
        k = len(S)
        cols = np.arange(k)
        depth = np.full((n, k), -1, np.int64)
        sigma = np.zeros((n, k))
        depth[S, cols] = 0
        sigma[S, cols] = 1.0
        front = np.zeros((n, k), bool)
        front[S, cols] = True
        d = 0
        while front.any():
            reach = AT @ np.where(front, sigma, 0.0)           # in-neighbours at depth d
            new = (reach > 0) & (depth < 0)
            sigma[new] = reach[new]
            depth[new] = d + 1
            front = new
            d += 1
        delta = np.zeros((n, k))
        for level in range(d - 1, 0, -1):
            at_next = depth == level + 1
            w = np.where(at_next, (1.0 + delta)/np.where(at_next, sigma, 1.0), 0.0)
            here = depth == level
            delta[here] = (sigma*(A @ w))[here]
            bc += np.where(here, delta, 0.0).sum(axis=1)
    return bc


def brute_force(rp, ci, sources=None):
    """bc from all-pairs BFS distances and path counts: sigma_st(v) = sigma_sv*sigma_vt
    when d(s, v) + d(v, t) = d(s, t).  For small graphs only."""
    n = len(rp) - 1
    src = np.arange(n) if sources is None else np.asarray(sources, np.int64).ravel()
    dist = np.full((n, n), -1, np.int64)
    count = np.zeros((n, n))
    for s in range(n):
        dist[s, s], count[s, s] = 0, 1.0
        front = [s]
        while front:
            nxt = []
            for u in front:
                for v in ci[rp[u]:rp[u + 1]]:
                    if v == u:
                        continue
                    if dist[s, v] < 0:
                        dist[s, v] = dist[s, u] + 1
                        nxt.append(v)
                    if dist[s, v] == dist[s, u] + 1:
                        count[s, v] += count[s, u]
            front = nxt
    bc = np.zeros(n)
    for s in src:
        for t in range(n):
            if t == s or dist[s, t] < 0:
                continue
            for v in range(n):
                if v in (s, t) or dist[s, v] < 0 or dist[v, t] < 0:
                    continue
                if dist[s, v] + dist[v, t] == dist[s, t]:
                    bc[v] += count[s, v]*count[v, t]/count[s, t]
    return bc
