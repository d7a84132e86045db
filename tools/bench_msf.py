"""Minimum spanning forest on the device (algorithm.msf): time per call against scipy's
minimum_spanning_tree on one host thread, cc on the same matrix and the time to stream
the CSR once.

  python tools/bench_msf.py [--iters 10] [--warmup 2] [--only NAME]

Workloads (R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, generator seed 0,
graphs.rmat_edges / build_csr, symmetrised, self-loops and duplicates removed; each
adopted as a CSR marked symmetric):
  rmat22_ties, rmat24_ties
                  weights 1..64 from the SSSP weight stream (host_uniform_weights, seed
                  1), one per stored entry, so A(i,j) and A(j,i) usually differ and the
                  minimum of the two counts: heavy ties, broken by the ids.
  rmat22_distinct distinct float weights: the floats whose bit patterns are 0x3f800000
                  (1.0) plus a seeded permutation of the stored entries, so no two
                  entries tie.
  grid27          the 27-point stencil on a 128^3 grid of tools/benchlib.py (its
                  self-loops ignored), weights 1..64 from the same stream: a mesh where
                  Boruvka's components grow evenly.
  pieces          the 4096 random pieces of 1024 vertices of tools/benchlib.py's
                  tree_pieces, ids interleaved, weights 1..64: a forest of 4096 trees.
No weight in these workloads is zero, so scipy, which treats stored zeros as missing
edges, sees the same graph.

Each line is one JSON record.  "ms" is the median of the CUDA-event times msf returns
for warm calls.  A time is quoted only after F equals the checker's
(tests/msf_reference.py, a CPU Kruskal under the same key) entry for entry, with the
same edge count and weight ("equals_checker"), and the weight equals scipy's
("weight_equals_scipy": exactly for integer weights, to a relative 1e-12 otherwise).
"scipy_ms" is scipy's minimum_spanning_tree on one host thread.  "cc_ms" is the median
time of algorithm.cc on the same matrix.  "rounds", "barriers" and "canon_ms" are
algorithm.msf_stats() of the last call.  "stream_bound_ms" is (4 (n + 1) + 8 nnz) bytes,
the CSR and its values read once, at 3.35 TB/s (the H100 SXM data-sheet HBM3
bandwidth): a bound, not an achieved rate.  "card" is the GPU's name and power limit,
read in the same run.
"""
import json
import time

import numpy as np
import torch

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import (card, device_ms, grid27, header, parser, rmat_csr, run,
                      stream_bound_ms, tree_pieces)
import graphblast_b200 as gb
from graphblast_b200 import algorithm, graphs
from msf_reference import msf as checker


def grid():
    n, rp, ci = grid27(128)
    rows = torch.repeat_interleave(torch.arange(n, device="cuda", dtype=torch.int32),
                                   (rp[1:] - rp[:-1]).long())
    keep = rows != ci                  # the stencil's self-loops
    rp2 = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    rp2[1:] = torch.cumsum(torch.bincount(rows[keep].long(), minlength=n), 0)
    return n, rp2.int(), ci[keep].contiguous()


def sssp_weights(nnz):
    return gb.api.host_uniform_weights(1, 1, 64, nnz)


def distinct_weights(nnz):
    bits = np.uint32(0x3f800000) + np.random.RandomState(3).permutation(nnz).astype(np.uint32)
    return bits.view(np.float32)


def scipy_msf(n, rp, ci, val):
    import scipy.sparse as sp
    from scipy.sparse.csgraph import minimum_spanning_tree
    A = sp.csr_matrix((val.astype(np.float64), ci, rp), shape=(n, n))
    t0 = time.perf_counter()
    T = minimum_spanning_tree(A)
    ms = (time.perf_counter() - t0)*1e3
    return float(T.sum()), int(T.nnz), ms


def measure(name, n, rp, ci, weights, args):
    nnz = int(ci.numel())
    h_val = weights(nnz)
    A = graphs.matrix_from_csr(n, rp, ci, torch.from_numpy(h_val).cuda())
    rec = {"workload": name, "n": n, "nnz": nnz, "card": card()}
    desc = gb.Descriptor()
    F = gb.Matrix(n, n)
    out = [0, 0.0]

    def run_msf():
        out[0], out[1], ms = algorithm.msf(F, A, desc)
        return ms
    run_msf()
    h_rp, h_ci = rp.cpu().numpy(), ci.cpu().numpy()
    (w_rp, w_ci, w_val), want_n, want_w = checker(h_rp, h_ci, h_val)
    got_rp, got_ci, got_val = F.extract_csr()
    integer = bool(np.all(h_val == np.round(h_val)))
    rec["equals_checker"] = bool(
        np.array_equal(got_rp, w_rp) and np.array_equal(got_ci, w_ci) and
        np.array_equal(got_val, w_val.astype(np.float32)) and out[0] == want_n and
        (out[1] == want_w if integer else abs(out[1] - want_w) <= 1e-12*abs(want_w)))
    rec["nedges"], rec["weight"] = out[0], out[1]
    s_weight, s_edges, rec["scipy_ms"] = scipy_msf(n, h_rp, h_ci, h_val)
    rec["weight_equals_scipy"] = bool(
        s_edges == out[0] and
        (s_weight == out[1] if integer else abs(s_weight - out[1]) <= 1e-12*abs(s_weight)))
    del got_rp, got_ci, got_val, w_rp, w_ci, w_val

    rec["ms"] = device_ms(run_msf, args.iters, args.warmup)
    rec["rounds"], rec["barriers"], rec["canon_ms"] = algorithm.msf_stats()
    cv = gb.Vector(n)
    rec["cc_ms"] = device_ms(lambda: algorithm.cc(cv, A, desc)[1], args.iters, args.warmup)
    rec["stream_bound_ms"] = stream_bound_ms(4.0*(n + 1) + 8.0*nnz)
    if rec["equals_checker"] and rec["weight_equals_scipy"]:
        rec["scipy_over_msf"] = rec["scipy_ms"]/rec["ms"]
    else:
        rec.pop("ms")                 # a wrong forest gets no time
    print(json.dumps(rec), flush=True)


def main():
    args = parser(iters=10, warmup=2,
                  only="rmat22_ties, rmat24_ties, rmat22_distinct, grid27 or "
                       "pieces").parse_args()
    gb.init(0)
    header()
    run([("rmat22_ties", lambda: rmat_csr(22, seed=0), sssp_weights),
         ("rmat24_ties", lambda: rmat_csr(24, seed=0), sssp_weights),
         ("rmat22_distinct", lambda: rmat_csr(22, seed=0), distinct_weights),
         ("grid27", grid, sssp_weights),
         ("pieces", tree_pieces, sssp_weights)], args, measure)


if __name__ == "__main__":
    main()
