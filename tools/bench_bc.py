"""Betweenness centrality on the device (algorithm.bc): time per call and per batch of 32
sources, against a BFS on the same graph and the float64 restatement of
tests/bc_reference.py on the host.

  python tools/bench_bc.py [--iters 5] [--warmup 1] [--only NAME] [--sources 32 256]
                           [--cpu-sources 1]

Workloads:
  rmat22          R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, symmetrised,
                  self-loops and duplicate edges removed, generator seed 0
                  (graphs.rmat_edges / build_csr / matrix_from_csr), marked symmetric: the
                  in-lists of the path-count pull are the CSR rows.
  rmat22_directed the same edges stored one way (self-loops and duplicates removed),
                  adopted with its CSR and CSC: a non-symmetric input.
  grid27          the 27-point stencil on a 128^3 grid of tools/benchlib.py (self-loops
                  included, which BC ignores): one component, up to 127 levels from a
                  source, so a batch runs many grid-wide levels.
Sources: a numpy RandomState(7) sample without repeats among the vertices with a stored
entry in their row.

Each line is one JSON record.  "ms" is the median of the CUDA-event times that bc
returns for warm calls, "ms_per_batch" that over the batches of 32.  A time is quoted
only after the result equals the checker's ("equals_checker"): every entry float32(want)
or one float step from it, zeros exact, where want is the restatement of
tests/bc_reference.py run on the device in float64 with torch sparse products (the same
passes; the host restatement would take minutes per workload).  "source_edges_per_s" is
nsources * nnz / time: each stored entry counted once per source, not the entries a
traversal reads.  "cpu_ms_per_source" is tests/bc_reference.py (numpy / scipy, float64)
on one host thread, measured on --cpu-sources sources and divided by their number.
"bfs_ms" is the median tight time of one direction-optimised algorithm.bfs from the
highest-degree vertex on the same matrix (the flags of bench.py), and
"batch_over_32_bfs" is ms_per_batch / (32 * bfs_ms): one batch against 32 single-source
BFS traversals, which compute no path counts or dependencies.  "card" is the GPU's name
and power limit, read in the same run.
"""
import json
import time
import warnings

import numpy as np
import torch

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import card, device_ms, grid27, header, parser, run
import bc_reference
import graphblast_b200 as gb
from graphblast_b200 import algorithm, graphs


def rmat(scale, undirected=True):
    src, dst = graphs.rmat_edges(scale, seed=0)
    n = 1 << scale
    rp, ci = graphs.build_csr(n, src, dst, undirected)
    cp, ri = (rp, ci) if undirected else graphs.build_csr(n, dst, src, False)
    return n, rp, ci, cp, ri


def grid(side=128):
    n, rp, ci = grid27(side)
    return n, rp, ci, rp, ci


def torch_pattern(n, ptr, ind):
    """The float64 pattern of (ptr, ind) on the device without its diagonal, as CSR."""
    rows = torch.repeat_interleave(torch.arange(n, device="cuda"), torch.diff(ptr.long()))
    cols = ind.long()
    keep = rows != cols
    rows, cols = rows[keep], cols[keep]
    counts = torch.bincount(rows, minlength=n)
    crow = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    crow[1:] = torch.cumsum(counts, 0)
    with warnings.catch_warnings():      # torch calls its sparse CSR support beta
        warnings.simplefilter("ignore")
        return torch.sparse_csr_tensor(crow, cols, torch.ones(cols.numel(), dtype=torch.float64,
                                                              device="cuda"), size=(n, n))


def torch_brandes(n, A, AT, sources, block=32):
    """tests/bc_reference.py brandes(), the same passes, with torch on the device."""
    bc = torch.zeros(n, dtype=torch.float64, device="cuda")
    src = torch.as_tensor(sources, dtype=torch.int64, device="cuda")
    for b in range(0, len(src), block):
        S = src[b:b + block]
        k = len(S)
        cols = torch.arange(k, device="cuda")
        depth = torch.full((n, k), -1, dtype=torch.int32, device="cuda")
        sigma = torch.zeros((n, k), dtype=torch.float64, device="cuda")
        depth[S, cols] = 0
        sigma[S, cols] = 1.0
        front = torch.zeros((n, k), dtype=torch.bool, device="cuda")
        front[S, cols] = True
        d = 0
        while bool(front.any()):
            reach = AT @ torch.where(front, sigma, 0.0)
            new = (reach > 0) & (depth < 0)
            sigma = torch.where(new, reach, sigma)
            depth[new] = d + 1
            front = new
            d += 1
        del reach, front
        delta = torch.zeros((n, k), dtype=torch.float64, device="cuda")
        for level in range(d - 1, 0, -1):
            at_next = depth == level + 1
            w = torch.where(at_next, (1.0 + delta)/torch.where(at_next, sigma, 1.0), 0.0)
            here = depth == level
            delta = torch.where(here, sigma*(A @ w), delta)
            bc += torch.where(here, delta, 0.0).sum(dim=1)
            del w, at_next, here
    return bc.cpu().numpy()


def equal_to_checker(got, want64):
    want = want64.astype(np.float32)
    got = np.asarray(got, np.float32)
    steps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    return bool(np.all(got[want == 0] == 0) and np.all(steps <= 1)), int(np.max(steps))


def measure(name, n, rp, ci, cp, ri, symmetric, args):
    if symmetric:
        A = graphs.matrix_from_csr(n, rp, ci, symmetric=True)
    else:
        A = gb.Matrix(n, n)
        ones = torch.ones(ci.numel(), dtype=torch.float32, device="cuda")
        A.build_device_csr(rp, ci, ones, ci.numel(), cp, ri, ones.clone(), symmetric=False)
    nnz = int(ci.numel())
    h_rp, h_ci = rp.cpu().numpy(), ci.cpu().numpy()
    deg = np.diff(h_rp)
    live = np.nonzero(deg > 0)[0]
    desc = gb.Descriptor()

    bdesc = gb.Descriptor(mxvmode=0, struconly=1, opreuse=1, earlyexit=1)
    lv = gb.Vector(n)
    top = int(np.argmax(deg))
    bfs_ms = device_ms(lambda: algorithm.bfs(lv, A, top, bdesc, timed=True), args.iters,
                       args.warmup)
    del lv

    TA = TAT = None
    for count in args.sources:
        sources = np.random.RandomState(7).choice(live, count, replace=False).astype(np.int32)
        rec = {"workload": name, "n": n, "nnz": nnz, "symmetric": symmetric,
               "nsources": count, "batches": (count + 31)//32, "card": card()}
        v = gb.Vector(n)
        rec["ms"] = device_ms(lambda: algorithm.bc(v, A, desc, sources), args.iters,
                              args.warmup)
        got = v.extractTuples()
        del v
        torch.cuda.empty_cache()
        if TA is None:
            TA = torch_pattern(n, rp, ci)
            TAT = torch_pattern(n, cp, ri) if not symmetric else TA
        want = torch_brandes(n, TA, TAT, sources)
        torch.cuda.empty_cache()
        rec["equals_checker"], rec["max_float_steps"] = equal_to_checker(got, want)
        rec["max_bc"] = float(np.max(got))
        rec["bfs_ms"] = bfs_ms
        if not rec["equals_checker"]:
            rec.pop("ms")                 # a wrong result gets no time
        else:
            rec["ms_per_batch"] = rec["ms"]/rec["batches"]
            rec["source_edges_per_s"] = count*nnz/(rec["ms"]*1e-3)
            rec["batch_over_32_bfs"] = rec["ms_per_batch"]/(32*bfs_ms)
        print(json.dumps(rec), flush=True)
    del TA, TAT

    if args.cpu_sources > 0:
        sources = np.random.RandomState(7).choice(live, args.cpu_sources, replace=False)
        t0 = time.perf_counter()
        bc_reference.brandes(h_rp, h_ci, sources)
        cpu = (time.perf_counter() - t0)*1e3
        print(json.dumps({"workload": name, "cpu_ms_per_source": cpu/args.cpu_sources,
                          "cpu_sources": args.cpu_sources,
                          "cpu": "tests/bc_reference.py, numpy/scipy float64, one host "
                                 "thread, pattern build included"}), flush=True)


def main():
    ap = parser(iters=5, warmup=1, only="rmat22, rmat22_directed or grid27")
    ap.add_argument("--sources", type=int, nargs="+", default=[32, 256])
    ap.add_argument("--cpu-sources", type=int, default=1)
    args = ap.parse_args()
    gb.init(0)
    header()
    run([("rmat22", lambda: rmat(22), True),
         ("rmat22_directed", lambda: rmat(22, undirected=False), False),
         ("grid27", grid, True)], args, measure)


if __name__ == "__main__":
    main()
