"""Strongly connected components on the device (algorithm.scc): time per call against
scipy's single-thread strong components, weak cc on the same matrix and the time to
stream the CSR and CSC once.

  python tools/bench_scc.py [--iters 10] [--warmup 2] [--only NAME] [--cycle-scale 20]

Workloads (R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, generator seed 0,
graphs.rmat_edges / build_csr, self-loops and duplicates removed):
  rmat22_directed, rmat24_directed
                  R-MAT edges one way; the CSC is build_csr on the swapped endpoints;
                  both adopted.  A giant component, a large trimmed fringe and many
                  small components.
  rmat22_sym_csc  the symmetrised R-MAT-22 adopted as CSR + CSC and not marked
                  symmetric: the kernel's path on one giant component (marked
                  symmetric, scc would run cc's kernel).
  pieces_directed 4096 pieces of 1024 vertices, each a directed Hamiltonian cycle plus
                  one random arc per vertex inside it, arcs only from lower to higher
                  piece index (4 per piece), ids interleaved by a fixed permutation
                  (seed 5): one pivot piece, the rest for the colouring.
  cycle           one directed cycle of 2^cycle-scale vertices (default 2^20), ids
                  permuted: every level of the pivot's reach is one vertex, the deep
                  worst case, one grid barrier per level.

Each line is one JSON record.  "ms" is the median of the CUDA-event times that scc
returns for warm calls.  A time is quoted only after the labels equal the checker's
(tests/scc_reference.py: scipy's strong components, each label mapped to its
component's minimum id) entry for entry and the counts agree ("equals_checker");
"cpu_ms" is that checker's time on one host thread.  "cc_ms" is the median time of
algorithm.cc (weak components) on the same matrix.  "trimmed", "pivot_size",
"colour_iterations" and "barriers" are algorithm.scc_stats() of the last call.
"stream_bound_ms" is (8 (n + 1) + 8 nnz) bytes, the CSR and CSC read once, at
3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth): a bound, not an achieved rate.
"card" is the GPU's name and power limit, read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))

from bench_mxm import card                        # noqa: E402
import graphblast_b200 as gb                      # noqa: E402
from graphblast_b200 import algorithm, graphs     # noqa: E402
from scc_reference import scc as checker          # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def median_ms(fn, iters, warmup):
    """Median of the device times fn() returns, after warmup calls."""
    for _ in range(warmup):
        fn()
    return float(np.median([fn() for _ in range(iters)]))


def adopt(n, src, dst, undirected=False):
    """CSR from (src, dst), CSC from the swapped endpoints, both adopted."""
    rp, ci = graphs.build_csr(n, src, dst, undirected)
    cp, ri = graphs.build_csr(n, dst, src, undirected)
    A = gb.Matrix(n, n)
    A.build_device_csr(rp, ci, torch.ones(ci.numel(), dtype=torch.float32, device="cuda"),
                       ci.numel(), cp, ri,
                       torch.ones(ri.numel(), dtype=torch.float32, device="cuda"))
    return A, rp, ci


def rmat(scale, undirected=False):
    src, dst = graphs.rmat_edges(scale, seed=0)
    return (1 << scale,) + adopt(1 << scale, src, dst, undirected)


def pieces(count=4096, size=1024, seed=5):
    rng = np.random.RandomState(seed)
    n = count*size
    base = (np.arange(count)*size)[:, None]
    local = np.arange(size)
    src = [(base + local).ravel(), (base + rng.randint(0, size, (count, size))).ravel()]
    dst = [(base + (local + 1) % size).ravel(),
           (base + rng.randint(0, size, (count, size))).ravel()]
    a, b = rng.randint(0, count, 4*count), rng.randint(0, count, 4*count)
    keep = a != b
    lo, hi = np.minimum(a, b)[keep], np.maximum(a, b)[keep]
    src.append(lo*size + rng.randint(0, size, len(lo)))
    dst.append(hi*size + rng.randint(0, size, len(hi)))
    perm = rng.permutation(n)
    src = torch.from_numpy(perm[np.concatenate(src)].astype(np.int32)).cuda()
    dst = torch.from_numpy(perm[np.concatenate(dst)].astype(np.int32)).cuda()
    return (n,) + adopt(n, src, dst)


def cycle(scale):
    n = 1 << scale
    ids = np.random.RandomState(6).permutation(n).astype(np.int32)
    src = torch.from_numpy(ids).cuda()
    dst = torch.from_numpy(np.roll(ids, -1)).cuda()
    return (n,) + adopt(n, src, dst)


def measure(name, n, A, rp, ci, args):
    nnz = int(ci.numel())
    rec = {"workload": name, "n": n, "nnz": nnz, "card": card()}
    desc = gb.Descriptor()
    v = gb.Vector(n)
    count = [0]

    def run_scc():
        count[0], ms = algorithm.scc(v, A, desc)
        return ms
    rec["ms"] = median_ms(run_scc, args.iters, args.warmup)
    rec["components"] = count[0]
    (rec["trimmed"], rec["pivot_size"], rec["colour_iterations"],
     rec["barriers"]) = algorithm.scc_stats()
    got = v.extractTuples()

    h_rp, h_ci = rp.cpu().numpy(), ci.cpu().numpy()
    t0 = time.perf_counter()
    want, want_k = checker(h_rp, h_ci)
    rec["cpu_ms"] = (time.perf_counter() - t0)*1e3
    rec["equals_checker"] = bool(np.array_equal(got.astype(np.int64), want) and
                                 count[0] == want_k)
    rec["largest_component"] = int(np.bincount(want).max())

    cv = gb.Vector(n)
    rec["cc_ms"] = median_ms(lambda: algorithm.cc(cv, A, desc)[1], args.iters, args.warmup)
    rec["stream_bound_ms"] = (8.0*(n + 1) + 8.0*nnz)/HBM_BYTES_PER_S*1e3
    if rec["equals_checker"]:
        rec["cpu_over_scc"] = rec["cpu_ms"]/rec["ms"]
    else:
        rec.pop("ms")                 # wrong labels get no time
    print(json.dumps(rec), flush=True)
    del A, v, cv
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cycle-scale", type=int, default=20)
    ap.add_argument("--only", default=None,
                    help="rmat22_directed, rmat24_directed, rmat22_sym_csc, "
                         "pieces_directed or cycle")
    args = ap.parse_args()
    gb.init(0)
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    builders = [("rmat22_directed", lambda: rmat(22)),
                ("rmat24_directed", lambda: rmat(24)),
                ("rmat22_sym_csc", lambda: rmat(22, undirected=True)),
                ("pieces_directed", pieces),
                ("cycle", lambda: cycle(args.cycle_scale))]
    for name, build in builders:
        if args.only in (None, name):
            n, A, rp, ci = build()
            measure(name, n, A, rp, ci, args)
            del A, rp, ci
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
