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
import json
import time

import numpy as np
import torch

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import (adopt_csr_csc, card, device_ms, header, parser, run,
                      stream_bound_ms)
import graphblast_b200 as gb
from graphblast_b200 import algorithm, graphs
from scc_reference import scc as checker


def rmat(scale, undirected=False):
    src, dst = graphs.rmat_edges(scale, seed=0)
    return (1 << scale,) + adopt_csr_csc(1 << scale, src, dst, undirected)


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
    return (n,) + adopt_csr_csc(n, src, dst, False)


def cycle(scale):
    n = 1 << scale
    ids = np.random.RandomState(6).permutation(n).astype(np.int32)
    src = torch.from_numpy(ids).cuda()
    dst = torch.from_numpy(np.roll(ids, -1)).cuda()
    return (n,) + adopt_csr_csc(n, src, dst, False)


def measure(name, n, A, rp, ci, args):
    nnz = int(ci.numel())
    rec = {"workload": name, "n": n, "nnz": nnz, "card": card()}
    desc = gb.Descriptor()
    v = gb.Vector(n)
    count = [0]

    def run_scc():
        count[0], ms = algorithm.scc(v, A, desc)
        return ms
    rec["ms"] = device_ms(run_scc, args.iters, args.warmup)
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
    rec["cc_ms"] = device_ms(lambda: algorithm.cc(cv, A, desc)[1], args.iters, args.warmup)
    rec["stream_bound_ms"] = stream_bound_ms(8.0*(n + 1) + 8.0*nnz)
    if rec["equals_checker"]:
        rec["cpu_over_scc"] = rec["cpu_ms"]/rec["ms"]
    else:
        rec.pop("ms")                 # wrong labels get no time
    print(json.dumps(rec), flush=True)


def main():
    ap = parser(iters=10, warmup=2,
                only="rmat22_directed, rmat24_directed, rmat22_sym_csc, pieces_directed "
                     "or cycle")
    ap.add_argument("--cycle-scale", type=int, default=20)
    args = ap.parse_args()
    gb.init(0)
    header()
    run([("rmat22_directed", lambda: rmat(22)),
         ("rmat24_directed", lambda: rmat(24)),
         ("rmat22_sym_csc", lambda: rmat(22, undirected=True)),
         ("pieces_directed", pieces),
         ("cycle", lambda: cycle(args.cycle_scale))], args, measure)


if __name__ == "__main__":
    main()
