"""Connected components on the device (algorithm.cc): time per call against scipy's
single-thread components, a BFS on the same graph and the time to stream the CSR once.

  python tools/bench_cc.py [--iters 10] [--warmup 2] [--only NAME]

Workloads:
  rmat22, rmat24  R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, symmetrised,
                  self-loops and duplicate edges removed, generator seed 0
                  (graphs.rmat_edges / build_csr / matrix_from_csr): a giant component
                  plus isolated vertices.  Marked symmetric, so the kernel may skip the
                  sampled component.
  rmat22_noskip   the same R-MAT-22 adopted with its CSR alone and not marked
                  symmetric: no skip, so every list is linked, the hubs' lists of up
                  to 10^5 entries and more each by one warp.
  rmat22_directed R-MAT-22 with each edge stored one way only (self-loops and
                  duplicates removed), CSR alone: a non-symmetric input.
  grid27          the 27-point stencil on a 128^3 grid of tools/bench_mxm.py (self-loops
                  included): one component of large diameter.
  pieces          4096 pieces of 1024 vertices, each a random spanning tree plus two
                  random edges per vertex, ids interleaved across the range by a fixed
                  permutation (seed 5), symmetrised: many components of equal size, so
                  skipping the largest sampled one saves little.

Each line is one JSON record.  "ms" is the median of the CUDA-event times that cc
returns for warm calls.  A time is quoted only after the labels equal the checker's
(tests/support.py components: scipy's weak components, each label mapped to its
component's minimum id) entry for entry and the counts agree ("equals_checker");
"cpu_ms" is that checker's time on one host thread.  "bfs_ms" is the median tight time
of algorithm.bfs from the highest-degree vertex on the same matrix (direction-optimised,
the flags of bench.py; not timed, null, for the matrices adopted with their CSR
alone).  "stream_bound_ms" is (4 (n + 1) + 4 nnz) bytes, the CSR read
once, at 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth): a bound, not an achieved
rate.  "card" is the GPU's name and power limit, read in the same run.
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

from bench_mxm import card, grid27                # noqa: E402
import graphblast_b200 as gb                      # noqa: E402
from graphblast_b200 import algorithm, graphs     # noqa: E402
from support import components                    # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def median_ms(fn, iters, warmup):
    """Median of the device times fn() returns, after warmup calls."""
    for _ in range(warmup):
        fn()
    return float(np.median([fn() for _ in range(iters)]))


def rmat(scale, undirected=True):
    src, dst = graphs.rmat_edges(scale, seed=0)
    rp, ci = graphs.build_csr(1 << scale, src, dst, undirected)
    return 1 << scale, rp, ci


def pieces(count=4096, size=1024, seed=5):
    rng = np.random.RandomState(seed)
    n = count*size
    local = np.arange(1, size)
    tree_parent = (rng.rand(count, size - 1)*local).astype(np.int64)   # < own index
    base = (np.arange(count)*size)[:, None]
    src = [(base + local).ravel(), (base + rng.randint(0, size, (count, 2*size))).ravel()]
    dst = [(base + tree_parent).ravel(), (base + rng.randint(0, size, (count, 2*size))).ravel()]
    perm = rng.permutation(n)
    src = perm[np.concatenate(src)].astype(np.int32)
    dst = perm[np.concatenate(dst)].astype(np.int32)
    rp, ci = graphs.build_csr(n, torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda(),
                              True)
    return n, rp, ci


def measure(name, n, rp, ci, args, symmetric=True):
    A = graphs.matrix_from_csr(n, rp, ci, symmetric=symmetric)
    nnz = int(ci.numel())
    rec = {"workload": name, "n": n, "nnz": nnz, "symmetric": symmetric, "card": card()}
    desc = gb.Descriptor()
    v = gb.Vector(n)
    count = [0]

    def run_cc():
        count[0], ms = algorithm.cc(v, A, desc)
        return ms
    rec["ms"] = median_ms(run_cc, args.iters, args.warmup)
    rec["components"] = count[0]
    got = v.extractTuples()

    h_rp, h_ci = rp.cpu().numpy(), ci.cpu().numpy()
    deg = np.diff(h_rp)
    t0 = time.perf_counter()
    want, want_k = components(n, h_rp, h_ci)
    rec["cpu_ms"] = (time.perf_counter() - t0)*1e3
    rec["equals_checker"] = bool(np.array_equal(got.astype(np.int64), want) and
                                 count[0] == want_k)
    rec["largest_component"] = int(np.bincount(want).max())
    rec["max_degree"] = int(deg.max())

    rec["bfs_ms"] = None
    if symmetric:
        src = int(np.argmax(deg))
        bdesc = gb.Descriptor(mxvmode=0, struconly=1, opreuse=1, earlyexit=1)
        lv = gb.Vector(n)
        rec["bfs_ms"] = median_ms(lambda: algorithm.bfs(lv, A, src, bdesc, timed=True),
                                  args.iters, args.warmup)
        del lv
    rec["stream_bound_ms"] = (4.0*(n + 1) + 4.0*nnz)/HBM_BYTES_PER_S*1e3
    if rec["equals_checker"]:
        rec["cpu_over_cc"] = rec["cpu_ms"]/rec["ms"]
        if rec["bfs_ms"] is not None:
            rec["cc_over_bfs"] = rec["ms"]/rec["bfs_ms"]
    else:
        rec.pop("ms")                 # wrong labels get no time
    print(json.dumps(rec), flush=True)
    del A, v
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default=None,
                    help="rmat22, rmat22_noskip, rmat22_directed, rmat24, grid27 or pieces")
    args = ap.parse_args()
    gb.init(0)
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    builders = [("rmat22", lambda: rmat(22), True),
                ("rmat22_noskip", lambda: rmat(22), False),
                ("rmat22_directed", lambda: rmat(22, undirected=False), False),
                ("rmat24", lambda: rmat(24), True),
                ("grid27", lambda: grid27(128), True), ("pieces", pieces, True)]
    for name, build, symmetric in builders:
        if args.only in (None, name):
            n, rp, ci = build()
            measure(name, n, rp, ci, args, symmetric)
            del rp, ci
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
