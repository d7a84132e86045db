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
  grid27          the 27-point stencil on a 128^3 grid of tools/benchlib.py (self-loops
                  included): one component of large diameter.
  pieces          tools/benchlib.py's tree_pieces: 4096 pieces of 1024 vertices, each a
                  random spanning tree plus two random edges per vertex, ids interleaved
                  across the range by a fixed permutation (seed 5), symmetrised: many
                  components of equal size, so skipping the largest sampled one saves
                  little.

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
import json
import time

import numpy as np

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import (card, device_ms, grid27, header, parser, rmat_csr, run,
                      stream_bound_ms, tree_pieces)
import graphblast_b200 as gb
from graphblast_b200 import algorithm, graphs
from support import components


def measure(name, n, rp, ci, symmetric, args):
    A = graphs.matrix_from_csr(n, rp, ci, symmetric=symmetric)
    nnz = int(ci.numel())
    rec = {"workload": name, "n": n, "nnz": nnz, "symmetric": symmetric, "card": card()}
    desc = gb.Descriptor()
    v = gb.Vector(n)
    count = [0]

    def run_cc():
        count[0], ms = algorithm.cc(v, A, desc)
        return ms
    rec["ms"] = device_ms(run_cc, args.iters, args.warmup)
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
        rec["bfs_ms"] = device_ms(lambda: algorithm.bfs(lv, A, src, bdesc, timed=True),
                                  args.iters, args.warmup)
        del lv
    rec["stream_bound_ms"] = stream_bound_ms(4.0*(n + 1) + 4.0*nnz)
    if rec["equals_checker"]:
        rec["cpu_over_cc"] = rec["cpu_ms"]/rec["ms"]
        if rec["bfs_ms"] is not None:
            rec["cc_over_bfs"] = rec["ms"]/rec["bfs_ms"]
    else:
        rec.pop("ms")                 # wrong labels get no time
    print(json.dumps(rec), flush=True)


def main():
    args = parser(iters=10, warmup=2,
                  only="rmat22, rmat22_noskip, rmat22_directed, rmat24, grid27 or "
                       "pieces").parse_args()
    gb.init(0)
    header()
    run([("rmat22", lambda: rmat_csr(22, seed=0), True),
         ("rmat22_noskip", lambda: rmat_csr(22, seed=0), False),
         ("rmat22_directed", lambda: rmat_csr(22, seed=0, undirected=False), False),
         ("rmat24", lambda: rmat_csr(24, seed=0), True),
         ("grid27", lambda: grid27(128), True),
         ("pieces", tree_pieces, True)], args, measure)


if __name__ == "__main__":
    main()
