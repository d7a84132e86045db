"""Community detection by label propagation on the device (algorithm.cdlp): time per call
and per iteration against the C checker on one thread and the time to stream the lists.

  python tools/bench_cdlp.py [--iters 10] [--warmup 2] [--only NAME]

Workloads:
  rmat22, rmat24  R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, symmetrised,
                  self-loops and duplicate edges removed, generator seed 0, marked
                  symmetric: the kernel reads the CSR alone.
  rmat22_directed R-MAT-22 with each edge stored one way only, CSR and CSC adopted:
                  every list is read twice, once from each side.
  grid27          the 27-point stencil on a 128^3 grid of tools/benchlib.py (self-loops
                  included): lists of 8 to 27 entries, all in the short class.
  pieces          the 4096 pieces of 1024 vertices of tools/benchlib.py's tree_pieces.

Settings: max_iter = 10 (the Graphalytics default), and one run with max_iter = 1000
that stops at the first iteration that changes nothing ("fix_iterations"; 1000 when no
fixpoint is reached, as on R-MAT, where synchronous propagation oscillates).

Each line is one JSON record.  "ms" is the median of the CUDA-event times that cdlp
returns for warm calls at max_iter = 10, "ms_per_iteration" that over the iterations
run.  A time is quoted only after the labels, community count and iteration count
equal the C checker's (tests/cdlp_reference.py) entry for entry ("equals_checker");
"cpu_ms" is the checker's time on one host thread (R-MAT-22 and smaller).  The run to
the fixpoint is timed once, after a warm call, and compared with the checker only when
it stops within 60 iterations ("fix_equals_checker", else null and no time).
"stream_bound_ms" is, per iteration, (4 (n + 1) + 4 nnz) bytes for each list read (the
CSR, and the CSC when it is held apart) at 3.35 TB/s, the H100 SXM data-sheet HBM3
bandwidth: computed from sizes, a bound and not an achieved rate.  "card" is the GPU's
name and power limit, read in the same run.
"""
import json
import time

import numpy as np

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import (adopt_csr_csc, card, device_ms, grid27, header, parser, rmat_csr, run,
                      stream_bound_ms, tree_pieces)
import cdlp_reference as R
import graphblast_b200 as gb
from graphblast_b200 import algorithm, graphs

MAX_ITER = 10
FIX_ITER = 1000
FIX_CHECK_MAX = 60


def symmetric(build):
    def make():
        n, rp, ci = build()
        return n, graphs.matrix_from_csr(n, rp, ci, symmetric=True), rp, ci
    return make


def directed(scale):
    n = 1 << scale
    return (n,) + adopt_csr_csc(n, *graphs.rmat_edges(scale, seed=0), False)


def measure(name, n, A, rp, ci, lists, args):
    nnz = int(ci.numel())
    rec = {"workload": name, "n": n, "nnz": nnz, "lists_read": lists, "card": card()}
    desc = gb.Descriptor()
    v = gb.Vector(n)
    out = {}

    def run_cdlp(max_iter):
        out["k"], out["it"], ms = algorithm.cdlp(v, A, max_iter, desc)
        return ms
    ms = device_ms(lambda: run_cdlp(MAX_ITER), args.iters, args.warmup)
    got = v.extractTuples().astype(np.int64)
    rec["communities"], rec["iterations"] = out["k"], out["it"]
    s = algorithm.cdlp_stats()
    rec["cdlp_stats"] = {"short_vertices": s[0], "warp_vertices": s[1], "long_vertices": s[2],
                         "long_items": s[3], "barriers": s[4]}
    h_rp, h_ci = rp.cpu().numpy(), ci.cpu().numpy()
    t0 = time.perf_counter()
    want, want_k, want_it = R.cdlp(h_rp, h_ci, MAX_ITER)
    cpu_ms = (time.perf_counter() - t0)*1e3
    if n <= (1 << 22):
        rec["cpu_ms"] = cpu_ms
    rec["equals_checker"] = bool(np.array_equal(got, want) and
                                 (out["k"], out["it"]) == (want_k, want_it))
    rec["stream_bound_ms"] = stream_bound_ms(lists*(4.0*(n + 1) + 4.0*nnz))
    if rec["equals_checker"]:
        rec["ms"] = ms
        rec["ms_per_iteration"] = rec["ms"]/max(out["it"], 1)
        rec["over_stream_bound"] = rec["ms_per_iteration"]/rec["stream_bound_ms"]
        if "cpu_ms" in rec:
            rec["cpu_over_cdlp"] = rec["cpu_ms"]/rec["ms"]

    run_cdlp(FIX_ITER)                              # warm
    fix_ms = run_cdlp(FIX_ITER)
    rec["fix_iterations"] = out["it"]
    rec["fix_equals_checker"] = None
    if out["it"] <= FIX_CHECK_MAX:
        got = v.extractTuples().astype(np.int64)
        want, want_k, want_it = R.cdlp(h_rp, h_ci, FIX_ITER)
        rec["fix_equals_checker"] = bool(np.array_equal(got, want) and
                                         (out["k"], out["it"]) == (want_k, want_it))
        if rec["fix_equals_checker"]:
            rec["fix_ms"] = fix_ms
    else:
        rec["fix_ms_per_iteration_unchecked"] = fix_ms/out["it"]
    print(json.dumps(rec), flush=True)


def main():
    args = parser(iters=10, warmup=2,
                  only="rmat22, rmat24, rmat22_directed, grid27 or pieces").parse_args()
    gb.init(0)
    header()
    run([("rmat22", symmetric(lambda: rmat_csr(22, seed=0)), 1),
         ("rmat24", symmetric(lambda: rmat_csr(24, seed=0)), 1),
         ("rmat22_directed", lambda: directed(22), 2),
         ("grid27", symmetric(lambda: grid27(128)), 1),
         ("pieces", symmetric(tree_pieces), 1)], args, measure)


if __name__ == "__main__":
    main()
