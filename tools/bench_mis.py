"""Maximal independent set on the device (algorithm.mis): time per call against the
graph colouring it replaces (algorithm.gc, whose colour class 1 is the same set) and
against the single-thread CPU oracle.

  python tools/bench_mis.py [--iters 10] [--warmup 2] [--gc-iters 3] [--only rmat22|rmat24]

Workloads: the graphs of tools/bench_gc.py, R-MAT (0.57, 0.19, 0.19, 0.05) of scale 22
and 24, edge factor 16, symmetrised, self-loops and duplicate edges removed
(graphs.rmat_edges / build_csr / matrix_from_csr), seed 0.

Each line is one JSON record.  "ms" is the median of the CUDA-event times that mis
returns for warm calls, "gc_ms" the same for gc on the same graph in the same run.
Before any time is quoted, the set must equal the CPU oracle's (tests/mis_oracle.c
orc_mis, the greedy MIS in the same priority order) entry for entry; "cpu_ms" is
that oracle's single-thread time and "luby_depth" its synchronous Luby round count.
"gc_class1_equal" says whether gc's colour class 1 is the same set.  "card" is the
GPU's name and power limit, read in the same run.
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
import greedy_oracle                              # noqa: E402


def median_ms(fn, iters, warmup):
    """Median of the device times fn() returns, after warmup calls."""
    for _ in range(warmup):
        fn()
    return float(np.median([fn() for _ in range(iters)]))


def measure(scale, args):
    n = 1 << scale
    src, dst = graphs.rmat_edges(scale)
    rp, ci = graphs.build_csr(n, src, dst, True)
    del src, dst
    A = graphs.matrix_from_csr(n, rp, ci)
    rec = {"workload": "rmat%d" % scale, "n": n, "nnz": int(ci.numel()), "card": card()}
    desc = gb.Descriptor()
    v = gb.Vector(n)
    size = [0]

    def run_mis():
        size[0], ms = algorithm.mis(v, A, 0, desc)
        return ms
    rec["ms"] = median_ms(run_mis, args.iters, args.warmup)
    rec["size"] = size[0]
    got = v.extractTuples()

    colours = gb.Vector(n)
    rec["gc_ms"] = median_ms(lambda: algorithm.gc(colours, A, 0, desc)[1],
                             args.gc_iters, 1)
    rec["gc_class1_equal"] = bool(np.array_equal(
        got, (colours.extractTuples() == 1).astype(np.float32)))
    rec["gc_over_mis"] = rec["gc_ms"]/rec["ms"]

    h_rp, h_ci = rp.cpu().numpy(), ci.cpu().numpy()
    t0 = time.perf_counter()
    want, want_size, depth = greedy_oracle.mis(h_rp, h_ci, 0)
    rec["cpu_ms"] = (time.perf_counter() - t0)*1e3
    rec["luby_depth"] = depth
    rec["oracle_size"] = want_size
    rec["equals_oracle"] = bool(np.array_equal(got, want.astype(np.float32)) and
                                size[0] == want_size)
    if not rec["equals_oracle"]:
        rec.pop("ms")                 # a wrong set gets no time
        rec.pop("gc_over_mis")
    print(json.dumps(rec), flush=True)
    del A, rp, ci, v, colours
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--gc-iters", type=int, default=3)
    ap.add_argument("--only", default=None, help="rmat22 or rmat24")
    args = ap.parse_args()
    gb.init(0)
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    for scale in (22, 24):
        if args.only in (None, "rmat%d" % scale):
            measure(scale, args)


if __name__ == "__main__":
    main()
