"""k-truss and truss decomposition on the device (algorithm.ktruss, algorithm.trussness):
time per call, with the peel rounds and levels each call ran, against the triangle
count (algorithm.tc) of the same graph.

  python tools/bench_ktruss.py [--scales 18 20 22] [--iters 5] [--warmup 1]

Workloads: R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, generator seed 1,
symmetrised, self-loops and duplicate edges removed (graphs.rmat_edges / build_csr /
matrix_from_csr), FP32, marked symmetric; INT32 results.  These are the graphs of
`bench.py --algo tc`, so the committed triangle counts apply to them.

Each line is one JSON record per scale.  Times are medians of the CUDA-event times the
calls return for warm calls.  "support_ms" is the support pass alone, timed inside the
kernel (algorithm.ktruss_stats); "k2_ms" a whole ktruss call with k = 2, which peels
nothing: the edge slots, the support pass and writing the result.  "ktruss" holds
k = 3, 8 and 32, and "trussness" the full decomposition, each with its rounds and
levels (algorithm.ktruss_stats: rounds that removed edges, levels that did).  "tc_ms" is
algorithm.tc on tril(A) of the same graph, built by the library's tril, with the
default descriptor.  Every result is checked before it is timed: up to scale 20
against the CPU bucket peel of tests/truss_oracle.c, entry for entry (the oracle's
calls run in threads at once, minutes at scale 20); at every scale, sum(C)/6 at k = 2
against "triangles_tril" of tests/golden/tc_golden.json where it has the graph, and the
pattern of each ktruss(k) against {tau >= k} of the trussness result.  "card" is the
GPU's name and power limit, read in the same run.
"""
import concurrent.futures
import json
import os

import numpy as np

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import ROOT, card, device_ms, parser, rmat_csr
import truss_reference
import graphblast_b200 as gb
from graphblast_b200 import algorithm, graphs

KS = (3, 8, 32)
ORACLE_MAX_SCALE = 20


def golden_triangles(scale, nnz):
    table = json.load(open(os.path.join(ROOT, "tests", "golden", "tc_golden.json")))
    g = table.get("rmat%d" % scale)
    return int(g["triangles_tril"]) if g is not None and g["nnz"] == nnz else None


def same_csr(M, want):
    got = M.extract_csr()
    return (np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and
            np.array_equal(got[2].astype(np.int64), np.asarray(want[2], np.int64)))


def run(scale, iters, warmup):
    n, rp, ci = rmat_csr(scale, seed=1)
    A = graphs.matrix_from_csr(n, rp, ci)
    h_rp, h_ci = rp.cpu().numpy(), ci.cpu().numpy()
    nnz = len(h_ci)
    desc = gb.Descriptor()
    out = gb.Matrix(n, n, dtype=gb.api.INT32)
    rec = {"workload": "rmat%d" % scale, "n": n, "nnz": nnz, "card": card()}

    # ---- checks ------------------------------------------------------------------------
    oracle = {}
    if scale <= ORACLE_MAX_SCALE:          # ctypes releases the GIL: the calls overlap
        pool = concurrent.futures.ThreadPoolExecutor(len(KS) + 2)
        oracle[0] = pool.submit(truss_reference.trussness, h_rp, h_ci)
        for k in (2,) + KS:
            oracle[k] = pool.submit(truss_reference.ktruss, h_rp, h_ci, k)
    algorithm.trussness(out, A, desc)
    t_rp, t_ci, tau = out.extract_csr()
    kmax = int(tau.max()) if len(tau) else 0
    checks = {}
    checks["trussness_pattern_is_A"] = bool(np.array_equal(t_rp, h_rp) and
                                            np.array_equal(t_ci, h_ci))
    if scale <= ORACLE_MAX_SCALE:
        want_tau, want_kmax = oracle[0].result()
        checks["trussness_equals_oracle"] = bool(
            np.array_equal(tau.astype(np.int64), want_tau) and kmax == want_kmax)
    rows = np.repeat(np.arange(n), np.diff(h_rp))
    for k in (2,) + KS:
        nedges, _ = algorithm.ktruss(out, A, k, desc)
        if scale <= ORACLE_MAX_SCALE:
            sup, kept = oracle[k].result()
            checks["ktruss%d_equals_oracle" % k] = bool(
                same_csr(out, truss_reference.kept_csr(h_rp, h_ci, sup)) and nedges == kept)
        c_rp, c_ci, c_v = out.extract_csr()
        keep = tau >= k
        want_rp = np.concatenate([[0], np.cumsum(np.bincount(rows[keep], minlength=n))])
        checks["ktruss%d_is_tau_level_set" % k] = bool(
            np.array_equal(c_rp, want_rp) and np.array_equal(c_ci, h_ci[keep]))
        if k == 2:
            tri = golden_triangles(scale, nnz)
            total = int(c_v.astype(np.int64).sum())
            rec["triangles"] = total//6
            if tri is not None:
                checks["support_sum_equals_golden_tc"] = bool(total == 6*tri)
    rec["checks"] = checks
    rec["kmax"] = kmax
    if not all(checks.values()):
        rec["error"] = "a check failed; nothing timed"
        return rec

    # ---- times -------------------------------------------------------------------------
    support = []

    def k2():
        ms = algorithm.ktruss(out, A, 2, desc)[1]
        support.append(algorithm.ktruss_stats()[2])
        return ms
    rec["k2_ms"] = device_ms(k2, iters, warmup)
    rec["support_ms"] = float(np.median(support[warmup:]))
    rec["ktruss"] = []
    for k in KS:
        ms = device_ms(lambda: algorithm.ktruss(out, A, k, desc)[1], iters, warmup)
        rounds, levels, _ = algorithm.ktruss_stats()
        rec["ktruss"].append({"k": k, "ms": ms, "edges": out.nvals()//2, "rounds": rounds})
    ms = device_ms(lambda: algorithm.trussness(out, A, desc)[1], iters, warmup)
    rounds, levels, _ = algorithm.ktruss_stats()
    rec["trussness"] = {"ms": ms, "rounds": rounds, "levels": levels}
    L = graphs.matrix_from_csr(n, rp, ci, dtype=gb.api.INT32, symmetric=True)
    L.tril(desc)
    B = gb.Matrix(n, n, dtype=gb.api.INT32)
    rec["tc_ms"] = device_ms(lambda: algorithm.tc(L, B, desc)[1], iters, warmup)
    return rec


def main():
    ap = parser(iters=5, warmup=1)
    ap.description = __doc__.split("\n\n")[0]
    ap.add_argument("--scales", type=int, nargs="+", default=[18, 20, 22])
    args = ap.parse_args()
    gb.init(0)
    for scale in args.scales:
        print(json.dumps(run(scale, args.iters, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
