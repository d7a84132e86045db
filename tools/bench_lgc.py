"""Local graph clustering on the device (algorithm.lgc and algorithm.lgc_sweep): time per
call on each route, checked bit for bit against the host restatement.

  python tools/bench_lgc.py [--scales 22 24] [--sources 2] [--iters 5] [--warmup 1]
                            [--driver-rounds 10] [--restate-max 22] [--glgc 16]

Workloads, on R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, symmetrised, self-loops
and duplicates removed, generator seed 0 (graphs.rmat_edges / build_csr /
matrix_from_csr), from --sources fixed-seed sources (seed 1) among the vertices with
d > 0:
  driver  the reference driver's parameters (example/glgc.cu): alpha from phi = 0.5,
          alpha = phi^2/(225 ln(100 sqrt(nnz))), eps = 1e-7.  The frontier spreads over
          most of the graph within a few rounds and the run lasts thousands of rounds,
          so it is cut at --driver-rounds rounds (desc max_niter) to keep the host check
          affordable: the dense-round side.
  local   alpha = 0.15, eps = 1e-6: a few dozen rounds over a small part of the graph,
          the sparse-round side.

Each line is one JSON record per (graph, setting, source).  "ms" maps the route
(default = mxvmode 0, push = 1, sparse rounds only, pull = 2, dense rounds only) to the
median CUDA-event time lgc returns over --iters warm calls; "sweep_ms" is the same for
lgc_sweep on the default route's p.  A time is quoted only after the result is checked
("checked"):
  - every route's p equals the reference's own SimpleReferenceLgc<float> (ref_lgc, one
    host thread, run with max_niter = the rounds the device ran) bit for bit, and every
    route ran the same rounds; "ref_ms" is that call's time;
  - up to --restate-max, also p, r and rounds against tests/lgc_reference.py's push()
    and the sweep's size and conductance against its sweep(); "pushed" (the sum over
    the rounds of the frontier's volume) comes from there.  Above it the sweep's
    size and conductance are not checked and get no time.
Without the reference library the restatement alone is the check.  "rounds",
"support", "cluster" and "conductance" describe the run.

--glgc SCALE also times the reference's own operation loop, the unchanged glgc driver
(oracle/_ref/dropin/glgc, algorithm/lgc.hpp over this backend), on an R-MAT of that
scale written as a Matrix Market file (tools/gen_rmat_mtx.py, seed 1), with the
driver's alpha and eps (computed in float there), max_niter = --driver-rounds, from the
highest-degree vertex; lgc runs the same problem on the matrix loaded from that file.
The two do not compute the same floats (the driver's loop is not the checker's order),
so only lgc's p is checked, against the restatement.  "card" is the GPU's name and power
limit, read in the same run.
"""
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import ROOT, card, device_ms, header, parser, rmat_csr
import graphblast_b200 as gb
from graphblast_b200 import algorithm, graphs
import lgc_reference as L

ROUTES = (("default", 0), ("push", 1), ("pull", 2))


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def measure(name, A, n, h_rp, h_ci, setting, alpha, eps, cap, s, restate, args):
    rec = {"workload": name, "setting": setting, "n": n, "nnz": int(len(h_ci)),
           "source": s, "alpha": alpha, "eps": eps, "max_niter": cap, "card": card()}
    p, r = gb.Vector(n), gb.Vector(n)
    got = {}
    for route, mode in ROUTES:
        desc = gb.Descriptor(mxvmode=mode, max_niter=cap)
        k, _ = algorithm.lgc(p, A, s, alpha, eps, desc, residual=r)
        got[route] = (k, p.extractTuples(), r.extractTuples())
    k = got["default"][0]
    ok = all(g[0] == k and np.array_equal(bits(g[1]), bits(got["default"][1])) and
             np.array_equal(bits(g[2]), bits(got["default"][2])) for g in got.values())
    rec["rounds"] = k
    if L.ref_lgc_available():
        t0 = time.perf_counter()
        want = L.ref_lgc(h_rp, h_ci, s, alpha, eps, k)
        rec["ref_ms"] = (time.perf_counter() - t0)*1e3
        ok = ok and np.array_equal(bits(got["default"][1]), bits(want))
    want_size = want_phi = None
    if restate:
        t0 = time.perf_counter()
        want_p, want_r, want_k, pushed = L.push(h_rp, h_ci, s, alpha, eps, cap)
        rec["host_ms"] = (time.perf_counter() - t0)*1e3
        rec["pushed"] = pushed
        ok = ok and (want_k == k and np.array_equal(bits(got["default"][1]), bits(want_p)) and
                     np.array_equal(bits(got["default"][2]), bits(want_r)))
        _, want_size, want_phi = L.sweep(h_rp, h_ci, want_p)
    elif not L.ref_lgc_available():
        ok = False                     # nothing to check against
    if ok:
        rec["ms"] = {}
        for route, mode in ROUTES:
            desc = gb.Descriptor(mxvmode=mode, max_niter=cap)
            rec["ms"][route] = device_ms(
                lambda: algorithm.lgc(p, A, s, alpha, eps, desc, residual=r)[1],
                args.iters, args.warmup)
    algorithm.lgc(p, A, s, alpha, eps, gb.Descriptor(max_niter=cap))
    cl = gb.Vector(n)
    size, phi, _ = algorithm.lgc_sweep(cl, p, A, gb.Descriptor())
    if restate:
        ok = ok and size == want_size and (phi == want_phi or
                                           (np.isnan(phi) and np.isnan(want_phi)))
    if ok and restate:
        rec["sweep_ms"] = device_ms(lambda: algorithm.lgc_sweep(cl, p, A, gb.Descriptor())[2],
                                    args.iters, args.warmup)
    h_p = got["default"][1]
    rec.update(support=int(np.count_nonzero((h_p > 0) & (np.diff(h_rp) > 0))),
               cluster=size, conductance=phi, checked=bool(ok))
    print(json.dumps(rec), flush=True)


def glgc(scale, args):
    """The unchanged glgc driver against lgc on one R-MAT Matrix Market file."""
    driver = os.path.join(ROOT, "oracle", "_ref", "dropin", "glgc")
    rec = {"workload": "rmat%d.mtx" % scale, "setting": "driver", "card": card()}
    if not os.path.exists(driver):
        rec["glgc"] = "not built"
        print(json.dumps(rec), flush=True)
        return
    with tempfile.TemporaryDirectory() as tmp:
        mtx = os.path.join(tmp, "rmat%d.mtx" % scale)
        subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "gen_rmat_mtx.py"),
                               str(scale), "16", mtx])
        A = gb.Matrix.from_mtx(mtx, directed=2)
        h_rp, h_ci, _ = A.extract_csr()
        n = len(h_rp) - 1
        s = int(np.argmax(np.diff(h_rp)))
        alpha = float(np.float32(0.25/(225.0*np.log(100.0*np.sqrt(float(len(h_ci)))))))
        eps = float(np.float32(1e-7))
        cap = args.driver_rounds
        out = subprocess.run([driver, "--mxvmode", "0", "--niter", str(args.iters),
                              "--timing", "1", "--directed", "2", "--max_niter", str(cap),
                              "--source", str(s), mtx],
                             capture_output=True, text=True, cwd=tmp).stdout
        m = re.search(r"^tight, ([0-9.eE+-]+)", out, re.M)
        rec.update(n=n, nnz=int(len(h_ci)), source=s, alpha=alpha, eps=eps, max_niter=cap,
                   glgc_ms=float(m.group(1)) if m else None)
    p = gb.Vector(n)
    desc = gb.Descriptor(max_niter=cap)
    k, _ = algorithm.lgc(p, A, s, alpha, eps, desc)
    want_p, _, want_k, _ = L.push(h_rp, h_ci, s, alpha, eps, cap)
    rec["rounds"] = k
    rec["checked"] = bool(k == want_k and np.array_equal(bits(p.extractTuples()),
                                                         bits(want_p)))
    if rec["checked"]:
        rec["lgc_ms"] = device_ms(lambda: algorithm.lgc(p, A, s, alpha, eps, desc)[1],
                                  args.iters, args.warmup)
    print(json.dumps(rec), flush=True)


def main():
    ap = parser(iters=5, warmup=1)
    ap.add_argument("--scales", type=int, nargs="+", default=[22, 24])
    ap.add_argument("--sources", type=int, default=2)
    ap.add_argument("--driver-rounds", type=int, default=10)
    ap.add_argument("--restate-max", type=int, default=22,
                    help="largest scale also checked against the numpy restatement")
    ap.add_argument("--glgc", type=int, default=None,
                    help="also time the glgc driver on an R-MAT .mtx of this scale")
    args = ap.parse_args()
    gb.init(0)
    header()
    for scale in args.scales:
        n, rp, ci = rmat_csr(scale, seed=0)
        A = graphs.matrix_from_csr(n, rp, ci, symmetric=True)
        h_rp, h_ci = rp.cpu().numpy(), ci.cpu().numpy()
        deg = np.diff(h_rp)
        srcs = np.random.RandomState(1).choice(np.nonzero(deg > 0)[0], args.sources,
                                               replace=False)
        settings = [("driver", L.driver_alpha(len(h_ci)), 1e-7, args.driver_rounds),
                    ("local", 0.15, 1e-6, 10000)]
        for setting, alpha, eps, cap in settings:
            for s in srcs:
                measure("rmat%d" % scale, A, n, h_rp, h_ci, setting, alpha, eps, cap,
                        int(s), scale <= args.restate_max, args)
        del A, rp, ci
        torch.cuda.empty_cache()
    if args.glgc is not None:
        glgc(args.glgc, args)


if __name__ == "__main__":
    main()
