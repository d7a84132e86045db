"""Unmasked SpGEMM C = A*A on the device: time per call, products/s, nnz(C),
against cuSPARSE (torch.sparse.mm on CUDA CSR tensors, plus-times) and, with
--scipy, single-threaded scipy; every output that is compared must agree.

  python tools/bench_mxm.py [--iters 10] [--warmup 2] [--scipy] [--only NAME]

Each line is one JSON record.  "product_ms" is a call whose C keeps only its CSR;
"mxm_ms" the default call, which also builds C's CSC; "csc_ms" their difference.
Times are medians of CUDA-event timings of single calls.  --profile adds
"phases_ms", kernel time per phase of one further call, taken after the timed ones.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import graphblast_b200 as gb                    # noqa: E402
from graphblast_b200 import graphs              # noqa: E402


def card():
    try:
        out = subprocess.check_output(
            ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
            text=True).strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001
        out = "unknown (%s)" % e
    return out


def rmat(scale):
    src, dst = graphs.rmat_edges(scale)
    rp, ci = graphs.build_csr(1 << scale, src, dst, True)
    return 1 << scale, rp, ci


def grid27(side):
    """3-D 27-point stencil on side^3 points, self loops included."""
    n = side ** 3
    idx = torch.arange(n, device="cuda", dtype=torch.int64)
    x, y, z = idx % side, (idx // side) % side, idx // (side * side)
    cols = []
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                ok = ((x + dx >= 0) & (x + dx < side) & (y + dy >= 0) & (y + dy < side) &
                      (z + dz >= 0) & (z + dz < side))
                cols.append(torch.where(ok, idx + dx + side * dy + side * side * dz,
                                        torch.full_like(idx, -1)))
    c = torch.stack(cols, 1)                    # ascending per row
    valid = c >= 0
    rp = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    rp[1:] = torch.cumsum(valid.sum(1), 0)
    return n, rp.int(), c[valid].int()


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def new_matrix(n, csr_only):
    if csr_only:
        os.environ["GRB_SPARSE_MATRIX_FORMAT"] = "1"
    try:
        return gb.Matrix(n, n)
    finally:
        os.environ.pop("GRB_SPARSE_MATRIX_FORMAT", None)


PHASES = [  # (phase, pattern on the kernel name), first match wins
    ("bounds+bins", r"mxmRowBound|mxmClassify"),
    ("symbolic S", r"mxmSymbolicKernel<256, true"),
    ("symbolic M", r"mxmSymbolicKernel<256, false"),
    ("symbolic L", r"mxmSymbolicKernel<1024"),
    ("symbolic D", r"mxmSymbolicDense"),
    ("numeric S", r"mxmNumericKernel<256, true"),
    ("numeric M", r"mxmNumericKernel<256, false"),
    ("numeric L", r"mxmNumericKernel<1024"),
    ("numeric D", r"mxmNumericDense|mxmFill"),
    ("scan", r"scanTile|scanTotals|scanAdd"),
    ("CSC build", r"ingest|radix"),
]


def phase_split(fn):
    """Device time per phase (ms) of one call of fn, from torch.profiler's CUDA
    kernel records; the scan kernels serve both C's row offsets and the CSC."""
    import re
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = (getattr(e, "self_device_time_total", None) or
              getattr(e, "self_cuda_time_total", 0.0))
        if not us:
            continue
        phase = next((p for p, pat in PHASES if re.search(pat, e.key)), "other")
        out[phase] = out.get(phase, 0.0) + us / 1e3
    return {k: round(v, 3) for k, v in out.items()}


def run(name, n, rp, ci, val, semiring, args):
    A = graphs.matrix_from_csr(n, rp, ci, val)
    deg = (rp[1:] - rp[:-1]).long()
    products = int(deg[ci.long()].sum().item())
    rec = {"workload": name, "n": n, "nnz_A": int(ci.numel()), "products": products,
           "semiring": semiring.name}
    desc = gb.Descriptor()
    C = new_matrix(n, True)
    rec["product_ms"] = timed(lambda: gb.mxm(C, None, None, semiring, A, A, desc),
                              args.iters, args.warmup)
    C2 = new_matrix(n, False)
    rec["mxm_ms"] = timed(lambda: gb.mxm(C2, None, None, semiring, A, A, desc),
                          args.iters, args.warmup)
    rec["csc_ms"] = rec["mxm_ms"] - rec["product_ms"]
    if args.profile:
        rec["phases_ms"] = phase_split(lambda: gb.mxm(C2, None, None, semiring, A, A, desc))
    rec["nnz_C"] = C2.nvals()
    rec["gproducts_per_s"] = products / rec["product_ms"] / 1e6
    grp, gci, gval = C.extract_csr()
    if semiring == gb.Semiring.PlusMultiplies:
        try:
            T = torch.sparse_csr_tensor(rp.long(), ci.long(),
                                        val if val is not None else
                                        torch.ones(ci.numel(), device="cuda"),
                                        size=(n, n))
            rec["cusparse_ms"] = timed(lambda: torch.sparse.mm(T, T), args.iters,
                                       args.warmup)
            R = torch.sparse.mm(T, T)
            rec["cusparse_agrees"] = bool(
                np.array_equal(R.crow_indices().cpu().numpy(), grp) and
                np.array_equal(R.col_indices().cpu().numpy(), gci) and
                np.array_equal(R.values().cpu().numpy(), gval))
        except Exception as e:                  # noqa: BLE001
            rec["cusparse"] = "not available: %s" % str(e).splitlines()[0][:120]
    if args.scipy and semiring == gb.Semiring.PlusMultiplies:
        import time
        import scipy.sparse as sp
        v = (val.cpu().numpy() if val is not None else np.ones(ci.numel(), np.float32))
        S = sp.csr_matrix((v, ci.cpu().numpy(), rp.cpu().numpy()), shape=(n, n))
        t0 = time.time()
        P = (S @ S).tocsr()
        rec["scipy_s"] = time.time() - t0
        P.sort_indices()
        # scipy drops entries that sum to 0; with positive values there are none
        rec["scipy_agrees"] = bool(np.array_equal(P.indptr, grp) and
                                   np.array_equal(P.indices, gci) and
                                   np.array_equal(P.data, gval))
    print(json.dumps(rec), flush=True)
    del C, C2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--scipy", action="store_true")
    ap.add_argument("--only", default=None)
    ap.add_argument("--profile", action="store_true",
                    help="one more call per workload under torch.profiler: device "
                         "time per phase (bins, symbolic, numeric, scan, CSC)")
    ap.add_argument("--rmat18", action="store_true", help="one R-MAT-18 A*A call")
    args = ap.parse_args()
    gb.init(0)
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    work = []
    n, rp, ci = rmat(14)
    work.append(("rmat14", n, rp, ci, None, gb.Semiring.PlusMultiplies))
    n, rp, ci = rmat(16)
    work.append(("rmat16", n, rp, ci, None, gb.Semiring.PlusMultiplies))
    w = torch.from_numpy(gb.api.host_uniform_weights(1, 1, 64, ci.numel())).cuda()
    work.append(("rmat16_minplus", n, rp, ci, w, gb.Semiring.MinimumPlus))
    for name, n, rp, ci, val, sr in work:
        if args.only is None or args.only == name:
            run(name, n, rp, ci, val, sr, args)
    del work
    if args.only in (None, "grid128"):
        n, rp, ci = grid27(128)
        run("grid128", n, rp, ci, None, gb.Semiring.PlusMultiplies, args)
    if args.rmat18:
        n, rp, ci = rmat(18)
        A = graphs.matrix_from_csr(n, rp, ci)
        C = new_matrix(n, True)
        try:
            ms = timed(lambda: gb.mxm(C, None, None, gb.Semiring.PlusMultiplies, A, A,
                                      gb.Descriptor()), 1, 0)
            print(json.dumps({"workload": "rmat18", "product_ms": ms,
                              "nnz_C": C.nvals()}), flush=True)
        except gb.api.GraphBLASError as e:
            print(json.dumps({"workload": "rmat18", "result": str(e)}), flush=True)


if __name__ == "__main__":
    main()
