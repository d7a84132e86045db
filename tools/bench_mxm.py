"""Unmasked SpGEMM C = A*A on the device: time per call, products/s, nnz(C),
against cuSPARSE (torch.sparse.mm on CUDA CSR tensors, plus-times) and, with
--scipy, single-threaded scipy; every output that is compared must agree.

  python tools/bench_mxm.py [--iters 10] [--warmup 2] [--scipy] [--only NAME]

Each line is one JSON record.  "product_ms" is a call whose C keeps only its CSR;
"mxm_ms" the default call, which also builds C's CSC; "csc_ms" their difference.
Times are medians of CUDA-event timings of single calls.  --profile adds
"phases_ms", kernel time per phase of one further call, taken after the timed ones.
"""
import json

import numpy as np
import torch

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import event_ms, grid27, header, new_matrix, parser, rmat_csr, run
import graphblast_b200 as gb
from graphblast_b200 import graphs

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


def measure(name, n, rp, ci, val, semiring, args):
    A = graphs.matrix_from_csr(n, rp, ci, val)
    deg = (rp[1:] - rp[:-1]).long()
    products = int(deg[ci.long()].sum().item())
    rec = {"workload": name, "n": n, "nnz_A": int(ci.numel()), "products": products,
           "semiring": semiring.name}
    desc = gb.Descriptor()
    C = new_matrix(n, n, True)
    rec["product_ms"] = event_ms(lambda: gb.mxm(C, None, None, semiring, A, A, desc),
                                 args.iters, args.warmup)
    C2 = new_matrix(n, n, False)
    rec["mxm_ms"] = event_ms(lambda: gb.mxm(C2, None, None, semiring, A, A, desc),
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
            rec["cusparse_ms"] = event_ms(lambda: torch.sparse.mm(T, T), args.iters,
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


def rmat16_minplus():
    n, rp, ci = rmat_csr(16, seed=1)
    w = torch.from_numpy(gb.api.host_uniform_weights(1, 1, 64, ci.numel())).cuda()
    return n, rp, ci, w


def main():
    ap = parser(iters=10, warmup=2, only="rmat14, rmat16, rmat16_minplus or grid128")
    ap.add_argument("--scipy", action="store_true")
    ap.add_argument("--profile", action="store_true",
                    help="one more call per workload under torch.profiler: device "
                         "time per phase (bins, symbolic, numeric, scan, CSC)")
    ap.add_argument("--rmat18", action="store_true", help="one R-MAT-18 A*A call")
    args = ap.parse_args()
    gb.init(0)
    header()
    run([("rmat14", lambda: rmat_csr(14, seed=1) + (None,), gb.Semiring.PlusMultiplies),
         ("rmat16", lambda: rmat_csr(16, seed=1) + (None,), gb.Semiring.PlusMultiplies),
         ("rmat16_minplus", rmat16_minplus, gb.Semiring.MinimumPlus),
         ("grid128", lambda: grid27(128) + (None,), gb.Semiring.PlusMultiplies)],
        args, measure)
    if args.rmat18:
        n, rp, ci = rmat_csr(18, seed=1)
        A = graphs.matrix_from_csr(n, rp, ci)
        C = new_matrix(n, n, True)
        try:
            ms = event_ms(lambda: gb.mxm(C, None, None, gb.Semiring.PlusMultiplies, A, A,
                                         gb.Descriptor()), 1, 0)
            print(json.dumps({"workload": "rmat18", "product_ms": ms,
                              "nnz_C": C.nvals()}), flush=True)
        except gb.api.GraphBLASError as e:
            print(json.dumps({"workload": "rmat18", "result": str(e)}), flush=True)


if __name__ == "__main__":
    main()
