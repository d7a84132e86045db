"""Element-wise union / intersection of two sparse matrices on the device
(gb.eWiseAdd / gb.eWiseMult with Matrix operands): time per call and bandwidth,
against cuSPARSE for the plus-times union (torch's CUDA CSR addition, csrgeam2).

  python tools/bench_ewise.py [--iters 10] [--warmup 2] [--only NAME]

Workloads (R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, values 1):
  rmat22_add / rmat22_mult  A + B and A .* B, A and B symmetrised, B a second seed
  rmat22_self               A + A (every entry matched)
  rmat22_sym                A + A' with A directed (GrB_INP1 = GrB_TRAN); A is
                            built by the device ingest without symmetrising, so
                            it carries a CSC
  rmat24_add                A + B at scale 24 (CSR-only C: building C's CSC
                            would not fit in 80 GB beside the operands)

Each line is one JSON record.  Times are medians of CUDA-event timings of single
warm calls, with C's CSC built (the default format) and without it (a CSR-only
C).  "GBps" divides the compulsory bytes by the CSR-only time: both passes read
both row pointer arrays and column lists, the fill pass also the values, and C's
row offsets and entries are written once:
  2(8(m+1) + 4 nnz_in) + 4 nnz_in + 4(m+1) + 8 nnz(C),  nnz_in = nnz(A) + nnz(B).
"peak_GBps" is a device-to-device copy measured in the same run (read + write).
cuSPARSE's result must equal ours entry for entry before its time is quoted.
"""
import ctypes
import json

import numpy as np
import torch

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import event_ms, hbm_peak_gbps, header, new_matrix, parser, rmat_csr, selected
import graphblast_b200 as gb
from graphblast_b200 import graphs

INGEST_DROP_LOOPS, INGEST_DEDUP = 2, 4


def compulsory_bytes(m, nnz_in, nnz_c):
    return 2*(8*(m + 1) + 4*nnz_in) + 4*nnz_in + 4*(m + 1) + 8*nnz_c


def symmetric(scale, seed):
    n, rp, ci = rmat_csr(scale, seed=seed)
    return graphs.matrix_from_csr(n, rp, ci), rp, ci


def directed(scale):
    """Directed R-MAT through the device ingest (loops and repeats dropped, not
    symmetrised): CSR and CSC owned by the matrix."""
    n = 1 << scale
    src, dst = graphs.rmat_edges(scale, seed=1)
    A = gb.Matrix(n, n)
    gb.api._check(A._lib.gb200_matrix_build_coo_device(
        A._h, ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), None,
        int(src.numel()), INGEST_DROP_LOOPS | INGEST_DEDUP), "ingest")
    del src, dst
    return A


def csr_tensor(rp, ci, n):
    return torch.sparse_csr_tensor(rp.long(), ci.long(),
                                   torch.ones(ci.numel(), device="cuda"), size=(n, n))


def measure(name, add, n, A, B, args, peak, desc=None, cusparse=None, with_csc=True):
    desc = gb.Descriptor() if desc is None else desc
    f = gb.eWiseAdd if add else gb.eWiseMult
    rec = {"workload": name, "op": "eWiseAdd" if add else "eWiseMult", "m": n,
           "nnz_A": A.nvals(), "nnz_B": B.nvals()}
    if with_csc:
        C = gb.Matrix(n, n)
        rec["ms_with_csc"] = event_ms(lambda: f(C, None, None, 1, A, B, desc), args.iters,
                                      args.warmup)
        del C
    C = new_matrix(n, n, True)
    rec["ms"] = event_ms(lambda: f(C, None, None, 1, A, B, desc), args.iters, args.warmup)
    rec["nnz_C"] = C.nvals()
    cb = compulsory_bytes(n, rec["nnz_A"] + rec["nnz_B"], rec["nnz_C"])
    rec["compulsory_GB"] = cb/1e9
    rec["GBps"] = cb/rec["ms"]/1e6
    rec["share_of_peak"] = rec["GBps"]/peak
    if cusparse is not None:
        rp, ci, val = C.extract_csr()
        del C
        try:
            TA, TB = cusparse()
            S = TA + TB
            agrees = (np.array_equal(S.crow_indices().cpu().numpy(), rp) and
                      np.array_equal(S.col_indices().cpu().numpy(), ci) and
                      np.array_equal(S.values().cpu().numpy(), val))
            rec["cusparse_agrees"] = bool(agrees)
            del S
            if agrees:
                rec["cusparse_ms"] = event_ms(lambda: TA + TB, args.iters, args.warmup)
            del TA, TB
        except torch.cuda.OutOfMemoryError:
            rec["cusparse"] = "out of memory"
    torch.cuda.empty_cache()
    print(json.dumps(rec), flush=True)


def main():
    args = parser(iters=10, warmup=2, only="rmat22, rmat22_sym or rmat24").parse_args()
    gb.init(0)
    peak = hbm_peak_gbps()
    header(peak_GBps=peak)
    if selected(args.only, "rmat22"):
        n = 1 << 22
        A, arp, aci = symmetric(22, 1)
        B, brp, bci = symmetric(22, 2)
        ts = lambda: (csr_tensor(arp, aci, n), csr_tensor(brp, bci, n))
        measure("rmat22_add", True, n, A, B, args, peak, cusparse=ts)
        measure("rmat22_mult", False, n, A, B, args, peak)
        measure("rmat22_self", True, n, A, A, args, peak)
        del A, B, arp, aci, brp, bci, ts
        torch.cuda.empty_cache()
    if selected(args.only, "rmat22_sym"):
        n = 1 << 22
        A = directed(22)
        tran1 = gb.Descriptor()
        tran1.set(gb.Desc_field.GrB_INP1, gb.Desc_value.GrB_TRAN)
        measure("rmat22_sym", True, n, A, A, args, peak, desc=tran1)
        del A
        torch.cuda.empty_cache()
    if selected(args.only, "rmat24"):
        n = 1 << 24
        A, arp, aci = symmetric(24, 1)
        B, brp, bci = symmetric(24, 2)
        ts = lambda: (csr_tensor(arp, aci, n), csr_tensor(brp, bci, n))
        # C's CSC (a radix sort of ~1 G entries) does not fit beside the operands
        measure("rmat24_add", True, n, A, B, args, peak, cusparse=ts, with_csc=False)


if __name__ == "__main__":
    main()
