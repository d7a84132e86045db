"""Submatrix extract on the device (gb.extract with Matrix operands): time per call and
bandwidth, against scipy's A[S][:, S] on one host thread.

  python tools/bench_extract.py [--iters 10] [--warmup 2] [--only NAME]

Workloads (R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, symmetrised, values 1;
vertex sets from numpy seed 7):
  rmat22_induced10 / rmat22_induced50  A(S,S), S a sorted random 10 % / 50 % of the
                                       vertices: C is symmetric and installed so
  rmat22_shuffled10                    the same 10 % S shuffled: the sort path
  rmat22_rows10                        A(S,:), the sorted 10 %: J = ALL, a copy
  rmat22_perm                          A(P,P) in place, P a random permutation
                                       (shuffled J: the sort path)
  rmat24_induced50                     as rmat22_induced50 at scale 24

Each line is one JSON record.  "ms" is the median of CUDA-event timings of single warm
calls with a CSR-only C (the CSC a CSRCSC C needs is the symmetric alias for the
induced workloads and a transpose otherwise, timed apart as "ms_with_csc").  "GBps"
divides the compulsory bytes by "ms": the selected rows' pointer pairs read (8|I|),
their entries' columns and values read (8 sel) by both passes when J is given and
once otherwise, one map lookup per selected entry when J is given (8 sel), the map
itself built once (8|J| + 4 ncols(A)), and C's row offsets and entries written once
(4(|I|+1) + 8 nnz(C)):
  8|I| + 8 sel (x2 with J) + [8 sel + 8|J| + 4 ncols] (with J) + 4(|I|+1) + 8 nnz(C).
"peak_GBps" is a device-to-device copy measured in the same run (read + write).
The device result must equal scipy's entry for entry before either time is quoted.
"""
import json
import time

import numpy as np
import torch

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import (event_ms, hbm_peak_gbps, header, new_matrix, parser, rmat_csr,
                      selected)
import graphblast_b200 as gb
from graphblast_b200 import graphs


def compulsory_bytes(n_i, n_j, ncols, sel, nnz_c):
    with_map = n_j is not None
    b = 8*n_i + 8*sel*(2 if with_map else 1) + 4*(n_i + 1) + 8*nnz_c
    if with_map:
        b += 8*sel + 8*n_j + 4*ncols
    return b


def symmetric(scale):
    n, rp, ci = rmat_csr(scale, seed=1)
    return graphs.matrix_from_csr(n, rp, ci), rp, ci


def scipy_of(rp, ci, n):
    import scipy.sparse as sp
    rp_h, ci_h = rp.cpu().numpy(), ci.cpu().numpy()
    return sp.csr_matrix((np.ones(len(ci_h), np.float32), ci_h, rp_h), shape=(n, n))


def measure(name, n, A, host, I, J, args, peak, in_place=False):
    desc = gb.Descriptor()
    n_i, n_j = len(I), (n if J is None else len(J))
    rp_h = host.indptr
    sel = int(np.sum(rp_h[I + 1] - rp_h[I]))
    rec = {"workload": name, "n": n, "nnz_A": int(host.nnz), "rows": n_i, "cols": n_j,
           "selected_entries": sel}
    t0 = time.perf_counter()
    want = host[I] if J is None else host[I][:, J]
    want = want.tocsr()
    want.sort_indices()
    rec["scipy_ms"] = (time.perf_counter() - t0)*1e3
    # the check runs on a separate C; the in-place workload then permutes A itself
    # on every timed call (the same work each time)
    C = new_matrix(n_i, n_j, True)
    gb.extract(C, None, None, A, I, n_i, J, n_j, desc)
    rp, ci, val = C.extract_csr()
    agrees = (np.array_equal(rp, want.indptr) and np.array_equal(ci, want.indices) and
              np.array_equal(val, want.data))
    rec["agrees_with_scipy"] = bool(agrees)
    rec["nnz_C"] = int(len(ci))
    del rp, ci, val
    if not agrees:
        print(json.dumps(rec), flush=True)
        raise SystemExit("%s: device result differs from scipy" % name)
    target = A if in_place else C
    rec["ms"] = event_ms(lambda: gb.extract(target, None, None, A, I, n_i, J, n_j, desc),
                         args.iters, args.warmup)
    if not in_place:
        del C
        C2 = gb.Matrix(n_i, n_j)
        rec["ms_with_csc"] = event_ms(lambda: gb.extract(C2, None, None, A, I, n_i, J, n_j,
                                                         desc), args.iters, args.warmup)
        del C2
    cb = compulsory_bytes(n_i, None if J is None else n_j, n, sel, rec["nnz_C"])
    rec["compulsory_GB"] = cb/1e9
    rec["GBps"] = cb/rec["ms"]/1e6
    rec["share_of_peak"] = rec["GBps"]/peak
    torch.cuda.empty_cache()
    print(json.dumps(rec), flush=True)


def main():
    args = parser(iters=10, warmup=2, only="rmat22 or rmat24").parse_args()
    gb.init(0)
    peak = hbm_peak_gbps()
    header(peak_GBps=peak)
    rng = np.random.RandomState(7)
    if selected(args.only, "rmat22"):
        n = 1 << 22
        A, rp, ci = symmetric(22)
        host = scipy_of(rp, ci, n)
        s10 = np.sort(rng.choice(n, n//10, replace=False)).astype(np.int32)
        s50 = np.sort(rng.choice(n, n//2, replace=False)).astype(np.int32)
        measure("rmat22_induced10", n, A, host, s10, s10, args, peak)
        measure("rmat22_induced50", n, A, host, s50, s50, args, peak)
        sh = rng.permutation(s10).astype(np.int32)
        measure("rmat22_shuffled10", n, A, host, sh, sh, args, peak)
        measure("rmat22_rows10", n, A, host, s10, None, args, peak)
        P = rng.permutation(n).astype(np.int32)
        measure("rmat22_perm", n, A, host, P, P, args, peak, in_place=True)
        del A, rp, ci, host
        torch.cuda.empty_cache()
    if selected(args.only, "rmat24"):
        n = 1 << 24
        A, rp, ci = symmetric(24)
        host = scipy_of(rp, ci, n)
        s50 = np.sort(rng.choice(n, n//2, replace=False)).astype(np.int32)
        measure("rmat24_induced50", n, A, host, s50, s50, args, peak)


if __name__ == "__main__":
    main()
