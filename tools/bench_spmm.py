"""SpMM C = A (+.x) B on the device (gb.mxm with a dense B): time per call and
bandwidth, against cuSPARSE (torch.sparse_csr_tensor(...) @ B, plus-times).

  python tools/bench_spmm.py [--iters 10] [--warmup 2] [--only NAME]

Workloads: R-MAT-22 (symmetrised) at N = 4, 16, 32, 64, 128, 256, which puts
widths on both sides of each class limit of kernels/spmm.cuh (64: groups of
fewer than 32 lanes; 128: columns tiled over the grid); R-MAT-24 at N = 32 and
64 (m*N must stay within INT32_MAX); the 27-point 128^3 grid at N = 32 and 128.
A holds the pattern (values 1), B uniform in [-1, 1].

Each line is one JSON record.  Times are medians of CUDA-event timings of single
warm calls (C already dense of its shape).  "GBps" divides the compulsory bytes
4(m+1) + 8 nnz + 4 k N + 4 m N by the time; "gather_GB" is 4 nnz N, the B rows
the kernel gathers (mostly from L2).  Plus-times must agree with cuSPARSE within
(deg_i + 1) 2^-23 (|A| |B|)_ij, twice the fp32 bound of a sum in any order.
MinimumPlus has no cuSPARSE counterpart; its sampled rows (the longest among
them) must equal a host min-plus exactly.
"""
import json

import numpy as np
import torch

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import event_ms, grid27, header, parser, rmat_csr, run
import graphblast_b200 as gb
from graphblast_b200 import graphs


def compulsory_bytes(m, k, nnz, n):
    return 4*(m + 1) + 8*nnz + 4*k*n + 4*m*n


def plus_times_agrees(T, Tabs, deg, B, got):
    want = torch.sparse.mm(T, B)
    scale = torch.sparse.mm(Tabs, B.abs())
    bound = (deg[:, None] + 1)*2.0**-23*scale + 1e-30
    return bool(((got - want).abs() <= bound).all().item()), want


def min_plus_agrees(rp, ci, B, got, rows):
    for i in rows:
        a, b = int(rp[i]), int(rp[i + 1])
        if a == b:
            want = np.full(B.shape[1], np.finfo(np.float32).max, np.float32)
        else:
            cols = ci[a:b].long()
            want = (B[cols] + 1.0).min(0).values.cpu().numpy()
        if not np.array_equal(got[i].cpu().numpy(), want):
            return False
    return True


def measure(name, n, rp, ci, widths, args):
    A = graphs.matrix_from_csr(n, rp, ci)
    nnz = int(ci.numel())
    deg = (rp[1:] - rp[:-1]).float()
    T = torch.sparse_csr_tensor(rp.long(), ci.long(), torch.ones(nnz, device="cuda"),
                                size=(n, n))
    rng = np.random.RandomState(1)
    rows = sorted(set(rng.randint(0, n, 63).tolist()) | {int(deg.argmax().item())})
    desc = gb.Descriptor()
    for w in widths:
        B = torch.rand(n, w, device="cuda")*2 - 1
        Bm = gb.Matrix(n, w)
        Bm.build_dense_device(B)
        C = gb.Matrix(n, w)
        rec = {"workload": name, "m": n, "nnz": nnz, "N": w}
        cb = compulsory_bytes(n, n, nnz, w)
        rec["compulsory_GB"] = cb/1e9
        rec["gather_GB"] = 4.0*nnz*w/1e9
        for sr in (gb.Semiring.PlusMultiplies, gb.Semiring.MinimumPlus):
            ms = event_ms(lambda: gb.mxm(C, None, None, sr, A, Bm, desc), args.iters,
                          args.warmup)
            got = torch.from_numpy(C.extract_dense()).cuda()
            key = "plus_times" if sr == gb.Semiring.PlusMultiplies else "min_plus"
            rec[key + "_ms"] = ms
            rec[key + "_GBps"] = cb/ms/1e6
            if sr == gb.Semiring.PlusMultiplies:
                rec["cusparse_ms"] = event_ms(lambda: torch.sparse.mm(T, B), args.iters,
                                              args.warmup)
                rec["cusparse_GBps"] = cb/rec["cusparse_ms"]/1e6
                rec["cusparse_agrees"], _ = plus_times_agrees(T, T, deg, B, got)
            else:
                rec["min_plus_agrees"] = min_plus_agrees(rp, ci, B, got, rows)
            del got
        print(json.dumps(rec), flush=True)
        del C, Bm, B
        torch.cuda.empty_cache()


def main():
    args = parser(iters=10, warmup=2, only="rmat22, rmat24 or grid128").parse_args()
    gb.init(0)
    header()
    run([("rmat22", lambda: rmat_csr(22, seed=1), [4, 16, 32, 64, 128, 256]),
         ("grid128", lambda: grid27(128), [32, 128]),
         ("rmat24", lambda: rmat_csr(24, seed=1), [32, 64])], args, measure)


if __name__ == "__main__":
    main()
