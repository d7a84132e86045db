"""Assign into a matrix on the device (gb.assign with a Matrix output): time per call and
bandwidth, with gb.eWiseAdd of C and a host-built embedded source as the yardstick.

  python tools/bench_assign.py [--iters 10] [--warmup 2] [--only rmat22|rmat24]

Workloads (R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, symmetrised, values 1; C
from seed 1, the assigned blocks cut from a second graph of seed 2; vertex sets from
numpy seed 7):
  rmat22_induced10         C(S,S) = B, S a sorted random 10 % of the vertices, no accum
  rmat22_induced10_plus    the same with PLUS as accum
  rmat22_shuffled10        the same S shuffled: the sort path
  rmat22_rows10            C(S,:) = B
  rmat22_hub_row           C(h,:) = u, h the highest-degree vertex, u its row in the
                           second graph: a small edit that still rewrites all of C
  rmat22_const4096         C(I,J) = 1, I and J sorted random 4 096-vertex sets
  rmat24_induced50         C(S,S) = B at scale 24, S a sorted 50 %

Each line is one JSON record.  Every result must equal tests/assign_reference.py entry
for entry before it is timed.  "ms" is the median of CUDA-event timings of single warm
calls with a CSR-only C; "ms_with_csc" is the same with a CSRCSC C (whose CSC is the
symmetric alias for the induced workloads, and is rebuilt otherwise).  C is rebuilt
from the same arrays before each timed call (outside the timing), so every call does
the same work.  "GBps" divides the compulsory bytes by "ms": C read, op(A) read, C'
written,
  4(m+1) + 8 nnz(C) + 4(nI+1) + 8 nnz(A) + 4(m+1) + 8 nnz(C').
"peak_GBps" is a device-to-device copy measured in the same run (read + write).
"ewise_add_ms" times gb.eWiseAdd of C with the embedded source E built on the host
(C ∪ E, the merge assign runs after building E), on the same CSR-only C.
"""
import json

import numpy as np
import torch

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import (event_ms, hbm_peak_gbps, header, new_matrix, parser, rmat_csr,
                      selected)
import graphblast_b200 as gb
from graphblast_b200 import graphs
import assign_reference as R


def compulsory_bytes(m, nnz_c, n_i, nnz_a, nnz_out):
    return 4*(m + 1) + 8*nnz_c + 4*(n_i + 1) + 8*nnz_a + 4*(m + 1) + 8*nnz_out


def matrix(n, ncols, rp, ci, val, csr_only, symmetric):
    """A Matrix over copies of the device CSR (rp, ci, val)."""
    M = new_matrix(n, ncols, csr_only)
    M.build_device_csr(rp.clone(), ci.clone(), val.clone(), ci.numel(), None, None, None,
                       symmetric=symmetric)
    return M


def host_csr(M):
    rp, ci, val = M.extract_csr()
    return rp, ci, val


class Case(object):
    """One workload: C's device CSR and the source, and how to call assign."""

    def __init__(self, name, n, c_arrays, call, want_fn, n_i, nnz_a, symmetric):
        self.name, self.n, self.c_arrays, self.call = name, n, c_arrays, call
        self.want_fn, self.n_i, self.nnz_a, self.symmetric = want_fn, n_i, nnz_a, symmetric


def measure(case, args, peak):
    n = case.n
    rp, ci, val = case.c_arrays
    rec = {"workload": case.name, "n": n, "nnz_C": int(ci.numel()), "rows": case.n_i,
           "nnz_source": case.nnz_a}
    C_ = matrix(n, n, rp, ci, val, True, case.symmetric)
    case.call(C_)
    got = host_csr(C_)
    del C_
    want = case.want_fn()
    agrees = (np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and
              np.array_equal(got[2].view(np.uint32), want[2].astype(np.float32).view(np.uint32)))
    rec["agrees_with_restatement"] = bool(agrees)
    rec["nnz_out"] = int(len(got[1]))
    if not agrees:
        print(json.dumps(rec), flush=True)
        raise SystemExit("%s: device result differs from the restatement" % case.name)
    # the embedded source E as host triples, for the eWiseAdd yardstick
    e_rows, e_cols, e_vals = want[3]
    del got, want

    def rebuilt_c_ms(csr_only):
        ts = []
        for it in range(args.warmup + args.iters):
            C_ = matrix(n, n, rp, ci, val, csr_only, case.symmetric)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            case.call(C_)
            b.record()
            b.synchronize()
            if it >= args.warmup:
                ts.append(a.elapsed_time(b))
            del C_
        return float(np.median(ts))
    rec["ms"] = rebuilt_c_ms(True)
    rec["ms_with_csc"] = rebuilt_c_ms(False)
    # yardstick: C ∪ E through the matrix eWiseAdd on a CSR-only C
    E = gb.Matrix(n, n)
    E.build(e_rows, e_cols, e_vals)
    C_ = matrix(n, n, rp, ci, val, True, case.symmetric)
    out = new_matrix(n, n, True)
    rec["ewise_add_ms"] = event_ms(lambda: gb.eWiseAdd(out, None, None,
                                                       gb.Semiring.PlusMultiplies, C_, E,
                                                       gb.Descriptor()),
                                   args.iters, args.warmup)
    del E, C_, out
    cb = compulsory_bytes(n, rec["nnz_C"], case.n_i, case.nnz_a, rec["nnz_out"])
    rec["compulsory_GB"] = cb/1e9
    rec["GBps"] = cb/rec["ms"]/1e6
    rec["share_of_peak"] = rec["GBps"]/peak
    torch.cuda.empty_cache()
    print(json.dumps(rec), flush=True)


def embedded(I, J, src, n):
    """(rows, cols, vals) of E: the host CSR src (ptr, ind, val) placed at (I, J)."""
    ptr, ind, val = src
    p = np.repeat(np.arange(len(ptr) - 1, dtype=np.int64), np.diff(ptr))
    cols = np.asarray(ind, np.int64) if J is None else np.asarray(J, np.int64)[ind]
    return (np.asarray(I, np.int64)[p].astype(np.int32), cols.astype(np.int32),
            np.asarray(val, np.float32))


def workloads(scale, rng, sets):
    n = 1 << scale
    _, rp, ci = rmat_csr(scale, seed=1)
    val = torch.ones(ci.numel(), dtype=torch.float32, device="cuda")
    c_arrays = (rp, ci, val)
    h_c = (rp.cpu().numpy(), ci.cpu().numpy(), np.ones(ci.numel(), np.float32))
    _, rp2, ci2 = rmat_csr(scale, seed=2)
    A2 = graphs.matrix_from_csr(n, rp2, ci2)
    d = gb.Descriptor()
    cases = []
    for name, S, accum in sets:
        # B = A2(S,S): for a shuffled S, C(S,S) = B places the same entries as for
        # the sorted S, through the sort path
        B = gb.Matrix(len(S), len(S))
        gb.extract(B, None, None, A2, S, len(S), S, len(S), d)
        hb = host_csr(B)
        acc = None if accum is None else gb.Monoid.Plus
        op = None if accum is None else "plus"

        def call(C_, B=B, S=S, acc=acc):
            gb.assign(C_, None, acc, B, S, len(S), S, len(S), d)

        def want(S=S, hb=hb, op=op):
            w = R.assign_matrix(h_c, n, n, (hb[0], hb[1], hb[2], len(S), len(S)), S, S,
                                accum=op)
            return w + (embedded(S, S, hb, n),)
        cases.append(Case(name, n, c_arrays, call, want, len(S), len(hb[1]), True))
    return n, A2, c_arrays, h_c, cases


def rmat22_extra(n, A2, c_arrays, h_c, rng, s10):
    d = gb.Descriptor()
    cases = []
    # C(S,:) = B
    B = gb.Matrix(len(s10), n)
    gb.extract(B, None, None, A2, s10, len(s10), None, n, d)
    hb = host_csr(B)
    cases.append(Case(
        "rmat22_rows10", n, c_arrays,
        lambda C_: gb.assign(C_, None, None, B, s10, len(s10), None, n, d),
        lambda: R.assign_matrix(h_c, n, n, (hb[0], hb[1], hb[2], len(s10), n), s10, None) +
        (embedded(s10, None, hb, n),),
        len(s10), len(hb[1]), False))
    # one hub row
    h = int(np.argmax(np.diff(h_c[0])))
    u = gb.Vector(n)
    gb.extract(u, None, None, A2, None, n, h, 0, d)
    u_ind, u_val = u.extractTuples(sparse=True)
    u_ind = np.asarray(u_ind, np.int64)
    u_val = np.asarray(u_val, np.float32)
    cases.append(Case(
        "rmat22_hub_row", n, c_arrays,
        lambda C_: gb.assign(C_, None, None, u, h, None, n, d),
        lambda: R.assign_row(h_c, n, n, u_ind, u_val, h, None) +
        ((np.full(len(u_ind), h, np.int32), u_ind.astype(np.int32), u_val),),
        1, len(u_ind), False))
    # a constant 4096 x 4096 block
    I = np.sort(rng.choice(n, 4096, replace=False)).astype(np.int32)
    J = np.sort(rng.choice(n, 4096, replace=False)).astype(np.int32)
    cases.append(Case(
        "rmat22_const4096", n, c_arrays,
        lambda C_: gb.assign(C_, None, None, 1.0, I, 4096, J, 4096, d),
        lambda: R.assign_constant(h_c, n, n, np.float32(1), I, J) +
        ((np.repeat(I, 4096), np.tile(J, 4096), np.ones(4096*4096, np.float32)),),
        4096, 4096*4096, False))
    return cases


def main():
    args = parser(iters=10, warmup=2, only="rmat22 or rmat24").parse_args()
    gb.init(0)
    peak = hbm_peak_gbps()
    header(peak_GBps=peak)
    rng = np.random.RandomState(7)
    if selected(args.only, "rmat22"):
        n = 1 << 22
        s10 = np.sort(rng.choice(n, n//10, replace=False)).astype(np.int32)
        sh = rng.permutation(s10).astype(np.int32)
        n, A2, c_arrays, h_c, cases = workloads(22, rng, [
            ("rmat22_induced10", s10, None),
            ("rmat22_induced10_plus", s10, "plus"),
            ("rmat22_shuffled10", sh, None)])
        cases += rmat22_extra(n, A2, c_arrays, h_c, rng, s10)
        for case in cases:
            measure(case, args, peak)
        del A2, c_arrays, h_c, cases
        torch.cuda.empty_cache()
    if selected(args.only, "rmat24"):
        n = 1 << 24
        s50 = np.sort(rng.choice(n, n//2, replace=False)).astype(np.int32)
        _, A2, c_arrays, h_c, cases = workloads(24, rng, [("rmat24_induced50", s50, None)])
        for case in cases:
            measure(case, args, peak)


if __name__ == "__main__":
    main()
