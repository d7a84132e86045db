"""Graph colouring on the device (algorithm.gc): time per call against cuSPARSE
csrcolor and against the single-thread CPU oracle.

  python tools/bench_gc.py [--iters 10] [--warmup 2] [--only rmat22|rmat24]

Workloads: R-MAT (0.57, 0.19, 0.19, 0.05) of scale 22 and 24, edge factor 16,
symmetrised, self-loops and duplicate edges removed (graphs.rmat_edges /
build_csr / matrix_from_csr), seed 1.

Each line is one JSON record.  "ms" is the median of the CUDA-event times that gc
returns for warm calls.  Before any time is quoted, the colouring must equal the
CPU oracle's (tests/gc_oracle.c, greedy first-fit in the same priority order) entry
for entry; "cpu_ms" is that oracle's single-thread time and "jp_depth" its Jones-Plassmann
round count.  cuSPARSE's cusparseScsrcolor (deprecated, still exported by the
libcusparse.so.12 that ships with torch) runs with fraction = 1.0; its colouring is
checked as proper before its time and colour count are quoted.  It is not greedy.
"""
import ctypes as C
import glob
import json
import os
import time

import numpy as np
import torch

# benchlib first: it puts the repository root and tests/ on sys.path
from benchlib import card, device_ms, event_ms, header, parser, rmat_csr, selected
import graphblast_b200 as gb
from graphblast_b200 import algorithm, graphs
import greedy_oracle


def cusparse_lib():
    import nvidia.cusparse
    for d in nvidia.cusparse.__path__:
        found = glob.glob(os.path.join(d, "lib", "libcusparse.so.12*"))
        if found:
            return C.CDLL(found[0])
    return C.CDLL("libcusparse.so.12")


class CsrColor:
    """cusparseScsrcolor on a device CSR (int32 row pointers and columns)."""

    def __init__(self, n, rp, ci):
        self.lib = cusparse_lib()
        self.n, self.rp, self.ci = n, rp, ci
        self.val = torch.ones(ci.numel(), dtype=torch.float32, device="cuda")
        self.coloring = torch.empty(n, dtype=torch.int32, device="cuda")
        self.reordering = torch.empty(n, dtype=torch.int32, device="cuda")
        self.handle, self.descr, self.info = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._ok(self.lib.cusparseCreate(C.byref(self.handle)), "cusparseCreate")
        self._ok(self.lib.cusparseSetStream(self.handle, C.c_void_p(
            torch.cuda.current_stream().cuda_stream)), "cusparseSetStream")
        self._ok(self.lib.cusparseCreateMatDescr(C.byref(self.descr)), "MatDescr")
        self._ok(self.lib.cusparseCreateColorInfo(C.byref(self.info)), "ColorInfo")
        self.ncolors = C.c_int(0)
        self.fraction = C.c_float(1.0)

    @staticmethod
    def _ok(status, what):
        if status != 0:
            raise RuntimeError("%s failed with cuSPARSE status %d" % (what, status))

    def __call__(self):
        self._ok(self.lib.cusparseScsrcolor(
            self.handle, C.c_int(self.n), C.c_int(self.ci.numel()), self.descr,
            C.c_void_p(self.val.data_ptr()), C.c_void_p(self.rp.data_ptr()),
            C.c_void_p(self.ci.data_ptr()), C.byref(self.fraction), C.byref(self.ncolors),
            C.c_void_p(self.coloring.data_ptr()), C.c_void_p(self.reordering.data_ptr()),
            self.info), "cusparseScsrcolor")

    def close(self):
        self.lib.cusparseDestroyColorInfo(self.info)
        self.lib.cusparseDestroyMatDescr(self.descr)
        self.lib.cusparseDestroy(self.handle)


def proper(colors, rows, ci):
    return not np.any(colors[rows] == colors[ci])


def measure(scale, args):
    n, rp, ci = rmat_csr(scale, seed=1)
    A = graphs.matrix_from_csr(n, rp, ci)
    rec = {"workload": "rmat%d" % scale, "n": n, "nnz": int(ci.numel()), "card": card()}
    v = gb.Vector(n)
    desc = gb.Descriptor()
    count = [0]

    def run_gc():
        count[0], ms = algorithm.gc(v, A, 0, desc)
        return ms
    rec["ms"] = device_ms(run_gc, args.iters, args.warmup)
    rec["ncolors"] = count[0]
    got = v.extractTuples()

    h_rp, h_ci = rp.cpu().numpy(), ci.cpu().numpy()
    t0 = time.perf_counter()
    want, want_n, depth = greedy_oracle.gc(h_rp, h_ci, 0)
    rec["cpu_ms"] = (time.perf_counter() - t0)*1e3
    rec["jp_depth"] = depth
    rec["oracle_ncolors"] = want_n
    rec["equals_oracle"] = bool(np.array_equal(got, want.astype(np.float32)) and
                                count[0] == want_n)
    rows = np.repeat(np.arange(n, dtype=np.int32), np.diff(h_rp))
    rec["proper"] = proper(got, rows, h_ci)
    if not rec["equals_oracle"]:
        rec.pop("ms")                 # a wrong colouring gets no time
    try:
        cs = CsrColor(n, rp, ci)
        cs()
        torch.cuda.synchronize()
        colors = cs.coloring.cpu().numpy()
        rec["cusparse_proper"] = proper(colors, rows, h_ci)
        if rec["cusparse_proper"]:
            rec["cusparse_ncolors"] = int(cs.ncolors.value)
            rec["cusparse_distinct_colors"] = int(np.unique(colors).size)
            rec["cusparse_ms"] = event_ms(cs, args.iters, args.warmup)
        cs.close()
        del cs
    except (OSError, RuntimeError, torch.cuda.OutOfMemoryError) as e:
        rec["cusparse"] = str(e)
    print(json.dumps(rec), flush=True)
    del A, rp, ci, v
    torch.cuda.empty_cache()


def main():
    args = parser(iters=10, warmup=2, only="rmat22 or rmat24").parse_args()
    gb.init(0)
    header()
    for scale in (22, 24):
        if selected(args.only, "rmat%d" % scale):
            measure(scale, args)


if __name__ == "__main__":
    main()
