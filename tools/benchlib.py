"""What the benchmark tools tools/bench_*.py share: the card query, the two timing rules,
the HBM figures, the graphs more than one tool runs, and the command line and run loop.

Importing it puts the repository root and tests/ on sys.path, so a tool imports it
before the package and the checkers.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import graphblast_b200 as gb                      # noqa: E402
from graphblast_b200 import graphs                # noqa: E402

# The H100 SXM data-sheet HBM3 bandwidth: a bound, not an achieved rate.
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.check_output(
            ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
            text=True).strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001
        out = "unknown (%s)" % e
    return out


def event_ms(fn, iters, warmup):
    """Median of CUDA-event times around single calls of fn, after warmup calls."""
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


def device_ms(fn, iters, warmup):
    """Median of the device times fn() returns, after warmup calls."""
    for _ in range(warmup):
        fn()
    return float(np.median([fn() for _ in range(iters)]))


def stream_bound_ms(nbytes):
    """Time to move nbytes at HBM_BYTES_PER_S."""
    return nbytes/HBM_BYTES_PER_S*1e3


def hbm_peak_gbps():
    """A device-to-device copy of 2 GiB, read + write, in GB/s."""
    x = torch.empty(1 << 29, dtype=torch.float32, device="cuda")     # 2 GiB
    y = torch.empty_like(x)
    ms = event_ms(lambda: y.copy_(x), 10, 2)
    del x, y
    torch.cuda.empty_cache()
    return 2*(1 << 31)/ms/1e6


def rmat_csr(scale, seed, undirected=True):
    """R-MAT (0.57, 0.19, 0.19, 0.05), edge factor 16, generator seed `seed`, self-loops
    and duplicates removed, symmetrised when undirected: (n, rowptr, colind) on the
    device."""
    src, dst = graphs.rmat_edges(scale, seed=seed)
    rp, ci = graphs.build_csr(1 << scale, src, dst, undirected)
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


def tree_pieces(count=4096, size=1024, seed=5):
    """count pieces of size vertices, each a random spanning tree plus two random edges
    per vertex, ids interleaved across the range by a fixed permutation, symmetrised:
    (n, rowptr, colind) on the device."""
    rng = np.random.RandomState(seed)
    n = count*size
    local = np.arange(1, size)
    tree_parent = (rng.rand(count, size - 1)*local).astype(np.int64)   # < own index
    base = (np.arange(count)*size)[:, None]
    src = [(base + local).ravel(), (base + rng.randint(0, size, (count, 2*size))).ravel()]
    dst = [(base + tree_parent).ravel(), (base + rng.randint(0, size, (count, 2*size))).ravel()]
    perm = rng.permutation(n)
    src = perm[np.concatenate(src)].astype(np.int32)
    dst = perm[np.concatenate(dst)].astype(np.int32)
    rp, ci = graphs.build_csr(n, torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda(),
                              True)
    return n, rp, ci


def new_matrix(nrows, ncols, csr_only):
    """An empty Matrix; csr_only keeps only the CSR of the results written to it."""
    if csr_only:
        os.environ["GRB_SPARSE_MATRIX_FORMAT"] = "1"
    try:
        return gb.Matrix(nrows, ncols)
    finally:
        os.environ.pop("GRB_SPARSE_MATRIX_FORMAT", None)


def adopt_csr_csc(n, src, dst, undirected):
    """CSR from (src, dst), CSC from the swapped endpoints, both adopted with values 1 and
    not marked symmetric: (A, rowptr, colind)."""
    rp, ci = graphs.build_csr(n, src, dst, undirected)
    cp, ri = graphs.build_csr(n, dst, src, undirected)
    A = gb.Matrix(n, n)
    A.build_device_csr(rp, ci, torch.ones(ci.numel(), dtype=torch.float32, device="cuda"),
                       ci.numel(), cp, ri,
                       torch.ones(ri.numel(), dtype=torch.float32, device="cuda"))
    return A, rp, ci


def parser(iters, warmup, only=None):
    """--iters and --warmup with these defaults and, when `only` names the workloads,
    --only: a comma-separated list of workload names, parsed to a set."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=iters)
    ap.add_argument("--warmup", type=int, default=warmup)
    if only is not None:
        ap.add_argument("--only", type=lambda s: set(s.split(",")), default=None,
                        help=only + " (comma-separated)")
    return ap


def selected(only, name):
    """Whether --only (None: every workload) selects name."""
    return only is None or name in only


def header(**extra):
    """The first line of a tool's output: the card, torch's version and extra."""
    print(json.dumps({"card": card(), "torch": torch.__version__, **extra}), flush=True)


def run(workloads, args, measure):
    """For each (name, build, *extra) of workloads that --only selects:
    measure(name, *build(), *extra, args), then free the workload and the cached device
    memory before the next one is built."""
    for name, build, *extra in workloads:
        if selected(args.only, name):
            measure(name, *build(), *extra, args)
            torch.cuda.empty_cache()
