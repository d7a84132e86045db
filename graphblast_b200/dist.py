"""1-D row-partitioned multi-GPU BFS, SSSP and PageRank (SURVEY.md §8e).

One process per GPU (torchrun), `torch.distributed` for rendezvous.  Rank p owns
the output vertices [bounds[p], bounds[p+1]) and stores the rows of A^T for them
as a rectangular local matrix M (n_local x n, CSR for the pull direction, CSC for
the push direction), so both directions produce only owned outputs and no
reduction across ranks is needed.  The replicated input vector of the next
step is exchanged through the library's own peer-memory exchange
(`PeerExchange`): every rank stores its owned slice into every other rank's
replica over NVLink.  The BFS is one persistent kernel per GPU with that exchange
inside (gb200_dist_bfs_fused: a bitmap, one bit per vertex); PageRank and SSSP
loop in C++ over it (gb200_dist_pr / gb200_dist_sssp: one float per vertex).

The reference has no distributed path at all (SURVEY.md §2 "Parallelism
strategies": none); the per-level operation sequence is the reference's BFS loop
(graphblas/algorithm/bfs.hpp:46-79) applied to the owned slice.
"""
import ctypes as C

import numpy as np
import torch


# ---------------------------------------------------------------------------
# Partition
# ---------------------------------------------------------------------------

# The one unit string of every bench line (both arms, every N): the driver divides
# lines only when their units agree.
UNIT = "MTEPS (stored entries of A / traversal time x 1e-6)"


def init_rank(local_rank):
    """Process group and CUDA device of this rank.  With more ranks on a node than
    GPUs, ranks share devices (local rank modulo the device count).  NCCL refuses
    two ranks on one device, so such a run uses gloo, whose collectives below go
    through host memory; the exchange of the traversal itself stays the library's
    peer-memory path."""
    import os
    import torch.distributed as dist
    ndev = torch.cuda.device_count()
    dev = torch.device("cuda", local_rank % ndev)
    if int(os.environ.get("LOCAL_WORLD_SIZE", "1")) <= ndev:
        dist.init_process_group("nccl", device_id=dev)
    else:
        dist.init_process_group("gloo")
    return dev


def _through_host(t):
    import torch.distributed as dist
    return t.is_cuda and dist.get_backend() == "gloo"


def all_reduce(t, op):
    import torch.distributed as dist
    if _through_host(t):
        h = t.cpu()
        dist.all_reduce(h, op=op)
        t.copy_(h)
    else:
        dist.all_reduce(t, op=op)


def all_gather(outs, t, group=None):
    import torch.distributed as dist
    if _through_host(t):
        hs = [torch.empty_like(o, device="cpu") for o in outs]
        dist.all_gather(hs, t.cpu(), group=group)
        for o, h in zip(outs, hs):
            o.copy_(h)
    else:
        dist.all_gather(outs, t, group=group)


def all_gather_into_tensor(out, t, group=None):
    import torch.distributed as dist
    if _through_host(t):
        parts = [torch.empty_like(t, device="cpu")
                 for _ in range(dist.get_world_size(group))]
        dist.all_gather(parts, t.cpu(), group=group)
        out.copy_(torch.cat(parts))
    else:
        dist.all_gather_into_tensor(out, t, group=group)


class _DevView(object):
    """A raw device pointer as something torch.as_tensor understands."""

    def __init__(self, ptr, count):
        self.__cuda_array_interface__ = {
            "shape": (count,), "typestr": "<f4", "data": (int(ptr), False),
            "version": 2}


class ResultGather(object):
    """End-to-end result path of the partitioned runs: the owned float slice of
    every rank is gathered over NCCL into one n-float vector on rank 0's GPU and
    copied into rank 0's pinned host buffer — the same 4n bytes of device->host
    traffic per step as the single-GPU run."""

    def __init__(self, bounds, world, rank, device):
        self.bounds, self.world, self.rank, self.device = bounds, world, rank, device
        self.sizes = [bounds[p + 1] - bounds[p] for p in range(world)]
        self.pad = max(self.sizes)
        self.n = bounds[world]
        self.buf = torch.zeros(self.pad, dtype=torch.float32, device=device)
        self.allv = torch.zeros(self.pad * world, dtype=torch.float32, device=device)
        self.host = (torch.empty(self.n, dtype=torch.float32).pin_memory()
                     if rank == 0 else None)

    def run(self, vec):
        """vec: gb.Vector holding this rank's owned slice.  Returns the host buffer
        on rank 0 (valid after the call), None elsewhere."""
        import torch.distributed as dist
        nl = self.sizes[self.rank]
        if nl > 0:
            view = torch.as_tensor(_DevView(vec.device_ptr(), nl), device=self.device)
            self.buf[:nl].copy_(view)
        all_gather_into_tensor(self.allv, self.buf)
        if self.rank == 0:
            for p in range(self.world):
                if self.sizes[p]:
                    self.host[self.bounds[p]:self.bounds[p + 1]].copy_(
                        self.allv[p * self.pad:p * self.pad + self.sizes[p]],
                        non_blocking=True)
            torch.cuda.synchronize()
            return self.host
        return None

    d2h_bytes = property(lambda self: 4 * self.n)


def timed_e2e(args, step, gather, vec, dev, h2d_bytes):
    """K steps through the public call path with host buffers: per step the step's
    input goes host->device from pinned memory, the traversal runs, and the full
    n-float result lands in rank 0's pinned host memory.  Wall clock, max over
    ranks.  Returns (ms per step, e2e dict without the value)."""
    import time
    import torch.distributed as dist
    host_in = torch.zeros(max(h2d_bytes // 4, 1), dtype=torch.int32).pin_memory()
    dev_in = torch.zeros_like(host_in, device=dev)
    for _ in range(2):
        step()
        gather.run(vec)
    torch.cuda.synchronize()
    dist.barrier()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        dev_in.copy_(host_in, non_blocking=True)
        step()
        gather.run(vec)
    torch.cuda.synchronize()
    wall = torch.tensor([(time.perf_counter() - t0) * 1e3], device=dev)
    all_reduce(wall, dist.ReduceOp.MAX)
    return float(wall.item()) / args.steps



def partition_bounds(rowptr, world, align=1024, row_weight=0.0):
    """Contiguous vertex ranges with (nearly) equal COST, cost of a vertex =
    its stored entries + row_weight; every boundary is a multiple of `align`
    (>= 32, so bitmap slices are whole words).  row_weight = 0 balances stored
    entries (what an SpMV iteration costs); the Boolean pull of a BFS mostly
    pays per ROW it has to look at (first-neighbour probe), so the BFS bench
    passes a row weight (GB200_DIST_ROW_WEIGHT; default 1e9 = equal vertex counts,
    measured best on R-MAT scale 24 at 2 GPUs: 0.464 ms entries-balanced, 0.428 at
    weight 32, 0.390 at 128, 0.385 with equal vertex counts).  rowptr: 1-D integer tensor/array of length n+1.  Returns a
    list of world+1 ints.

    No slice is empty: a bound that would not pass the one before it (a row
    heavier than 1/world of the cost) moves forward by `align`, and one that would
    leave a later rank empty moves back, as far as needed to leave one block to
    each later rank but the last and one vertex to the last.  A graph with fewer
    than world * align vertices raises ValueError."""
    rp = rowptr if isinstance(rowptr, np.ndarray) else rowptr.cpu().numpy()
    n = len(rp) - 1
    assert align % 32 == 0
    if n < world * align:
        raise ValueError("partition_bounds: %d vertices cannot give each of %d ranks "
                         "a slice of at least %d" % (n, world, align))
    cost = rp.astype(np.float64) + row_weight * np.arange(n + 1, dtype=np.float64)
    total = float(cost[-1])
    bounds = [0]
    for p in range(1, world):
        target = total * p / world
        v = int(np.searchsorted(cost, target, side="left"))
        v = (v + align // 2) // align * align
        # one block past the previous bound at least, one block left for each rank
        # after this one but the last, one vertex for the last (n >= world * align
        # keeps both possible)
        last = (n - 1 - (world - p - 1) * align) // align * align
        bounds.append(min(max(v, bounds[-1] + align), last))
    bounds.append(n)
    return bounds


def local_slice(rowptr, colind, lo, hi, n, return_order=False):
    """CSR and CSC (device tensors when the inputs are) of rows [lo, hi) of a
    structurally symmetric matrix, i.e. of A^T restricted to the owned outputs.
    Returns rp_local[n_local+1], ci_local[nnz_l], colptr[n+1], rowind[nnz_l]
    (+ the CSR->CSC permutation of the local entries when return_order)."""
    e0 = int(rowptr[lo])
    e1 = int(rowptr[hi])
    rp_local = (rowptr[lo:hi + 1] - rowptr[lo]).to(torch.int32).contiguous()
    ci_local = colind[e0:e1].contiguous()
    nl = hi - lo
    rows = torch.repeat_interleave(
        torch.arange(nl, device=colind.device, dtype=torch.int64),
        (rp_local[1:] - rp_local[:-1]).to(torch.int64))
    key = ci_local.to(torch.int64) * nl + rows
    order = torch.argsort(key)
    rowind = rows[order].to(torch.int32).contiguous()
    counts = torch.bincount(ci_local.to(torch.int64), minlength=n)
    colptr = torch.zeros(n + 1, dtype=torch.int64, device=colind.device)
    torch.cumsum(counts, 0, out=colptr[1:])
    if return_order:
        return (rp_local, ci_local, colptr.to(torch.int32).contiguous(), rowind,
                order)
    return rp_local, ci_local, colptr.to(torch.int32).contiguous(), rowind


def pagerank_local_matrix(gb, n, rowptr, colind, lo, hi, alpha):
    """(owned x n) CSR of the owned rows [lo, hi) of (alpha * A ./ outdeg)^T for a
    structurally symmetric A: entry (i, j) = alpha / deg(j), what gb200_dist_pr
    multiplies.  The matrix keeps its arrays alive."""
    e0, e1 = int(rowptr[lo]), int(rowptr[hi])
    rp_l = (rowptr[lo:hi + 1] - rowptr[lo]).to(torch.int32).contiguous()
    ci_l = colind[e0:e1].contiguous()
    deg = (rowptr[1:] - rowptr[:-1]).to(torch.float32)
    val_l = (alpha / deg[ci_l.to(torch.int64)]).contiguous()
    M = gb.Matrix(hi - lo, n)
    M._keep = [rp_l, ci_l, val_l]
    rc = gb._lib.load().gb200_matrix_adopt_csr(
        M._h, C.c_void_p(rp_l.data_ptr()), C.c_void_p(ci_l.data_ptr()),
        C.c_void_p(val_l.data_ptr()), int(ci_l.numel()))
    if rc != 0:
        raise RuntimeError("gb200_matrix_adopt_csr failed: %d" % rc)
    return M


def weighted_local_matrix(gb, n, rowptr, colind, cscval, lo, hi):
    """(owned x n) matrix of the owned rows [lo, hi) of A^T: CSR entries
    (j_owned, i) = A(i, j) = cscval of the symmetric structure's entry (ones when
    cscval is None: the BFS reads only the structure), CSC = the same entries by
    source column.  Returns (Matrix, tensors to keep alive)."""
    rp_l, ci_l, colptr, rowind, order = local_slice(rowptr, colind, lo, hi, n,
                                                    return_order=True)
    e0, e1 = int(rowptr[lo]), int(rowptr[hi])
    if cscval is None:
        val_l = torch.ones(e1 - e0, dtype=torch.float32, device=colind.device)
    else:
        val_l = cscval[e0:e1].contiguous()
    cval_l = val_l[order].contiguous()
    nl = hi - lo
    M = gb.Matrix(max(nl, 1), n)
    if nl > 0 and ci_l.numel() > 0:
        M.build_device_csr(rp_l, ci_l, val_l, ci_l.numel(), colptr, rowind, cval_l,
                           symmetric=False)
    return M, [rp_l, ci_l, colptr, rowind, val_l, cval_l]


# ---------------------------------------------------------------------------
# Exchange
# ---------------------------------------------------------------------------

class PeerExchange(object):
    """The library's own exchange (include/graphblast_b200.h, gb200_xchg_*): every
    rank maps every other rank's exchange block through CUDA IPC; the owner's
    kernel stores its slice, partial and epoch flag into all peers over NVLink.
    torch.distributed is used once, to pass the 64-byte IPC handles around and
    to agree that every rank connected."""

    def __init__(self, gb, bounds, device, bits):
        """bounds: the vertex partition (world + 1 increasing ints, multiples of 32
        but the last; of 128 with bits, since the BFS kernel stores the owned
        bitmap slice 16 bytes at a time).  bits: the replicated array holds one bit
        per vertex (BFS) instead of one 32-bit word (float payloads)."""
        import torch.distributed as dist
        self._h = C.c_void_p()
        self.world = len(bounds) - 1
        unit = 128 if bits else 32
        if any(b % unit for b in bounds[:-1]):
            raise ValueError("PeerExchange: every bound but the last must be a multiple "
                             "of %d vertices%s: %s" % (
                                 unit, " for a bitmap exchange" if bits else "", bounds))
        if any(bounds[p + 1] <= bounds[p] for p in range(self.world)):
            raise ValueError("PeerExchange: every rank must own at least one vertex: %s"
                             % bounds)
        self.lib = gb._lib.load()
        self.rank = dist.get_rank() if self.world > 1 else 0
        offsets = [(b + 31) // 32 for b in bounds] if bits else bounds
        offs = (C.c_longlong * (self.world + 1))(*[int(o) for o in offsets])
        mine = (C.c_ubyte * 64)()
        why = None
        rc = self.lib.gb200_xchg_create(C.byref(self._h), self.world, self.rank,
                                        offs)
        if rc == 0:
            rc = self.lib.gb200_xchg_handle(self._h, mine)
            if rc != 0:
                why = "gb200_xchg_handle failed: %d" % rc
        else:
            why = "gb200_xchg_create failed: %d" % rc
        # Every rank takes part in the handle gather and in the agreement below, so
        # a rank that cannot set up makes every rank raise instead of leaving the
        # others to wait for its stores.
        t = torch.tensor(list(mine), dtype=torch.uint8, device=device)
        allh = torch.zeros(64 * self.world, dtype=torch.uint8, device=device)
        if self.world > 1:
            all_gather_into_tensor(allh, t)
        else:
            allh.copy_(t)
        if why is None:
            rc = self.lib.gb200_xchg_connect(self._h, allh.cpu().numpy().tobytes())
            if rc != 0:
                why = "gb200_xchg_connect failed: %d" % rc
        if self.world > 1:
            ok = torch.tensor([0 if why else 1], device=device)
            all_reduce(ok, dist.ReduceOp.MIN)
            if why is None and int(ok.item()) == 0:
                why = "the peer exchange could not be set up on another rank"
        if why is not None:
            self.close()
            raise RuntimeError(why)

    def _call(self, name, *args):
        out = C.c_int(0)
        rc = getattr(self.lib, name)(self._h, *args, C.byref(out))
        if rc != 0:
            raise RuntimeError("%s failed: %d" % (name, rc))
        return out.value

    def bfs(self, v_own, M, n, source, desc):
        """Levels of the owned vertices into v_own; returns the number of levels."""
        return self._call("gb200_dist_bfs_fused", v_own._h, M._h, n, source, desc._h)

    def pr(self, p_own, M, n, alpha, eps, desc):
        """Owned ranks into p_own; returns the number of iterations."""
        return self._call("gb200_dist_pr", p_own._h, M._h, n, alpha, eps, desc._h)

    def sssp(self, v_own, M, n, source, desc):
        """Owned distances into v_own; returns the number of rounds."""
        return self._call("gb200_dist_sssp", v_own._h, M._h, n, source, desc._h)

    def close(self):
        if self._h:
            self.lib.gb200_xchg_free(self._h)
            self._h = C.c_void_p()


# ---------------------------------------------------------------------------
# Bench (bench.py --gpus N)
# ---------------------------------------------------------------------------

def _all_ranks(values, dev):
    """float64 tensor of `values` from every rank, in rank order."""
    import torch.distributed as dist
    t = torch.tensor(values, device=dev, dtype=torch.float64)
    out = [torch.zeros_like(t) for _ in range(dist.get_world_size())]
    all_gather(out, t)
    return out


# Each setup partitions the graph, builds this rank's local matrix, vector and
# exchange, and returns what the harness needs as plain values: bounds, xchg,
# vec, run (one traversal; returns its level / iteration / round count), verify
# (kind and context of bench.py's checker), profile (the kernel kind whose
# launches give the roofline), kernel (its name), config (the run count -> the
# algorithm's config entries), e2e (what a step does and what the gathered
# slices hold, for the e2e note), extra (the checker's extra output -> result keys).

def _setup_bfs(gb, args, n, rowptr, colind, world, rank, dev):
    """Direction-optimised BFS: the whole traversal, exchange included, as one
    persistent kernel per GPU."""
    import os
    source = int(torch.argmax(rowptr[1:] - rowptr[:-1]).item())
    weight = os.environ.get("GB200_DIST_ROW_WEIGHT", "1e9")
    bounds = partition_bounds(rowptr, world, row_weight=float(weight))
    lo, hi = bounds[rank], bounds[rank + 1]
    M, _ = weighted_local_matrix(gb, n, rowptr, colind, None, lo, hi)
    nnz_local = int(rowptr[hi]) - int(rowptr[lo])
    nnz_per_rank = [int(t.item()) for t in _all_ranks([nnz_local], dev)]
    v = gb.Vector(max(hi - lo, 1))
    desc = gb.Descriptor(mxvmode=0, struconly=1, opreuse=0, earlyexit=1)
    xchg = PeerExchange(gb, bounds, dev, bits=True)
    return dict(
        bounds=bounds, xchg=xchg, vec=v,
        run=lambda: xchg.bfs(v, M, n, source, desc),
        verify=("bfs", {"source": source}),
        profile=1, kernel="bfsFusedDistKernel (whole traversal with the exchange), "
                          "slowest rank",
        config=lambda levels: {
            "workload": "direction-optimised BFS (LogicalOrAnd mxv, push<->pull) "
                        "on R-MAT scale-%d ef-%d seed %d, symmetrised"
                        % (args.scale, args.edgefactor, args.seed),
            "source": source, "levels": levels,
            "partition": "1-D row slices balanced on stored entries + %s per row, "
                         "bounds %s" % (weight, bounds),
            "nnz_per_rank": nnz_per_rank,
            "exchange": "peer-memory stores of the owned frontier slice into "
                        "every rank's replica (CUDA IPC over NVLink), flag + "
                        "count per level, level loop in C++",
            "flags": "--struconly 1 --earlyexit 1; pull levels probe the "
                     "replicated cumulative visited bitmap (global operand reuse)"},
        e2e=("source id H2D, traversal", "level"),
        extra=lambda check: {})


def _setup_pr(gb, args, n, rowptr, colind, world, rank, dev):
    """PageRank (10 power iterations): local merge-path SpMV on the owned rows, p
    exchanged through peer memory after every mxv."""
    alpha, niter = 0.85, 10
    bounds = partition_bounds(rowptr, world)
    lo, hi = bounds[rank], bounds[rank + 1]
    M = pagerank_local_matrix(gb, n, rowptr, colind, lo, hi, alpha)
    p_own = gb.Vector(hi - lo)
    desc = gb.Descriptor(mxvmode=0, max_niter=niter)
    xchg = PeerExchange(gb, bounds, dev, bits=False)
    return dict(
        bounds=bounds, xchg=xchg, vec=p_own,
        run=lambda: xchg.pr(p_own, M, n, alpha, 0.0, desc),
        verify=("pr", {"alpha": alpha, "niter": niter}),
        profile=0, kernel="spmvMergeKernel (merge-path pull SpMV), slowest rank",
        config=lambda iters: {
            "workload": "PageRank (PlusMultiplies mxv, %d iterations) on R-MAT "
                        "scale-%d ef-%d seed %d, symmetrised"
                        % (niter, args.scale, args.edgefactor, args.seed),
            "iterations": iters,
            "partition": "1-D nnz-balanced row slices, bounds %s" % bounds,
            "exchange": "peer-memory stores of the owned float slice into every "
                        "rank's replica (CUDA IPC over NVLink) + residual partial "
                        "per iteration, loop in C++"},
        e2e=("one PageRank run", "rank"),
        extra=lambda check: {
            "max_rel_err": check.get("max_rel_err_vs_reference") if check else None,
            "pagerank_check": check})


def _setup_sssp(gb, args, n, rowptr, colind, world, rank, dev):
    """SSSP: frontier values exchanged through peer memory after every mxv,
    direction chosen per round by mxv."""
    from graphblast_b200 import graphs
    nnz = int(colind.numel())
    source = int(torch.argmax(rowptr[1:] - rowptr[:-1]).item())
    w = gb.api.host_uniform_weights(args.seed, 1, 64, nnz)
    d_wt = graphs.transpose_values(n, rowptr, colind, torch.from_numpy(w).to(dev))
    bounds = partition_bounds(rowptr, world)
    lo, hi = bounds[rank], bounds[rank + 1]
    M, _ = weighted_local_matrix(gb, n, rowptr, colind, d_wt, lo, hi)
    v_own = gb.Vector(max(hi - lo, 1))
    desc = gb.Descriptor(mxvmode=0, switchpoint=0.025)
    xchg = PeerExchange(gb, bounds, dev, bits=False)
    return dict(
        bounds=bounds, xchg=xchg, vec=v_own,
        run=lambda: xchg.sssp(v_own, M, n, source, desc),
        verify=("sssp", {"source": source, "weights": w}),
        profile=0, kernel="spmvMergeKernel (merge-path pull SpMV), slowest rank",
        config=lambda rounds: {
            "workload": "SSSP (MinimumPlus mxv, push<->pull) on R-MAT scale-%d "
                        "ef-%d seed %d, symmetrised, uniform integer weights 1..64"
                        % (args.scale, args.edgefactor, args.seed),
            "source": source, "rounds": rounds,
            "partition": "1-D nnz-balanced row slices, bounds %s" % bounds,
            "exchange": "peer-memory stores of the owned frontier values into every "
                        "rank's replica (CUDA IPC over NVLink) + improved count per "
                        "round, loop in C++"},
        e2e=("source id H2D, traversal", "distance"),
        extra=lambda check: {})


def bench_distributed(args, world, rank, local_rank):
    """bench.py body for WORLD_SIZE > 1: strong scaling of the headline BFS, of
    SSSP or of PageRank (--algo) over the 1-D row partition."""
    setups = {"bfs": _setup_bfs, "sssp": _setup_sssp, "pr": _setup_pr}
    if args.algo not in setups:
        raise SystemExit("--algo %s has no multi-GPU path (bfs, sssp, pr)" % args.algo)
    import os
    import time
    import torch.distributed as dist
    import graphblast_b200 as gb
    from graphblast_b200 import graphs

    # keep stdout to the single JSON line: NCCL's banner goes to stderr
    os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
    dev = init_rank(local_rank)

    n = 1 << args.scale
    src, dst = graphs.rmat_edges(args.scale, args.edgefactor, seed=args.seed,
                                 device=dev)
    rowptr, colind = graphs.build_csr(n, src, dst, undirected=True)
    del src, dst
    nnz = int(colind.numel())
    a = setups[args.algo](gb, args, n, rowptr, colind, world, rank, dev)
    run, vec, bounds = a["run"], a["vec"], a["bounds"]
    h_rowptr = rowptr.cpu().numpy() if rank == 0 else None
    h_colind = colind.cpu().numpy() if rank == 0 else None
    del rowptr, colind
    torch.cuda.empty_cache()

    torch.cuda.synchronize()
    dist.barrier()
    for _ in range(max(args.warmup, 1)):
        run()
    torch.cuda.synchronize()
    dist.barrier()

    lib = gb._lib.load()
    launches0 = C.c_ulonglong(0)
    lib.gb200_launch_count(C.byref(launches0))
    lib.gb200_profile_enable(1)
    lib.gb200_profile_reset()
    sampler = None
    try:
        from bench import ClockSampler, measured_peak_hbm
        sampler = ClockSampler(dev.index)
        sampler.start()
    except Exception:                        # noqa: BLE001
        measured_peak_hbm = lambda: (3350.0, "H100 SXM data sheet, not measured")  # noqa: E731
    ev0 = torch.cuda.Event(enable_timing=True)
    ev1 = torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    dist.barrier()
    t0 = time.perf_counter()
    ev0.record()
    count = 0
    for _ in range(args.steps):
        count = run()
    ev1.record()
    torch.cuda.synchronize()
    wall_ms = (time.perf_counter() - t0) * 1e3
    clocks = sampler.stop() if sampler is not None else None
    dist.barrier()
    # the roofline kernel on this rank: CUDA-event time and algorithmic bytes
    k_ms, k_n, k_b = C.c_double(0), C.c_longlong(0), C.c_double(0)
    lib.gb200_profile_read(a["profile"], C.byref(k_ms), C.byref(k_n), C.byref(k_b))
    lib.gb200_profile_enable(0)
    kern_all = _all_ranks([k_ms.value, float(k_n.value), k_b.value], dev)
    ms = torch.tensor([ev0.elapsed_time(ev1), wall_ms], device=dev)
    all_reduce(ms, dist.ReduceOp.MAX)
    launches1 = C.c_ulonglong(0)
    lib.gb200_launch_count(C.byref(launches1))
    ms_per_step = float(ms[0].item()) / args.steps

    # end to end: step input H2D, run, full result vector to rank 0's host memory
    gather = ResultGather(bounds, world, rank, dev)
    e2e_ms = timed_e2e(args, run, gather, vec, dev, 4)
    # parity: the gathered result against the CPU code (the checker lives in
    # bench.py: nothing in this package touches oracle/)
    host = gather.run(vec)
    parity = None
    cpu_baseline = None
    check = None
    verify = getattr(args, "verify", None)
    if rank == 0 and verify is not None and not args.no_cpu_baseline:
        kind, ctx = a["verify"]
        parity, cpu_baseline, check = verify(kind, h_rowptr, h_colind, host.numpy(),
                                             ctx)
    # roofline of the dominant kernel on the slowest rank (same definition as N=1)
    slow = max(kern_all, key=lambda k: float(k[0].item()))
    s_ms, s_n, s_b = (float(slow[0].item()), float(slow[1].item()),
                      float(slow[2].item()))
    peak, peak_src = measured_peak_hbm()
    ach = (s_b / 1e9) / (s_ms / 1e3) if s_ms > 0 else 0.0
    config = {"n": n, "nnz": nnz}
    config.update(a["config"](count))
    config["l2_policy"] = "inputs larger than L2"
    step, slices = a["e2e"]
    result = {
        "metric": "MTEPS", "value": nnz / (ms_per_step * 1e3),
        "unit": UNIT,
        "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_per_step, "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": "f32",
        "data": "synthetic",
        "config": config,
        "e2e": {"value": nnz / (e2e_ms * 1e3), "unit": "MTEPS",
                "ms_per_step": e2e_ms, "h2d_bytes_per_step": 4,
                "d2h_bytes_per_step": gather.d2h_bytes,
                "note": "per step: %s, NCCL gather of the owned %s slices to rank 0 "
                        "and the n-float result D2H into rank 0's pinned memory; "
                        "wall clock, max over ranks" % (step, slices)},
        "gpu_launches": int(launches1.value - launches0.value),
        "roofline": {
            "kernel": a["kernel"], "bound": "hbm", "achieved": ach, "peak": peak,
            "unit": "GB/s", "frac": ach / peak if peak else None,
            "peak_source": peak_src, "launches": int(s_n),
            "ms_per_launch": s_ms / s_n if s_n else 0.0,
            "bytes_per_launch": s_b / s_n if s_n else 0.0,
            "share_of_step": s_ms / (ms_per_step * args.steps) if ms_per_step else 0.0,
            "traffic": None},
        "cpu_baseline": cpu_baseline,
        "parity_vs_cpu_reference": parity,
        "clocks": clocks,
    }
    result.update(a["extra"](check))
    a["xchg"].close()
    dist.destroy_process_group()
    return result
