"""Every operation on a caller's stream: a non-blocking torch stream S, set with
gb.set_stream, with a gate queued on it ahead of the work.

The legacy default stream (stream 0, where every other suite runs) is ordered with
every blocking stream, which hides a kernel, memset or copy issued on stream 0
instead of the library's stream, a host read that waits on the wrong stream, a
set_stream that does not drain, and a host buffer still being read after a call
returns.  S is non-blocking, so work issued on any other stream runs while S spins
in the gate (torch.cuda._sleep, one thread) and reads inputs that have not landed:
each of those bugs becomes a wrong answer every time.

1. Every producer x consumer pair of operand_states.RUN behind a short gate.
2. Every compute entry outside that table behind a short gate, checked against the
   reference its own suite uses and bit for bit against the same call on stream 0.
3. Host buffers in pinned memory: builds may overwrite their source once the call
   returns, extracts are complete on return, host-returned scalars are final.
4. Stream switches: set_stream drains the stream it replaces, objects cross streams,
   set_stream to the current stream returns at once, and the Python ingest helpers
   give the same CSR on S.
5. The mailbox's timed-out reads (util.hpp Runtime::mailWait), once per slot: a gate
   longer than the 2 s limit makes each one fall back to its own cell.
6. The profiler's counters on S equal those of the same sequence on stream 0.

Inputs are seeded per case and the library's memory pool is scrubbed with NaN before
each gate, so a stale copy of the answer cannot stand in for one that was not
computed.  The runtime is process-global: every test returns it to stream 0.
"""
import contextlib
import ctypes as C
import os
import time

import numpy as np
import pytest

import operand_states as st
import oracle_binding as orc
from support import Csr, components, device_matrix, gb, make_matrix, mtx_graph  # noqa: F401

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SHORT_MS = 3          # the gate ahead of each case of 1 and 2
LONG_MS = 200         # the gate of 3 and 4
MAIL_MS = 2500        # longer than mailWait's 2 s limit
MAIL_LIMIT_S = 2.0
FUSED = dict(struconly=1, opreuse=1, earlyexit=1)
PLUS = 1


class Streams(object):
    """Two non-blocking streams and a gate calibrated on this device's clock."""

    def __init__(self, torch):
        self.torch = torch
        self.S = torch.cuda.Stream()
        self.S2 = torch.cuda.Stream()
        self.cycles_per_ms = self._calibrate()

    def _calibrate(self):
        torch = self.torch
        cycles = 20000000
        with torch.cuda.stream(self.S):
            torch.cuda._sleep(1000)
            a = torch.cuda.Event(enable_timing=True)
            b = torch.cuda.Event(enable_timing=True)
            a.record()
            torch.cuda._sleep(cycles)
            b.record()
        b.synchronize()
        return cycles/max(a.elapsed_time(b), 1e-3)

    def gate(self, ms):
        """Spin one thread on the current torch stream for about ms milliseconds."""
        self.torch.cuda._sleep(int(ms*self.cycles_per_ms))

    @contextlib.contextmanager
    def on(self, gb, stream):
        """The library and torch on `stream` (None: stream 0); back to stream 0 and
        everything drained on the way out, whatever happens inside."""
        torch = self.torch
        try:
            gb.set_stream(0 if stream is None else stream.cuda_stream)
            with torch.cuda.stream(stream if stream is not None else
                                   torch.cuda.default_stream()):
                yield
        finally:
            gb.set_stream(0)
            torch.cuda.synchronize()


@pytest.fixture(scope="module")
def streams(gb):
    import torch
    s = Streams(torch)
    try:
        yield s
    finally:
        gb.set_stream(0)
        torch.cuda.synchronize()


def scrub(gb, n):
    """NaN into the pool blocks a case of up to n values may be handed next: blocks
    of n, n/4, n/16, ... values, all held at once, then freed."""
    held = []
    while True:
        v = gb.Vector(max(int(n), 1))
        v.fill(float("nan"))
        held.append(v)
        if n <= 1024:
            break
        n //= 4
    del held


def same_bits(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, "%s: %r %r vs %r %r" % (
        what, a.dtype, a.shape, b.dtype, b.shape)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "%s differs" % what


def elapsed(call):
    t0 = time.perf_counter()
    out = call()
    return out, time.perf_counter() - t0


# ---------------------------------------------------------------------------
# the setup itself
# ---------------------------------------------------------------------------

def test_the_side_stream_does_not_block_stream_0(gb, streams):
    """Gate S for 200 ms; a tiny op on torch's default stream (the legacy stream 0,
    where a stray library launch would go) must finish well before the gate ends,
    so that such a launch runs during the gate."""
    torch = streams.torch
    assert streams.cycles_per_ms > 1e5
    # a kernel's first launch may load its module, which waits for the whole device
    (torch.ones(4, device="cuda") + 1).sum()
    torch.cuda.synchronize()
    with torch.cuda.stream(streams.S):
        streams.gate(LONG_MS)
    t0 = time.perf_counter()
    x = torch.ones(4, device="cuda") + 1
    torch.cuda.default_stream().synchronize()
    took = time.perf_counter() - t0
    busy = not streams.S.query()
    streams.S.synchronize()
    assert float(x.sum()) == 8.0
    assert busy and took < 0.1, took


def test_the_gate_lasts_as_calibrated(gb, streams):
    torch = streams.torch
    with torch.cuda.stream(streams.S):
        t0 = time.perf_counter()
        streams.gate(LONG_MS)
        streams.S.synchronize()
    took = time.perf_counter() - t0
    assert 0.5*LONG_MS/1e3 < took < 4*LONG_MS/1e3, took


# ---------------------------------------------------------------------------
# 1. producer x consumer behind the gate
# ---------------------------------------------------------------------------

@pytest.fixture(scope="module")
def ctx(gb):
    rng = np.random.RandomState(2025)
    src = rng.randint(0, st.N, 3*st.N).astype(np.int32)
    dst = rng.randint(0, st.N, 3*st.N).astype(np.int32)
    rp, ci = orc.build_csr(st.N, src, dst, True)

    class Ctx(object):
        pass
    c = Ctx()
    c.S = Csr(st.N, st.N, rp, ci, rng.choice(np.float32([-3, -2, -1, 1, 2, 3]), len(ci)))
    c.M = device_matrix(gb, c.S)
    c.src = int(np.argmax(np.diff(rp)))
    # the matrix's cached summaries (merge tiles, first-neighbour and max-degree
    # summaries) are built here, on stream 0: the pairs gate the operations alone
    from test_operand_states_gpu import use_every_route
    use_every_route(gb, c.M, c.S, "warm-up")
    gb.sync()
    return c


@pytest.mark.parametrize("consumer", list(st.CONSUMERS))
def test_operand_pairs_behind_the_gate(gb, streams, ctx, consumer, monkeypatch):
    """Gate, producer, gate, consumer, the pair's host model.  A call that returns a
    value to the host waits for S and so ends the gate ahead of it.  Each host build
    (the inputs of most producers and consumers) queues a new gate, and one is queued
    between producer and consumer, so the producer's operation and the consumer's
    first call each wait behind a gate.  Work after another host read inside one
    producer or consumer (a reduce, a compaction's total) runs ungated."""
    build = gb.Vector.build

    def build_and_gate(self, *args):
        build(self, *args)
        streams.gate(1)
    monkeypatch.setattr(gb.Vector, "build", build_and_gate)
    failed = []
    with streams.on(gb, streams.S):
        for p in [p for p, c in st.RUN if c == consumer]:
            try:
                scrub(gb, st.N)
                streams.gate(SHORT_MS)
                op = st.PRODUCERS[p](gb, ctx, p)
                streams.gate(SHORT_MS)
                st.CONSUMERS[consumer](gb, ctx, op)
            except Exception as e:
                failed.append("%s -> %s: %s: %s" % (p, consumer, type(e).__name__, e))
    assert not failed, "\n".join(failed)


# ---------------------------------------------------------------------------
# 2. every other compute entry behind the gate, and bit for bit as on stream 0
# ---------------------------------------------------------------------------

def run_both(gb, streams, prepare, run, size):
    """prepare(gb) builds the inputs on the current stream; run(gb, inputs, gate)
    calls the operations, each one right after gate(), and returns host arrays.
    First on stream 0, where gate() does nothing: a kernel's first launch in the
    process may load its module, which waits for the whole device and so would end
    a gate.  Then, after a scrub of the pool, on S: the inputs are written behind a
    gate, and gate() queues a new one before each call, since every call that
    returns a value to the host waits for S and so ends the gate before it.  The two
    must agree bit for bit.  Returns the result on S."""
    with streams.on(gb, None):
        inputs = prepare(gb)
        want = [np.asarray(x) for x in run(gb, inputs, lambda: None)]
        del inputs
    with streams.on(gb, streams.S):
        scrub(gb, size)
        streams.gate(SHORT_MS)
        inputs = prepare(gb)
        got = [np.asarray(x) for x in run(gb, inputs, lambda: streams.gate(SHORT_MS))]
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        same_bits(g, w, "output %d on S and on stream 0" % i)
    return got


def rmat(scale, seed=1):
    rp, ci = orc.rmat_csr(scale, 16, seed)
    return rp, ci


def weighted(rp, ci, seed, values=np.float32([-3, -2, -1, 1, 2, 3])):
    n = len(rp) - 1
    return Csr(n, n, rp, ci, np.random.RandomState(seed).choice(values, len(ci)))


def csr_list(M):
    return list(M.extract_csr())


def test_mxm_unmasked_behind_the_gate(gb, streams):
    import mxm_reference as mref
    rp, ci = rmat(9, seed=11)
    A = weighted(rp, ci, 1)
    n = A.nrows
    got = run_both(gb, streams, lambda gb: device_matrix(gb, A),
                   lambda gb, M, gate: csr_list(_mxm(gb, M, M, n, gate)), A.nnz*4)
    for g, w in zip(got, mref.mxm(PLUS, A.ptr, A.ind, A.val, A.ptr, A.ind, A.val, n)):
        assert np.array_equal(g, w)


def _mxm(gb, A, B, n, gate):
    C_ = gb.Matrix(n, n)
    gate()
    gb.mxm(C_, None, None, PLUS, A, B, gb.Descriptor())
    return C_


def test_masked_mxm_and_triangle_count_behind_the_gate(gb, streams):
    rp, ci = rmat(10, seed=12)
    n = len(rp) - 1
    lr, lc = orc.tril(rp, ci)
    L = Csr(n, n, lr, lc, np.ones(len(lc), np.int32))
    want = orc.tc(lr, lc)

    def run(gb, Ld, gate):
        B = gb.Matrix(n, n, dtype=gb.api.INT32)
        gate()
        ntris, _ = gb.algorithm.tc(Ld, B, gb.Descriptor())
        # the masked mxm itself: C<L> = L * L'
        Cm = gb.Matrix(n, n, dtype=gb.api.INT32)
        desc = gb.Descriptor()
        desc.set(gb.Desc_field.GrB_INP1, gb.Desc_value.GrB_TRAN)
        gate()
        gb.mxm(Cm, Ld, None, PLUS, Ld, Ld, desc)
        return [np.int64([ntris])] + csr_list(B) + csr_list(Cm)
    got = run_both(gb, streams, lambda gb: device_matrix(gb, L, integer=True), run, 4*L.nnz)
    assert int(got[0][0]) == want
    assert int(got[3].astype(np.int64).sum()) == want
    assert int(got[6].astype(np.int64).sum()) == want


def test_spmm_behind_the_gate(gb, streams):
    import mxm_reference as mref
    rp, ci = rmat(10, seed=13)
    A = weighted(rp, ci, 2)
    n, k = A.nrows, 24
    Bh = np.random.RandomState(3).choice(np.float32([-2, -1, 0.5, 1, 2]), (n, k))

    def prepare(gb):
        B = gb.Matrix(n, k)
        B.build_dense(Bh)
        return device_matrix(gb, A), B

    def run(gb, inputs, gate):
        Ad, B = inputs
        AB = gb.Matrix(n, k)
        gate()
        gb.mxm(AB, None, None, PLUS, Ad, B, gb.Descriptor())
        return [AB.extract_dense()]
    got = run_both(gb, streams, prepare, run, n*k)
    b_ptr = np.arange(n + 1, dtype=np.int64)*k
    b_ind = np.tile(np.arange(k, dtype=np.int64), n)
    w_rp, w_ci, w_v = mref.mxm(PLUS, A.ptr, A.ind, A.val, b_ptr, b_ind, Bh.reshape(-1), k)
    want = np.zeros((n, k), np.float32)
    want[np.repeat(np.arange(n), np.diff(w_rp)), w_ci] = w_v
    assert np.array_equal(got[0], want)


def test_matrix_ewise_and_transpose_behind_the_gate(gb, streams):
    import ewise_matrix_reference as xref
    rp, ci = rmat(10, seed=14)
    A = weighted(rp, ci, 4)
    rp2, ci2 = rmat(10, seed=15)
    B = weighted(rp2, ci2, 5)
    n = A.nrows

    def run(gb, inputs, gate):
        Ad, Bd = inputs
        out = []
        for add in (True, False):
            C_ = gb.Matrix(n, n)
            gate()
            (gb.eWiseAdd if add else gb.eWiseMult)(C_, None, None, PLUS, Ad, Bd,
                                                   gb.Descriptor())
            out += csr_list(C_)
        T = gb.Matrix(n, n)
        gate()
        gb.transpose(T, None, None, Ad, gb.Descriptor())
        return out + csr_list(T)
    got = run_both(gb, streams, lambda gb: (device_matrix(gb, A), device_matrix(gb, B)),
                   run, 2*(A.nnz + B.nnz))
    for i, add in enumerate((True, False)):
        want = xref.ewise(add, PLUS, A.ptr, A.ind, A.val, B.ptr, B.ind, B.val, n)
        for g, w in zip(got[3*i:3*i + 3], want):
            assert np.array_equal(g, w)
    T = A.T
    for g, w in zip(got[6:], (T.ptr, T.ind, T.val)):
        assert np.array_equal(g, w)


def test_matrix_extract_and_assign_behind_the_gate(gb, streams):
    import assign_reference as aref
    import extract_reference as eref
    rp, ci = rmat(10, seed=16)
    A = weighted(rp, ci, 6)
    n = A.nrows
    rng = np.random.RandomState(7)
    I = rng.choice(n, 700, replace=False).astype(np.int32)
    J = rng.choice(n, 500, replace=False).astype(np.int32)
    src = weighted(*rmat(9, seed=17), 8)
    Ia = np.sort(rng.choice(n, src.nrows, replace=False)).astype(np.int32)
    Ja = rng.choice(n, src.ncols, replace=False).astype(np.int32)

    def run(gb, inputs, gate):
        Ad, Cd, Sd = inputs
        E = gb.Matrix(len(I), len(J))
        gate()
        gb.extract(E, None, None, Ad, I, len(I), J, len(J), gb.Descriptor())
        gate()
        gb.assign(Cd, None, None, Sd, Ia, len(Ia), Ja, len(Ja), gb.Descriptor())
        return csr_list(E) + csr_list(Cd)
    got = run_both(gb, streams, lambda gb: (device_matrix(gb, A), device_matrix(gb, A),
                                           device_matrix(gb, src)), run, 4*A.nnz)
    for g, w in zip(got[:3], eref.extract_matrix(A.ptr, A.ind, A.val, n, n, I, J)):
        assert np.array_equal(g, w)
    want = aref.assign_matrix((A.ptr, A.ind, A.val), n, n,
                              (src.ptr, src.ind, src.val, src.nrows, src.ncols), Ia, Ja)
    for g, w in zip(got[3:], want):
        assert np.array_equal(np.asarray(g), np.asarray(w).astype(np.asarray(g).dtype))


def test_matrix_reductions_and_value_writers_behind_the_gate(gb, streams):
    import ewise_reference as vref
    rp, ci = rmat(10, seed=18)
    A = weighted(rp, ci, 9)
    n = A.nrows
    alpha = np.float32(0.85)

    def run(gb, inputs, gate):
        Ad, Ld, Rd, Pd = inputs
        gate()
        total = gb.reduce(None, 0, Ad, gb.Descriptor())
        w = gb.Vector(n)
        gate()
        gb.reduce(None, 0, Ad, gb.Descriptor(), out=w)
        gate()
        Ld.tril(gb.Descriptor())
        gate()
        Rd.apply_uniform_random(gb.Descriptor(), seed=5, lo=1, hi=64)
        gate()
        Pd.pr_normalize(float(alpha), gb.Descriptor())
        return ([np.float64([total]), w.extractTuples()] + csr_list(Ld) + csr_list(Rd) +
                csr_list(Pd))
    got = run_both(gb, streams, lambda gb: tuple(device_matrix(gb, A) for _ in range(4)),
                   run, 2*A.nnz)
    assert got[0][0] == A.val.astype(np.float64).sum()
    assert np.array_equal(got[1], vref.reduce_rows(0, A.ptr, A.val)[0].astype(np.float32))
    tr, tc_ = orc.tril(A.ptr, A.ind)
    assert np.array_equal(got[2], tr) and np.array_equal(got[3], tc_)
    assert np.array_equal(got[4], A.val[A.rows() >= A.ind])
    assert np.array_equal(got[5], A.ptr) and np.array_equal(got[6], A.ind)
    r = got[7]
    assert np.all((r >= 1) & (r <= 64) & (r == np.round(r))) and len(np.unique(r)) > 32
    outdeg = vref.reduce_rows(0, A.ptr, A.val)[0].astype(np.float32)
    want = vref.scale_rows(4, A.ptr, vref.scale_csr(1, A.val, alpha), outdeg)
    assert np.array_equal(got[10], np.asarray(want, np.float32))


def test_ingest_behind_the_gate(gb, streams):
    import torch
    from graphblast_b200 import _lib, graphs
    REF = np.load(os.path.join(GOLDEN, "reference_cpu.npz"))
    scale = 11
    n = 1 << scale
    rng = np.random.RandomState(19)
    keys = rng.randint(0, 1 << 62, 50000, dtype=np.int64)
    keys[rng.randint(0, len(keys), 10000)] = keys[3]

    def prepare(gb):
        return (torch.from_numpy(keys).cuda(),
                torch.arange(len(keys), dtype=torch.int32, device="cuda"))

    def run(gb, inputs, gate):
        d_k, d_p = inputs
        gate()
        src, dst = graphs.rmat_edges(scale, 16, seed=2)
        gate()
        rp, ci = graphs.build_csr(n, src, dst, undirected=True)
        val = torch.arange(1, ci.numel() + 1, dtype=torch.float32, device="cuda")
        gate()
        tv = graphs.transpose_values(n, rp, ci, val)
        gate()
        assert _lib.load().gb200_sort_pairs_u64(C.c_void_p(d_k.data_ptr()),
                                                C.c_void_p(d_p.data_ptr()), len(keys), 40) == 0
        M = gb.Matrix(n, n)
        gate()
        gb.api._check(M._lib.gb200_matrix_build_coo_device(
            M._h, C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), None, src.numel(),
            graphs.INGEST_DROP_LOOPS | graphs.INGEST_DEDUP | graphs.INGEST_SYMMETRIZE),
            "build_coo_device")
        gate()
        L = gb.Matrix.from_mtx(os.path.join(GOLDEN, "chesapeake.mtx"), directed=0)
        return ([src.cpu().numpy(), dst.cpu().numpy(), rp.cpu().numpy(), ci.cpu().numpy(),
                 tv.cpu().numpy(), d_k.cpu().numpy(), d_p.cpu().numpy()] + csr_list(M)[:2] +
                csr_list(L))
    got = run_both(gb, streams, prepare, run, 32*n)
    osrc, odst = orc.rmat_edges(scale, 16, 2)
    assert np.array_equal(got[0], osrc) and np.array_equal(got[1], odst)
    orp, oci = orc.build_csr(n, osrc, odst, True)
    assert np.array_equal(got[2], orp) and np.array_equal(got[3], oci)
    rows = np.repeat(np.arange(n), np.diff(orp))
    order = np.lexsort((rows, oci))
    assert np.array_equal(got[4], np.arange(1, len(oci) + 1, dtype=np.float32)[order])
    low = keys.view(np.uint64) & np.uint64((1 << 40) - 1)
    perm = np.argsort(low, kind="stable")
    assert np.array_equal(got[5], keys[perm]) and np.array_equal(got[6], perm.astype(np.int32))
    assert np.array_equal(got[7], orp) and np.array_equal(got[8], oci)
    key = "load/chesapeake.mtx/0/"
    for g, name in zip(got[9:], ("rowptr", "colind", "val")):
        assert np.array_equal(g, REF[key + name])


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_bfs_behind_the_gate(gb, streams, mode):
    """Timed, then the enqueue-only form twice on one descriptor (both results read
    after the second call)."""
    rp, ci = rmat(12, seed=20)
    n = len(rp) - 1
    deg = np.diff(rp)
    s1, s2 = int(np.argmax(deg)), int(np.nonzero(deg)[0][-1])

    def run(gb, A, gate):
        desc = gb.Descriptor(mxvmode=mode, **FUSED)
        v, v1, v2 = gb.Vector(n), gb.Vector(n), gb.Vector(n)
        gate()
        ms = gb.algorithm.bfs(v, A, s2, desc, timed=True)
        assert ms > 0
        gate()
        assert gb.algorithm.bfs(v1, A, s1, desc) is None
        gate()
        assert gb.algorithm.bfs(v2, A, s2, desc) is None
        return [v.extractTuples(), v1.extractTuples(), v2.extractTuples()]
    got = run_both(gb, streams, lambda gb: make_matrix(gb, rp, ci), run, n)
    assert np.array_equal(got[0].astype(np.int32), orc.bfs(rp, ci, s2))
    assert np.array_equal(got[1].astype(np.int32), orc.bfs(rp, ci, s1))
    assert np.array_equal(got[2], got[0])


def test_sssp_and_pagerank_behind_the_gate(gb, streams):
    rp, ci = rmat(11, seed=21)
    n = len(rp) - 1
    w = np.random.RandomState(22).randint(1, 64, len(ci)).astype(np.float32)
    src = int(np.argmax(np.diff(rp)))

    def run(gb, inputs, gate):
        W, P = inputs
        d = gb.Vector(n)
        gate()
        gb.algorithm.sssp(d, W, src, gb.Descriptor(mxvmode=0))
        desc = gb.Descriptor(mxvmode=0, max_niter=10)
        gate()
        P.pr_normalize(0.85, desc)
        p = gb.Vector(n)
        gate()
        gb.algorithm.pr(p, P, 0.85, 0.0, desc)
        return [d.extractTuples(), p.extractTuples()]
    got = run_both(gb, streams, lambda gb: (make_matrix(gb, rp, ci, w, symmetric=False),
                                           make_matrix(gb, rp, ci, symmetric=False)), run, n)
    assert np.array_equal(got[0], orc.sssp(rp, ci, w, src))
    want = orc.pr(rp, ci, 0.85, 0.0, 10).astype(np.float64)
    rel = np.abs(got[1] - want)/np.maximum(np.abs(want), 1e-30)
    assert rel.max() < 1e-5, rel.max()


def test_cooperative_algorithms_behind_the_gate(gb, streams):
    """cc, gc, mis, lgc with its sweep, bc, ktruss, trussness and scc: every
    cooperative kernel launched on S."""
    import bc_reference
    import greedy_oracle
    import lgc_reference
    import scc_reference
    import truss_reference
    rp, ci = rmat(10, seed=23)
    n = len(rp) - 1
    cc_rp, cc_ci = mtx_graph("test_cc")
    drp, dci = orc.build_csr(1 << 11, *orc.rmat_edges(11, 8, 24), False)
    nd = len(drp) - 1
    s = int(np.argmax(np.diff(rp)))
    sources = np.random.RandomState(25).choice(n, 40, replace=False)
    psources = pinned(sources.astype(np.int32))

    def prepare(gb):
        return (make_matrix(gb, rp, ci), make_matrix(gb, cc_rp, cc_ci),
                make_matrix(gb, drp, dci, symmetric=False))

    def run(gb, inputs, gate):
        A, G, D = inputs
        out = []
        for M, k in ((A, n), (G, len(cc_rp) - 1)):
            v = gb.Vector(k)
            gate()
            ncomp, _ = gb.algorithm.cc(v, M, gb.Descriptor())
            out += [np.int64([ncomp]), v.extractTuples()]
        v = gb.Vector(n)
        gate()
        ncol, _ = gb.algorithm.gc(v, A, 3, gb.Descriptor())
        out += [np.int64([ncol]), v.extractTuples()]
        v = gb.Vector(n)
        gate()
        nm, _ = gb.algorithm.mis(v, A, 3, gb.Descriptor())
        out += [np.int64([nm]), v.extractTuples()]
        p, r = gb.Vector(n), gb.Vector(n)
        gate()
        rounds, _ = gb.algorithm.lgc(p, A, s, 0.15, 1e-6, gb.Descriptor(), residual=r)
        cl = gb.Vector(n)
        gate()
        size, phi, _ = gb.algorithm.lgc_sweep(cl, p, A, gb.Descriptor())
        out += [np.int64([rounds, size]), np.float64([phi]), p.extractTuples(),
                r.extractTuples(), cl.extractTuples()]
        v = gb.Vector(n)
        # the sources from pinned memory: staging a pageable copy may wait for S
        ms = C.c_float(0)
        gate()
        assert gb.api._lib.load().gb200_bc(v._h, A._h, psources.ctypes.data_as(C.c_void_p),
                                           len(psources), gb.Descriptor()._h,
                                           C.byref(ms)) == 0
        out.append(v.extractTuples())
        K = gb.Matrix(n, n, dtype=gb.api.INT32)
        gate()
        nedges, _ = gb.algorithm.ktruss(K, A, 4, gb.Descriptor())
        T = gb.Matrix(n, n, dtype=gb.api.INT32)
        gate()
        kmax, _ = gb.algorithm.trussness(T, A, gb.Descriptor())
        out += [np.int64([nedges, kmax])] + csr_list(K) + csr_list(T)
        v = gb.Vector(nd)
        gate()
        nscc, _ = gb.algorithm.scc(v, D, gb.Descriptor())
        out += [np.int64([nscc]), v.extractTuples()]
        return out
    got = run_both(gb, streams, prepare, run, 4*len(ci))
    lab, k = components(n, rp, ci)
    assert got[0][0] == k and np.array_equal(got[1], lab.astype(np.float32))
    lab, k = components(len(cc_rp) - 1, cc_rp, cc_ci)
    assert got[2][0] == k and np.array_equal(got[3], lab.astype(np.float32))
    col, ncol, _ = greedy_oracle.gc(rp, ci, 3)
    assert got[4][0] == ncol and np.array_equal(got[5], col.astype(np.float32))
    mem, size, _ = greedy_oracle.mis(rp, ci, 3)
    assert got[6][0] == size and np.array_equal(got[7], mem.astype(np.float32))
    want_p, want_r, want_rounds, _ = lgc_reference.push(rp, ci, s, 0.15, 1e-6)
    want_cl, want_size, want_phi = lgc_reference.sweep(rp, ci, want_p)
    assert list(got[8]) == [want_rounds, want_size] and got[9][0] == want_phi
    same_bits(got[10], want_p, "lgc p")
    same_bits(got[11], want_r, "lgc residual")
    assert np.array_equal(got[12], want_cl)
    want_bc = bc_reference.brandes(rp, ci, sources)
    assert np.allclose(got[13], want_bc, rtol=1e-6, atol=1e-6)
    sup, nedges = truss_reference.ktruss(rp, ci, 4)
    tau, kmax = truss_reference.trussness(rp, ci)
    assert list(got[14]) == [nedges, kmax]
    for g, w in zip(got[15:18], truss_reference.kept_csr(rp, ci, sup)):
        assert np.array_equal(g, w)
    for g, w in zip(got[18:21], truss_reference.kept_csr(rp, ci, tau)):
        assert np.array_equal(g, w)
    lab, k = scc_reference.scc(drp, dci)
    assert got[21][0] == k and np.array_equal(got[22].astype(np.int64), lab)


# ---------------------------------------------------------------------------
# 3. host buffers in pinned memory
# ---------------------------------------------------------------------------

def pinned(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).pin_memory().numpy()


def test_builds_may_overwrite_pinned_sources_on_return(gb, streams):
    """A build returns only once its host values are on the device: the caller may
    overwrite the buffer at once."""
    rng = np.random.RandomState(30)
    n = 1 << 16
    x = rng.choice(st.VALS, n)
    ind = np.sort(rng.choice(n, n//7, replace=False)).astype(np.int32)
    val = rng.choice(st.VALS, len(ind))
    rows = rng.randint(0, 3000, 40000).astype(np.int32)
    cols = rng.randint(0, 2000, 40000).astype(np.int32)
    keys = np.unique(rows.astype(np.int64)*2000 + cols)
    rows, cols = (keys//2000).astype(np.int32), (keys % 2000).astype(np.int32)
    mval = rng.choice(np.float32([-2, -1, 1, 2, 5]), len(rows))
    dense = rng.choice(np.float32([-2, -1, 0.5, 1, 2]), (3000, 16))
    rp, ci = rmat(9, seed=31)
    srcs = rng.choice(len(rp) - 1, 20, replace=False).astype(np.int32)
    bufs = [pinned(a) for a in (x, ind, val, rows, cols, mval, dense, srcs)]
    px, pind, pval, prows, pcols, pmval, pdense, psrcs = bufs
    with streams.on(gb, streams.S):
        A = make_matrix(gb, rp, ci)
        scrub(gb, n)
        vd, vs = gb.Vector(n), gb.Vector(n)
        M, Dm = gb.Matrix(3000, 2000), gb.Matrix(3000, 16)
        # a gate ahead of each build: its copy waits behind it
        streams.gate(LONG_MS)
        vd.build(px)
        px[:] = -9
        streams.gate(LONG_MS)
        vs.build(pind, pval)
        pind[:] = 0
        pval[:] = -9
        streams.gate(LONG_MS)
        M.build(prows, pcols, pmval)
        prows[:] = 0
        pcols[:] = 0
        pmval[:] = -9
        streams.gate(LONG_MS)
        Dm.build_dense(pdense)
        pdense[:] = -9
        streams.gate(LONG_MS)
        bcv = gb.Vector(len(rp) - 1)
        ms = C.c_float(0)
        assert gb.api._lib.load().gb200_bc(bcv._h, A._h, psrcs.ctypes.data_as(C.c_void_p),
                                           len(psrcs), gb.Descriptor()._h, C.byref(ms)) == 0
        psrcs[:] = 0
        assert np.array_equal(vd.extractTuples(), x)
        gi, gv = vs.extractTuples(sparse=True)
        assert np.array_equal(gi, ind) and np.array_equal(gv, val)
        mr, mc, mv = M.extract_csr()
        order = np.lexsort((cols, rows))
        assert np.array_equal(mc, cols[order]) and np.array_equal(mv, mval[order])
        assert np.array_equal(np.repeat(np.arange(3000), np.diff(mr)), rows[order])
        assert np.array_equal(Dm.extract_dense(), dense)
        import bc_reference
        assert np.allclose(bcv.extractTuples(), bc_reference.brandes(rp, ci, srcs),
                           rtol=1e-6, atol=1e-6)


def test_extracts_into_pinned_memory_are_complete_on_return(gb, streams):
    """A gate is queued after the operation producing the values returns and before
    the extract is called: the pinned buffer must hold every value when the extract
    returns."""
    lib = gb.api._lib.load()
    rp, ci = rmat(11, seed=32)
    A = weighted(rp, ci, 33)
    n = A.nrows
    rng = np.random.RandomState(34)
    u = rng.choice(st.VALS, n)
    Bh = rng.choice(np.float32([-1, 0.5, 2]), (n, 8))
    want_w = (A.scipy() @ u.astype(np.float64)).astype(np.float32)
    import mxm_reference as mref
    want_c = mref.mxm(PLUS, A.ptr, A.ind, A.val, A.ptr, A.ind, A.val, n)
    with streams.on(gb, streams.S):
        Ad = device_matrix(gb, A)
        ud = st._dense(gb, u)
        B = gb.Matrix(n, 8)
        B.build_dense(Bh)
        scrub(gb, 8*n)
        w = gb.Vector(n)
        gb.mxv(w, None, None, PLUS, Ad, ud, gb.Descriptor(mxvmode=2))
        out = pinned(np.full(n, -7, np.float32))
        streams.gate(LONG_MS)
        w.extract_into(out)
        assert np.array_equal(out, want_w)

        w2 = gb.Vector(n)
        gb.mxv(w2, None, None, PLUS, Ad, ud, gb.Descriptor(mxvmode=2))
        w2.dense2sparse(0.0, gb.Descriptor())
        cnt = C.c_int(n)
        pi, pv = pinned(np.full(n, -1, np.int32)), pinned(np.full(n, -7, np.float32))
        streams.gate(LONG_MS)
        assert lib.gb200_vector_extract_sparse(w2._h, pi.ctypes.data_as(C.c_void_p),
                                               pv.ctypes.data_as(C.c_void_p),
                                               C.byref(cnt)) == 0
        nz = np.nonzero(want_w)[0]
        assert cnt.value == len(nz)
        assert np.array_equal(pi[:len(nz)], nz) and np.array_equal(pv[:len(nz)], want_w[nz])

        Cm = gb.Matrix(n, n)
        gb.mxm(Cm, None, None, PLUS, Ad, Ad, gb.Descriptor())
        nv = Cm.nvals()
        assert nv == len(want_c[1])
        prp = pinned(np.full(n + 1, -1, np.int32))
        pci, pcv = pinned(np.full(nv, -1, np.int32)), pinned(np.full(nv, -7, np.float32))
        streams.gate(LONG_MS)
        assert lib.gb200_matrix_extract_csr(Cm._h, prp.ctypes.data_as(C.c_void_p),
                                            pci.ctypes.data_as(C.c_void_p),
                                            pcv.ctypes.data_as(C.c_void_p)) == 0
        for g, w_ in zip((prp, pci, pcv), want_c):
            assert np.array_equal(g, w_)

        AB = gb.Matrix(n, 8)
        gb.mxm(AB, None, None, PLUS, Ad, B, gb.Descriptor())
        pd = pinned(np.full((n, 8), -7, np.float32))
        streams.gate(LONG_MS)
        assert lib.gb200_matrix_extract_dense(AB._h, pd.ctypes.data_as(C.c_void_p),
                                              pd.size) == 0
        assert np.array_equal(pd, (A.scipy() @ Bh.astype(np.float64)).astype(np.float32))


def test_host_scalars_are_final_on_return(gb, streams):
    rp, ci = rmat(11, seed=35)
    n = len(rp) - 1
    lr, lc = orc.tril(rp, ci)
    rng = np.random.RandomState(36)
    x = rng.choice(st.VALS, n)
    src = int(np.argmax(np.diff(rp)))
    with streams.on(gb, streams.S):
        A = make_matrix(gb, rp, ci)
        L = make_matrix(gb, lr, lc, symmetric=False, integer=True)
        xd = st._dense(gb, x)
        scrub(gb, 4*len(ci))
        streams.gate(LONG_MS)
        w = gb.Vector(n)
        gb.eWiseAdd(w, None, None, PLUS, xd, xd, gb.Descriptor())
        w.dense2sparse(0.0, gb.Descriptor())
        assert w.nvals() == int(np.count_nonzero(x))
        streams.gate(LONG_MS)
        y = gb.Vector(n)
        gb.eWiseAdd(y, None, None, PLUS, xd, xd, gb.Descriptor())
        assert gb.reduce(None, 0, y, gb.Descriptor()) == 2*x.astype(np.float64).sum()
        streams.gate(LONG_MS)
        B = gb.Matrix(n, n, dtype=gb.api.INT32)
        assert gb.algorithm.tc(L, B, gb.Descriptor())[0] == orc.tc(lr, lc)
        streams.gate(LONG_MS)
        v = gb.Vector(n)
        assert gb.algorithm.cc(v, A, gb.Descriptor())[0] == components(n, rp, ci)[1]
        streams.gate(LONG_MS)
        v = gb.Vector(n)
        t0 = time.perf_counter()
        ms = gb.algorithm.bfs(v, A, src, gb.Descriptor(mxvmode=0, **FUSED), timed=True)
        took = time.perf_counter() - t0
        # the time is read after the traversal ended, so the gate ahead of it is over
        assert 0 < ms and took >= 0.5*LONG_MS/1e3
        assert np.array_equal(v.extractTuples().astype(np.int32), orc.bfs(rp, ci, src))


# ---------------------------------------------------------------------------
# 4. stream switches
# ---------------------------------------------------------------------------

def test_set_stream_drains_the_stream_it_replaces(gb, streams):
    """An op on S1 behind a gate writes x; after set_stream(S2) an op reads x.
    Without the drain the read would run while S1 still waits in the gate."""
    torch = streams.torch
    rp, ci = rmat(11, seed=40)
    A = weighted(rp, ci, 41)
    n = A.nrows
    u = np.random.RandomState(42).choice(st.VALS, n)
    want = (A.scipy() @ u.astype(np.float64)).astype(np.float32)
    with streams.on(gb, streams.S):
        Ad = device_matrix(gb, A)
        ud = st._dense(gb, u)
        # one pull first builds Ad's merge tiles and the descriptor's scratch (freeing
        # or growing that scratch waits for the whole device), so that the gated pull
        # waits for nothing
        desc, d2 = gb.Descriptor(mxvmode=2), gb.Descriptor()
        # (on other values: the pool may hand its output's block to x)
        gb.mxv(gb.Vector(n), None, None, PLUS, Ad, st._dense(gb, np.ones(n)), desc)
        # y's storage too: a pool allocation on S2 that reuses a block freed on S1 may
        # make S2 wait for S1 and so stand in for the drain
        y = gb.Vector(n)
        gb.eWiseAdd(y, None, None, PLUS, ud, ud, d2)
        gb.reduce(None, 0, ud, d2)
        scrub(gb, n)
        gb.sync()
        streams.gate(LONG_MS)
        x = gb.Vector(n)
        gb.mxv(x, None, None, PLUS, Ad, ud, desc)
        assert not streams.S.query(), "the pull waited for the gate"
        gb.set_stream(streams.S2.cuda_stream)
        with torch.cuda.stream(streams.S2):
            gb.eWiseAdd(y, None, None, PLUS, x, x, d2)
            total = gb.reduce(None, 0, x, d2)
            assert np.array_equal(y.extractTuples(), 2*want)
            assert total == want.astype(np.float64).sum()


def test_objects_cross_streams(gb, streams):
    """S1 -> S2 -> 0 -> S1: objects made on one stream, used and freed on another."""
    torch = streams.torch
    rp, ci = rmat(10, seed=43)
    A = weighted(rp, ci, 44)
    n = A.nrows
    u = np.random.RandomState(45).choice(st.VALS, n)
    Au = A.scipy() @ u.astype(np.float64)
    with streams.on(gb, streams.S):
        Ad = device_matrix(gb, A)
        streams.gate(SHORT_MS)
        w1 = gb.Vector(n)
        gb.mxv(w1, None, None, PLUS, Ad, st._dense(gb, u), gb.Descriptor(mxvmode=2))
        gb.set_stream(streams.S2.cuda_stream)
        with torch.cuda.stream(streams.S2):
            streams.gate(SHORT_MS)
            w2 = gb.Vector(n)
            gb.eWiseAdd(w2, None, None, PLUS, w1, w1, gb.Descriptor())
            del w1
            C1 = gb.Matrix(n, n)
            gb.eWiseAdd(C1, None, None, PLUS, Ad, Ad, gb.Descriptor())
        gb.set_stream(0)
        w3 = gb.Vector(n)
        gb.mxv(w3, None, None, PLUS, C1, w2, gb.Descriptor(mxvmode=2))
        del w2
        gb.set_stream(streams.S.cuda_stream)
        streams.gate(SHORT_MS)
        w4 = gb.Vector(n)
        gb.eWiseAdd(w4, None, None, PLUS, w3, w3, gb.Descriptor())
        del w3, C1
        total = gb.reduce(None, 0, w4, gb.Descriptor())
        got = w4.extractTuples()
    want = 2*(2*A.scipy()) @ (2*Au)
    assert np.array_equal(got, want.astype(np.float32))
    assert total == want.sum()


def test_set_stream_to_the_current_stream_returns_at_once(gb, streams):
    with streams.on(gb, streams.S):
        streams.gate(LONG_MS)
        _, took = elapsed(lambda: gb.set_stream(streams.S.cuda_stream))
        busy = not streams.S.query()
    assert busy and took < 0.1, took


def test_python_ingest_on_the_side_stream(gb, streams):
    """graphs.build_csr, matrix_from_csr and transpose_values under
    torch.cuda.stream(S) give the CSR they give on the default stream."""
    import torch
    from graphblast_b200 import graphs
    scale = 12
    n = 1 << scale

    def run():
        src, dst = graphs.rmat_edges(scale, 16, seed=4)
        rp, ci = graphs.build_csr(n, src, dst, undirected=True)
        val = torch.arange(1, ci.numel() + 1, dtype=torch.float32, device="cuda")
        tv = graphs.transpose_values(n, rp, ci, val)
        M = graphs.matrix_from_csr(n, rp, ci, val, cscval=tv)
        return [rp.cpu().numpy(), ci.cpu().numpy(), tv.cpu().numpy()] + csr_list(M)
    with streams.on(gb, streams.S):
        scrub(gb, 32*n)
        streams.gate(SHORT_MS)
        got = run()
    with streams.on(gb, None):
        want = run()
    for i, (g, w) in enumerate(zip(got, want)):
        same_bits(g, w, "ingest output %d" % i)


# ---------------------------------------------------------------------------
# 5. the mailbox's timed-out reads
# ---------------------------------------------------------------------------

def mailbox_case(gb, streams, make, check):
    """make(gb, seed) queues the inputs and returns read(), the call that waits on the
    mailbox; check(seed, value) checks what read() returned.  Behind a gate longer
    than the wait limit nothing is posted in time, so the read can only return the
    right value from its own cell once the gate is over: the call must be right and
    take at least the limit.  (The time alone does not tell the fallback from a wait
    that ends when the late post arrives; a fallback that reads a wrong cell or value
    fails the check.)  The same call at once without a gate, on other inputs, must
    get its own value, not the late post of the timed-out ticket."""
    with streams.on(gb, streams.S):
        read = make(gb, 1)
        scrub(gb, 1 << 16)
        streams.gate(MAIL_MS)
        fire = read()
        value, took = elapsed(fire)
        check(1, value)
        assert took >= MAIL_LIMIT_S, "the read did not wait out the limit: %.3f s" % took
        read = make(gb, 2)
        value, took = elapsed(read())
        check(2, value)
        assert took < MAIL_LIMIT_S


def test_mailbox_fallback_compaction_total(gb, streams):
    """Slot 0: dense2sparse's total."""
    n = 1 << 16
    xs = {k: np.random.RandomState(50 + k).choice(np.float32([0, 0, 0, 1, -2]), n)
          for k in (1, 2)}

    def make(gb, k):
        v = st._dense(gb, xs[k])

        def read():
            def go():
                v.dense2sparse(0.0, gb.Descriptor())
                return v.extractTuples(sparse=True)
            return go
        return read

    def check(k, got):
        ind, val = got
        nz = np.nonzero(xs[k])[0]
        assert np.array_equal(ind, nz) and np.array_equal(val, xs[k][nz])
    mailbox_case(gb, streams, make, check)


def test_mailbox_fallback_boolean_pull_count(gb, streams, ctx):
    """Slot 1: the fused Boolean pull's pending count, read by a plus-reduce; two
    vectors are left with pending counts and the first one is read."""
    def make(gb, k):
        rng = np.random.RandomState(60 + k)
        vis = [(rng.rand(st.N) < 0.4).astype(np.float32) for _ in range(2)]
        us = [(rng.rand(st.N) < d).astype(np.float32) for d in (0.02, 0.3)]
        masks = [st._shadowed(gb, m) for m in vis]
        ins = [st._dense(gb, u) for u in us]
        want = [st.ref.bool_pull(ctx.S.ptr, ctx.S.ind, m, u, 0.0, True, False)
                for m, u in zip(vis, us)]
        desc = gb.Descriptor(mxvmode=2, fusedmask=1, earlyexit=1)
        desc.toggle(gb.Desc_field.GrB_MASK)
        plain = gb.Descriptor()

        def pulls():
            ws = []
            for m, u in zip(masks, ins):
                w = gb.Vector(st.N)
                gb.mxv(w, m, None, st.LOR, ctx.M, u, desc)
                ws.append(w)
            return ws

        def go(ws):
            first = gb.reduce(None, 0, ws[0], plain)
            second = gb.reduce(None, 0, ws[1], plain)
            return first, second, want
        go(pulls())          # the descriptors' scratch and every kernel, before the gate
        gb.sync()

        def read():
            ws = pulls()
            return lambda: go(ws)
        return read

    def check(k, got):
        first, second, want = got
        assert first == want[0].sum() and second == want[1].sum()
        assert want[0].sum() != want[1].sum()
    mailbox_case(gb, streams, make, check)


def test_mailbox_fallback_reduce(gb, streams):
    """Slot 2: the vector reduce's fold."""
    n = 1 << 16
    xs = {k: np.random.RandomState(70 + k).choice(st.VALS, n) for k in (1, 2)}

    def make(gb, k):
        x = st._dense(gb, xs[k])

        def read():
            y = gb.Vector(n)
            gb.eWiseAdd(y, None, None, PLUS, x, x, gb.Descriptor())
            return lambda: gb.reduce(None, 0, y, gb.Descriptor())
        return read

    def check(k, got):
        assert got == 2*xs[k].astype(np.float64).sum()
    mailbox_case(gb, streams, make, check)


def test_mailbox_fallback_push_edge_count(gb, streams):
    """Slot 4: the push's edge count for the direction check, a frontier of more than
    4096 entries under push-pull."""
    import test_mxv_gpu as mx
    rng = np.random.RandomState(80)
    m = 6000
    lens = rng.randint(0, 3, m)
    lens[:5000] = rng.randint(5, 12, 5000)
    H = mx.structure(rng, lens, m, "int")
    fronts = {1: np.arange(5000), 2: np.sort(rng.choice(m, 4500, replace=False))}
    fvals = {k: rng.choice(st.VALS[st.VALS != 0], len(f)) for k, f in fronts.items()}

    def make(gb, k):
        Hd = device_matrix(gb, H)
        f = gb.Vector(m)
        f.build(np.asarray(fronts[k], np.int32), np.asarray(fvals[k], np.float32))

        def read():
            def go():
                w = gb.Vector(m)
                desc = gb.Descriptor(mxvmode=0, switchpoint=0.9)
                gb.vxm(w, None, None, PLUS, f, Hd, desc)
                return w.extractTuples(), desc.lastmxv
            return go
        return read

    def check(k, got):
        w, route = got
        ind, val = st.ref.push(PLUS, H.ptr, H.ind, H.val, fronts[k], fvals[k], m)
        assert np.array_equal(w, st.eref.densify(m, ind, val, 0))
        # the count read decides the direction alone: more than 33 % of the entries
        # (GB200_EDGE_SWITCH_PCT) hands the push back to the pull
        edges = int(np.diff(H.ptr)[fronts[k]].sum())
        assert abs(edges - 0.33*H.nnz) > 0.01*H.nnz
        want = (gb.Desc_value.GrB_PULLONLY if edges > 0.33*H.nnz else
                gb.Desc_value.GrB_PUSHONLY)
        assert route == want, (route, edges, H.nnz)
    mailbox_case(gb, streams, make, check)


# ---------------------------------------------------------------------------
# 6. the profiler on S
# ---------------------------------------------------------------------------

def test_profiler_counts_on_the_side_stream(gb, streams):
    lib = gb.api._lib.load()
    rp, ci = orc.build_csr(1 << 11, *orc.rmat_edges(11, 8, 3), False)
    n = len(rp) - 1
    s = int(np.argmax(np.diff(rp)))

    def profiled(gated):
        A = make_matrix(gb, rp, ci, symmetric=False)
        desc = gb.Descriptor(mxvmode=0, **FUSED)
        v = gb.Vector(n)
        lib.gb200_profile_enable(1)
        try:
            lib.gb200_profile_reset()
            if gated:
                streams.gate(SHORT_MS)
            gb.algorithm.bfs(v, A, s, desc)
            out = []
            for kind in range(5):
                ms, launches, nbytes = C.c_double(0), C.c_longlong(0), C.c_double(0)
                assert lib.gb200_profile_read(kind, C.byref(ms), C.byref(launches),
                                              C.byref(nbytes)) == 0
                out.append((launches.value, nbytes.value))
        finally:
            lib.gb200_profile_enable(0)
        assert np.array_equal(v.extractTuples().astype(np.int32), orc.bfs(rp, ci, s))
        return out
    with streams.on(gb, streams.S):
        got = profiled(True)
    with streams.on(gb, None):
        want = profiled(False)
    assert got == want and got[1][0] >= 1 and got[1][1] > 0
