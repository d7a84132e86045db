"""Operations on the operands other operations leave behind, against the float64 and
integer references of the operation suites.

1. Vector producer x consumer table (operand_states.py): every pair of RUN, each
   consumer over every producer it applies to.
2. One Descriptor through a seeded sequence of pushes with different identities,
   zero-product masked pushes, scmp masks, struct-only on and off, output sizes that
   grow and shrink, a push that hands back to the pull, refused INT32 operands, SSSP,
   a fused BFS, reduce and compactions: the push arenas ("accumulator all identity,
   touched bitmap all zero" between calls) and the counter cells must come out of
   each call as the next one expects.  The same steps on fresh Descriptors must give
   the same bits.
3. One Matrix through every writer that replaces it in place: the merge tiles, the
   Boolean-pull first-neighbour summary, the fused-BFS max-degree summary and (in a
   child process with the hub thresholds at 0) the hub index must be rebuilt, and the
   host CSR mirror must follow value-only changes too.
4. Writing through device_ptr or a build_device tensor: re-adopting (INTEGRATION.md)
   is what makes the library see the new contents.

Values are integers (every comparison bit-exact) except after pr_normalize, where
pulls are held to the reference's float64 bound.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import ewise_reference as eref
import mxm_reference as mref
import mxv_reference as ref
import operand_states as st
import oracle_binding as orc
from support import Csr, check_csr, csr, device_matrix, gb  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HUB_FORCED = (os.environ.get("GB200_SPMV_HUB_MIN_NNZ") == "0" and
              os.environ.get("GB200_SPMV_HUB_MIN_PCT") == "0")
PLUS, MINPLUS, MAXMUL, LOR = 1, 2, 3, 0
INTS = np.float32([v for v in range(-8, 9) if v != 0])


def symmetric_graph(rng, n, m):
    src = rng.randint(0, n, m).astype(np.int32)
    dst = rng.randint(0, n, m).astype(np.int32)
    return orc.build_csr(n, src, dst, True)


class Context(object):
    pass


@pytest.fixture(scope="module")
def ctx(gb):
    c = Context()
    rng = np.random.RandomState(2024)
    rp, ci = symmetric_graph(rng, st.N, 3*st.N)
    c.S = Csr(st.N, st.N, rp, ci, rng.choice(INTS, len(ci)))
    c.M = device_matrix(gb, c.S)
    c.src = int(np.argmax(np.diff(rp)))
    return c


# ---------------------------------------------------------------------------
# 1. producer x consumer
# ---------------------------------------------------------------------------

def static_tags(p):
    return {"sparse": p in st.SPARSE_PRODUCERS, "pattern": p in st.PATTERN_PRODUCERS,
            "huge": p in st.HUGE_PRODUCERS}


@pytest.mark.gpu
@pytest.mark.parametrize("consumer", list(st.CONSUMERS))
def test_consumer_over_every_producer(gb, ctx, consumer):
    failed = []
    for p in [p for p, c in st.RUN if c == consumer]:
        try:
            op = st.PRODUCERS[p](gb, ctx, p)
            assert {k: k in op.tags for k in ("sparse", "pattern", "huge")} == \
                static_tags(p), "static tags"
            st.CONSUMERS[consumer](gb, ctx, op)
        except Exception as e:
            failed.append("%s -> %s: %s: %s" % (p, consumer, type(e).__name__, e))
    assert not failed, "\n".join(failed)


# ---------------------------------------------------------------------------
# 2. one descriptor across a sequence of calls
# ---------------------------------------------------------------------------

class Step(object):
    """knobs and scmp configure the descriptor; run(gb, desc) returns a tuple of
    arrays, want the reference's."""

    def __init__(self, name, knobs, run, want, scmp=False):
        self.name, self.knobs, self.run, self.want, self.scmp = name, knobs, run, want, scmp


KNOBS = dict(mxvmode=1, struconly=0, opreuse=0, earlyexit=0, fusedmask=0)


def configure(gb, desc, step):
    """Every knob a step may set, to the step's value or the default."""
    knobs = dict(KNOBS, switchpoint=gb.Descriptor().get_knob("switchpoint"))
    for k, v in dict(knobs, **step.knobs).items():
        desc.set_knob(k, v)
    desc.set(gb.Desc_field.GrB_MASK,
             gb.Desc_value.GrB_SCMP if step.scmp else gb.Desc_value.GrB_DEFAULT)


def densified(n, ind, val):
    return eref.densify(n, ind, val, 0)


def sequence_steps(gb):
    import test_mxv_gpu as mx
    rng = np.random.RandomState(31)
    m, k = 1500, 700
    A = mx.structure(rng, np.minimum(rng.randint(0, 25, m), k), k, "int")
    A1 = A.with_values(np.ones(A.nnz, np.float32))
    Ad, A1d = device_matrix(gb, A), device_matrix(gb, A1)
    Aint = device_matrix(gb, A.with_values(rng.randint(-5, 6, A.nnz).astype(np.int32)),
                         integer=True)
    nh = 6000
    lens = rng.randint(0, 3, nh)
    lens[:5000] = rng.randint(5, 12, 5000)
    H = mx.structure(rng, lens, nh, "int")
    Hd = device_matrix(gb, H)
    grp, gci = symmetric_graph(rng, 2000, 6000)
    gw = rng.randint(1, 9, len(gci)).astype(np.float32)
    G = device_matrix(gb, Csr(2000, 2000, grp, gci, gw))
    big = rng.choice(np.float32([0, 0, 0, 1, -3]), 40000)

    def push(M, orient, sem, f, fv, n_out, mask=None):
        def run(gb, desc):
            u = gb.Vector(M.nrows() if orient == "vxm" else M.ncols())
            u.build(np.asarray(f, np.int32), np.asarray(fv, np.float32))
            w = gb.Vector(n_out)
            mv = None if mask is None else st._dense(gb, mask)
            if orient == "vxm":
                gb.vxm(w, mv, None, sem, u, M, desc)
            else:
                gb.mxv(w, mv, None, sem, M, u, desc)
            return (w.extractTuples(),)
        return run

    steps = []

    def add_push(name, S, M, orient, sem, size, vals=None, mask=None, scmp=False,
                 struconly=False, mode=1):
        T = S if orient == "vxm" else S.T            # vxm pushes along A's rows
        f = np.sort(rng.choice(T.nrows, size, replace=False))
        fv = rng.choice(INTS, size) if vals is None else np.full(size, vals, np.float32)
        n_out = T.ncols
        if struconly:
            ind, val = st.struct_push(sem, T, f, fv, n_out, mask, scmp)
        elif mask is not None:
            ind, val = st.masked_push(sem, T, f, fv, n_out, mask, scmp)
        else:
            ind, val = ref.push(sem, T.ptr, T.ind, T.val, f, fv, n_out)
        steps.append(Step(name, dict(struconly=int(struconly), mxvmode=mode),
                          push(M, orient, sem, f, fv, n_out, mask),
                          (densified(n_out, ind, val),), scmp))
        return f

    add_push("plus vxm", A, Ad, "vxm", PLUS, 300)
    add_push("minplus mxv (grows)", A, Ad, "mxv", MINPLUS, 200)
    # every product 1 + -1 = 0: every touched word of the keyed masked push is dropped,
    # and finish() alone must put FLT_MAX back into its accumulator cells
    mask = (rng.rand(k) < 0.6).astype(np.float32)
    steps_before = len(steps)
    f0 = add_push("minplus zero products, mask (shrinks)", A1, A1d, "vxm", MINPLUS, 400,
                  vals=-1.0, mask=mask)
    add_push("minplus zero products, scmp", A1, A1d, "vxm", MINPLUS, 400, vals=-1.0,
             mask=mask, scmp=True)
    assert not steps[steps_before].want[0].any() and not steps[-1].want[0].any()
    # the same cells again, products 2: min(identity, 2) = 2
    ind, val = ref.push(MINPLUS, A1.ptr, A1.ind, A1.val, f0, np.ones(len(f0)), k)
    assert np.all(val == 2)
    steps.append(Step("minplus over the dropped cells", {},
                      push(A1d, "vxm", MINPLUS, f0, np.ones(len(f0), np.float32), k),
                      (densified(k, ind, val),)))
    add_push("maxmul mxv", A, Ad, "mxv", MAXMUL, 250)
    add_push("struct-only plus vxm", A, Ad, "vxm", PLUS, 300, struconly=True)
    add_push("plus mxv, mask", A, Ad, "mxv", PLUS, 250,
             mask=(rng.rand(m) < 0.5).astype(np.float32))
    add_push("minplus vxm", A, Ad, "vxm", MINPLUS, 300)

    # INT32: mxv / vxm refuse an INT32 A (capi.cu: GrB_DOMAIN_MISMATCH before any
    # work, so no push accumulator of another type or identity exists); the matrix
    # reduce and the vector reduce run on the same descriptor's counter cells
    def int32_run(gb, desc):
        w = st._dense(gb, np.full(m, 7, np.float32))
        u = gb.Vector(k)
        u.build(np.int32([1, 2]), np.float32([1, 1]))
        try:
            gb.mxv(w, None, None, PLUS, Aint, u, desc)
            refused = False
        except gb.GraphBLASError as e:
            refused = e.info == gb.Info.GrB_DOMAIN_MISMATCH
        total = gb.reduce(None, 0, Aint, desc)
        return (w.extractTuples(), np.float64([refused, total]))
    _, _, aval = Aint.extract_csr()
    steps.append(Step("int32 refused, int32 reduce", {}, int32_run,
                      (np.full(m, 7, np.float32), np.float64([1, aval.sum()]))))
    add_push("plus vxm after int32", A, Ad, "vxm", PLUS, 300)

    # a frontier of 5000 owning more than a third of H's entries: handed to the pull
    f = np.arange(5000)
    fv = rng.choice(INTS, 5000)
    assert H.ptr[5000] > H.nnz/3
    ind, val = ref.push(PLUS, H.ptr, H.ind, H.val, f, fv, nh)

    def handback(gb, desc):
        out = push(Hd, "vxm", PLUS, f, fv, nh)(gb, desc)
        return out + (np.float64([int(desc.lastmxv)]),)
    steps.append(Step("hand-back to the pull (grows)", dict(mxvmode=0, switchpoint=0.9),
                      handback, (densified(nh, ind, val),
                                 np.float64([int(gb.Desc_value.GrB_PULLONLY)]))))
    add_push("plus vxm over H", H, Hd, "vxm", PLUS, 3000)

    def sssp(gb, desc):
        v = gb.Vector(2000)
        gb.algorithm.sssp(v, G, 0, desc)
        return (v.extractTuples(),)
    steps.append(Step("sssp", dict(mxvmode=0), sssp, (orc.sssp(grp, gci, gw, 0),)))
    add_push("minplus vxm after sssp (shrinks)", A, Ad, "vxm", MINPLUS, 300)

    def bfs(gb, desc):
        v = gb.Vector(2000)
        gb.algorithm.bfs(v, G, 3, desc)
        return (v.extractTuples(),)
    # opreuse goes with fusedmask, as in the reference's scripts: without the fused
    # pull, the push-to-pull switch under opreuse leaves the dense frontier unwritten
    # (Vector::sparse2dense) and the generic pull reads it
    steps.append(Step("fused bfs", dict(mxvmode=0, struconly=1, opreuse=1, earlyexit=1,
                                        fusedmask=1),
                      bfs, (orc.bfs(grp, gci, 3).astype(np.float32),)))
    steps.append(Step("bfs operation by operation", dict(mxvmode=0, struconly=1),
                      bfs, (orc.bfs(grp, gci, 3).astype(np.float32),)))

    def compact_reduce(gb, desc):
        v = st._dense(gb, big)
        total = gb.reduce(None, 0, st._dense(gb, big), desc)
        v.dense2sparse(0.0, desc)
        ind, val = v.extractTuples(sparse=True)
        return (ind.astype(np.float64), val, np.float64([total]))
    want_i, want_v = eref.dense2sparse(big, 0.0)
    steps.append(Step("reduce and dense2sparse", {}, compact_reduce,
                      (want_i.astype(np.float64), want_v,
                       np.float64([big.astype(np.float64).sum()]))))
    add_push("plus vxm at the end", A, Ad, "vxm", PLUS, 300)
    add_push("minplus mxv, scmp mask, at the end", A, Ad, "mxv", MINPLUS, 250,
             mask=(rng.rand(m) < 0.5).astype(np.float32), scmp=True)
    return steps


@pytest.mark.gpu
def test_one_descriptor_across_a_sequence(gb):
    steps = sequence_steps(gb)
    shared = gb.Descriptor()
    for s in steps:
        configure(gb, shared, s)
        got = s.run(gb, shared)
        fresh = gb.Descriptor()
        configure(gb, fresh, s)
        again = s.run(gb, fresh)
        assert len(got) == len(again) == len(s.want), s.name
        for i, (g, a, w) in enumerate(zip(got, again, s.want)):
            g, a = np.asarray(g), np.asarray(a)
            for run, out in (("shared", g), ("fresh", a)):
                try:
                    st.same(out, w)
                except AssertionError as e:
                    raise AssertionError("%s, output %d, %s descriptor: %s" % (
                        s.name, i, run, e)) from e
            assert g.dtype == a.dtype and np.array_equal(g.view(np.uint8), a.view(np.uint8)), \
                "%s: the shared and the fresh descriptor differ" % s.name


# ---------------------------------------------------------------------------
# 3. matrix caches and the host mirror across in-place changes
# ---------------------------------------------------------------------------

def symmetric_pattern(S):
    T = S.T
    return np.array_equal(S.ptr, T.ptr) and np.array_equal(S.ind, T.ind)


def use_every_route(gb, C, S, where):
    """The generic pull (merge tiles or hub index), the Boolean pull (first-neighbour
    summary) and, on a symmetric pattern, the fused BFS (max-degree summary) over C,
    against the references of S; C's host CSR equals S."""
    check_csr(C, S)
    rng = np.random.RandomState(S.nnz % 1000)
    u = rng.choice(INTS, S.ncols)
    w = gb.Vector(S.nrows)
    gb.mxv(w, None, None, PLUS, C, st._dense(gb, u), gb.Descriptor(mxvmode=2))
    want, bound = ref.pull(PLUS, S.ptr, S.ind, S.val, u)
    got = w.extractTuples()
    assert np.all(np.abs(got - want) <= bound), "%s: generic pull" % where
    mk = rng.choice(np.float32([0, 1, 2.5]), S.nrows)
    ub = (rng.rand(S.ncols) < 0.2).astype(np.float32)
    desc = gb.Descriptor(mxvmode=2, fusedmask=1, earlyexit=1)
    desc.toggle(gb.Desc_field.GrB_MASK)
    w = gb.Vector(S.nrows)
    gb.mxv(w, st._dense(gb, mk), None, LOR, C, st._dense(gb, ub), desc)
    assert np.array_equal(w.extractTuples(),
                          ref.bool_pull(S.ptr, S.ind, mk, ub, 0.0, True, False)), \
        "%s: Boolean pull" % where
    if symmetric_pattern(S):
        src = int(np.argmax(np.diff(S.ptr)))
        v = gb.Vector(S.nrows)
        gb.algorithm.bfs(v, C, src, gb.Descriptor(mxvmode=0, struconly=1, opreuse=1,
                                                   earlyexit=1))
        assert np.array_equal(v.extractTuples(), orc.bfs(S.ptr, S.ind, src)
                              .astype(np.float32)), "%s: fused BFS" % where


def relabelled(S, perm):
    """S with vertex i renamed perm[i]: the same entry count, another structure."""
    rows = perm[S.rows()]
    cols = perm[S.ind]
    return csr(S.nrows, S.ncols, rows, cols, S.val, np.float32)


@pytest.mark.gpu
def test_caches_and_host_mirror_follow_every_writer(gb):
    rng = np.random.RandomState(77)
    n = 1500
    rp, ci = symmetric_graph(rng, n, 5*n)
    S = Csr(n, n, rp, ci, rng.choice(INTS, len(ci)))
    C = device_matrix(gb, S)
    desc = gb.Descriptor()
    use_every_route(gb, C, S, "adopted")

    # assign C(:, :) = B, B a relabelling of S: the same nvals, another structure
    B = relabelled(S, rng.permutation(n).astype(np.int64))
    assert B.nnz == S.nnz and not np.array_equal(B.ptr, S.ptr)
    gb.assign(C, None, None, device_matrix(gb, B), None, n, None, n, desc)
    S = B
    use_every_route(gb, C, S, "assign")

    gb.eWiseAdd(C, None, None, PLUS, C, C, desc)
    S = S.with_values(S.val*2)
    use_every_route(gb, C, S, "eWiseAdd C = C + C")
    gb.eWiseMult(C, None, None, PLUS, C, C, desc)
    S = S.with_values(S.val*S.val)
    use_every_route(gb, C, S, "eWiseMult C = C .* C")

    # value-only writers: the same arrays, new values; the host mirror must follow
    alpha = np.float32(0.85)
    C.pr_normalize(float(alpha), desc)
    outdeg, _ = eref.reduce_rows(0, S.ptr, S.val)
    S = S.with_values(eref.scale_rows(4, S.ptr, eref.scale_csr(1, S.val, alpha),
                                      outdeg.astype(np.float32)))
    use_every_route(gb, C, S, "pr_normalize")
    C.apply_uniform_random(desc, seed=5, lo=1, hi=9)
    _, _, val = C.extract_csr()
    assert np.all((val >= 1) & (val <= 9) & (val == np.round(val)))
    assert not np.array_equal(val, S.val)
    S = S.with_values(val)
    use_every_route(gb, C, S, "apply_uniform_random")

    # mxm into a reused matrix that has caches, then with C = A = B
    X = device_matrix(gb, S)
    use_every_route(gb, X, S, "before mxm")
    gb.mxm(X, None, None, PLUS, C, C, desc)
    P = Csr(n, n, *mref.mxm(PLUS, S.ptr, S.ind, S.val, S.ptr, S.ind, S.val, n))
    use_every_route(gb, X, P, "mxm into a reused C")
    gb.mxm(C, None, None, PLUS, C, C, desc)
    S = P
    use_every_route(gb, C, S, "mxm C = C * C")

    gb.transpose(C, None, None, C, desc)
    S = S.T
    use_every_route(gb, C, S, "transpose in place")

    import truss_reference
    nedges, _ = gb.algorithm.ktruss(C, C, 3, desc)
    sup, want_edges = truss_reference.ktruss(S.ptr, S.ind, 3)
    assert nedges == want_edges
    S = Csr(n, n, *truss_reference.kept_csr(S.ptr, S.ind, sup))
    S = S.with_values(S.val.astype(np.float32))
    use_every_route(gb, C, S, "ktruss out = A")

    C.tril(desc)
    keep = S.rows() >= S.ind
    S = csr(n, n, S.rows()[keep], S.ind[keep], S.val[keep], np.float32)
    use_every_route(gb, C, S, "tril")


@pytest.mark.gpu
@pytest.mark.skipif(HUB_FORCED, reason="already a child")
def test_hub_index_follows_every_writer_in_a_child():
    """The same writers with the hub thresholds at 0: the generic pulls take the hub
    kernel, whose index must be rebuilt after each."""
    env = dict(os.environ, GB200_SPMV_HUB="1", GB200_SPMV_HUB_MIN_NNZ="0",
               GB200_SPMV_HUB_MIN_PCT="0")
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider",
           os.path.abspath(__file__), "-k", "follow_every_writer and not child"]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:]
    assert " passed" in r.stdout


# ---------------------------------------------------------------------------
# 4. writing through device memory: re-adopt after writing
# ---------------------------------------------------------------------------

@pytest.mark.gpu
def test_readopt_after_writing_through_device_memory(gb, ctx):
    """INTEGRATION.md: after writing a vector's values through device_ptr or an
    adopted tensor, build_device the tensor again; the library then reads the new
    values on every route, including the ones that read a shadow or a count."""
    import torch
    n = st.N
    rng = np.random.RandomState(4)
    # a Boolean-pull result (bitmap shadow and pending count), written through
    # device_ptr, then re-adopted
    w, x = st._bits_pull(gb, ctx, rng, False, False)
    ptr = w.device_ptr()
    gb.sync()
    t = torch.as_tensor(st._Cuda(ptr, n), device="cuda")
    new = rng.choice(st.VALS, n)
    t.copy_(torch.from_numpy(new).cuda())
    torch.cuda.synchronize()
    owned = t.clone()
    w.build_device(owned)
    assert np.array_equal(w.extractTuples(), new)
    assert np.float32(gb.reduce(None, 0, w, gb.Descriptor())) == new.astype(np.float64).sum()
    assert np.array_equal(st.exported_bits(gb, w), new != 0)
    # an adopted tensor written in place, re-adopted: shadow, count and host mirror
    a = torch.from_numpy(rng.choice(np.float32([0, 1]), n)).cuda()
    v = gb.Vector(n)
    v.build_device(a)
    v.fill(1.0)                                    # bitmap shadow all ones
    assert v.extractTuples().sum() == n            # host mirror current
    y = rng.choice(st.VALS, n)
    a.copy_(torch.from_numpy(y).cuda())
    torch.cuda.synchronize()
    v.build_device(a)
    assert np.array_equal(v.extractTuples(), y)
    assert np.array_equal(st.exported_bits(gb, v), y != 0)
    four = np.full(n, 4, np.float32)
    tgt = st._dense(gb, four)
    gb.assign(tgt, v, None, 3.0, None, 0, gb.Descriptor())
    assert np.array_equal(tgt.extractTuples(), eref.assign_dense(four, y, 3.0))
    v.dense2sparse(0.0, gb.Descriptor())
    ind, val = v.extractTuples(sparse=True)
    want_i, want_v = eref.dense2sparse(y, 0.0)
    assert np.array_equal(ind, want_i) and np.array_equal(val, want_v)


@pytest.mark.gpu
def test_swap_of_an_adopted_vector_keeps_the_tensor_alive(gb):
    """Vector.swap hands the contents over, and with them the tensor the other vector
    adopted: once that vector is gone, the tensor must not be freed (and its memory
    handed to the next allocation) under the contents."""
    import gc
    import torch
    x = np.arange(st.N, dtype=np.float32)
    a = gb.Vector(st.N)
    a.build_device(torch.from_numpy(x).cuda())
    b = st._dense(gb, np.zeros(st.N, np.float32))
    b.swap(a)
    del a
    gc.collect()
    junk = [torch.full((st.N,), -1.0, device="cuda") for _ in range(4)]
    torch.cuda.synchronize()
    assert np.array_equal(b.extractTuples(), x)
    assert np.array_equal(st.exported_bits(gb, b), x != 0)
    del junk
