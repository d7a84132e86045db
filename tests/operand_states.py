"""Operands as other operations leave them behind, and the operations that read them.

A dense vector carries facts about its contents (backend/cuda/dense_vector.hpp): the
count of entries != 0, possibly still pending on the device or in the mailbox;
"contents are exactly 0/1" (a plus-reduce is then that count); a bitmap shadow that
masks and conversions read instead of the values; and "only the bitmap is current"
after the bits form of the fused Boolean pull.  Each PRODUCER below returns a vector
in one such state together with a host model of its contents, and each CONSUMER
reads a vector through one route and checks what it reads against the model.
test_operand_states_gpu.py runs every pair of RUN; EXCLUDED names the pairs that
are not run and why.  Nothing here needs a device until a producer or consumer is
called.

Quirks kept on purpose, modelled here as the code does them:
  * sparse2dense under --opreuse writes nothing: the dense array keeps what it held
    (vector.hpp Vector::sparse2dense, reference vector.hpp:344-357);
  * a masked key-value push drops entries whose value is 0 (spmspv.hpp, reference
    spmspv.hpp:203-243);
  * a struct-only push stores 1 for every entry (spmspv.hpp, reference
    spmspv.hpp:15-257), and a struct-only dense2sparse writes no values at all
    (kernels/compact.cuh DenseCompactSource): only its pattern is defined.
"""
import zlib

import numpy as np

import ewise_reference as eref
import mxv_reference as ref
from mxm_reference import FLT_MAX

N = 1003                     # not a multiple of 32: the last bitmap word is partial
VALS = np.float32([-2, -1, 0, 0, 1, 2, 3])
PLUS = 1
LOR, CLESS_PLUS, NE_PLUS, CLESS_LESS = 0, 9, 12, 15
MONOID_NAMES = ["plus", "mul", "min", "max", "or", "and", "gt", "lt", "ne"]


class Operand(object):
    """A vector and its model.  x: the values extractTuples() reads (a sparse vector
    densified with 0).  ind / val: a sparse vector's stored entries (val None when
    only the pattern is defined).  tags: what the state is."""

    def __init__(self, v, x=None, ind=None, val=None, tags=()):
        self.v = v
        self.ind = None if ind is None else np.asarray(ind, np.int32)
        self.val = None if val is None else np.asarray(val, np.float32)
        if x is None and ind is not None:
            x = np.zeros(N, np.float32)
            if val is not None:
                x[self.ind] = self.val
        self.x = None if x is None else np.asarray(x, np.float32)
        self.tags = set(tags) | ({"sparse"} if ind is not None else {"dense"})
        if val is None and ind is not None:
            self.tags.add("pattern")
        if self.x is not None and np.any(np.abs(self.x) >= 2.0**24):
            self.tags.add("huge")

    @property
    def sparse(self):
        return "sparse" in self.tags


# ---------------------------------------------------------------------------
# host models of the quirks (checked without a device in test_operand_states_cpu.py)
# ---------------------------------------------------------------------------

def opreuse_sparse2dense(dense_before):
    """sparse2dense under --opreuse: the dense array is left as it was."""
    return np.asarray(dense_before, np.float32).copy()


def masked_push(semiring, S, f, fv, n, mask, scmp=False):
    """A masked key-value push: the reference push with the zeros dropped."""
    ind, val = ref.push(semiring, S.ptr, S.ind, S.val, f, fv, n, mask, scmp)
    return ind[val != 0], val[val != 0]


def struct_push(semiring, S, f, fv, n, mask=None, scmp=False):
    """A struct-only push: the reference's pattern, every value 1."""
    ind, _ = ref.push(semiring, S.ptr, S.ind, S.val, f, fv, n, mask, scmp)
    return ind, np.ones(len(ind), np.float32)


def mul_reduce_defined(x):
    """A Multiplies fold of float32 x has one answer in every order when every value
    is 0 or a power of two and no partial product can leave the float32 range."""
    x = np.asarray(x, np.float32)
    nz = x[x != 0]
    m, _ = np.frexp(np.abs(nz))
    if not np.all(m == 0.5):
        return False
    return float(np.abs(np.log2(np.abs(nz))).sum()) < 120


def reduce_launches(op, monoid):
    """Kernel launches of reduce(monoid, v) on a dense operand, or None where the code
    leaves the count open.  A plus-reduce of a vector the fused Boolean pull wrote
    reads the count that pull left (mailbox or device cell, no launch); after dup the
    count is gone but "0/1" is kept, so one countNonIdentityKernel runs
    (reduce.hpp reduceDense, dense_vector.hpp computeNnz)."""
    if monoid != 0 or op.sparse:
        return None
    if "counted" in op.tags:
        return 0
    if "zero_one" in op.tags:
        return 1
    return None


# ---------------------------------------------------------------------------
# producers
# ---------------------------------------------------------------------------

def _rng(name):
    return np.random.RandomState(zlib.crc32(name.encode()) & 0x7fffffff)


def _dense(gb, x):
    v = gb.Vector(len(x))
    v.build(np.asarray(x, np.float32))
    return v


def _sparse(gb, ind, val):
    v = gb.Vector(N)
    v.build(np.asarray(ind, np.int32), np.asarray(val, np.float32))
    return v


def _pattern(rng, k=None):
    k = N//5 if k is None else k
    return np.sort(rng.choice(N, k, replace=False)).astype(np.int32)


def _mask01(rng):
    return (rng.rand(N) < 0.4).astype(np.float32)


def _shadowed(gb, x01):
    """A 0/1 vector whose bitmap shadow is current: fill(0), then a sparse-mask
    assign of 1 (both keep the shadow)."""
    m = gb.Vector(N)
    m.fill(0.0)
    nz = np.nonzero(x01)[0].astype(np.int32)
    if len(nz):
        gb.assign(m, _sparse(gb, nz, np.ones(len(nz))), None, 1.0, None, 0, gb.Descriptor())
    return m


def p_build_dense(gb, c, name):
    x = _rng(name).choice(VALS, N)
    return Operand(_dense(gb, x), x)


def p_build_sparse(gb, c, name):
    rng = _rng(name)
    ind = _pattern(rng)
    val = rng.choice(VALS, len(ind))
    return Operand(_sparse(gb, ind, val), ind=ind, val=val)


def p_fill(value):
    def make(gb, c, name):
        v = gb.Vector(N)
        v.fill(value)
        return Operand(v, np.full(N, value, np.float32))
    return make


def p_assign(mask_kind, scmp):
    """fill(0), then w<mask> = 2 (scmp: where the mask is 0)."""
    def make(gb, c, name):
        rng = _rng(name)
        desc = gb.Descriptor()
        if scmp:
            desc.toggle(gb.Desc_field.GrB_MASK)
        w = gb.Vector(N)
        w.fill(0.0)
        zeros = np.zeros(N, np.float32)
        if mask_kind == "sparse":
            m_ind = _pattern(rng)
            m_val = rng.choice(np.float32([0, 1]), len(m_ind))
            gb.assign(w, _sparse(gb, m_ind, m_val), None, 2.0, None, 0, desc)
            # every stored index is written; GrB_SCMP is refused and writes nothing
            x = zeros if scmp else eref.assign_dense_sparse_mask(zeros, m_ind, 2.0)
        elif mask_kind == "shadow":
            mk = _mask01(rng)
            gb.assign(w, _shadowed(gb, mk), None, 2.0, None, 0, desc)
            x = eref.assign_dense(zeros, mk, 2.0, scmp)
        else:
            mk = rng.choice(np.float32([0, -0.0, 1, 2.5]), N)
            gb.assign(w, _dense(gb, mk), None, 2.0, None, 0, desc)
            x = eref.assign_dense(zeros, mk, 2.0, scmp)
        return Operand(w, x)
    return make


def _bits_pull(gb, c, rng, earlyexit, opreuse):
    """BFS-shaped: w<!visited> = A (or.and) frontier, the bits form."""
    visited = _mask01(rng)
    u = (rng.rand(N) < 0.1).astype(np.float32)
    desc = gb.Descriptor(mxvmode=2, fusedmask=1, earlyexit=int(earlyexit),
                         opreuse=int(opreuse))
    desc.toggle(gb.Desc_field.GrB_MASK)
    w = gb.Vector(N)
    gb.mxv(w, _shadowed(gb, visited), None, LOR, c.M, _dense(gb, u), desc)
    assert desc.lastmxv == gb.Desc_value.GrB_PULLONLY
    return w, ref.bool_pull(c.S.ptr, c.S.ind, visited, u, 0.0, True, opreuse)


def p_bool_bits(earlyexit, opreuse):
    def make(gb, c, name):
        w, x = _bits_pull(gb, c, _rng(name), earlyexit, opreuse)
        return Operand(w, x, tags=("counted", "zero_one"))
    return make


def p_bool_value(semiring):
    def make(gb, c, name):
        rng = _rng(name)
        mk = rng.choice(np.float32([0, -0.0, 2.5, -1, FLT_MAX]), N)
        u = rng.choice(np.float32([FLT_MAX, FLT_MAX, 0, -0.0, 1, -2]), N)
        desc = gb.Descriptor(mxvmode=2, fusedmask=1)
        w = gb.Vector(N)
        gb.mxv(w, _dense(gb, mk), None, semiring, c.M, _dense(gb, u), desc)
        assert desc.lastmxv == gb.Desc_value.GrB_PULLONLY
        return Operand(w, ref.bool_pull(c.S.ptr, c.S.ind, mk, u, FLT_MAX, False, False),
                       tags=("counted", "zero_one"))
    return make


def p_pull(masked, accum):
    def make(gb, c, name):
        rng = _rng(name)
        u = rng.choice(VALS, N)
        mk = rng.choice(np.float32([0, -0.0, 1, -3]), N) if masked else None
        w_old = rng.choice(VALS, N) if accum else None
        w = _dense(gb, w_old) if accum else gb.Vector(N)
        gb.mxv(w, None if mk is None else _dense(gb, mk), "accum" if accum else None, PLUS,
               c.M, _dense(gb, u), gb.Descriptor(mxvmode=2))
        want, _ = ref.pull(PLUS, c.S.ptr, c.S.ind, c.S.val, u, mask=mk, w_old=w_old)
        return Operand(w, want.astype(np.float32))
    return make


def p_push(kind):
    """vxm over A (push along its CSR rows) from a sparse frontier."""
    def make(gb, c, name):
        rng = _rng(name)
        f = _pattern(rng, N//8)
        fv = rng.choice(VALS, len(f))
        desc = gb.Descriptor(mxvmode=1, struconly=int(kind == "struct"))
        mk = _mask01(rng) if kind == "masked" else None
        w = gb.Vector(N)
        gb.vxm(w, None if mk is None else _dense(gb, mk), None, PLUS, _sparse(gb, f, fv),
               c.M, desc)
        assert desc.lastmxv == gb.Desc_value.GrB_PUSHONLY
        if kind == "struct":
            ind, val = struct_push(PLUS, c.S, f, fv, N)
        elif kind == "masked":
            ind, val = masked_push(PLUS, c.S, f, fv, N, mk)
        else:
            ind, val = ref.push(PLUS, c.S.ptr, c.S.ind, c.S.val, f, fv, N)
        return Operand(w, ind=ind, val=val)
    return make


def p_sparse2dense(identity, struconly):
    def make(gb, c, name):
        rng = _rng(name)
        ind = _pattern(rng)
        val = rng.choice(VALS, len(ind))
        v = _sparse(gb, ind, val)
        v.sparse2dense(identity, gb.Descriptor(struconly=struconly))
        return Operand(v, eref.sparse2dense(N, ind, val, identity, bool(struconly)))
    return make


def p_sparse2dense_opreuse(gb, c, name):
    """fill(5); a push turns w sparse; sparse2dense under opreuse: still all 5."""
    rng = _rng(name)
    w = gb.Vector(N)
    w.fill(5.0)
    f = _pattern(rng, 40)
    gb.vxm(w, None, None, PLUS, _sparse(gb, f, np.ones(len(f))), c.M,
           gb.Descriptor(mxvmode=1))
    assert w.getStorage() == gb.Storage.GrB_SPARSE
    w.sparse2dense(0.0, gb.Descriptor(opreuse=1))
    return Operand(w, opreuse_sparse2dense(np.full(N, 5, np.float32)))


def p_dense2sparse(identity, struconly):
    def make(gb, c, name):
        x = _rng(name).choice(VALS, N)
        if identity != 0:
            x = np.where(x == 0, FLT_MAX, x).astype(np.float32)
        v = _dense(gb, x)
        v.dense2sparse(identity, gb.Descriptor(struconly=struconly))
        ind, val = eref.dense2sparse(x, identity)
        return Operand(v, ind=ind, val=None if struconly else val)
    return make


def p_dense2sparse_bits(struconly):
    """The bits form of the Boolean pull compacted from its bitmap."""
    def make(gb, c, name):
        w, x = _bits_pull(gb, c, _rng(name), True, False)
        w.dense2sparse(0.0, gb.Descriptor(struconly=struconly))
        ind, val = eref.dense2sparse(x, 0.0)
        return Operand(w, ind=ind, val=None if struconly else val)
    return make


def p_set_after_fill(gb, c, name):
    v = gb.Vector(N)
    v.fill(0.0)
    x = np.zeros(N, np.float32)
    for k, val in ((5, 3.0), (N - 1, -2.0), (64, 1.0)):
        v.setElement(val, k)
        x[k] = val
    return Operand(v, x)


def p_set_after_bits(gb, c, name):
    w, x = _bits_pull(gb, c, _rng(name), False, False)
    one = int(np.nonzero(x)[0][0])
    zero = int(np.nonzero(x == 0)[0][-1])
    w.setElement(2.0, zero)
    w.setElement(0.0, one)
    x = x.copy()
    x[zero], x[one] = 2.0, 0.0
    return Operand(w, x)


def p_dup(base):
    def make(gb, c, name):
        src = PRODUCERS[base](gb, c, base)
        g = gb.Vector(N)
        g.dup(src.v)
        tags = src.tags - {"counted"}
        return Operand(g, src.x, src.ind, src.val, tags)
    return make


def p_swap(base):
    def make(gb, c, name):
        src = PRODUCERS[base](gb, c, base)
        other = (_sparse(gb, [0, 7], [9, 9]) if src.sparse else
                 _dense(gb, np.full(N, 9, np.float32)))
        other.swap(src.v)
        return Operand(other, src.x, src.ind, src.val, src.tags)
    return make


def p_adopt(gb, c, name):
    import torch
    x = _rng(name).choice(VALS, N)
    v = gb.Vector(N)
    v.build_device(torch.from_numpy(x).cuda())
    return Operand(v, x)


def p_reduce_rows(gb, c, name):
    w = gb.Vector(N)
    gb.reduce(None, 0, c.M, gb.Descriptor(), out=w)
    want, _ = eref.reduce_rows(0, c.S.ptr, c.S.val)
    return Operand(w, want.astype(np.float32))


def p_ewise_add(gb, c, name):
    rng = _rng(name)
    a, b = rng.choice(VALS, N), rng.choice(VALS, N)
    w = gb.Vector(N)
    gb.eWiseAdd(w, None, None, PLUS, _dense(gb, a), _dense(gb, b), gb.Descriptor())
    return Operand(w, eref.ewise_add_dense(PLUS, a, b))


def p_extract(gb, c, name):
    rng = _rng(name)
    u = rng.choice(VALS, N)
    rows = rng.permutation(N).astype(np.int32)
    w = gb.Vector(N)
    gb.extract(w, None, None, _dense(gb, u), rows, N, None, 0, gb.Descriptor())
    return Operand(w, u[rows])


def p_bfs(gb, c, name):
    import oracle_binding as orc
    v = gb.Vector(N)
    gb.algorithm.bfs(v, c.M, c.src, gb.Descriptor(mxvmode=0, struconly=1, opreuse=1,
                                                   earlyexit=1))
    return Operand(v, orc.bfs(c.S.ptr, c.S.ind, c.src).astype(np.float32))


def p_cc(gb, c, name):
    import support
    v = gb.Vector(N)
    gb.algorithm.cc(v, c.M, gb.Descriptor())
    return Operand(v, support.components(N, c.S.ptr, c.S.ind)[0].astype(np.float32))


PRODUCERS = {
    "build_dense": p_build_dense,
    "build_sparse": p_build_sparse,
    "fill_0": p_fill(0.0),
    "fill_1": p_fill(1.0),
    "fill_2.5": p_fill(2.5),
}
for _kind in ("shadow", "values", "sparse"):
    for _scmp in (False, True):
        PRODUCERS["assign_%s_scmp%d" % (_kind, _scmp)] = p_assign(_kind, _scmp)
for _ee in (0, 1):
    for _or in (0, 1):
        PRODUCERS["bool_bits_ee%d_or%d" % (_ee, _or)] = p_bool_bits(_ee, _or)
for _sem in (CLESS_PLUS, NE_PLUS, CLESS_LESS):
    PRODUCERS["bool_value_%d" % _sem] = p_bool_value(_sem)
PRODUCERS.update({
    "pull": p_pull(False, False),
    "pull_mask": p_pull(True, False),
    "pull_accum": p_pull(False, True),
    "pull_mask_accum": p_pull(True, True),
    "push_keyed": p_push("keyed"),
    "push_keyed_masked": p_push("masked"),
    "push_struct": p_push("struct"),
    "sparse2dense_opreuse": p_sparse2dense_opreuse,
})
for _id, _idn in ((0.0, "0"), (float(FLT_MAX), "fltmax")):
    for _so in (0, 1):
        PRODUCERS["sparse2dense_%s_so%d" % (_idn, _so)] = p_sparse2dense(_id, _so)
        PRODUCERS["dense2sparse_%s_so%d" % (_idn, _so)] = p_dense2sparse(_id, _so)
for _so in (0, 1):
    PRODUCERS["dense2sparse_bits_so%d" % _so] = p_dense2sparse_bits(_so)
PRODUCERS.update({
    "set_after_fill": p_set_after_fill,
    "set_after_bits": p_set_after_bits,
    "adopt": p_adopt,
    "reduce_rows": p_reduce_rows,
    "ewise_add": p_ewise_add,
    "extract": p_extract,
    "bfs": p_bfs,
    "cc": p_cc,
})
# dup and swap of every kind of state
STATES = ["build_dense", "build_sparse", "fill_1", "assign_shadow_scmp0",
          "assign_values_scmp0", "bool_bits_ee1_or0", "bool_value_9", "push_keyed",
          "push_struct", "sparse2dense_0_so1", "set_after_bits", "adopt"]
for _b in STATES:
    PRODUCERS["dup_" + _b] = p_dup(_b)
    PRODUCERS["swap_" + _b] = p_swap(_b)

# Tags a producer's operand carries, without running it (for the coverage table).
SPARSE_PRODUCERS = {"build_sparse", "push_keyed", "push_keyed_masked", "push_struct",
                    "dense2sparse_0_so0", "dense2sparse_0_so1", "dense2sparse_fltmax_so0",
                    "dense2sparse_fltmax_so1", "dense2sparse_bits_so0",
                    "dense2sparse_bits_so1"} | \
    {p + b for p in ("dup_", "swap_") for b in ("build_sparse", "push_keyed", "push_struct")}
PATTERN_PRODUCERS = {"dense2sparse_0_so1", "dense2sparse_fltmax_so1", "dense2sparse_bits_so1"}
HUGE_PRODUCERS = {"sparse2dense_fltmax_so0", "sparse2dense_fltmax_so1"}


# ---------------------------------------------------------------------------
# consumers
# ---------------------------------------------------------------------------

class _Cuda(object):
    """A device array wrapped for torch.as_tensor (no copy)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4",
                                         "data": (ptr, False), "version": 2}


def same(got, want):
    """Equal entry by entry, NaN equal to NaN, -0 equal to +0."""
    got = np.atleast_1d(np.asarray(got, np.float32))
    want = np.atleast_1d(np.asarray(want, np.float32))
    ok = (got == want) | (np.isnan(got) & np.isnan(want))
    assert got.shape == want.shape and ok.all(), \
        "%d of %d differ, first at %d: got %r want %r" % (
            int((~ok).sum()), len(ok), int(np.argmin(ok)), got[np.argmin(ok)],
            want[np.argmin(ok)])


def refused(gb, info, call):
    try:
        call()
    except gb.GraphBLASError as e:
        assert e.info == info, e.info
        return
    raise AssertionError("not refused")


def exported_bits(gb, v):
    import ctypes as C
    import torch
    bits = torch.zeros((N + 31)//32 + 1, dtype=torch.int32, device="cuda")
    assert gb.api._lib.load().gb200_vector_export_bits(
        v._h, C.c_void_p(bits.data_ptr()), None) == 0
    words = bits.cpu().numpy().view(np.uint32)[:(N + 31)//32]
    got = np.unpackbits(words.view(np.uint8), bitorder="little")
    assert not got[N:].any(), "bits past the end"
    return got[:N].astype(bool)


def c_extract_dense(gb, c, op):
    same(op.v.extractTuples(), op.x)


def c_extract_sparse(gb, c, op):
    if not op.sparse:
        refused(gb, gb.Info.GrB_INVALID_OBJECT, lambda: op.v.extractTuples(sparse=True))
        return
    ind, val = op.v.extractTuples(sparse=True)
    assert np.array_equal(ind, op.ind)
    if op.val is not None:
        same(val, op.val)


def c_extract_into(gb, c, op):
    out = np.full(N, -7, np.float32)
    op.v.extract_into(out)
    same(out, op.x)


def c_device_ptr(gb, c, op):
    if op.sparse:
        refused(gb, gb.Info.GrB_INVALID_OBJECT, op.v.device_ptr)
        return
    import torch
    ptr = op.v.device_ptr()
    gb.sync()
    same(torch.as_tensor(_Cuda(ptr, N), device="cuda").cpu().numpy(), op.x)


def c_bits(gb, c, op):
    got = exported_bits(gb, op.v)
    want = np.isin(np.arange(N), op.ind) if op.sparse else op.x != 0
    assert np.array_equal(got, want), "bitmap differs at %d" % int(np.argmax(got != want))


def c_reduce(monoid):
    def consume(gb, c, op):
        vals = op.val if op.sparse else op.x
        if monoid == 1 and not mul_reduce_defined(vals):
            return
        from support import launch_count
        before = launch_count(gb)
        got = np.float32(gb.reduce(None, monoid, op.v, gb.Descriptor()))
        launches = launch_count(gb) - before
        want, bound = eref.reduce(monoid, vals)
        if bound is None:
            same(got, want)
        elif np.isinf(np.float32(want)):
            assert got == np.float32(want), (got, want)
        else:
            assert abs(float(got) - want) <= bound, (got, want)
        expected = reduce_launches(op, monoid)
        if expected is not None:
            assert launches == expected, (launches, expected)
    return consume


def _other(name):
    return _rng("other " + name).choice(VALS, N)


def c_ewise_add_other(gb, c, op):
    d = _other("add")
    w = gb.Vector(N)
    gb.eWiseAdd(w, None, None, PLUS, op.v, _dense(gb, d), gb.Descriptor())
    want = (eref.ewise_add_sparse_dense(PLUS, op.ind, op.val, d) if op.sparse else
            eref.ewise_add_dense(PLUS, op.x, d))
    same(w.extractTuples(), want)


def c_ewise_add_as_w(gb, c, op):
    d = _other("add w")
    gb.eWiseAdd(op.v, None, None, PLUS, op.v, _dense(gb, d), gb.Descriptor())
    want = (eref.ewise_add_aliased_sparse(PLUS, N, op.ind, op.val, d, True) if op.sparse
            else eref.ewise_add_dense(PLUS, op.x, d))
    same(op.v.extractTuples(), want)


def c_ewise_add_self(gb, c, op):
    gb.eWiseAdd(op.v, None, None, PLUS, op.v, op.v, gb.Descriptor())
    same(op.v.extractTuples(), eref.ewise_add_dense(PLUS, op.x, op.x))


def c_ewise_mult_other(gb, c, op):
    d = _other("mult")
    w = gb.Vector(N)
    gb.eWiseMult(w, None, None, PLUS, op.v, _dense(gb, d), gb.Descriptor())
    if op.sparse:
        ind, val = eref.ewise_mult_sparse_dense(PLUS, op.ind, op.val, d)
        want = eref.densify(N, ind, val, 0)
    else:
        want = eref.ewise_mult_dense(PLUS, op.x, d)
    same(w.extractTuples(), want)


def c_ewise_mult_self(gb, c, op):
    gb.eWiseMult(op.v, None, None, PLUS, op.v, op.v, gb.Descriptor())
    same(op.v.extractTuples(), eref.ewise_mult_dense(PLUS, op.x, op.x))


def c_assign_mask(scmp):
    """w<v> = 3 into a filled w (bitmap shadow current) and into a built one (none);
    either way w's shadow must equal its values afterwards."""
    def consume(gb, c, op):
        desc = gb.Descriptor()
        if scmp:
            desc.toggle(gb.Desc_field.GrB_MASK)
        four = np.full(N, 4, np.float32)
        if op.sparse:
            want = four if scmp else eref.assign_dense_sparse_mask(four, op.ind, 3.0)
        else:
            want = eref.assign_dense(four, op.x, 3.0, scmp)
        for filled in (True, False):
            if filled:
                w = gb.Vector(N)
                w.fill(4.0)
            else:
                w = _dense(gb, four)
            gb.assign(w, op.v, None, 3.0, None, 0, desc)
            same(w.extractTuples(), want)
            assert np.array_equal(exported_bits(gb, w), want != 0)
    return consume


def c_gather(gb, c, op):
    idx = _rng("gather").permutation(N).astype(np.float32)
    w, iv, desc = _dense(gb, np.zeros(N, np.float32)), _dense(gb, idx), gb.Descriptor()
    assert gb.api._lib.load().gb200_extract_gather(w._h, op.v._h, iv._h, desc._h) == 0
    same(w.extractTuples(), op.x[idx.astype(np.int64)])


def c_scatter(gb, c, op):
    idx = _rng("scatter").permutation(N).astype(np.float32)
    w, iv, desc = _dense(gb, np.zeros(N, np.float32)), _dense(gb, idx), gb.Descriptor()
    assert gb.api._lib.load().gb200_assign_scatter(w._h, op.v._h, iv._h, desc._h) == 0
    want = np.zeros(N, np.float32)
    want[idx.astype(np.int64)] = op.x
    same(w.extractTuples(), want)


def c_mxv_u_pull(gb, c, op):
    w = gb.Vector(N)
    desc = gb.Descriptor(mxvmode=2)
    gb.mxv(w, None, None, PLUS, c.M, op.v, desc)
    assert desc.lastmxv == gb.Desc_value.GrB_PULLONLY
    want, _ = ref.pull(PLUS, c.S.ptr, c.S.ind, c.S.val, op.x)
    same(w.extractTuples(), want)


def c_vxm_u_push(gb, c, op):
    w = gb.Vector(N)
    desc = gb.Descriptor(mxvmode=1)
    gb.vxm(w, None, None, PLUS, op.v, c.M, desc)
    assert desc.lastmxv == gb.Desc_value.GrB_PUSHONLY
    if op.sparse:
        f, fv = op.ind, op.val
    else:
        f = np.nonzero(op.x)[0]
        fv = op.x[f]
    ind, val = ref.push(PLUS, c.S.ptr, c.S.ind, c.S.val, f, fv, N)
    same(w.extractTuples(), eref.densify(N, ind, val, 0))


def c_mxv_mask_pull(gb, c, op):
    u = _other("pull u")
    w = gb.Vector(N)
    call = lambda: gb.mxv(w, op.v, None, PLUS, c.M, _dense(gb, u), gb.Descriptor(mxvmode=2))
    if op.sparse:
        refused(gb, gb.Info.GrB_NOT_IMPLEMENTED, call)
        return
    call()
    want, _ = ref.pull(PLUS, c.S.ptr, c.S.ind, c.S.val, u, mask=op.x)
    same(w.extractTuples(), want)


def c_vxm_mask_push(gb, c, op):
    rng = _rng("push frontier")
    f = _pattern(rng, N//8)
    fv = rng.choice(VALS, len(f))
    w = gb.Vector(N)
    call = lambda: gb.vxm(w, op.v, None, PLUS, _sparse(gb, f, fv), c.M,
                          gb.Descriptor(mxvmode=1))
    if op.sparse:
        refused(gb, gb.Info.GrB_NOT_IMPLEMENTED, call)
        return
    call()
    ind, val = masked_push(PLUS, c.S, f, fv, N, op.x)
    got_i, got_v = w.extractTuples(sparse=True)
    assert np.array_equal(got_i, ind)
    same(got_v, val)


def c_mxv_w_accum(gb, c, op):
    u = _other("accum u")
    gb.mxv(op.v, None, "accum", PLUS, c.M, _dense(gb, u), gb.Descriptor(mxvmode=2))
    want, _ = ref.pull(PLUS, c.S.ptr, c.S.ind, c.S.val, u, w_old=op.x)
    same(op.v.extractTuples(), want)


def c_dense2sparse(gb, c, op):
    desc = gb.Descriptor()
    if op.sparse:
        refused(gb, gb.Info.GrB_INVALID_OBJECT, lambda: op.v.dense2sparse(0.0, desc))
        return
    op.v.dense2sparse(0.0, desc)
    ind, val = op.v.extractTuples(sparse=True)
    want_i, want_v = eref.dense2sparse(op.x, 0.0)
    assert np.array_equal(ind, want_i)
    same(val, want_v)


def _mis_want(c, x):
    import greedy_oracle
    member, size, _ = greedy_oracle.mis(c.S.ptr, c.S.ind, 3,
                                        candidates=(x != 0).astype(np.int32))
    return member.astype(np.float32), size


def c_mis_candidates(gb, c, op):
    out = gb.Vector(N)
    k, _ = gb.algorithm.mis(out, c.M, 3, gb.Descriptor(), candidates=op.v)
    want, size = _mis_want(c, op.x)
    assert k == size
    same(out.extractTuples(), want)


def c_mis_self(gb, c, op):
    k, _ = gb.algorithm.mis(op.v, c.M, 3, gb.Descriptor(), candidates=op.v)
    want, size = _mis_want(c, op.x)
    assert k == size
    same(op.v.extractTuples(), want)


def c_lgc_sweep(gb, c, op):
    import lgc_reference
    cl = gb.Vector(N)
    size, phi, _ = gb.algorithm.lgc_sweep(cl, op.v, c.M, gb.Descriptor())
    want_cl, want_size, want_phi = lgc_reference.sweep(c.S.ptr, c.S.ind, op.x)
    assert size == want_size
    assert phi == want_phi or (np.isnan(phi) and np.isnan(want_phi))
    same(cl.extractTuples(), want_cl)


CONSUMERS = {
    "extract_dense": c_extract_dense,
    "extract_sparse": c_extract_sparse,
    "extract_into": c_extract_into,
    "device_ptr": c_device_ptr,
    "bits": c_bits,
}
for _m, _name in enumerate(MONOID_NAMES):
    CONSUMERS["reduce_" + _name] = c_reduce(_m)
CONSUMERS.update({
    "ewise_add_other": c_ewise_add_other,
    "ewise_add_as_w": c_ewise_add_as_w,
    "ewise_add_self": c_ewise_add_self,
    "ewise_mult_other": c_ewise_mult_other,
    "ewise_mult_self": c_ewise_mult_self,
    "assign_mask": c_assign_mask(False),
    "assign_mask_scmp": c_assign_mask(True),
    "gather": c_gather,
    "scatter": c_scatter,
    "mxv_u_pull": c_mxv_u_pull,
    "vxm_u_push": c_vxm_u_push,
    "mxv_mask_pull": c_mxv_mask_pull,
    "vxm_mask_push": c_vxm_mask_push,
    "mxv_w_accum": c_mxv_w_accum,
    "dense2sparse": c_dense2sparse,
    "mis_candidates": c_mis_candidates,
    "mis_self": c_mis_self,
    "lgc_sweep": c_lgc_sweep,
})

# ---------------------------------------------------------------------------
# the table: every pair runs except these
# ---------------------------------------------------------------------------

REASONS = {
    "order": "the fold of a non-associative monoid depends on the grid; "
             "ewise_reference.reduce defines it on empty input only",
    "pattern": "a struct-only dense2sparse writes no values: only the pattern is defined",
    "dense_only": "gather and scatter take dense float vectors (graphblast_b200.h)",
    "two_sparse": "eWise of a sparse vector with itself: both operands sparse, a route "
                  "ewise_reference.py does not define",
    "sparse_w": "mxv_reference.pull accumulates into a dense w only",
    "huge": "FLT_MAX entries: products and sums leave the exactly representable range",
}
VALUE_CONSUMERS = {"extract_dense", "extract_into", "ewise_add_other", "ewise_add_as_w",
                   "ewise_mult_other", "mxv_u_pull", "vxm_u_push", "mis_candidates",
                   "mis_self", "lgc_sweep", "gather", "scatter", "mxv_w_accum"} | \
    {"reduce_" + m for m in MONOID_NAMES}
MXV_CONSUMERS = {"mxv_u_pull", "vxm_u_push", "mxv_w_accum"}


def exclusion(p, c):
    """The reason pair (producer p, consumer c) is not run, or None."""
    if c in ("reduce_gt", "reduce_lt", "reduce_ne"):
        return "order"
    if p in PATTERN_PRODUCERS and c in VALUE_CONSUMERS:
        return "pattern"
    if p in SPARSE_PRODUCERS:
        if c in ("gather", "scatter"):
            return "dense_only"
        if c in ("ewise_add_self", "ewise_mult_self"):
            return "two_sparse"
        if c == "mxv_w_accum":
            return "sparse_w"
    if p in HUGE_PRODUCERS and c in MXV_CONSUMERS:
        return "huge"
    return None


ALL_PAIRS = [(p, c) for p in PRODUCERS for c in CONSUMERS]
EXCLUDED = {pc: exclusion(*pc) for pc in ALL_PAIRS if exclusion(*pc) is not None}
RUN = [pc for pc in ALL_PAIRS if pc not in EXCLUDED]

# What the table must hold: the producers and consumers operations leave behind.
REQUIRED_PRODUCERS = [
    "build_dense", "build_sparse", "fill_0", "fill_1", "fill_2.5",
    "assign_shadow_scmp0", "assign_shadow_scmp1", "assign_values_scmp0",
    "assign_values_scmp1", "assign_sparse_scmp0", "assign_sparse_scmp1",
    "bool_bits_ee0_or0", "bool_bits_ee0_or1", "bool_bits_ee1_or0", "bool_bits_ee1_or1",
    "bool_value_9", "bool_value_12", "bool_value_15",
    "pull", "pull_mask", "pull_accum", "push_keyed", "push_keyed_masked", "push_struct",
    "sparse2dense_0_so0", "sparse2dense_0_so1", "sparse2dense_fltmax_so0",
    "sparse2dense_fltmax_so1", "sparse2dense_opreuse",
    "dense2sparse_0_so0", "dense2sparse_0_so1", "dense2sparse_fltmax_so0",
    "dense2sparse_fltmax_so1", "dense2sparse_bits_so0", "dense2sparse_bits_so1",
    "set_after_fill", "set_after_bits", "adopt", "reduce_rows", "ewise_add", "extract",
    "bfs", "cc"] + ["dup_" + s for s in STATES] + ["swap_" + s for s in STATES]
REQUIRED_CONSUMERS = list(CONSUMERS)
