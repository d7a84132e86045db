"""eWiseAdd, eWiseMult, assign, reduce and the vector conversions entry by entry on
every storage route, against ewise_reference.py.

Values: integers in -8..8 (every route bit-exact), arbitrary floats of both signs
(plus-folds within the float64 bound of ewise_reference.reduce), and the
identities themselves (0, 1, FLT_MAX, FLT_MIN), so that every short-circuit and
every "drop entries equal to" rule fires.  Signed zeros compare equal (==): min
and max of +0.0 and -0.0 may return either.

Designed lengths (test_ewise_reference_cpu.py checks them against the kernels):
  value compaction  VALUE_CTA = COMPACT_NT * 8 = 2048 elements a CTA;
                    VALUE_CHUNKED: more than COMPACT_NT CTAs, so the last CTA of
                    the count pass scans the block counts in chunks
  bitmap compaction BITS_CTA = COMPACT_NT * 4 words * 32 = 32768 elements a CTA;
                    BITS_CHUNKED likewise
  reduce            the grid stops growing at REDUCE_NT * 4 * SMs elements and
                    strides beyond
Lengths that do not match are run on vectors adopted from longer tensors whose
tail holds a sentinel: an overrun lands inside the tensor, and shows there.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":
    sys.path.insert(0, ROOT)

import ewise_reference as ref  # noqa: E402
import mxm_reference as mref  # noqa: E402
from support import device_matrix, gb, make_matrix, ragged_graph, same  # noqa: E402

COMPACT_NT = 256
VALUE_CTA = COMPACT_NT*8
BITS_CTA = COMPACT_NT*4*32
REDUCE_NT = 256
GRID_CTAS_PER_SM = 8
REDUCE_CTAS_PER_SM = 4
VALUE_CHUNKED = 600_001
BITS_CHUNKED = 9_000_001
LENGTHS = [1, 7, 8, 9, 31, 32, 33, VALUE_CTA - 1, VALUE_CTA, VALUE_CTA + 1]
BIG_LENGTHS = [BITS_CTA - 1, BITS_CTA, BITS_CTA + 1, VALUE_CHUNKED, BITS_CHUNKED]
SPARSE_LENGTHS = [1, 33, VALUE_CTA + 1, BITS_CTA + 1]
ROW_LENGTHS = [0, 1, 31, 32, 33, 5000, 0, 0, 0, 64, 65, 7, 0, 2, 5000, 1]

FLT_MAX, FLT_MIN = mref.FLT_MAX, mref.FLT_MIN
IDENTITIES = np.float32([0, 1, FLT_MAX, FLT_MIN])
SENTINEL = np.uint32(0x5EA5A5A5)
DIM_MISMATCH = 6


def reduce_edge(sms):
    return REDUCE_NT*REDUCE_CTAS_PER_SM*sms


def reduce_lengths(sms):
    e = reduce_edge(sms)
    return [e - 1, e, e + 1]


def values(rng, regime, n):
    if regime == "int":
        return rng.randint(-8, 9, n).astype(np.float32)
    if regime == "float":
        sign = np.where(rng.rand(n) < 0.5, -1, 1)
        return (sign*rng.uniform(0.5, 2.0, n)*2.0**rng.randint(-3, 4, n)).astype(np.float32)
    x = rng.randint(-8, 9, n).astype(np.float32)
    pick = rng.rand(n) < 0.4
    x[pick] = rng.choice(IDENTITIES, int(pick.sum()))
    return x


def pattern(rng, n, kind):
    """Sorted indices: empty, one entry, all, the last partial word, random."""
    if kind == "empty":
        return np.zeros(0, np.int32)
    if kind == "one":
        return np.int32([rng.randint(n)])
    if kind == "all":
        return np.arange(n, dtype=np.int32)
    if kind == "tail":
        return np.arange(n - (n % 32 or 32), n, dtype=np.int32)[::2].copy()
    return np.sort(rng.choice(n, max(1, n//3), replace=False)).astype(np.int32)


def dense(gb, x):
    v = gb.Vector(len(x))
    v.build(np.asarray(x, np.float32))
    return v


def sparse(gb, n, ind, val):
    v = gb.Vector(n)
    if len(ind) == 0:                 # an empty sparse vector: compact an all-zero one
        v.fill(0.0)
        v.dense2sparse(0.0, gb.Descriptor())
    else:
        v.build(np.asarray(ind, np.int32), np.asarray(val, np.float32))
    assert v.getStorage() == gb.Storage.GrB_SPARSE
    return v


def tuples(v):
    ind, val = v.extractTuples(sparse=True)
    return ind, val


def check_shadow(gb, v):
    """The bitmap shadow of a dense vector equals values != 0."""
    import torch
    n = v.size()
    bits = torch.zeros((n + 31)//32 + 1, dtype=torch.int32, device="cuda")
    assert gb.api._lib.load().gb200_vector_export_bits(
        v._h, C.c_void_p(bits.data_ptr()), None) == 0
    words = bits.cpu().numpy().view(np.uint32)[:(n + 31)//32]
    got = np.unpackbits(words.view(np.uint8), bitorder="little")
    assert not got[n:].any(), "bits past the end"
    assert np.array_equal(got[:n].astype(bool), v.extractTuples() != 0)


def reduce_val(gb, monoid, src, desc=None):
    return np.float32(gb.reduce(None, monoid, src, desc or gb.Descriptor()))


# ---------------------------------------------------------------------------
# eWiseAdd
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["int", "float", "ident"])
def test_ewise_add_dense_dense(gb, regime):
    desc = gb.Descriptor()
    for n in LENGTHS + [BITS_CTA + 1]:
        rng = np.random.RandomState(n)
        u, v = values(rng, regime, n), values(rng, regime, n)
        for s in range(17):
            want = ref.ewise_add_dense(s, u, v)
            w = gb.Vector(n)
            gb.eWiseAdd(w, None, None, s, dense(gb, u), dense(gb, v), desc)
            assert same(w.extractTuples(), want), (n, s)
            # w is u, w is v, w is both
            du, dv = dense(gb, u), dense(gb, v)
            gb.eWiseAdd(du, None, None, s, du, dv, desc)
            assert same(du.extractTuples(), want), (n, s, "w=u")
            du, dv = dense(gb, u), dense(gb, v)
            gb.eWiseAdd(dv, None, None, s, du, dv, desc)
            assert same(dv.extractTuples(), want), (n, s, "w=v")
            du = dense(gb, u)
            gb.eWiseAdd(du, None, None, s, du, du, desc)
            assert same(du.extractTuples(), ref.ewise_add_dense(s, u, u)), (n, s, "w=u=v")


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["int", "ident"])
def test_ewise_add_sparse_dense_and_aliasing(gb, regime):
    desc = gb.Descriptor()
    for n in SPARSE_LENGTHS:
        for kind in ("one", "tail", "random"):
            rng = np.random.RandomState(n + len(kind))
            ind = pattern(rng, n, kind)
            val = values(rng, regime, len(ind))
            v = values(rng, regime, n)
            for s in range(17):
                for reverse in (False, True):
                    su, dv = sparse(gb, n, ind, val), dense(gb, v)
                    w = gb.Vector(n)
                    args = (dv, su) if reverse else (su, dv)
                    gb.eWiseAdd(w, None, None, s, *args, desc)
                    want = ref.ewise_add_sparse_dense(s, ind, val, v, reverse)
                    assert w.getStorage() == gb.Storage.GrB_DENSE
                    assert same(w.extractTuples(), want), (n, kind, s, reverse)
                    # w is the dense operand: the sparse pass reads the rewritten v
                    su, dv = sparse(gb, n, ind, val), dense(gb, v)
                    args = (dv, su) if reverse else (su, dv)
                    gb.eWiseAdd(dv, None, None, s, *args, desc)
                    want = ref.ewise_add_sparse_dense(s, ind, val, v, reverse, w_is_v=True)
                    assert same(dv.extractTuples(), want), (n, kind, s, reverse, "w=v")
                    # w is the sparse operand: densified with the identity first
                    su, dv = sparse(gb, n, ind, val), dense(gb, v)
                    args = (dv, su) if reverse else (su, dv)
                    gb.eWiseAdd(su, None, None, s, *args, desc)
                    want = ref.ewise_add_aliased_sparse(s, n, ind, val, v,
                                                        w_is_first=not reverse)
                    assert su.getStorage() == gb.Storage.GrB_DENSE
                    assert same(su.extractTuples(), want), (n, kind, s, reverse, "w=u")


@pytest.mark.gpu
def test_ewise_add_scalar(gb):
    desc = gb.Descriptor()
    for n in [1, 31, 33, VALUE_CTA + 1]:
        rng = np.random.RandomState(n)
        u = values(rng, "ident", n)
        ind = pattern(rng, n, "random")
        val = values(rng, "ident", len(ind))
        for s in range(17):
            for scalar in (np.float32(3), np.float32(-0.5), mref.SEMIRINGS[s][2]):
                w = gb.Vector(n)
                gb.eWiseAdd(w, None, None, s, dense(gb, u), float(scalar), desc)
                assert same(w.extractTuples(), ref.ewise_add_scalar_dense(s, u, scalar))
                du = dense(gb, u)
                gb.eWiseAdd(du, None, None, s, du, float(scalar), desc)
                assert same(du.extractTuples(), ref.ewise_add_scalar_dense(s, u, scalar))
                want = ref.ewise_add_scalar_sparse(s, n, ind, val, scalar)
                w = gb.Vector(n)
                gb.eWiseAdd(w, None, None, s, sparse(gb, n, ind, val), float(scalar), desc)
                assert same(w.extractTuples(), want), (n, s, scalar)
                su = sparse(gb, n, ind, val)
                gb.eWiseAdd(su, None, None, s, su, float(scalar), desc)
                assert same(su.extractTuples(), want), (n, s, scalar, "w=u")


@pytest.mark.gpu
def test_refused_ewise_add_leaves_w_as_it_was(gb):
    """sparse + sparse and every masked eWiseAdd are not built: they report it,
    return success, and leave w's storage and contents alone."""
    desc = gb.Descriptor()
    n = 100
    ind, val = np.int32([3, 50, 99]), np.float32([1, -2, 4])
    w_ind, w_val = np.int32([0, 7]), np.float32([5, 6])
    rng = np.random.RandomState(0)
    u, v = values(rng, "int", n), values(rng, "int", n)
    cases = [
        ("sparse+sparse", lambda w: gb.eWiseAdd(w, None, None, 1, sparse(gb, n, ind, val),
                                                sparse(gb, n, ind, val), desc)),
        ("masked dense+dense", lambda w: gb.eWiseAdd(w, dense(gb, np.ones(n)), None, 1,
                                                     dense(gb, u), dense(gb, v), desc)),
        ("masked sparse+dense", lambda w: gb.eWiseAdd(w, dense(gb, np.ones(n)), None, 1,
                                                      sparse(gb, n, ind, val),
                                                      dense(gb, v), desc)),
    ]
    for name, call in cases:
        w = sparse(gb, n, w_ind, w_val)
        call(w)
        assert w.getStorage() == gb.Storage.GrB_SPARSE, name
        got_i, got_v = tuples(w)
        assert np.array_equal(got_i, w_ind) and np.array_equal(got_v, w_val), name
        w = dense(gb, u)
        call(w)
        assert np.array_equal(w.extractTuples(), u), name


# ---------------------------------------------------------------------------
# eWiseMult
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["int", "ident"])
def test_ewise_mult_dense_dense(gb, regime):
    desc = gb.Descriptor()
    for n in LENGTHS + [BITS_CTA + 1]:
        rng = np.random.RandomState(n + 1)
        u, v = values(rng, regime, n), values(rng, regime, n)
        mk = rng.choice(np.float32([0, -0.0, 1, 2.5]), n)
        m_ind = pattern(rng, n, "random")
        m_val = rng.choice(np.float32([0, 1, -3]), len(m_ind))
        for s in range(17):
            want = ref.ewise_mult_dense(s, u, v)
            w = gb.Vector(n)
            gb.eWiseMult(w, None, None, s, dense(gb, u), dense(gb, v), desc)
            assert same(w.extractTuples(), want), (n, s)
            du, dv = dense(gb, u), dense(gb, v)
            gb.eWiseMult(du, None, None, s, du, dv, desc)
            assert same(du.extractTuples(), want), (n, s, "w=u")
            du, dv = dense(gb, u), dense(gb, v)
            gb.eWiseMult(dv, None, None, s, du, dv, desc)
            assert same(dv.extractTuples(), want), (n, s, "w=v")
            du = dense(gb, u)
            gb.eWiseMult(du, None, None, s, du, du, desc)
            assert same(du.extractTuples(), ref.ewise_mult_dense(s, u, u)), (n, s, "w=u=v")
            # dense mask: the identity where the mask is 0
            w = gb.Vector(n)
            gb.eWiseMult(w, dense(gb, mk), None, s, dense(gb, u), dense(gb, v), desc)
            assert same(w.extractTuples(), ref.ewise_mult_dense(s, u, v, mk)), (n, s)
            # sparse mask: the mask's pattern, 0 where the mask value is 0
            w = gb.Vector(n)
            gb.eWiseMult(w, sparse(gb, n, m_ind, m_val), None, s, dense(gb, u),
                         dense(gb, v), desc)
            assert w.getStorage() == gb.Storage.GrB_SPARSE
            wi, wv = ref.ewise_mult_dense_sparse_mask(s, u, v, m_ind, m_val)
            got_i, got_v = tuples(w)
            assert np.array_equal(got_i, wi) and same(got_v, wv), (n, s)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["int", "ident"])
def test_ewise_mult_sparse_dense(gb, regime):
    desc = gb.Descriptor()
    for n in SPARSE_LENGTHS:
        for kind in ("one", "tail", "random"):
            rng = np.random.RandomState(n + 7*len(kind))
            ind = pattern(rng, n, kind)
            val = values(rng, regime, len(ind))
            v = values(rng, regime, n)
            mk = rng.choice(np.float32([0, -0.0, 1, 2.5]), n)
            m_ind = pattern(rng, n, "random")
            m_val = rng.choice(np.float32([0, 1, -3]), len(m_ind))
            for s in range(17):
                for reverse in (False, True):
                    def run(w, mask, first=None):
                        su, dv = sparse(gb, n, ind, val), dense(gb, v)
                        if first == "u":
                            w = su
                        elif first == "v":
                            w = dv
                        args = (dv, su) if reverse else (su, dv)
                        gb.eWiseMult(w, mask, None, s, *args, desc)
                        assert w.getStorage() == gb.Storage.GrB_SPARSE
                        return tuples(w)
                    wi, wv = ref.ewise_mult_sparse_dense(s, ind, val, v, reverse)
                    for alias in (None, "u", "v"):
                        got_i, got_v = run(gb.Vector(n), None, alias)
                        assert np.array_equal(got_i, wi) and same(got_v, wv), \
                            (n, kind, s, reverse, alias)
                    wi, wv = ref.ewise_mult_sparse_dense(s, ind, val, v, reverse, mk)
                    got_i, got_v = run(gb.Vector(n), dense(gb, mk))
                    assert np.array_equal(got_i, wi) and same(got_v, wv), (n, kind, s)
                    wi, wv = ref.ewise_mult_sparse_dense_sparse_mask(
                        s, ind, val, v, m_ind, m_val, reverse)
                    got_i, got_v = run(gb.Vector(n), sparse(gb, n, m_ind, m_val))
                    assert np.array_equal(got_i, wi) and same(got_v, wv), (n, kind, s)


@pytest.mark.gpu
def test_matrix_scale_and_broadcast_through_pr_normalize(gb):
    """pr_normalize: outdeg = row reduce, A = alpha * A, A = A ./ outdeg (row
    broadcast), on the CSR and the CSC value arrays."""
    import test_mxv_gpu as mx
    rng = np.random.RandomState(3)
    S = mx.structure(rng, ROW_LENGTHS, 6000)
    vals = rng.randint(1, 9, S.nnz).astype(np.float32)
    S = S.with_values(vals)
    M = device_matrix(gb, S)
    alpha = np.float32(0.85)
    M.pr_normalize(float(alpha), gb.Descriptor())
    outdeg, _ = ref.reduce_rows(0, S.ptr, S.val)
    want = ref.scale_rows(4, S.ptr, ref.scale_csr(1, S.val, alpha), outdeg.astype(np.float32))
    rp, ci, got = M.extract_csr()
    assert np.array_equal(rp, S.ptr) and np.array_equal(ci, S.ind)
    assert same(got, want)
    # the CSC side: a pull over it (vxm) of min(0 + a) is each column's minimum
    w = gb.Vector(S.ncols)
    gb.vxm(w, None, None, 2, dense(gb, np.zeros(S.nrows, np.float32)), M,
           gb.Descriptor(mxvmode=2))
    col_min = np.full(S.ncols, FLT_MAX, np.float32)
    np.minimum.at(col_min, S.ind, want)
    assert np.array_equal(w.extractTuples(), col_min)


# ---------------------------------------------------------------------------
# reduce
# ---------------------------------------------------------------------------

def monoid_values(rng, monoid, n):
    """Inputs on which every fold order gives one answer."""
    if monoid == 1:                      # powers of two: products exact in any order
        x = np.ones(n, np.float32)
        k = min(n, 40)
        at = rng.choice(n, k, replace=False)
        x[at[:k//2]] = 2
        x[at[k//2:]] = 0.5
        x[rng.choice(n, min(n, 3), replace=False)] *= -1
        return x
    x = rng.randint(-8, 9, n).astype(np.float32)
    x[rng.rand(n) < 0.1] = -0.0
    return x


@pytest.mark.gpu
def test_reduce_vector_every_monoid_and_storage(gb):
    desc = gb.Descriptor()
    lengths = LENGTHS + reduce_lengths(gb.sm_count()) + [VALUE_CHUNKED]
    for n in lengths:
        rng = np.random.RandomState(n)
        for m in range(9):
            if m in ref.ORDER_DEPENDENT_MONOIDS:
                continue
            x = monoid_values(rng, m, n)
            want, _ = ref.reduce(m, x)
            assert reduce_val(gb, m, dense(gb, x), desc) == want, (n, m)
            ind = pattern(rng, n, "random")
            want, _ = ref.reduce(m, x[ind])
            assert reduce_val(gb, m, sparse(gb, n, ind, x[ind]), desc) == want, (n, m)
        # max over negatives is the identity 0; logical-and is always 0
        neg = -rng.randint(1, 9, n).astype(np.float32)
        assert reduce_val(gb, 3, dense(gb, neg), desc) == 0
        assert reduce_val(gb, 5, dense(gb, np.ones(n, np.float32)), desc) == 0
        # plus over floats: within the float64 bound
        x = values(rng, "float", n)
        want, bound = ref.reduce(0, x)
        assert abs(float(reduce_val(gb, 0, dense(gb, x), desc)) - want) <= bound, n
        # struct-only: a sparse vector reduces to its entry count, any monoid
        ind = pattern(rng, n, "random")
        for m in range(9):
            got = reduce_val(gb, m, sparse(gb, n, ind, x[ind]), gb.Descriptor(struconly=1))
            assert got == len(ind), (n, m)
    # an empty input returns the identity; the only case the order-dependent
    # monoids (Greater, CustomLess, NotEqualTo) are checked on
    for m in range(9):
        assert reduce_val(gb, m, sparse(gb, 50, [], []), desc) == ref.MONOIDS[m][1]


@pytest.mark.gpu
def test_reduce_matrix_to_scalar(gb):
    import test_mxv_gpu as mx
    rng = np.random.RandomState(11)
    S = mx.structure(rng, ROW_LENGTHS*20, 6000)
    M = device_matrix(gb, S)
    desc = gb.Descriptor()
    for m in (0, 2, 3, 4, 5):
        want, _ = ref.reduce(m, S.val)
        assert reduce_val(gb, m, M, desc) == want, m
    F = S.with_values(values(rng, "float", S.nnz))
    MF = device_matrix(gb, F)
    want, bound = ref.reduce(0, F.val)
    assert abs(float(reduce_val(gb, 0, MF, desc)) - want) <= bound
    assert reduce_val(gb, 0, MF, gb.Descriptor(struconly=1)) == S.nnz
    # int matrix, plus: exact
    MI = gb.Matrix(S.nrows, S.ncols, dtype=gb.api.INT32)
    rows = np.repeat(np.arange(S.nrows), np.diff(S.ptr))
    MI.build(rows, S.ind, S.val.astype(np.int32))
    assert gb.reduce(None, 0, MI, desc) == int(S.val.astype(np.int64).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["int", "float"])
def test_reduce_rows(gb, regime):
    import test_mxv_gpu as mx
    rng = np.random.RandomState(12)
    S = mx.structure(rng, ROW_LENGTHS, 6000)
    M = device_matrix(gb, S)
    desc = gb.Descriptor()
    monoids = [0] if regime == "float" else [0, 1, 2, 3, 4, 5]
    for m in monoids:
        if regime == "float":
            val = values(rng, "float", S.nnz)
        else:
            val = np.concatenate([monoid_values(rng, m, S.ptr[i + 1] - S.ptr[i])
                                  for i in range(S.nrows)]).astype(np.float32)
        M = device_matrix(gb, S.with_values(val))
        w = gb.Vector(S.nrows)
        gb.reduce(None, m, M, desc, out=w)
        want, bound = ref.reduce_rows(m, S.ptr, val)
        got = w.extractTuples()
        if bound is None or regime == "int":
            assert np.array_equal(got, np.asarray(want, np.float32)), m
        else:
            assert np.all(np.abs(got - want) <= bound), m
    # struct-only leaves w untouched
    w = dense(gb, np.full(S.nrows, 7, np.float32))
    gb.reduce(None, 0, M, gb.Descriptor(struconly=1), out=w)
    assert np.all(w.extractTuples() == 7)


# ---------------------------------------------------------------------------
# conversions
# ---------------------------------------------------------------------------

def bits_vector(gb, n, ind, val):
    """Dense vector whose bitmap shadow is current: fill(0), then a sparse-mask
    assign of val at ind (both keep the shadow)."""
    v = gb.Vector(n)
    v.fill(0.0)
    if len(ind):
        gb.assign(v, sparse(gb, n, ind, np.ones(len(ind))), None, float(val), None, 0,
                  gb.Descriptor())
    return v


@pytest.mark.gpu
def test_dense2sparse_and_back_on_every_source(gb):
    for n in LENGTHS + BIG_LENGTHS:
        rng = np.random.RandomState(n % 100003)
        kinds = ("empty", "one", "all", "tail", "random")
        if n > BITS_CTA + 1:
            kinds = ("tail", "random")           # the chunked scans
        for kind in kinds:
            ind = pattern(rng, n, kind)
            x = np.zeros(n, np.float32)
            x[ind] = values(rng, "int", len(ind))
            x[ind[x[ind] == 0]] = 3
            for struconly in (0, 1):
                desc = gb.Descriptor(struconly=struconly)
                # the value source, identity 0 and FLT_MAX
                for identity in (0.0, FLT_MAX):
                    xi = x if identity == 0 else np.where(x == 0, FLT_MAX, x).astype(np.float32)
                    v = dense(gb, xi)
                    v.dense2sparse(identity, desc)
                    got_i, got_v = tuples(v)
                    want_i, want_v = ref.dense2sparse(xi, identity)
                    assert np.array_equal(got_i, want_i), (n, kind, struconly)
                    if not struconly:
                        assert np.array_equal(got_v, want_v), (n, kind)
                        v.sparse2dense(identity, desc)
                        assert np.array_equal(v.extractTuples(), xi), (n, kind)
                # the bitmap source
                v = bits_vector(gb, n, ind, 5.0)
                v.dense2sparse(0.0, desc)
                got_i, got_v = tuples(v)
                assert np.array_equal(got_i, ind), (n, kind, struconly, "bits")
                if not struconly:
                    assert np.all(got_v == 5)
                # back to dense: struct-only writes 1 and keeps the bitmap shadow
                v.sparse2dense(0.0, desc)
                want = ref.sparse2dense(n, ind, np.full(len(ind), 5, np.float32), 0.0,
                                        struconly=bool(struconly))
                assert np.array_equal(v.extractTuples(), want), (n, kind, struconly)
                check_shadow(gb, v)


@pytest.mark.gpu
def test_reduce_and_dense2sparse_share_one_descriptor(gb):
    """Both use the descriptor's block-sum scratch, back to back."""
    desc = gb.Descriptor()
    rng = np.random.RandomState(5)
    n = VALUE_CHUNKED
    x = rng.randint(-8, 9, n).astype(np.float32)
    y = rng.randint(-8, 9, n).astype(np.float32)
    for _ in range(2):
        a, b = dense(gb, x), dense(gb, y)
        a.dense2sparse(0.0, desc)
        assert reduce_val(gb, 0, b, desc) == y.astype(np.float64).sum()
        got_i, got_v = tuples(a)
        want_i, want_v = ref.dense2sparse(x, 0)
        assert np.array_equal(got_i, want_i) and np.array_equal(got_v, want_v)
        assert reduce_val(gb, 0, a, desc) == x.astype(np.float64).sum()
        b.dense2sparse(0.0, desc)
        assert np.array_equal(tuples(b)[0], ref.dense2sparse(y, 0)[0])


# ---------------------------------------------------------------------------
# assign
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("scmp", [False, True])
def test_assign_dense_target_every_mask(gb, scmp):
    import test_mxv_gpu as mx
    for n in [1, 31, 33, VALUE_CTA + 1, BITS_CTA + 1]:
        rng = np.random.RandomState(n)
        for val in (0.0, 3.0):
            desc = gb.Descriptor()
            if scmp:
                desc.toggle(gb.Desc_field.GrB_MASK)
            w0 = values(rng, "int", n)
            mk = rng.choice(np.float32([0, -0.0, 1, 2.5]), n)
            # value mask, target without a current shadow
            w = dense(gb, w0)
            gb.assign(w, dense(gb, mk), None, val, None, 0, desc)
            assert np.array_equal(w.extractTuples(), ref.assign_dense(w0, mk, val, scmp))
            # mask read as a bitmap (fill + assign), target with a current shadow
            m_ind = pattern(rng, n, "random")
            m01 = np.zeros(n, np.float32)
            m01[m_ind] = 1
            w = bits_vector(gb, n, pattern(rng, n, "tail"), 2.0)
            before = w.extractTuples()
            gb.assign(w, bits_vector(gb, n, m_ind, 1.0), None, val, None, 0, desc)
            assert np.array_equal(w.extractTuples(), ref.assign_dense(before, m01, val, scmp))
            check_shadow(gb, w)
            # mask from a fused Boolean pull (lazily held 0/1 values)
            S = mx.square(rng, n)
            M = device_matrix(gb, S)
            u = rng.choice(np.float32([0, 1]), n)
            pm = rng.choice(np.float32([0, 1]), n)
            f = mx.bool_pull(gb, M, "mxv", 0, u, mx.dense_vector(gb, pm), False, False, False)
            fm = mx.ref.bool_pull(S.ptr, S.ind, pm, u, 0.0, False, False)
            w = gb.Vector(n)
            w.fill(4.0)
            gb.assign(w, f, None, val, None, 0, desc)
            assert np.array_equal(w.extractTuples(),
                                  ref.assign_dense(np.full(n, 4, np.float32), fm, val, scmp))
            check_shadow(gb, w)
            # sparse mask: every stored index, whatever its value; refused under scmp
            m_val = rng.choice(np.float32([0, 1]), len(m_ind))
            for start in ("fill", "values"):
                w = bits_vector(gb, n, [], 0) if start == "fill" else dense(gb, w0)
                before = w.extractTuples()
                gb.assign(w, sparse(gb, n, m_ind, m_val), None, val, None, 0, desc)
                want = before if scmp else ref.assign_dense_sparse_mask(before, m_ind, val)
                assert np.array_equal(w.extractTuples(), want), (n, val, start)
                check_shadow(gb, w)


@pytest.mark.gpu
@pytest.mark.parametrize("scmp", [False, True])
def test_assign_sparse_target_is_a_masked_delete(gb, scmp):
    for n in [9, 33, VALUE_CTA + 1, BITS_CTA + 1]:
        rng = np.random.RandomState(n)
        ind = pattern(rng, n, "random")
        val = rng.choice(np.float32([1, 2, 3, -1]), len(ind))
        mk = rng.choice(np.float32([0, -0.0, 1]), n)
        for v in (2.0, 7.0):
            desc = gb.Descriptor()
            if scmp:
                desc.toggle(gb.Desc_field.GrB_MASK)
            w = sparse(gb, n, ind, val)
            gb.assign(w, dense(gb, mk), None, v, None, 0, desc)
            want_i, want_v = ref.assign_sparse(ind, val, mk, v, scmp)
            got_i, got_v = tuples(w)
            assert np.array_equal(got_i, want_i) and np.array_equal(got_v, want_v)
        # a sparse mask is converted with switch point 0.3 first: at or below it
        # the mask stays sparse and nothing happens; above it, the dense form masks
        for fill in (0.2, 0.6):
            m_ind = np.sort(rng.choice(n, max(1, int(fill*n)), replace=False)).astype(np.int32)
            mask = sparse(gb, n, m_ind, np.ones(len(m_ind)))
            desc = gb.Descriptor()
            if scmp:
                desc.toggle(gb.Desc_field.GrB_MASK)
            w = sparse(gb, n, ind, val)
            gb.assign(w, mask, None, 2.0, None, 0, desc)
            sparse_after, _ = ref.convert(True, len(m_ind), n, 0.3, 0.0)
            got_i, got_v = tuples(w)
            if sparse_after:
                assert mask.getStorage() == gb.Storage.GrB_SPARSE
                assert np.array_equal(got_i, ind) and np.array_equal(got_v, val)
            else:
                assert mask.getStorage() == gb.Storage.GrB_DENSE
                md = ref.sparse2dense(n, m_ind, np.ones(len(m_ind)), 0.0)
                want_i, want_v = ref.assign_sparse(ind, val, md, 2.0, scmp)
                assert np.array_equal(got_i, want_i) and np.array_equal(got_v, want_v)


# ---------------------------------------------------------------------------
# state carried between operations
# ---------------------------------------------------------------------------

@pytest.mark.gpu
def test_count_of_a_zero_one_vector_follows_every_change(gb):
    """A fused Boolean pull leaves a 0/1 vector that carries its count, and a
    plus-reduce over it reads the count: each change must forget it."""
    import test_mxv_gpu as mx
    n = BITS_CTA + 1
    rng = np.random.RandomState(9)
    S = mx.square(rng, n)
    M = device_matrix(gb, S)
    desc = gb.Descriptor()

    def fresh():
        u = rng.choice(np.float32([0, 1]), n)
        pm = rng.choice(np.float32([0, 1]), n)
        f = mx.bool_pull(gb, M, "mxv", 0, u, mx.dense_vector(gb, pm), False, False, False)
        return f, mx.ref.bool_pull(S.ptr, S.ind, pm, u, 0.0, False, False)

    f, x = fresh()
    assert reduce_val(gb, 0, f, desc) == x.sum()
    f.setElement(2.0, 5)
    x[5] = 2
    assert reduce_val(gb, 0, f, desc) == x.sum()
    f, x = fresh()
    mk = rng.choice(np.float32([0, 1]), n)
    gb.assign(f, dense(gb, mk), None, 3.0, None, 0, desc)
    x = ref.assign_dense(x, mk, 3.0)
    assert reduce_val(gb, 0, f, desc) == x.sum()
    f, x = fresh()
    v = values(rng, "int", n)
    gb.eWiseAdd(f, None, None, 1, f, dense(gb, v), desc)
    assert reduce_val(gb, 0, f, desc) == (x + v).astype(np.float64).sum()
    f, x = fresh()
    g = dense(gb, v)
    g.dup(f)
    assert reduce_val(gb, 0, g, desc) == x.sum()
    f, x = fresh()
    h = dense(gb, v)
    h.swap(f)
    assert reduce_val(gb, 0, f, desc) == v.astype(np.float64).sum()
    assert reduce_val(gb, 0, h, desc) == x.sum()
    check_shadow(gb, h)


# ---------------------------------------------------------------------------
# lengths that do not match
# ---------------------------------------------------------------------------

def adopted(gb, n, tail, fill):
    """Vector of length n adopting the head of a tensor of n + tail floats: the
    head holds `fill`, the tail the sentinel bit pattern."""
    import torch
    host = np.empty(n + tail, np.float32)
    host[:n] = fill
    host[n:] = SENTINEL.view(np.float32)
    t = torch.from_numpy(host).cuda()
    v = gb.Vector(n)
    v.build_device(t, nvals=n)
    return v, t


def tail_intact(t, n):
    tail = t[n:].cpu().numpy().view(np.uint32)
    return bool(np.all(tail == SENTINEL))


def info_of(gb, call):
    """The Info code a Python-level call ends with (0 on success)."""
    try:
        call()
    except gb.GraphBLASError as e:
        return int(e.info)
    return 0


# Each case checks the tensor tail before the return code: without the shape
# check the operation runs and its overrun shows there.

@pytest.mark.gpu
def test_ewise_add_into_a_shorter_w_is_refused(gb):
    desc = gb.Descriptor()
    n, nw = 1000, 600
    rng = np.random.RandomState(1)
    u, v = values(rng, "int", n), values(rng, "int", n)
    ind = pattern(rng, n, "all")
    for name, args in [("dense+dense", lambda: (dense(gb, u), dense(gb, v))),
                       ("sparse+dense", lambda: (sparse(gb, n, ind, u), dense(gb, v)))]:
        w, t = adopted(gb, nw, n, 9.0)
        a, b = args()
        code = info_of(gb, lambda: gb.eWiseAdd(w, None, None, 1, a, b, desc))
        assert tail_intact(t, nw), name
        assert code == DIM_MISMATCH, name
        assert np.all(w.extractTuples() == 9), name


@pytest.mark.gpu
def test_row_reduce_into_a_shorter_w_is_refused(gb):
    import test_mxv_gpu as mx
    rng = np.random.RandomState(2)
    S = mx.structure(rng, ROW_LENGTHS*4, 6000)
    M = device_matrix(gb, S)
    nw = S.nrows - 17
    w, t = adopted(gb, nw, S.nrows, 9.0)
    code = info_of(gb, lambda: gb.reduce(None, 0, M, gb.Descriptor(), out=w))
    assert tail_intact(t, nw)
    assert code == DIM_MISMATCH
    assert np.all(w.extractTuples() == 9)


@pytest.mark.gpu
def test_extract_gather_with_more_indices_than_w_is_refused(gb):
    """w[i] = u[ind[i]] for i < nvals(ind): more indices than w would write past w."""
    lib = gb.api._lib.load()
    n, nw = 500, 300
    u = dense(gb, np.arange(n, dtype=np.float32) + 1)
    ind = dense(gb, np.arange(n, dtype=np.float32)[::-1].copy())
    w, t = adopted(gb, nw, n, -1.0)
    desc = gb.Descriptor()
    code = lib.gb200_extract_gather(w._h, u._h, ind._h, desc._h)
    assert tail_intact(t, nw)
    assert code == DIM_MISMATCH
    assert np.all(w.extractTuples() == -1)


@pytest.mark.gpu
def test_assign_scatter_with_more_indices_than_u_is_refused(gb):
    """w[ind[i]] = u[i] for i < nvals(ind): more indices than u would read past u
    (here: the sentinel tail, which would land in w)."""
    lib = gb.api._lib.load()
    n, nu = 500, 300
    u, t = adopted(gb, nu, n, 4.0)
    w = dense(gb, np.zeros(n, np.float32))
    ind = dense(gb, np.random.RandomState(3).permutation(n).astype(np.float32))
    desc = gb.Descriptor()
    code = lib.gb200_assign_scatter(w._h, u._h, ind._h, desc._h)
    got = w.extractTuples()
    assert not np.any(got.view(np.uint32) == SENTINEL)
    assert code == DIM_MISMATCH
    assert np.all(got == 0) and tail_intact(t, nu)


@pytest.mark.gpu
def test_extract_gather_reads_only_inside_u(gb):
    """A source index in [size(u), size(w)) leaves w[i] as it was instead of
    reading past u (here: the sentinel tail)."""
    lib = gb.api._lib.load()
    nu, nw = 100, 200
    u, t = adopted(gb, nu, nw, 5.0)
    src = np.float32([0, nu - 1, nu, nw - 1, 150, -1, 3])
    w = dense(gb, np.full(nw, -2, np.float32))
    ind, desc = dense(gb, src), gb.Descriptor()
    assert lib.gb200_extract_gather(w._h, u._h, ind._h, desc._h) == 0
    want = np.full(nw, -2, np.float32)
    for i, s in enumerate(src.astype(np.int64)):
        if 0 <= s < nu:
            want[i] = 5.0
    assert np.array_equal(w.extractTuples(), want)
    assert tail_intact(t, nu)


# ---------------------------------------------------------------------------
# the fused loop steps against the operation route
# ---------------------------------------------------------------------------

def pr_zero_rank_graph():
    """Directed: vertices 0..h-1 have no in-edges and one out-edge each, to h+i;
    h..n-1 have in-edges and no out-edges.  At alpha = 1 the first iteration
    gives rank 0 to the first half and leaves the second half at 1/n."""
    h = 512
    src = np.arange(h, dtype=np.int32)
    dst = src + h
    n = 2*h
    rp = np.zeros(n + 1, np.int32)
    rp[1:h + 1] = np.arange(1, h + 1)
    rp[h + 1:] = h
    return n, rp, dst


def pr_first_errors(n, rp, ci):
    """First-iteration error of PageRank at alpha = 1, both definitions, float64:
    the operation route's (eWiseMult: 0 wherever either rank is 0) and the plain
    difference."""
    outdeg = np.diff(rp).astype(np.float64)
    p0 = np.full(n, 1.0/n)
    p1 = np.zeros(n)
    rows = np.repeat(np.arange(n), np.diff(rp))
    np.add.at(p1, ci, p0[rows]/outdeg[rows])
    diff = p1 - p0
    op = np.where((p1 == 0) | (p0 == 0), 0.0, diff)
    return np.sqrt((op**2).sum()), np.sqrt((diff**2).sum()), p1


def _child(out, eps):
    import graphblast_b200 as g
    from graphblast_b200 import algorithm
    import oracle_binding as orc
    g.init(0)
    res = {}
    rp, ci = ragged_graph()
    n = len(rp) - 1
    w = g.api.host_uniform_weights(1, 1, 64, len(ci))
    d = g.Vector(n)
    algorithm.sssp(d, make_matrix(g, rp, ci, w, symmetric=False), 3,
                   g.Descriptor(mxvmode=2))
    res["sssp"] = d.extractTuples()
    res["sssp_oracle"] = orc.sssp(rp, ci, w, 3)
    A = make_matrix(g, rp, ci, np.ones(len(ci), np.float32), symmetric=False)
    desc = g.Descriptor(mxvmode=2, max_niter=10)
    A.pr_normalize(0.85, desc)
    p = g.Vector(n)
    algorithm.pr(p, A, 0.85, 0.0, desc)
    res["pr"] = p.extractTuples()
    n, rp, ci = pr_zero_rank_graph()
    A = make_matrix(g, rp, ci, np.ones(len(ci), np.float32), symmetric=False)
    desc = g.Descriptor(mxvmode=2, max_niter=20)
    A.pr_normalize(1.0, desc)
    p = g.Vector(n)
    algorithm.pr(p, A, 1.0, eps, desc)
    res["pr_zero"] = p.extractTuples()
    np.savez(out, **res)


def _run_child(tmp_path, loop_steps, eps):
    env = dict(os.environ)
    env.pop("GB200_LOOP_STEPS", None)
    if loop_steps is not None:
        env["GB200_LOOP_STEPS"] = loop_steps
    out = str(tmp_path / ("steps_%s.npz" % loop_steps))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), out, repr(float(eps))],
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:]
    return np.load(out)


@pytest.mark.gpu
def test_loop_steps_give_the_scalars_of_the_operation_route(tmp_path):
    """SSSP and PageRank pull-only with the fused tails (default) and with the
    operation-by-operation route (GB200_LOOP_STEPS=0), bit for bit.  PageRank at
    alpha = 1 on a graph whose vertices without in-edges reach rank 0: eps lies
    between the two definitions of the first error, so a step that computed the
    plain difference would run a second iteration."""
    n, rp, ci = pr_zero_rank_graph()
    err_op, err_plain, p1 = pr_first_errors(n, rp, ci)
    assert err_plain > 2*err_op
    eps = (err_op + err_plain)/2
    fused = _run_child(tmp_path, None, eps)
    ops = _run_child(tmp_path, "0", eps)
    for key in ("sssp", "pr", "pr_zero"):
        assert np.array_equal(fused[key].view(np.uint32), ops[key].view(np.uint32)), key
    assert np.array_equal(fused["sssp"], fused["sssp_oracle"])
    # the operation route stops after one iteration: the ranks are p1
    assert np.array_equal(ops["pr_zero"], p1.astype(np.float32))


if __name__ == "__main__":
    _child(sys.argv[1], float(sys.argv[2]))
