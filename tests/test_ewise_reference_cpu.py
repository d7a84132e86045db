"""The CPU reference of the element-wise operations (ewise_reference.py) against
the C oracle's scalar operations and against the identities stddef.hpp defines;
the quirks it pins; and the kernel constants the designed shapes of
test_ewise_gpu.py depend on, against the kernel headers."""
import os
import re

import numpy as np
import pytest

import ewise_reference as ref
import mxm_reference as mref
import oracle_binding as orc
from support import same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.path.join(ROOT, "graphblast_b200", "csrc", "graphblas", "backend", "cuda")
STDDEF = os.path.join(ROOT, "include", "graphblas", "stddef.hpp")

GRID = np.float32([-8, -2, -1, -0.5, -0.0, 0, 0.5, 1, 2, 3, 8, mref.FLT_MAX, mref.FLT_MIN])

MONOID_NAMES = ["PlusMonoid", "MultipliesMonoid", "MinimumMonoid", "MaximumMonoid",
                "LogicalOrMonoid", "LogicalAndMonoid", "GreaterMonoid",
                "CustomLessMonoid", "NotEqualToMonoid"]


def _stddef_lists():
    text = open(STDDEF).read()
    monoids = dict((name, ident.strip()) for name, _, ident in re.findall(
        r"X\((\w+Monoid),\s*(\w+),\s*(.+?)\)\s*(?:\\|$)", text, re.M))
    semirings = re.findall(r"X\((\w+Semiring),\s*(\w+Monoid),\s*(\w+)\)", text)
    return monoids, semirings


def _identity_value(expr):
    return {"0": 0.0, "1": 1.0, "false": 0.0,
            "std::numeric_limits<T_out>::max()": float(mref.FLT_MAX),
            "std::numeric_limits<T_out>::min()": float(mref.FLT_MIN)}[expr]


def test_monoid_identities_are_the_ones_stddef_defines():
    monoids, _ = _stddef_lists()
    assert list(monoids) == MONOID_NAMES
    for m, name in enumerate(MONOID_NAMES):
        assert float(ref.MONOIDS[m][1]) == _identity_value(monoids[name]), name
    # the quirks: max and logical-and start from 0, greater from the smallest
    # positive normal
    assert ref.MONOIDS[3][1] == 0 and ref.MONOIDS[5][1] == 0
    assert ref.MONOIDS[6][1] == np.finfo(np.float32).tiny > 0


@pytest.mark.parametrize("semiring", range(17))
def test_each_semiring_add_is_its_monoid_and_matches_the_oracle(semiring):
    """The semiring's add and identity (mxm_reference.SEMIRINGS) are its monoid's
    (ewise_reference.MONOIDS, through stddef.hpp's semiring list), and agree with
    the oracle's orc_add / orc_mul / orc_identity on a grid of values."""
    _, semirings = _stddef_lists()
    monoid = MONOID_NAMES.index(semirings[semiring][1])
    add_name, mul_name, ident = mref.SEMIRINGS[semiring]
    assert ref.MONOIDS[monoid][0] == add_name
    assert ref.MONOIDS[monoid][1] == ident
    assert np.float32(orc.identity(semiring)) == ident
    lib = orc.lib()
    a, b = np.meshgrid(GRID, GRID)
    a, b = a.ravel(), b.ravel()
    want_add = np.float32([lib.orc_add(semiring, float(x), float(y)) for x, y in zip(a, b)])
    want_mul = np.float32([lib.orc_mul(semiring, float(x), float(y)) for x, y in zip(a, b)])
    with np.errstate(all="ignore"):
        assert same(ref.ewise_add_dense(semiring, a, b), want_add)
        assert same(mref.OPS[mul_name](a, b), want_mul)
        # eWiseMult dense x dense: the oracle's product wherever no operand is the
        # identity, the identity elsewhere
        got = ref.ewise_mult_dense(semiring, a, b)
        live = (a != ident) & (b != ident)
        assert same(got[live], want_mul[live])
        assert np.all(got[~live] == ident)


def test_reduce_folds_from_the_identity():
    neg = np.float32([-3, -1, -8])
    assert ref.reduce(3, neg)[0] == 0                    # max over negatives is 0
    assert ref.reduce(2, neg)[0] == -8
    assert ref.reduce(5, np.float32([1, 1, 1]))[0] == 0  # logical-and is always 0
    assert ref.reduce(4, np.float32([0, -0.0, 2]))[0] == 1
    assert ref.reduce(4, np.float32([0, -0.0]))[0] == 0
    assert ref.reduce(1, np.float32([2, -0.5, 4]))[0] == -4
    for m in range(9):
        assert ref.reduce(m, [])[0] == ref.MONOIDS[m][1]
    for m in ref.ORDER_DEPENDENT_MONOIDS:
        with pytest.raises(ValueError):
            ref.reduce(m, [1.0])
    s, bound = ref.reduce(0, np.float32([1e8, 1, -1e8]))
    assert s == 1.0 and bound > 1
    # the fold order-dependent monoids do: greater(FLT_MIN, 0) and greater(0,
    # FLT_MIN) differ, so no grid-independent answer exists for them
    gt = mref.OPS["gt"]
    assert gt(mref.FLT_MIN, np.float32(0)) != gt(np.float32(0), mref.FLT_MIN)


def test_ewise_add_quirks():
    # CustomLessPlus (add = less, identity FLT_MAX): the aliased call densifies the
    # sparse w with the identity first, the non-aliased one rewrites the dense
    # operand with add(v, identity) first -- different results
    FM = mref.FLT_MAX
    n, ind, val = 4, [1, 3], np.float32([5, -1])
    v = np.float32([2, 7, -3, 0])
    aliased = ref.ewise_add_aliased_sparse(9, n, ind, val, v)
    plain = ref.ewise_add_sparse_dense(9, ind, val, v)
    assert list(aliased) == [0, 1, 0, 1]        # lt(FM, v) = 0, lt(5, 7), lt(-1, 0)
    assert list(plain) == [1, 1, 1, 1]          # lt(v, FM) = 1, then lt(u, v)
    assert not np.array_equal(aliased, plain)
    # reverse: the constant pass is add(id, v); the sparse pass keeps (u, v) order
    rev = ref.ewise_add_sparse_dense(9, ind, val, v, reverse=True)
    assert list(rev) == [0, 1, 0, 1]
    # w is v: the sparse pass reads the rewritten v
    wv = ref.ewise_add_sparse_dense(9, ind, val, v, w_is_v=True)
    assert list(wv) == [1, 0, 1, 1]             # lt(5, 1), lt(-1, 1)
    assert ref.ewise_add_scalar_sparse(1, 3, [2], [4], 0.5).tolist() == [0.5, 0.5, 4.5]
    assert ref.ewise_add_scalar_dense(2, np.float32([FM, 1]), 3).tolist() == [3, 1]


def test_ewise_mult_quirks():
    # identity short-circuit of the dense kernel vs the 0 of the sparse routes
    u = np.float32([0, 2, 3, 4])
    v = np.float32([5, 0, 2, 1])
    assert ref.ewise_mult_dense(1, u, v).tolist() == [0, 0, 6, 4]
    assert ref.ewise_mult_dense(10, np.float32([mref.FLT_MAX, 2]),
                                np.float32([3, 4])).tolist() == [mref.FLT_MAX, 8]
    assert ref.ewise_mult_dense(1, u, v, mask=np.float32([1, 1, 0, -0.0])).tolist() == \
        [0, 0, 0, 0]
    _, w = ref.ewise_mult_dense_sparse_mask(10, u, v, [0, 2], np.float32([0, 1]))
    assert w.tolist() == [0, 6]                 # 0, not the identity FLT_MAX
    _, w = ref.ewise_mult_sparse_dense(10, [0, 2], np.float32([mref.FLT_MAX, 3]), v)
    assert w.tolist() == [0, 6]
    _, w = ref.ewise_mult_sparse_dense(7, [0, 2], np.float32([1, 3]), v, reverse=True)
    assert w.tolist() == [4, -1]                # minus(v, u)
    _, w = ref.ewise_mult_sparse_dense(1, [0, 2], np.float32([1, 3]), v,
                                       mask=np.float32([0, 1, 1, 1]))
    assert w.tolist() == [0, 6]
    ind, w = ref.ewise_mult_sparse_dense_sparse_mask(
        1, [0, 2], np.float32([1, 3]), v, [1, 2, 3], np.float32([1, 1, 0]))
    assert ind.tolist() == [1, 2, 3] and w.tolist() == [0, 6, 0]


def test_assign_and_conversion_rules():
    w = np.float32([1, 2, 3, 4])
    m = np.float32([0, -0.0, 5, 1])
    assert ref.assign_dense(w, m, 9).tolist() == [1, 2, 9, 9]
    assert ref.assign_dense(w, m, 9, scmp=True).tolist() == [9, 9, 3, 4]
    assert ref.assign_dense_sparse_mask(w, [0, 3], 0).tolist() == [0, 2, 3, 0]
    ind, val = ref.assign_sparse([0, 1, 2, 3], np.float32([7, 2, 3, 2]),
                                 np.float32([1, 0, 0, 0]), 2)
    assert ind.tolist() == [2] and val.tolist() == [3]
    ind, val = ref.dense2sparse(np.float32([0, -0.0, 3, 0, 1]), 0)
    assert ind.tolist() == [2, 4] and val.tolist() == [3, 1]
    assert ref.sparse2dense(4, [1, 3], np.float32([5, 6]), 0, struconly=True).tolist() == \
        [0, 1, 0, 1]
    # hysteresis: growing past the switch point turns dense, shrinking at or
    # below it turns sparse; otherwise the fill seen is remembered
    assert ref.convert(True, 5, 10, 0.3, 0.0) == (False, 0.0)
    assert ref.convert(True, 5, 10, 0.3, 0.6) == (True, 0.5)
    assert ref.convert(False, 3, 10, 0.3, 0.5) == (True, 0.5)
    assert ref.convert(False, 3, 10, 0.3, 0.2)[0] is False
    assert ref.convert(True, 3, 10, 0.3, 0.0)[0] is True


# ---- kernel constants ---------------------------------------------------------------

def _read(name):
    return open(os.path.join(CUDA, name)).read()


def _define(name, key):
    return int(re.search(r"^#define\s+%s\s+(\d+)" % key, _read(name), re.M).group(1))


def _kgroup(source):
    text = _read("kernels/compact.cuh")
    body = text[text.index("struct %s {" % source):]
    return int(re.search(r"kGroup\s*=\s*(\d+)", body).group(1))


def test_kernel_constants_match_the_gpu_test():
    """The designed sizes of test_ewise_gpu.py sit on these limits; a change to a
    limit must come with a change to the sizes, and this fails first."""
    import test_ewise_gpu as g
    nt = _define("kernels/compact.cuh", "GB_COMPACT_NT")
    assert nt == g.COMPACT_NT
    assert _kgroup("DenseCompactSource") == 1
    assert _kgroup("DenseBitsCompactSource") == 4
    assert "base = item*8" in _read("kernels/compact.cuh")       # 8 values an item
    assert g.VALUE_CTA == nt*1*8
    assert g.BITS_CTA == nt*4*32
    assert _define("kernels/reduce.cuh", "GB_REDUCE_NT") == g.REDUCE_NT
    cap = re.search(r"ctas_per_sm\s*=\s*(\d+)", _read("util.hpp")).group(1)
    assert int(cap) == g.GRID_CTAS_PER_SM
    assert re.search(r"gridFor\(nvals, GB_REDUCE_NT, (\d+)\)",
                     _read("reduce.hpp")).group(1) == str(g.REDUCE_CTAS_PER_SM)
    # the designed lengths straddle each boundary
    for cta in (g.VALUE_CTA, g.BITS_CTA):
        assert {cta - 1, cta, cta + 1} <= set(g.LENGTHS + g.BIG_LENGTHS)
    # the last CTA of the count pass scans the per-CTA counts nt at a time: more
    # than nt CTAs means more than one chunk
    assert -(-g.VALUE_CHUNKED // g.VALUE_CTA) > nt
    assert -(-g.BITS_CHUNKED // g.BITS_CTA) > nt
    assert g.BITS_CHUNKED // g.VALUE_CTA > nt
    # the reduce grid stops growing at REDUCE_NT * REDUCE_CTAS_PER_SM * SMs
    for sms in (114, 132):
        edge = g.reduce_edge(sms)
        lens = g.reduce_lengths(sms)
        assert edge - 1 in lens and edge in lens and edge + 1 in lens
        assert -(-(edge + 1) // g.REDUCE_NT) > sms*g.REDUCE_CTAS_PER_SM
        assert -(-(edge - 1) // g.REDUCE_NT) == sms*g.REDUCE_CTAS_PER_SM
    # the row lengths of the row reduce cross a warp's 32 lanes
    assert {0, 1, 31, 32, 33} <= set(g.ROW_LENGTHS) and max(g.ROW_LENGTHS) > 32*100
