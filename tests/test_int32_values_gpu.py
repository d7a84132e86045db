"""Every INT32 operation entry by entry with values float32 cannot hold, against an
int64 reference.

The other suites use INT32 values of a few units: every one of them, and every sum
and product they produce, is exact in float32, so a value that passed through float
anywhere (a float staging buffer or scratch array, a float accumulator, a
static_cast<float> in a template shared with FP32, a functor on the wrong type, the
wrong 32 bits out of the host mailbox) would go unseen.  Here:

  * products: A's values have 2^12 <= |a| < 2^15, mostly odd, both signs, stored
    zeros; B's magnitude is chosen per row of B (unmasked) or per column of B (masked)
    from the largest sum of |a| over the folds that row or column feeds, so that the
    sum of |a*b| over every output entry, a bound on every partial sum of the fold in
    any order, stays below 2^31.  Long folds thus take small products, but of one
    sign mostly, so their sums still lie far outside the float-exact range;
  * operations that do not multiply (eWiseAdd, assign, extract, build, transpose,
    reduce) take values up to 2^30 (both operands of a sum) or over all of int32,
    with +-(2^24 + 1), the smallest integer float32 cannot hold, planted; eWiseMult
    pairs +-(2^24 + 1) with a +-1 partner;
  * reduce: totals of exactly INT32_MAX, INT32_MIN and a negative odd total beyond
    2^24, over lengths below, at and past one CTA and the cap of the reduce grid.

The reference is the int64 result, asserted to lie in int32, and every comparison is
bit for bit, pattern and values (support.check_csr).  The CPU tests check the regime
itself: at least 90 % of the nonzero reference outputs are not float32-exact, no fold
can leave int32, each case still reaches the routes and limits its source suite
designed it for, and the reference sent through float32 and back is rejected by the
same comparison.  The cooperative algorithms, which read A's pattern only, must give
the same bytes on an INT32 A holding INT32_MIN, -1, 0 and INT32_MAX as on the pattern
with FP32 ones.
"""
import functools
import os
import re

import numpy as np
import pytest

import assign_reference as R
import extract_reference as X
import mxm_reference
import oracle_binding as orc
import ewise_matrix_reference
from support import Csr, check_csr, csr, device_matrix, gb, random_csr  # noqa: F401
from test_extract_gpu import index_sets
from test_ewise_matrix_gpu import IPT, TILE, overlap, straddling
from test_mxm_gpu import (CHUNK, HEAVY, LENS, Problem, designed_problem, oracle, routes)
from test_mxm_unmasked_gpu import DESIGNED, NUM, SYM, designed_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.path.join(ROOT, "graphblast_b200", "csrc", "graphblas", "backend", "cuda")

I32_MIN, I32_MAX = int(np.iinfo(np.int32).min), int(np.iinfo(np.int32).max)
EDGE = 2**24 + 1                  # the smallest integer float32 cannot hold
A_LO, A_HI = 2**12, 2**15         # |a| of a product's first operand: [A_LO, A_HI)
REDUCE_NT = 256                   # GB_REDUCE_NT; the grid is gridFor(n, NT, 4)
H100_SMS = 132                    # the cap the CPU tests design the lengths for


# ---------------------------------------------------------------------------
# values
# ---------------------------------------------------------------------------

def magnitudes(rng, n, lo, hi):
    """n integers in [lo, hi] (scalars or arrays of n), seven in eight odd."""
    lo = np.broadcast_to(np.asarray(lo, np.int64), (n,))
    hi = np.broadcast_to(np.asarray(hi, np.int64), (n,))
    v = np.minimum(lo + np.floor(rng.rand(n)*(hi - lo + 1)).astype(np.int64), hi)
    even = (v % 2 == 0) & (rng.rand(n) < 7/8)
    v[even] = np.where(v[even] < hi[even], v[even] + 1, v[even] - 1)
    return v


def signed(rng, mag, neg=0.25, zeros=0.05):
    """mag with a share `neg` negated and a share `zeros` stored as 0 (int64)."""
    n = len(mag)
    v = np.where(rng.rand(n) < neg, -mag, mag).astype(np.int64)
    v[rng.rand(n) < zeros] = 0
    return v


def wide(rng, n, top=2**30, zeros=0.05):
    """Summands: 2^24 <= |v| < top, +-(2^24 + 1) planted, both signs, stored zeros."""
    v = signed(rng, magnitudes(rng, n, 2**24, top - 1), neg=0.4, zeros=zeros)
    at = rng.rand(n) < 0.03
    v[at] = rng.choice([-EDGE, EDGE], at.sum())
    return v


def full_range(rng, n):
    """Any int32, with INT32_MIN, INT32_MAX, +-(2^24 + 1), -1 and 0 planted."""
    v = rng.randint(I32_MIN, I32_MAX, n, dtype=np.int64)
    planted = np.array([I32_MIN, I32_MAX, EDGE, -EDGE, -1, 0], np.int64)
    at = rng.choice(n, min(n, 6*len(planted)), replace=False)
    v[at] = np.resize(planted, len(at))
    return v


def big_a(rng, n):
    return signed(rng, magnitudes(rng, n, A_LO, A_HI - 1), neg=0.1)


def b_for_folds(rng, reach):
    """B values for entries whose folds sum at most `reach` (per entry) of |a|:
    |b| <= bmax with reach * bmax <= INT32_MAX, from the top quarter; one in ten
    negative, so that long folds of small products still add up."""
    bmax = I32_MAX // np.maximum(reach, 1).astype(np.int64)
    return signed(rng, magnitudes(rng, len(bmax), (3*bmax + 3)//4, bmax), neg=0.1)


def ones(S):
    return S.with_values(np.ones(S.nnz, np.int64))


def absolute(S):
    return S.with_values(np.abs(S.val.astype(np.int64)))


def int64(S):
    return S.with_values(S.val.astype(np.int64))


def row_max(S):
    out = np.zeros(S.nrows, np.int64)
    np.maximum.at(out, S.rows(), S.val.astype(np.int64))
    return out


# ---------------------------------------------------------------------------
# references and checks
# ---------------------------------------------------------------------------

def mxm(A, B):
    rp, ci, val = mxm_reference.mxm(1, A.ptr, A.ind, A.val, B.ptr, B.ind, B.val,
                                    B.ncols, integer=True)
    return Csr(A.nrows, B.ncols, rp, ci, val)


def ewise(add, A, B):
    rp, ci, val = ewise_matrix_reference.ewise(add, 1, A.ptr, A.ind, A.val, B.ptr, B.ind,
                                               B.val, A.ncols, integer=True)
    return Csr(A.nrows, A.ncols, rp, ci, val)


def in_int32(x):
    x = np.asarray(x, np.int64)
    return bool(np.all((x >= I32_MIN) & (x <= I32_MAX)))


def check(C, want):
    """C is INT32 and equals the int64 reference want (in int32) bit for bit."""
    assert C.extract_csr()[2].dtype == np.int32, "C is not INT32"
    assert in_int32(want.val), "the reference leaves int32"
    check_csr(C, want)


class Host(object):
    """A host CSR in the place of a device matrix, for check_csr."""

    def __init__(self, S):
        self.S = S

    def extract_csr(self):
        return self.S.ptr, self.S.ind, self.S.val.astype(np.int32)


def through_float(S):
    """S with every value staged through float32 and converted back, saturating."""
    v = S.val.astype(np.float32).astype(np.float64)
    return S.with_values(np.clip(v, I32_MIN, I32_MAX).astype(np.int64))


def inexact_share(vals):
    v = np.asarray(vals, np.int64)
    v = v[v != 0]
    return np.mean(v.astype(np.float32).astype(np.int64) != v) if len(v) else 0.0


# ---------------------------------------------------------------------------
# operand sets: each returns (operands..., want, bound), bound the largest partial
# sum any order of any fold can reach
# ---------------------------------------------------------------------------

def product_operands(rng, A, B):
    """A and B revalued: A big, B scaled per row k by the largest sum of |a| over the
    folds of the rows of A that use k."""
    A = A.with_values(big_a(rng, A.nnz))
    reach_i = row_max(mxm(absolute(A), ones(B)))
    reach = np.zeros(B.nrows, np.int64)
    np.maximum.at(reach, A.ind, reach_i[A.rows()])
    B = B.with_values(b_for_folds(rng, reach[B.rows()]))
    return A, B


def unmasked(A, B):
    return mxm(A, B), int(mxm(absolute(A), absolute(B)).val.max(initial=0))


@functools.lru_cache(None)
def unmasked_designed():
    A, B = designed_rows(DESIGNED)
    A, B = product_operands(np.random.RandomState(1), A, B)
    return (A, B) + unmasked(A, B)


@functools.lru_cache(None)
def unmasked_random(square=False):
    rng = np.random.RandomState(2 + square)
    m, k, n = (257, 257, 257) if square else (300, 500, 200)
    A = random_csr(rng, m, k, 0.03, np.ones(1, np.int64), zeros=0)
    B = random_csr(rng, k, n, 0.03, np.ones(1, np.int64), zeros=0)
    A, B = product_operands(rng, A, B)
    return (A, B) + unmasked(A, B)


def mask_values(rng, n):
    """One in eight an explicit 0, the others beyond 2^24, both signs."""
    v = wide(rng, n, top=2**31, zeros=0)
    v[rng.rand(n) < 1/8] = 0
    return v


def masked_operands(rng, p):
    """A big, B scaled per column j by the largest sum of |a| over the folds of the
    mask entries of column j."""
    A = p.A.with_values(big_a(rng, p.A.nnz).astype(np.int32))
    fold = oracle(Problem(absolute(A).astype(np.int32), ones(p.Bt).astype(np.int32),
                          ones(p.M).astype(np.int32)))
    reach = np.zeros(p.Bt.nrows, np.int64)
    np.maximum.at(reach, p.M.ind, fold)
    return Problem(A, p.Bt.with_values(b_for_folds(rng, reach[p.Bt.rows()]).astype(np.int32)),
                   p.M.with_values(mask_values(rng, p.M.nnz).astype(np.int32)))


@functools.lru_cache(None)
def masked_designed():
    p = masked_operands(np.random.RandomState(3), designed_problem())
    bound = oracle(Problem(absolute(p.A).astype(np.int32), absolute(p.Bt).astype(np.int32),
                           ones(p.M).astype(np.int32)))
    return p, p.M.with_values(oracle(p)), int(bound.max(initial=0))


@functools.lru_cache(None)
def triangles():
    """A lower triangle L of a sparse random graph, values scaled so that the sum of
    |L(i,k) L(j,k)| over every triangle, a bound on the count's fold and on every
    entry of B, stays in int32."""
    rng = np.random.RandomState(4)
    n = 400
    src, dst = rng.randint(0, n, 1200), rng.randint(0, n, 1200)
    rp, ci = orc.build_csr(n, src.astype(np.int32), dst.astype(np.int32), True)
    lr, lc = orc.tril(rp, ci)
    ntri = orc.tc(lr, lc)
    vmax = int(np.sqrt(I32_MAX // max(ntri, 1)))       # products beyond 2^25
    mag = magnitudes(rng, len(lc), (3*vmax + 3)//4, vmax)
    mag -= mag % 2 == 0              # all odd: an entry of one triangle is odd
    L = Csr(n, n, lr, lc, signed(rng, mag, neg=0.3, zeros=0.02).astype(np.int32))
    want = orc.mxm_masked(L.ptr, L.ind, L.val, L.ptr, L.ind, L.val, L.ptr, L.ind, L.val)
    a = absolute(L).astype(np.int32)
    bound = orc.mxm_masked(a.ptr, a.ind, a.val, a.ptr, a.ind, a.val, L.ptr, L.ind,
                           np.ones(L.nnz, np.int32))
    return L, L.with_values(want), int(bound.sum())


def ewise_values(rng, add, A, B):
    if add:
        return A.with_values(wide(rng, A.nnz)), B.with_values(wide(rng, B.nnz))
    a = big_a(rng, A.nnz)
    b = signed(rng, magnitudes(rng, B.nnz, A_HI, 2*A_HI), neg=0.4)
    ka = A.rows().astype(np.int64)*A.ncols + A.ind
    kb = B.rows().astype(np.int64)*B.ncols + B.ind
    _, ia, ib = np.intersect1d(ka, kb, return_indices=True)
    edge = rng.rand(len(ia)) < 0.05                 # +-(2^24 + 1) against +-1
    a[ia[edge]] = rng.choice([-EDGE, EDGE], edge.sum())
    b[ib[edge]] = rng.choice([-1, 1], edge.sum())
    return A.with_values(a), B.with_values(b)


def ewise_bound(add, A, B):
    return int(np.abs(ewise(add, absolute(A), absolute(B)).val).max(initial=0))


EWISE = (["overlap_" + k for k in ("disjoint", "identical", "nested", "partial")] +
         ["straddling_1", "straddling_3", "transposed"])


@functools.lru_cache(None)
def ewise_case(name, add):
    rng = np.random.RandomState(EWISE.index(name)*2 + add)
    if name.startswith("overlap_"):
        A, B = overlap(EWISE.index(name), name[8:], 1)
    elif name.startswith("straddling_"):
        A, B = straddling(int(name[11:]))
    else:
        A = random_csr(rng, 70, 110, 0.1, np.ones(1, np.float32))
        B = random_csr(rng, 70, 110, 0.1, np.ones(1, np.float32))
    A, B = ewise_values(rng, add, A, B)      # "identical": one pattern, two value sets
    return A, B, ewise(add, A, B), ewise_bound(add, A, B)


ASSIGN_M, ASSIGN_N = 90, 70


@functools.lru_cache(None)
def assign_target():
    rng = np.random.RandomState(5)
    C = random_csr(rng, ASSIGN_M, ASSIGN_N, 0.1, np.ones(1, np.int64), zeros=0)
    return C.with_values(wide(rng, C.nnz, zeros=0.2))


def assign_regions():
    """(name, I, J): sorted and unsorted lists, GrB_ALL, one row and one column."""
    rng = np.random.RandomState(6)
    m, n = ASSIGN_M, ASSIGN_N
    return [("sorted", np.sort(rng.choice(m, 30, replace=False)),
             np.sort(rng.choice(n, 25, replace=False))),
            ("unsorted", rng.permutation(m)[:40], rng.permutation(n)[:35]),
            ("all_rows", None, rng.permutation(n)[:20]),
            ("row", np.array([17]), rng.permutation(n)[:50]),
            ("column", rng.permutation(m)[:60], np.array([33]))]


@functools.lru_cache(None)
def assign_case(region, accum, tran=False):
    C = assign_target()
    name, I, J = [r for r in assign_regions() if r[0] == region][0]
    nI = ASSIGN_M if I is None else len(I)
    nJ = ASSIGN_N if J is None else len(J)
    rng = np.random.RandomState(7 + 2*len(region) + accum + 4*tran)
    shape = (nJ, nI) if tran else (nI, nJ)
    A = random_csr(rng, shape[0], shape[1], 0.3, np.ones(1, np.int64), zeros=0)
    A = A.with_values(wide(rng, A.nnz, zeros=0.2))
    def placed(C, A):
        return R.assign_matrix((C.ptr, C.ind, C.val), ASSIGN_M, ASSIGN_N,
                               (A.ptr, A.ind, A.val, A.nrows, A.ncols), I, J,
                               accum="plus" if accum else None, tran=tran)
    rp, ci, val = placed(C, A)
    bound = int(placed(absolute(C), absolute(A))[2].max(initial=0))
    return C, A, I, J, Csr(ASSIGN_M, ASSIGN_N, rp, ci, val), bound


SCALARS = [-EDGE, EDGE, 3*EDGE + 2]


@functools.lru_cache(None)
def assign_scalar_case(val, accum):
    C = assign_target()
    _, I, J = assign_regions()[1]
    rp, ci, out = R.assign_constant((C.ptr, C.ind, C.val), ASSIGN_M, ASSIGN_N, np.int64(val),
                                    I, J, accum="plus" if accum else None)
    return C, I, J, Csr(ASSIGN_M, ASSIGN_N, rp, ci, out), int(np.abs(out).max())


@functools.lru_cache(None)
def extract_source():
    rng = np.random.RandomState(8)
    S = random_csr(rng, 120, 97, 0.08, np.ones(1, np.int64), zeros=0)
    return S.with_values(full_range(rng, S.nnz))


def extract_cases():
    S = extract_source()
    rng = np.random.RandomState(9)
    out = []
    for tran in (False, True):
        for name, I in index_sets(rng, S.ncols if tran else S.nrows):
            for nameJ, J in index_sets(rng, S.nrows if tran else S.ncols):
                if "repeated" in name or "repeated" in nameJ or name == nameJ == "all":
                    out.append((tran, I, J))
    return out


def extract_want(S, I, J, tran):
    rp, ci, val = X.extract_matrix(S.ptr, S.ind, S.val, S.nrows, S.ncols, I, J, tran=tran)
    nr, nc = (S.ncols, S.nrows) if tran else (S.nrows, S.ncols)
    return Csr(nr if I is None else len(I), nc if J is None else len(J), rp, ci, val)


@functools.lru_cache(None)
def build_tuples():
    """Unsorted host COO of a 150 x 110 matrix over all of int32, no position twice."""
    rng = np.random.RandomState(10)
    S = random_csr(rng, 150, 110, 0.05, np.ones(1, np.int64), zeros=0)
    S = S.with_values(full_range(rng, S.nnz))
    order = rng.permutation(S.nnz)
    return S, S.rows()[order], S.ind[order], S.val[order]


@functools.lru_cache(None)
def dedup_tuples():
    """Device COO for DEDUP | SYMMETRIZE: no loops, repeated positions with other
    values; the reference keeps the first forward tuple, then the first mirror."""
    rng = np.random.RandomState(11)
    n, t = 300, 4000
    r, c = rng.randint(0, n, t), rng.randint(0, n, t)
    keep = r != c
    r, c = r[keep], c[keep]
    rep = rng.choice(len(r), len(r)//5)
    r, c = np.concatenate([r, r[rep]]), np.concatenate([c, c[rep]])
    v = full_range(rng, len(r))
    rows, cols, vals = np.concatenate([r, c]), np.concatenate([c, r]), np.concatenate([v, v])
    key = rows.astype(np.int64)*n + cols
    _, first = np.unique(key, return_index=True)
    S = csr(n, n, rows[first], cols[first], vals[first], np.int64)
    return n, r, c, v, S


def reduce_lengths(sms):
    """Below, at and past one CTA and the grid's cap of 4 CTAs per SM."""
    cap = REDUCE_NT*4*sms
    return [1, REDUCE_NT - 1, REDUCE_NT, REDUCE_NT + 1, cap - 1, cap, cap + 1, 3*cap + 5]


TOTALS = ["max", "min", "negative"]


def reduce_values(n, total):
    """n values whose sum is INT32_MAX, INT32_MIN, or odd, negative and beyond 2^24;
    the positive and the negative values each sum inside int32, so no order of the
    fold leaves it."""
    rng = np.random.RandomState(n*3 + TOTALS.index(total))
    if total in ("max", "min"):
        want = I32_MAX if total == "max" else I32_MIN
        w = rng.rand(n) + 0.05
        v = np.floor(w/w.sum()*abs(want)).astype(np.int64)
        v[:abs(want) - int(v.sum())] += 1
        v[rng.rand(n) < 0.05] = 0 if n > 1 else v[0]
        v[0] += abs(want) - int(v.sum())
        return v if total == "max" else -v
    want = -(2**28 + 12345)
    if n == 1:
        return np.array([want], np.int64)
    v = signed(rng, magnitudes(rng, n, 1, max(2, 2**29 // n)), neg=0.5)
    v[rng.choice(n - 1, min(n - 1, 4), replace=False)] = -EDGE
    v[-1] += want - int(v.sum())
    return v


def reduce_matrix_of(v):
    n = len(v)
    cols = 1024
    idx = np.arange(n)
    return csr(-(-n // cols), cols, idx // cols, idx % cols, v, np.int64)


# ---------------------------------------------------------------------------
# the cases every CPU check runs over: name -> (want, bound)
# ---------------------------------------------------------------------------

def _cases():
    out = {"unmasked_designed": lambda: unmasked_designed()[2:],
           "unmasked_random": lambda: unmasked_random()[2:],
           "unmasked_square": lambda: unmasked_random(True)[2:],
           "masked_designed": lambda: masked_designed()[1:],
           "triangles": lambda: triangles()[1:]}
    for name in EWISE:
        for add in (True, False):
            if not add and name == "overlap_disjoint":
                continue                        # an empty intersection: no values
            out["%s_%s" % ("add" if add else "mult", name)] = \
                functools.partial(lambda n, a: ewise_case(n, a)[2:], name, add)
    for region, *_ in assign_regions():
        for accum in (False, True):
            out["assign_%s_%s" % (region, "plus" if accum else "replace")] = \
                functools.partial(lambda r, a: assign_case(r, a)[4:], region, accum)
    out["assign_unsorted_transposed"] = lambda: assign_case("unsorted", True, True)[4:]
    for val in SCALARS:
        for accum in (False, True):
            out["assign_scalar_%d_%s" % (val, "plus" if accum else "replace")] = \
                functools.partial(lambda x, a: assign_scalar_case(x, a)[3:], val, accum)
    out["extract_all"] = lambda: (int64(extract_source()), 0)
    out["build"] = lambda: (build_tuples()[0], 0)
    out["build_dedup_symmetric"] = lambda: (dedup_tuples()[4], 0)
    return out


CASES = _cases()


# ---------------------------------------------------------------------------
# CPU: the regime holds, the designed routes are reached, float is caught
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(CASES))
def test_values_lie_outside_float32(name):
    want, _ = CASES[name]()
    assert want.val.dtype.kind == "i"
    assert inexact_share(want.val) >= 0.9, inexact_share(want.val)


@pytest.mark.parametrize("name", sorted(CASES))
def test_no_fold_leaves_int32(name):
    want, bound = CASES[name]()
    assert in_int32(want.val)
    assert bound <= I32_MAX


@pytest.mark.parametrize("name", sorted(CASES))
def test_float_round_trip_is_rejected(name):
    want, _ = CASES[name]()
    check_csr(Host(want), want)
    with pytest.raises(pytest.fail.Exception):
        check_csr(Host(through_float(want)), want)


def test_products_and_edges_are_there():
    """Most products exceed 2^24; both signs, stored zeros and +-(2^24 + 1) appear."""
    A, B = unmasked_designed()[:2]
    big = 0
    for e in range(0, A.nnz):
        k = A.ind[e]
        prods = np.abs(A.val[e]*B.val[B.ptr[k]:B.ptr[k + 1]].astype(np.int64))
        big += np.count_nonzero(prods > 2**24)
    assert big > 0.5*B.nnz
    for S in (A, B, masked_designed()[0].M, assign_target(), extract_source()):
        assert (S.val == 0).any() and (S.val < 0).any() and (S.val > 0).any()
    for S in (assign_target(), extract_source(), build_tuples()[0]):
        assert (S.val == EDGE).any() and (S.val == -EDGE).any()
    a, b = ewise_case("overlap_partial", False)[:2]
    assert (np.abs(a.val) == EDGE).any() and (np.abs(b.val) == 1).any()
    for S in (extract_source(), build_tuples()[0], dedup_tuples()[4]):
        assert S.val.min() == I32_MIN and S.val.max() == I32_MAX


def test_unmasked_operands_reach_every_bin_limit():
    """The check of test_mxm_unmasked_gpu on the revalued operands."""
    A, B, want, _ = unmasked_designed()
    blen = np.diff(B.ptr).astype(np.int64)
    bound = np.minimum(np.add.reduceat(blen[A.ind], A.ptr[:-1]), B.ncols)
    count = np.diff(want.ptr)
    assert list(zip(bound.tolist(), count.tolist())) == \
        [(min(u, B.ncols), d) for u, d in DESIGNED]
    for lim in SYM + NUM:
        assert {lim - 1, lim, lim + 1} <= set(bound.tolist()) | set(count.tolist())
    assert count.max() == B.ncols > 2*NUM[2]


def test_masked_operands_reach_every_class_and_route():
    """The classes, passes, segments and the heavy threshold of test_mxm_gpu, with
    large values in the mask beside its explicit zeros."""
    p, want, _ = masked_designed()
    r = routes(p)
    for ps in (1, 2):
        in_pass = r["pass_"] == ps
        assert set(LENS) - {0} <= set(r["owner_len"][in_pass].tolist())
        for cls in "SML":
            sel = in_pass & (r["cls"] == cls)
            c = CHUNK[cls]
            assert {c - 1, c, c + 1} <= set(r["partners"][sel].tolist()), (ps, cls)
            assert (r["mval"][sel] == 0).any() and (np.abs(r["mval"][sel]) > 2**24).any()
            assert (want.val[sel] != 0).any()
        assert set(r["nseg"][in_pass & (r["cls"] == "L")].tolist()) == {1, 2, 3}
    shorter = np.minimum(r["a_len"], r["b_len"])
    assert {HEAVY, HEAVY + 1} <= set(shorter.tolist())
    assert (want.val[shorter > HEAVY] != 0).any() and (want.val[shorter <= HEAVY] != 0).any()
    L, B, _ = triangles()
    assert (B.val != 0).sum() > 20


def test_ewise_straddling_pairs_cross_tile_and_thread_boundaries():
    for lead in (1, 3):
        A, B = ewise_case("straddling_%d" % lead, True)[:2]
        k = np.arange(B.nnz)
        a_pos, b_pos = lead + 2*k, lead + 2*k + 1
        assert ((a_pos // IPT) != (b_pos // IPT)).sum() >= B.nnz // IPT - 1
        assert ((a_pos // TILE) != (b_pos // TILE)).sum() >= 2


def test_assign_regions_cover_the_unsorted_path():
    regions = {name: (I, J) for name, I, J in assign_regions()}
    J = regions["unsorted"][1]
    assert not np.all(np.diff(J) > 0) and np.all(np.diff(regions["sorted"][1]) > 0)
    assert len(regions["row"][0]) == 1 and len(regions["column"][1]) == 1


def test_extract_lists_repeat_and_are_unsorted():
    cases = extract_cases()
    assert {t for t, _, _ in cases} == {False, True}
    rep = [I for _, I, _ in cases if I is not None and len(np.unique(I)) < len(I)]
    assert rep and any(not np.all(np.diff(I) >= 0) for I in rep)


def test_reduce_lengths_and_totals():
    src = open(os.path.join(CUDA, "kernels", "reduce.cuh")).read()
    assert int(re.search(r"#define GB_REDUCE_NT\s+(\d+)", src).group(1)) == REDUCE_NT
    assert "gridFor(nvals, GB_REDUCE_NT, 4)" in open(os.path.join(CUDA, "reduce.hpp")).read()
    cap = 4*H100_SMS
    grids = [min(-(-n // REDUCE_NT), cap) for n in reduce_lengths(H100_SMS)]
    assert {1, cap} <= set(grids) and max(-(-n // REDUCE_NT) for n in
                                          reduce_lengths(H100_SMS)) > 3*cap
    for n in reduce_lengths(H100_SMS):
        for total in TOTALS:
            v = reduce_values(n, total)
            assert len(v) == n and in_int32(v)
            assert v[v > 0].sum() <= I32_MAX and v[v < 0].sum() >= I32_MIN
            t = int(v.sum())
            if total == "max":
                assert t == I32_MAX and float(np.float32(t)) != t
            elif total == "min":
                assert t == I32_MIN
            else:
                assert t < -2**24 and t % 2 == 1 and float(np.float32(t)) != t


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------

def dev(gb, S, csc=True):
    return device_matrix(gb, S.astype(np.int32), csc=csc, integer=True)


def imatrix(gb, m, n):
    return gb.Matrix(m, n, dtype=gb.api.INT32)


def tran_desc(gb, field=None):
    desc = gb.Descriptor()
    if field is not None:
        desc.set(field, gb.Desc_value.GrB_TRAN)
    return desc


@pytest.mark.gpu
def test_unmasked_every_bin_limit(gb):
    A, B, want, _ = unmasked_designed()
    C = imatrix(gb, A.nrows, B.ncols)
    gb.mxm(C, None, None, gb.Semiring.PlusMultiplies, dev(gb, A), dev(gb, B), gb.Descriptor())
    check(C, want)


@pytest.mark.gpu
@pytest.mark.parametrize("tran", [None, "inp0", "inp1", "both"])
def test_unmasked_random_and_transposed(gb, tran):
    A, B, want, _ = unmasked_random(tran is not None)
    sA = A.T if tran in ("inp0", "both") else A
    sB = B.T if tran in ("inp1", "both") else B
    desc = gb.Descriptor()
    if tran in ("inp0", "both"):
        desc.set(gb.Desc_field.GrB_INP0, gb.Desc_value.GrB_TRAN)
    if tran in ("inp1", "both"):
        desc.set(gb.Desc_field.GrB_INP1, gb.Desc_value.GrB_TRAN)
    C = imatrix(gb, A.nrows, B.ncols)
    gb.mxm(C, None, None, gb.Semiring.PlusMultiplies, dev(gb, sA), dev(gb, sB), desc)
    check(C, want)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["hash", "search"])
def test_masked_designed(gb, route):
    p, want, _ = masked_designed()
    C = imatrix(gb, p.M.nrows, p.M.ncols)
    gb.mxm(C, dev(gb, p.M, csc=(route == "hash")), None, gb.Semiring.PlusMultiplies,
           dev(gb, p.A), dev(gb, p.Bt.T), gb.Descriptor())
    check(C, want)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["hash", "search"])
def test_triangle_count(gb, route):
    """algorithm.tc on a large-valued L: B entry by entry, and the returned scalar the
    int64 sum of B."""
    from graphblast_b200 import algorithm
    L, want, _ = triangles()
    dL = dev(gb, L, csc=(route == "hash"))
    B = imatrix(gb, L.nrows, L.nrows)
    for _ in range(2):
        total, _ = algorithm.tc(dL, B, gb.Descriptor(mxvmode=0))
        check(B, want)
        assert total == int(want.val.astype(np.int64).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("add", [True, False])
@pytest.mark.parametrize("name", EWISE)
def test_ewise(gb, name, add):
    A, B, want, _ = ewise_case(name, add)
    desc, sA, sB = gb.Descriptor(), A, B
    if name == "transposed":
        desc.set(gb.Desc_field.GrB_INP0 if add else gb.Desc_field.GrB_INP1,
                 gb.Desc_value.GrB_TRAN)
        sA, sB = (A.T, B) if add else (A, B.T)
    C = imatrix(gb, A.nrows, A.ncols)
    (gb.eWiseAdd if add else gb.eWiseMult)(C, None, None, gb.Semiring.PlusMultiplies,
                                           dev(gb, sA), dev(gb, sB), desc)
    check(C, want)


@pytest.mark.gpu
@pytest.mark.parametrize("accum", [False, True])
def test_assign(gb, accum):
    plus = gb.Monoid.Plus if accum else None
    cases = [(r[0], False) for r in assign_regions()] + [("unsorted", True)]
    for region, tran in cases:
        C, A, I, J, want, _ = assign_case(region, accum, tran)
        dC = dev(gb, C)
        gb.assign(dC, None, plus, dev(gb, A), I, ASSIGN_M if I is None else len(I), J,
                  ASSIGN_N if J is None else len(J),
                  tran_desc(gb, gb.Desc_field.GrB_INP0 if tran else None))
        check(dC, want)
    for val in SCALARS:
        C, I, J, want, _ = assign_scalar_case(val, accum)
        dC = dev(gb, C)
        gb.assign(dC, None, plus, val, I, len(I), J, len(J), gb.Descriptor())
        check(dC, want)


@pytest.mark.gpu
def test_extract(gb):
    S = extract_source()
    A = dev(gb, S)
    for tran, I, J in extract_cases():
        want = extract_want(S, I, J, tran)
        C = imatrix(gb, want.nrows, want.ncols)
        gb.extract(C, None, None, A, I, want.nrows, J, want.ncols,
                   tran_desc(gb, gb.Desc_field.GrB_INP0 if tran else None))
        check(C, want)


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["built", "adopted"])
def test_transpose_and_the_csc_in_a_product(gb, source):
    """The CSC of a matrix built from host COO (ingestCsrToCsc<int>) or adopted,
    read back through transpose and through an mxm with GrB_INP0 = GrB_TRAN."""
    S, r, c, v = build_tuples()
    A, B, want, _ = unmasked_random()
    if source == "built":
        M = imatrix(gb, S.nrows, S.ncols)
        M.build(r, c, v.astype(np.int32))
        At = imatrix(gb, A.ncols, A.nrows)
        rows = A.rows()
        order = np.random.RandomState(12).permutation(A.nnz)
        At.build(A.ind[order], rows[order], A.val[order].astype(np.int32))
    else:
        M, At = dev(gb, S), dev(gb, A.T)
    check(M, S)
    T = imatrix(gb, S.ncols, S.nrows)
    gb.transpose(T, None, None, M, gb.Descriptor())
    check(T, S.T)
    C = imatrix(gb, A.nrows, B.ncols)
    gb.mxm(C, None, None, gb.Semiring.PlusMultiplies, At, dev(gb, B),
           tran_desc(gb, gb.Desc_field.GrB_INP0))
    check(C, want)


@pytest.mark.gpu
def test_build_dedup_symmetrize_and_the_symmetric_form(gb):
    """Device COO with repeated positions (the first tuple wins, a forward tuple
    before a mirror) and symmetrised; then the same values through the host build
    marked undirected, whose CSC aliases the CSR."""
    import torch
    from graphblast_b200 import graphs
    n, r, c, v, want = dedup_tuples()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()
    dr, dc, dv = t(r), t(c), t(v)
    M = imatrix(gb, n, n)
    gb.api._check(M._lib.gb200_matrix_build_coo_device(
        M._h, gb.api._dev(dr), gb.api._dev(dc), gb.api._dev(dv), len(r),
        graphs.INGEST_DEDUP | graphs.INGEST_SYMMETRIZE), "build_coo_device")
    check(M, want)
    T = imatrix(gb, n, n)
    gb.transpose(T, None, None, M, gb.Descriptor())
    check(T, want.T)
    # the pattern is symmetric, so want.T lists the mirror of each entry in place
    Sym = want.with_values(np.where(want.rows() <= want.ind, want.val, want.T.val))
    assert np.array_equal(Sym.T.val, Sym.val)
    U = imatrix(gb, n, n)
    U.build(Sym.rows(), Sym.ind, Sym.val.astype(np.int32), undirected=True)
    check(U, Sym)
    gb.transpose(T, None, None, U, gb.Descriptor())
    check(T, Sym)


@pytest.mark.gpu
def test_reduce_totals_through_the_mailbox(gb):
    """PlusMonoid over every length and total, each matrix twice in a row and the
    totals one after another, so that every call takes a fresh mailbox ticket."""
    for n in reduce_lengths(gb.sm_count()):
        mats = [(reduce_values(n, total), total) for total in TOTALS]
        for v, total in mats:
            A = dev(gb, reduce_matrix_of(v), csc=False)
            want = int(v.sum())
            for _ in range(2):
                got = gb.reduce(None, gb.PlusMonoid, A, gb.Descriptor())
                assert got == want, (n, total, got, want)


def _pattern_outputs(gb, A, n, src):
    from graphblast_b200 import algorithm
    desc = gb.Descriptor
    out = {}
    for name, f in (("cc", algorithm.cc), ("scc", algorithm.scc)):
        v = gb.Vector(n)
        k, _ = f(v, A, desc())
        out[name] = (k, v.extractTuples().tobytes())
    for name, f in (("mis", algorithm.mis), ("gc", algorithm.gc)):
        v = gb.Vector(n)
        k, _ = f(v, A, 7, desc())
        out[name] = (k, v.extractTuples().tobytes())
    K = gb.Matrix(n, n)
    k, _ = algorithm.ktruss(K, A, 4, desc())
    out["ktruss"] = (k,) + tuple(x.tobytes() for x in K.extract_csr())
    K = gb.Matrix(n, n)
    k, _ = algorithm.trussness(K, A, desc())
    out["trussness"] = (k,) + tuple(x.tobytes() for x in K.extract_csr())
    v = gb.Vector(n)
    algorithm.bc(v, A, desc(), sources=range(0, n, 7))
    out["bc"] = v.extractTuples().tobytes()
    p, res = gb.Vector(n), gb.Vector(n)
    k, _ = algorithm.lgc(p, A, src, 0.15, 1e-6, desc(), residual=res)
    out["lgc"] = (k, p.extractTuples().tobytes(), res.extractTuples().tobytes())
    return out


@pytest.mark.gpu
def test_cooperative_algorithms_read_no_values(gb):
    rp, ci = orc.rmat_csr(9)
    n = len(rp) - 1
    extremes = np.resize(np.array([I32_MIN, -1, 0, I32_MAX], np.int32), len(ci))
    src = int(np.argmax(np.diff(rp)))
    got = _pattern_outputs(gb, device_matrix(gb, Csr(n, n, rp, ci, extremes), integer=True),
                           n, src)
    want = _pattern_outputs(gb, device_matrix(gb, Csr(n, n, rp, ci, np.ones(len(ci),
                                                                           np.float32))),
                            n, src)
    assert sorted(got) == sorted(want)
    for name in want:
        assert got[name] == want[name], name
