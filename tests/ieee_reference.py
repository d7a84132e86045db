"""The FP32 contract every route keeps, and the comparison that checks it (test
infrastructure only).

  * min and max ignore a NaN operand (fminf / fmaxf, np.fmin / np.fmax); if both
    operands are NaN the result is NaN.  The sign of a min or max of +0 and -0 is
    not specified: there, and only there, +-0 compare equal.
  * Every other operation is IEEE binary32 with round-to-nearest: subnormals are
    kept (no flush to zero) and every product is rounded before it is added (no
    multiply-add contraction), on every route.  A fold starts from the identity,
    so a plus fold of zeros is +0.
  * Values no arithmetic touches keep their exact bits, a NaN's payload and sign
    and the sign of a zero included: host and device builds and extractTuples
    (ingest keeps the first of duplicate tuples), extract, assign without accum,
    transpose and dup, the entries sparse2dense / dense2sparse keep, eWiseAdd's
    entries outside the overlap, a dense -> sparse round trip.
  * A NaN that arithmetic produces is compared as "is NaN": the device's canonical
    NaN (0x7fffffff) and x86's (0xffc00000) differ in payload and sign.
  * Masks treat NaN as nonzero and -0.0 as zero, in the value form and in the
    bitmap shadow.  The push's identity short-circuit is an == test, so a NaN never
    short-circuits.

A signaling NaN (PAYLOAD_NAN) is a NaN like any other: min and max ignore it too,
and arithmetic gives some quiet NaN.

The route references (mxm_reference, mxv_reference, ewise_reference) share one ops
table, mxm_reference.OPS, whose min and max are np.fmin / np.fmax.  ops() swaps
that table for the length of a with-block, which is how the CPU tests build the
mutants the comparison must reject: FTZ, TERNARY (min / max as a < b ? a : b) and,
for plus-times folds, fused_fold (a*b + c rounded once).
"""
import contextlib
import fractions

import numpy as np
import pytest

import mxm_reference as mref
import mxv_reference as vref

F32 = np.float32
FLT_MAX = mref.FLT_MAX
FLT_MIN = mref.FLT_MIN


def f32(bits):
    return np.asarray(bits, np.uint32).view(F32)


NAN = f32(0x7fc00000)           # numpy's np.nan, the device's NaN of a quiet input
NEG_NAN = f32(0xffc00000)       # x86's default NaN (numpy's 0/0)
PAYLOAD_NAN = f32(0x7fa00001)   # a payload no arithmetic produces
TINY = f32(0x00000001)          # 2^-149, the smallest subnormal
MAX_SUB = f32(0x007fffff)       # the largest subnormal
INF = F32(np.inf)
NEG_ZERO = F32(-0.0)
SPECIALS = {"nan": NAN, "-nan": NEG_NAN, "inf": INF, "-inf": -INF, "-0": NEG_ZERO,
            "tiny": TINY, "max_sub": MAX_SUB, "flt_max": FLT_MAX}
# a product that overflows: 2^64 * 2^64 beside a partial sum of -FLT_MAX (unfused inf,
# fused about 2^104); and two inexact products of opposite sign (unfused 0, fused
# +-2^-24): (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24 rounds to 1 + 2^-11
BIG = F32(2.0**64)
ONE_EPS = F32(1 + 2.0**-12)
# |partial sums| below this, of multiples of 2^-149, are exact in any order
FIXED_LIMIT = 2.0**-125


def bits(x):
    return np.asarray(x, F32).view(np.uint32)


def is_subnormal(x):
    x = np.asarray(x, F32)
    return (x != 0) & (np.abs(x) < FLT_MIN)


def holds(x, name):
    """x (any float32 array) contains the special value `name`, by its bits, or, for
    the NaNs, a NaN of that sign."""
    x = np.asarray(x, F32).ravel()
    if name in ("nan", "-nan"):
        return bool((np.isnan(x) & (np.signbit(x) == (name == "-nan"))).any())
    return bool((bits(x) == bits(SPECIALS[name])).any())


# ---------------------------------------------------------------------------
# the comparison
# ---------------------------------------------------------------------------

def agree(got, want, minmax=False):
    """Entry by entry: equal bits, both NaN, or (minmax) both zero."""
    g, w = np.asarray(got, F32), np.asarray(want, F32)
    ok = (bits(g) == bits(w)) | (np.isnan(g) & np.isnan(w))
    if minmax:
        ok |= (g == 0) & (w == 0)
    return ok


def check(got, want, minmax=False, where=""):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, "%s: shape %r, want %r" % (where, got.shape, want.shape)
    ok = agree(got, want, minmax)
    if not ok.all():
        i = int(np.argmin(ok.ravel()))
        pytest.fail("%s: %d of %d differ, first at %d: got %r (0x%08x) want %r (0x%08x)" % (
            where, int((~ok).sum()), ok.size, i, got.ravel()[i], bits(got).ravel()[i],
            want.ravel()[i], bits(want).ravel()[i]))


def check_bits(got, want, where=""):
    """Carried values: every bit, NaN payloads and zero signs included."""
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, where
    bad = np.nonzero(bits(got) != bits(want))[0]
    if len(bad):
        i = bad[0]
        pytest.fail("%s: %d of %d differ in their bits, first at %d: 0x%08x want 0x%08x" % (
            where, len(bad), got.size, i, bits(got)[i], bits(want)[i]))


def check_csr(C, want, minmax=False, where=""):
    rp, ci, val = C.extract_csr()
    assert np.array_equal(rp, want.ptr), "%s: row offsets differ" % where
    assert np.array_equal(ci, want.ind), "%s: column indices differ" % where
    check(val, want.val, minmax, where)


def is_minmax(semiring):
    return mref.SEMIRINGS[semiring][0] in ("min", "max")


# ---------------------------------------------------------------------------
# references under the contract
# ---------------------------------------------------------------------------

def pull(semiring, ptr, ind, val, u, **kw):
    """mxv_reference.pull as float32, for operands whose folds every order rounds
    alike (plus folds of multiples of 2^-149 below FIXED_LIMIT, NaN and inf, or two
    terms): the exact float64 sum rounded once, from the identity +0."""
    w, bound = vref.pull(semiring, ptr, ind, val, u, **kw)
    if bound is not None:
        with np.errstate(all="ignore"):
            w = (w + 0.0).astype(F32)
    return w


# ---------------------------------------------------------------------------
# the mutants
# ---------------------------------------------------------------------------

def ftz(x):
    x = np.asarray(x, F32)
    return np.where(is_subnormal(x), np.copysign(F32(0), x), x).astype(F32)


def _flushing(op):
    return lambda a, b: ftz(op(ftz(a), ftz(b)))


FTZ = {k: _flushing(op) for k, op in mref.OPS.items()}
TERNARY = dict(mref.OPS, min=lambda a, b: np.where(a < b, a, b).astype(F32),
               max=lambda a, b: np.where(a > b, a, b).astype(F32))
TERNARY["min"].reduceat = lambda x, at: np.minimum.reduceat(x, at)
TERNARY["max"].reduceat = lambda x, at: np.maximum.reduceat(x, at)
TERNARY["min"].reduce = np.minimum.reduce
TERNARY["max"].reduce = np.maximum.reduce


@contextlib.contextmanager
def ops(table):
    """Every route reference computes with `table` inside the block."""
    saved = dict(mref.OPS)
    mref.OPS.update(table)
    try:
        yield
    finally:
        mref.OPS.update(saved)


def fma32(a, b, c):
    """a*b + c rounded once to float32 (Python 3.12 has no math.fma)."""
    a, b, c = F32(a), F32(b), F32(c)
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        with np.errstate(all="ignore"):
            return F32(np.float64(a)*np.float64(b) + np.float64(c))
    exact = fractions.Fraction(float(a))*fractions.Fraction(float(b)) + \
        fractions.Fraction(float(c))
    # float64 holds a*b exactly only if it fits 48 bits: round through Fraction
    return _round32(exact)


def _round32(q):
    """The float32 nearest the rational q, ties to even, overflow to inf."""
    if q == 0:
        return F32(0.0)
    sign = -1 if q < 0 else 1
    q = abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    while fractions.Fraction(2)**e > q:
        e -= 1
    while fractions.Fraction(2)**(e + 1) <= q:
        e += 1
    e = max(e, -126)
    ulp = fractions.Fraction(2)**(e - 23)
    m = q/ulp
    n = int(m)
    rem = m - n
    if rem > fractions.Fraction(1, 2) or (rem == fractions.Fraction(1, 2) and n % 2):
        n += 1
    v = n*ulp
    if v >= fractions.Fraction(2)**128:
        return F32(sign*np.inf)
    return F32(sign*float(v))


def fused_fold(ptr, ind, val, u):
    """The plus-times pull with every product fused into its add, rows in order
    from the identity +0."""
    out = np.zeros(len(ptr) - 1, F32)
    for i in range(len(ptr) - 1):
        acc = F32(0)
        for e in range(ptr[i], ptr[i + 1]):
            acc = fma32(val[e], u[ind[e]], acc)
        out[i] = acc
    return out
