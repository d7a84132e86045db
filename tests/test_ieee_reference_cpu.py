"""The FP32 contract of ieee_reference.py on closed forms, the designed operands of
test_ieee_values_gpu.py checked for what they are meant to hold, and the
comparison shown to reject an FTZ, a fused and a ternary-min reference on them."""
import numpy as np
import pytest

import ewise_reference as eref
import ieee_reference as ieee
import mxm_reference as mref
import oracle_binding as orc
import test_ieee_values_gpu as V
from ieee_reference import (BIG, F32, FLT_MAX, INF, MAX_SUB, NAN, NEG_NAN, NEG_ZERO,
                            ONE_EPS, TINY)

PLUS, MINPLUS, MAXMUL, MINSECOND = 1, 2, 3, 13


def test_closed_forms():
    fmin, fmax = mref.OPS["min"], mref.OPS["max"]
    for nan in (NAN, NEG_NAN):
        assert fmin(nan, F32(1)) == 1 and fmin(F32(-2), nan) == -2
        assert fmax(nan, F32(1)) == 1 and fmax(F32(-2), nan) == -2
        assert np.isnan(fmin(nan, nan)) and np.isnan(fmax(nan, nan))
    with np.errstate(all="ignore"):
        assert np.isnan(INF + -INF) and np.isnan(F32(0)*INF)
    assert ieee.bits(TINY + TINY) == 2 and ieee.is_subnormal(TINY + TINY)
    assert ieee.bits(MAX_SUB + TINY) == ieee.bits(mref.FLT_MIN)
    # the overflow edge: unfused inf, fused 2^104
    S, u = V.pull_operands()
    pair = lambda a1, a2: (np.array([0, 2]), np.array([0, 1]), F32([a1, a2]))
    ptr, ind, val = pair(-FLT_MAX, BIG)
    uu = F32([1, BIG])
    assert ieee.pull(PLUS, ptr, ind, val, uu)[0] == INF
    assert ieee.fused_fold(ptr, ind, val, uu)[0] == F32(2.0**104)
    # two inexact products of opposite sign: unfused 0, fused -2^-24
    ptr, ind, val = pair(ONE_EPS, -ONE_EPS)
    uu = F32([ONE_EPS, ONE_EPS])
    assert ieee.pull(PLUS, ptr, ind, val, uu)[0] == 0
    assert ieee.fused_fold(ptr, ind, val, uu)[0] == F32(-2.0**-24)


def test_fma32_rounds_once():
    assert ieee.fma32(F32(1), F32(1), F32(2.0**-24)) == F32(1)       # tie to even
    assert ieee.fma32(F32(1), F32(1), F32(2.0**-24 + 2.0**-40)) == F32(1 + 2.0**-23)
    assert ieee.fma32(TINY, F32(0.5), F32(0)) == 0                   # 2^-150: tie to 0
    assert ieee.fma32(MAX_SUB, F32(1), TINY) == mref.FLT_MIN
    assert ieee.fma32(FLT_MAX, F32(2), F32(0)) == INF


def test_oracle_min_and_max_ignore_nan():
    """orc_add's OP_MIN / OP_MAX are fminf / fmaxf, as the device's min / max."""
    lib = orc.lib()
    for sem, op in ((MINPLUS, mref.OPS["min"]), (MAXMUL, mref.OPS["max"])):
        for a, b in ((NAN, F32(3)), (F32(3), NAN), (NEG_NAN, F32(-3)), (F32(-3), NEG_NAN),
                     (F32(1), F32(2)), (INF, -INF)):
            got = F32(lib.orc_add(sem, float(a), float(b)))
            assert got == op(a, b), (sem, a, b, got)
        assert np.isnan(lib.orc_add(sem, float(NAN), float(NEG_NAN)))


def test_masks_and_the_identity_test():
    import mxv_reference as vref
    m = F32([NAN, NEG_NAN, NEG_ZERO, 0, TINY])
    assert list(vref._kept(m, False)) == [True, True, False, False, True]
    # the push's identity short-circuit is ==: -0.0 short-circuits under 0, NaN never
    w_ind, w_val = vref.push(PLUS, np.array([0, 3]), np.array([0, 1, 2]),
                             F32([INF, INF, INF]), [0], [NEG_ZERO], 3)
    assert list(w_val) == [0, 0, 0]
    w_ind, w_val = vref.push(PLUS, np.array([0, 3]), np.array([0, 1, 2]),
                             F32([INF, 1, -INF]), [0], [NAN], 3)
    assert np.isnan(w_val).all()


# ---------------------------------------------------------------------------
# the designed cases: name -> (inputs, reference outputs, reference under a mutant)
# ---------------------------------------------------------------------------

def _pull(sem):
    S, u = V.pull_operands()
    return (S.val, u), lambda: V.pull_want(sem, S, u)


def _push(sem):
    S, u = V.pull_operands()
    return (S.val, u), lambda: V.push_want(sem, S, u)[1]


def _unmasked(sem):
    A, B = V.unmasked_operands()
    return (A.val, B.val), lambda: V.mxm_want(sem, A, B).val


def _spmm(n, sem):
    A, B = V.spmm_operands(n)
    return (A.val, B), lambda: V.spmm_want(sem, A, B)


def _ewise(name, sem):
    A, B = V.ewise_operands(name)
    return (A.val, B.val), lambda: V.ewise_want(True, sem, A, B).val


def _reduce():
    xs = [V.reduce_input(k, n) for k in sorted(V.REDUCE_SETS) for n in V.REDUCE_LENGTHS]
    return tuple(xs), lambda: F32([V.reduce_want(m, x) for x in xs for m in (0, 2, 3)])


CASES = {"pull_plus": lambda: _pull(PLUS), "pull_minplus": lambda: _pull(MINPLUS),
         "pull_maxmul": lambda: _pull(MAXMUL), "push_plus": lambda: _push(PLUS),
         "push_maxmul": lambda: _push(MAXMUL), "push_minsecond": lambda: _push(MINSECOND),
         "unmasked_plus": lambda: _unmasked(PLUS), "unmasked_maxmul": lambda: _unmasked(MAXMUL),
         "reduce": _reduce}
for _n in V.SPMM_WIDTHS:
    CASES["spmm_%d_plus" % _n] = (lambda n: lambda: _spmm(n, PLUS))(_n)
for _name in V.EWISE_CASES:
    CASES["ewise_%s_plus" % _name] = (lambda n: lambda: _ewise(n, PLUS))(_name)
    CASES["ewise_%s_minplus" % _name] = (lambda n: lambda: _ewise(n, MINPLUS))(_name)
# (case, mutant) pairs the comparison must reject: the FTZ mutant wherever subnormal
# arithmetic happens, the ternary one wherever a min or max meets a NaN
MUTANTS = ([(c, "ftz") for c in sorted(CASES) if c.endswith("plus") and "minplus" not in c
            and c != "ewise_disjoint_plus"] +                # no arithmetic there
           [(c, "ternary") for c in ("pull_minplus", "pull_maxmul", "push_maxmul",
                                     "push_minsecond", "unmasked_maxmul")] +
           [(c, "ternary") for c in sorted(CASES) if c.startswith("ewise_")
            and c.endswith("minplus") and "disjoint" not in c])


@pytest.mark.parametrize("name", sorted(CASES))
def test_every_case_holds_every_special(name):
    inputs, _ = CASES[name]()
    for special in ieee.SPECIALS:
        assert any(ieee.holds(x, special) for x in inputs), (name, special)


@pytest.mark.parametrize("name", sorted(CASES))
def test_every_case_has_a_subnormal_output(name):
    _, want = CASES[name]()
    assert ieee.is_subnormal(want()).any(), name


def test_fixed_point_folds_stay_exact():
    """Every plus fold of the designed finite products stays below 2^-125 (in units
    of 2^-149: below 2^24), so that any order of it is exact."""
    S, u = V.pull_operands()
    fin = np.isfinite(S.val) & (np.abs(S.val) < 2.0**-100)
    unit = fin & np.isfinite(u[S.ind]) & (np.abs(u[S.ind]) <= 4)
    prods = np.where(unit, np.abs(np.where(unit, S.val, 0).astype(np.float64)*
                                  np.where(unit, u[S.ind], 0)), 0)
    sums = np.add.reduceat(prods, S.ptr[:-1][np.diff(S.ptr) > 0])
    assert sums.max() < ieee.FIXED_LIMIT
    A, B = V.unmasked_operands()
    small = lambda v: np.where(np.isfinite(v) & (np.abs(v) <= 4), np.abs(v), 0).astype(F32)
    bound = V.mxm_want(PLUS, A.with_values(small(A.val)),
                       B.with_values(np.where(np.abs(B.val) < 2.0**-140, np.abs(B.val), 0)))
    assert bound.val.max() < ieee.FIXED_LIMIT
    for n in V.SPMM_WIDTHS:
        A, B = V.spmm_operands(n)
        a = np.where(np.abs(A.val) < 2.0**-140, np.abs(A.val), 0).astype(np.float64)
        row = np.add.reduceat(a, A.ptr[:-1][np.diff(A.ptr) > 0])
        assert 4*row.max() < ieee.FIXED_LIMIT


def test_pair_folds_are_designed():
    """An overflowing product beside -FLT_MAX, and two inexact products of opposite
    sign, in the pull operand and in the mxm / SpMM pair rows."""
    S, u = V.pull_operands()
    found = set()
    for i in range(S.nrows):
        lo, hi = S.ptr[i], S.ptr[i + 1]
        terms = list(zip(S.val[lo:hi], u[S.ind[lo:hi]]))
        if len(terms) == 2:
            if (-FLT_MAX, 1) in terms and (BIG, BIG) in terms:
                found.add("overflow")
            if (ONE_EPS, ONE_EPS) in terms and (-ONE_EPS, ONE_EPS) in terms:
                found.add("contraction")
    assert found == {"overflow", "contraction"}
    assert (F32(1), BIG) in V.PAIR_A and V.B1[0] == -FLT_MAX and V.B2[0] == BIG
    assert (ONE_EPS, -ONE_EPS) in V.PAIR_A and V.B1[1] == V.B2[1] == ONE_EPS


def _mutant_want(name, mutant):
    _, want = CASES[name]()
    with ieee.ops(ieee.FTZ if mutant == "ftz" else ieee.TERNARY):
        return want()


@pytest.mark.parametrize("name,mutant", MUTANTS)
def test_the_comparison_rejects_the_mutant(name, mutant):
    _, want = CASES[name]()
    w = want()
    assert ieee.agree(w, w).all()
    bad = _mutant_want(name, mutant)
    minmax = mutant == "ternary"
    assert not ieee.agree(bad, w, minmax).all(), (name, mutant)
    with pytest.raises(pytest.fail.Exception):
        ieee.check(bad, w, minmax)


def test_the_comparison_rejects_the_fused_mutant():
    S, u = V.pull_operands()
    pairs = np.nonzero(np.diff(S.ptr) == 2)[0]
    sub = np.concatenate([np.arange(S.ptr[i], S.ptr[i + 2 - 1 + 1]) for i in pairs])
    ptr = np.arange(0, 2*len(pairs) + 1, 2)
    want = ieee.pull(PLUS, ptr, S.ind[sub], S.val[sub], u)
    fused = ieee.fused_fold(ptr, S.ind[sub], S.val[sub], u)
    assert not ieee.agree(fused, want).all()
    with pytest.raises(pytest.fail.Exception):
        ieee.check(fused, want)
    # the mxm pair rows: C(P1, 0) = 1 * -FLT_MAX + 2^64 * 2^64, C(P2, 1) = 0
    A, B = V.unmasked_operands()
    C = V.mxm_want(PLUS, A, B)
    m = A.nrows - len(V.PAIR_A)
    at = lambda i, j: C.val[C.ptr[i] + np.searchsorted(C.ind[C.ptr[i]:C.ptr[i + 1]], j)]
    assert at(m, 0) == INF and at(m + 1, 1) == 0
    assert ieee.fma32(BIG, BIG, -FLT_MAX) == F32(2.0**104)
    assert ieee.fma32(-ONE_EPS, ONE_EPS, ieee.fma32(ONE_EPS, ONE_EPS, F32(0))) != 0


def test_reduce_reference_ignores_nan_under_min_and_max():
    x = F32([NAN, 3, NEG_NAN, ieee.PAYLOAD_NAN, -1, TINY])
    assert mref.OPS["min"](ieee.PAYLOAD_NAN, NEG_ZERO) == 0       # signaling: ignored too
    assert eref.reduce(2, x)[0] == -1 and eref.reduce(3, x)[0] == 3
    assert eref.reduce(3, F32([NAN, NEG_NAN]))[0] == 0       # fmax(identity 0, NaN)
