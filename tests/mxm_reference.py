"""Unmasked semiring product C = A (+.x) B on the CPU (test infrastructure only).

Gustavson, row by row: a dense accumulator over the columns of C and a record of
the columns touched; products are folded from the semiring's identity in
ascending k, mul taking A's value first.  The scalar operations restate the C
oracle's (oracle/gb_oracle.c: orc_add, orc_mul, orc_identity) with numpy float32
arithmetic, so that one entry of A costs one vector operation;
test_mxm_unmasked_oracle.py checks both against each other on every semiring.
C comes out as a sorted CSR: (rowptr, colind, val).
"""
import numpy as np

F32 = np.float32
FLT_MAX = F32(np.finfo(np.float32).max)
FLT_MIN = F32(np.finfo(np.float32).tiny)


def _flag(x):
    return x.astype(F32)


class _NanIgnoring(object):
    """np.fmin / np.fmax on operands multiplied by 1 first: numpy's fmin returns NaN
    for a signaling NaN operand, where fminf and the device's min ignore it as they
    ignore a quiet one.  x * 1 quiets a signaling NaN and leaves every other value,
    a zero's sign included, as it is."""

    def __init__(self, ufunc):
        self.ufunc = ufunc

    def __call__(self, a, b):
        return self.ufunc(_quiet(a), _quiet(b))

    def reduce(self, x):
        return self.ufunc.reduce(_quiet(x))

    def reduceat(self, x, at):
        return self.ufunc.reduceat(_quiet(x), at)


def _quiet(x):
    x = np.asarray(x)
    return x*x.dtype.type(1)


OPS = {
    "or": lambda a, b: _flag((a != 0) | (b != 0)),
    "and": lambda a, b: _flag((a != 0) & (b != 0)),
    "plus": lambda a, b: a + b,
    "minus": lambda a, b: a - b,
    "mul": lambda a, b: a * b,
    "div": lambda a, b: a / b,
    "min": _NanIgnoring(np.fmin),     # a NaN operand is ignored (fminf; ieee_reference)
    "max": _NanIgnoring(np.fmax),
    "gt": lambda a, b: _flag(a > b),
    "lt": lambda a, b: _flag(a < b),
    "ne": lambda a, b: _flag(a != b),
    "second": lambda a, b: b + np.zeros_like(a),
}

# (add, mul, identity) by semiring id (graphblast_b200.api.Semiring order)
SEMIRINGS = [
    ("or", "and", F32(0)),          # LogicalOrAnd
    ("plus", "mul", F32(0)),        # PlusMultiplies
    ("min", "plus", FLT_MAX),       # MinimumPlus
    ("max", "mul", F32(0)),         # MaximumMultiplies
    ("plus", "div", F32(0)),        # PlusDivides
    ("plus", "gt", F32(0)),         # PlusGreater
    ("gt", "plus", FLT_MIN),        # GreaterPlus
    ("plus", "minus", F32(0)),      # PlusMinus
    ("plus", "lt", F32(0)),         # PlusLess
    ("lt", "plus", FLT_MAX),        # CustomLessPlus
    ("min", "mul", FLT_MAX),        # MinimumMultiplies
    ("mul", "mul", F32(1)),         # MultipliesMultiplies
    ("ne", "plus", FLT_MAX),        # NotEqualToPlus
    ("min", "second", FLT_MAX),     # MinimumSelectSecond
    ("plus", "ne", F32(0)),         # PlusNotEqualTo
    ("lt", "lt", FLT_MAX),          # CustomLessLess
    ("min", "ne", FLT_MAX),         # MinimumNotEqualTo
]

# semirings whose add is not associative: the device refuses them
ORDER_DEPENDENT = (6, 9, 12, 15)


def mxm(semiring, a_ptr, a_ind, a_val, b_ptr, b_ind, b_val, ncols, integer=False):
    """C = A (+.x) B with A and B as CSR arrays.  integer=True: int plus-times in
    int64 (semiring must be PlusMultiplies)."""
    if integer:
        assert semiring == 1
        add, mul, ident = OPS["plus"], OPS["mul"], np.int64(0)
        a_val = np.asarray(a_val, np.int64)
        b_val = np.asarray(b_val, np.int64)
        dtype = np.int64
    else:
        add_name, mul_name, ident = SEMIRINGS[semiring]
        add, mul = OPS[add_name], OPS[mul_name]
        a_val = np.asarray(a_val, F32)
        b_val = np.asarray(b_val, F32)
        dtype = F32
    a_ptr, a_ind = np.asarray(a_ptr, np.int64), np.asarray(a_ind, np.int64)
    b_ptr, b_ind = np.asarray(b_ptr, np.int64), np.asarray(b_ind, np.int64)
    nrows = len(a_ptr) - 1
    acc = np.full(ncols, ident, dtype)
    rowptr = np.zeros(nrows + 1, np.int64)
    cols, vals = [], []
    with np.errstate(all="ignore"):
        for i in range(nrows):
            touched = []
            for e in range(a_ptr[i], a_ptr[i + 1]):
                k = a_ind[e]
                lo, hi = b_ptr[k], b_ptr[k + 1]
                if lo == hi:
                    continue
                cj = b_ind[lo:hi]
                acc[cj] = add(acc[cj], mul(np.full(hi - lo, a_val[e], dtype),
                                           b_val[lo:hi]))
                touched.append(cj)
            if touched:
                ci = np.unique(np.concatenate(touched))
                cols.append(ci)
                vals.append(acc[ci].copy())
                acc[ci] = ident
                rowptr[i + 1] = rowptr[i] + len(ci)
            else:
                rowptr[i + 1] = rowptr[i]
    colind = np.concatenate(cols) if cols else np.zeros(0, np.int64)
    val = np.concatenate(vals) if vals else np.zeros(0, dtype)
    return rowptr.astype(np.int64), colind.astype(np.int32), val
