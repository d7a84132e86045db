"""Element-wise union / intersection of two sparse matrices on the CPU (test
infrastructure only).

C = A (+) B: the union of the two patterns; where both hold an entry the
semiring's ADD of (a, b), A's value first; where one does, that value unchanged.
C = A (x) B: the intersection, the semiring's MUL of (a, b), A's value first.
The scalar operations are mxm_reference's OPS / SEMIRINGS, which
test_mxm_unmasked_oracle.py pins to the C oracle.  Nothing is pruned: stored
zeros and results equal to 0 or NaN stay.  C comes out as a sorted CSR:
(rowptr, colind, val).
"""
import numpy as np

from mxm_reference import F32, OPS, SEMIRINGS


def _keys(ptr, ind, ncols):
    ptr = np.asarray(ptr, np.int64)
    rows = np.repeat(np.arange(len(ptr) - 1, dtype=np.int64), np.diff(ptr))
    return rows*max(ncols, 1) + np.asarray(ind, np.int64)


def ewise(add, semiring, a_ptr, a_ind, a_val, b_ptr, b_ind, b_val, ncols,
          integer=False):
    """add=True: A (+) B, add=False: A (x) B, A and B as CSR arrays of one shape.
    integer=True: int plus-times in int64 (semiring must be PlusMultiplies)."""
    if integer:
        assert semiring == 1
        f = OPS["plus"] if add else OPS["mul"]
        dtype = np.int64
    else:
        add_name, mul_name, _ = SEMIRINGS[semiring]
        f = OPS[add_name] if add else OPS[mul_name]
        dtype = F32
    a_val = np.asarray(a_val, dtype)
    b_val = np.asarray(b_val, dtype)
    ka, kb = _keys(a_ptr, a_ind, ncols), _keys(b_ptr, b_ind, ncols)
    keys = np.union1d(ka, kb) if add else np.intersect1d(ka, kb)
    ia = np.searchsorted(ka, keys)
    ib = np.searchsorted(kb, keys)
    in_a = ia < len(ka)
    in_a[in_a] = ka[ia[in_a]] == keys[in_a]
    in_b = ib < len(kb)
    in_b[in_b] = kb[ib[in_b]] == keys[in_b]
    both = in_a & in_b
    val = np.zeros(len(keys), dtype)
    val[in_a & ~in_b] = a_val[ia[in_a & ~in_b]]
    val[in_b & ~in_a] = b_val[ib[in_b & ~in_a]]
    with np.errstate(all="ignore"):
        val[both] = f(a_val[ia[both]], b_val[ib[both]])
    nrows = len(a_ptr) - 1
    rows = keys // max(ncols, 1)
    rowptr = np.zeros(nrows + 1, np.int64)
    np.cumsum(np.bincount(rows, minlength=nrows), out=rowptr[1:])
    return rowptr, (keys % max(ncols, 1)).astype(np.int32), val
