"""eWiseAdd, eWiseMult, assign, reduce and the vector conversions on the CPU, one
function per device route (test infrastructure only).

The scalar operations are the OPS / SEMIRINGS tables of mxm_reference.py (numpy
float32, checked against the C oracle there); MONOIDS below adds the monoids with
the identities include/graphblas/stddef.hpp gives them.  Those identities are
the reference's, quirks included: Maximum and LogicalAnd start from 0, Greater
from FLT_MIN (the smallest positive normal, not the lowest value).  Every device
fold starts from the identity, so max over all-negative values is 0 and a
LogicalAnd reduction is always 0.  test_ewise_reference_cpu.py checks the
tables against the oracle and pins these quirks; test_ewise_gpu.py runs every
route against the functions here.

Sparse vectors are (ind, val) pairs with sorted indices; dense ones float32 arrays.

  ewise_add_dense / _sparse_dense / _scalar_*   ewiseadd.hpp, kernels/elementwise.cuh
  ewise_mult_dense / _sparse_mask / _sparse_dense / _sparse_dense_sparse_mask
                                                ewisemult.hpp, kernels/elementwise.cuh
  scale_csr / scale_rows / scale_cols           matrix (x) scalar / broadcast vector
  assign_dense / assign_dense_sparse_mask / assign_sparse    assign.hpp
  reduce                                        reduce.hpp, kernels/reduce.cuh
  dense2sparse / sparse2dense / convert         vector.hpp, kernels/compact.cuh
"""
import numpy as np

from mxm_reference import F32, FLT_MAX, FLT_MIN, OPS, SEMIRINGS

# (op, identity) by monoid id (graphblast_b200.api.Monoid order)
MONOIDS = [
    ("plus", F32(0)),        # Plus
    ("mul", F32(1)),         # Multiplies
    ("min", FLT_MAX),        # Minimum
    ("max", F32(0)),         # Maximum: identity 0, not -FLT_MAX
    ("or", F32(0)),          # LogicalOr
    ("and", F32(0)),         # LogicalAnd: identity false, so every fold gives 0
    ("gt", FLT_MIN),         # Greater: numeric_limits<float>::min()
    ("lt", FLT_MAX),         # CustomLess
    ("ne", FLT_MAX),         # NotEqualTo
]

# Monoids whose operator is neither associative nor commutative: the device's
# tree fold gives an answer that depends on the grid, so the tests check them only
# where no fold runs (an empty input returns the identity).
ORDER_DEPENDENT_MONOIDS = (6, 7, 8)


def _add(semiring):
    return OPS[SEMIRINGS[semiring][0]]


def _mul(semiring):
    return OPS[SEMIRINGS[semiring][1]]


def _ident(semiring):
    return SEMIRINGS[semiring][2]


def _f(x):
    return np.asarray(x, F32)


def densify(n, ind, val, fill):
    w = np.full(n, fill, F32)
    w[np.asarray(ind, np.int64)] = _f(val)
    return w


# ---- eWiseAdd (always a dense result) ------------------------------------------

def ewise_add_dense(semiring, u, v):
    """dense (+) dense: w[i] = add(u[i], v[i])."""
    with np.errstate(all="ignore"):
        return _add(semiring)(_f(u), _f(v))


def ewise_add_sparse_dense(semiring, ind, val, v, reverse=False, w_is_v=False):
    """sparse u (+) dense v.  First every w[i] = add(v[i], id), or add(id, v[i])
    when the dense operand came first (reverse); then at u's stored positions
    w[j] = add(u_val, v[j]), always in (sparse, dense) order.  That second pass
    reads the original v unless w is v, which the first pass has rewritten."""
    add, ident = _add(semiring), _ident(semiring)
    v = _f(v)
    ind = np.asarray(ind, np.int64)
    with np.errstate(all="ignore"):
        w = add(np.full_like(v, ident), v) if reverse else add(v, np.full_like(v, ident))
        src = w if w_is_v else v
        w[ind] = add(_f(val), src[ind])
    return w


def ewise_add_aliased_sparse(semiring, n, ind, val, other, w_is_first=True):
    """w (+) other where w is a sparse operand: w is densified with the
    semiring's identity first, then dense (+) dense."""
    wd = densify(n, ind, val, _ident(semiring))
    return ewise_add_dense(semiring, wd, other) if w_is_first else \
        ewise_add_dense(semiring, other, wd)


def ewise_add_scalar_dense(semiring, u, s):
    with np.errstate(all="ignore"):
        return _add(semiring)(_f(u), np.full(len(u), s, F32))


def ewise_add_scalar_sparse(semiring, n, ind, val, s):
    """w = add(id, s) everywhere, then w[j] = add(u_val, w[j]) at u's entries."""
    add = _add(semiring)
    ind = np.asarray(ind, np.int64)
    with np.errstate(all="ignore"):
        w = np.full(n, add(np.float32([_ident(semiring)]), np.float32([s]))[0], F32)
        w[ind] = add(_f(val), w[ind])
    return w


# ---- eWiseMult ---------------------------------------------------------------------

def ewise_mult_dense(semiring, u, v, mask=None):
    """dense (x) dense: the identity wherever either operand is the identity
    (no product), else mul(u, v); under a dense mask the identity where the mask
    is 0."""
    mul, ident = _mul(semiring), _ident(semiring)
    u, v = _f(u), _f(v)
    with np.errstate(all="ignore"):
        w = np.where((u == ident) | (v == ident), ident, mul(u, v)).astype(F32)
    if mask is not None:
        w[_f(mask) == 0] = ident
    return w


def ewise_mult_dense_sparse_mask(semiring, u, v, m_ind, m_val):
    """dense (x) dense under a sparse mask: the mask's pattern; mul(u, v) where
    the mask value is nonzero, 0 (not the identity) where it is 0, and no
    identity short-circuit."""
    m_ind = np.asarray(m_ind, np.int64)
    with np.errstate(all="ignore"):
        prod = _mul(semiring)(_f(u)[m_ind], _f(v)[m_ind])
    return m_ind, np.where(_f(m_val) != 0, prod, F32(0)).astype(F32)


def ewise_mult_sparse_dense(semiring, ind, val, v, reverse=False, mask=None):
    """sparse u (x) dense v: u's pattern; mul(u, v), or mul(v, u) under reverse;
    0 where u holds the identity; under a dense mask the identity where the mask
    is 0 (the entry stays)."""
    mul, ident = _mul(semiring), _ident(semiring)
    ind = np.asarray(ind, np.int64)
    a, b = _f(val), _f(v)[ind]
    with np.errstate(all="ignore"):
        prod = mul(b, a) if reverse else mul(a, b)
    w = np.where(a != ident, prod, F32(0)).astype(F32)
    if mask is not None:
        w[_f(mask)[ind] == 0] = ident
    return ind, w


def ewise_mult_sparse_dense_sparse_mask(semiring, ind, val, v, m_ind, m_val,
                                        reverse=False):
    """sparse u (x) dense v under a sparse mask: the mask's pattern; an entry is
    mul(u, v) where the mask value is nonzero, v is not the identity and u
    stores that index (binary search in u's sorted indices), 0 elsewhere."""
    mul, ident = _mul(semiring), _ident(semiring)
    ind = np.asarray(ind, np.int64)
    m_ind = np.asarray(m_ind, np.int64)
    v = _f(v)
    at = np.searchsorted(ind, m_ind)
    found = at < len(ind)
    found[found] = ind[at[found]] == m_ind[found]
    a = np.zeros(len(m_ind), F32)
    a[found] = _f(val)[at[found]]
    b = v[m_ind]
    with np.errstate(all="ignore"):
        prod = mul(b, a) if reverse else mul(a, b)
    live = (_f(m_val) != 0) & (b != ident) & found
    return m_ind, np.where(live, prod, F32(0)).astype(F32)


def scale_csr(semiring, val, s):
    """matrix (x) scalar: every stored value becomes mul(a, s)."""
    with np.errstate(all="ignore"):
        return _mul(semiring)(_f(val), np.full(len(val), s, F32))


def scale_rows(semiring, ptr, val, b):
    """matrix (x) column vector: A(i, j) = mul(A(i, j), b[i])."""
    rows = np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
    with np.errstate(all="ignore"):
        return _mul(semiring)(_f(val), _f(b)[rows])


def scale_cols(semiring, ind, val, b):
    """matrix (x) row vector: A(i, j) = mul(A(i, j), b[j])."""
    with np.errstate(all="ignore"):
        return _mul(semiring)(_f(val), _f(b)[np.asarray(ind, np.int64)])


# ---- assign --------------------------------------------------------------------------

def selected(mask, scmp):
    """Positions a dense mask selects: nonzero ones, zero ones under GrB_SCMP."""
    nz = _f(mask) != 0
    return ~nz if scmp else nz


def assign_dense(w, mask, val, scmp=False):
    """Dense target, dense mask (read as values or as its bitmap shadow)."""
    w = _f(w).copy()
    w[selected(mask, scmp)] = val
    return w


def assign_dense_sparse_mask(w, m_ind, val):
    """Dense target, sparse mask: every stored mask index is written, whatever
    the mask value there (GrB_SCMP is refused and changes nothing)."""
    w = _f(w).copy()
    w[np.asarray(m_ind, np.int64)] = val
    return w


def assign_sparse(ind, val, mask, v, scmp=False):
    """Sparse target, dense mask: a masked delete.  Entries the mask selects and
    entries equal to v are dropped; the rest keep their order."""
    ind = np.asarray(ind, np.int64)
    val = _f(val)
    keep = ~selected(_f(mask)[ind], scmp) & (val != F32(v))
    return ind[keep], val[keep]


# ---- reduce --------------------------------------------------------------------------

def reduce(monoid, x):
    """Fold of x from the monoid's identity.  Returns (value, bound): for Plus
    the float64 sum and the float32 fold's bound (n + 1) 2^-24 sum |x|; for the
    others a float32 value and bound None (exact: min / max / or / and in any
    order, Multiplies on powers of two).  Order-dependent monoids are defined here
    only on empty input."""
    op, ident = MONOIDS[monoid]
    x = _f(x)
    if len(x) == 0:
        return F32(ident), None
    if monoid in ORDER_DEPENDENT_MONOIDS:
        raise ValueError("order-dependent monoid %d: defined on empty input only" % monoid)
    if op == "plus":
        x64 = x.astype(np.float64)
        return float(x64.sum()), (len(x) + 1)*2.0**-24*float(np.abs(x64).sum())
    if op == "mul":
        return F32(np.prod(x.astype(np.float64))), None
    if op in ("min", "max"):
        return F32(OPS[op](F32(ident), OPS[op].reduce(x))), None   # NaN ignored
    if op == "or":
        return F32(bool(np.any(x != 0))), None
    return F32(0), None                            # and: and(false, ...) is false


def reduce_rows(monoid, ptr, val):
    """w[i] = reduce(monoid, row i); every row, empty ones give the identity.
    Returns (w, bound) with bound None unless the monoid is Plus."""
    n = len(ptr) - 1
    w = np.zeros(n, np.float64)
    bound = np.zeros(n, np.float64) if MONOIDS[monoid][0] == "plus" else None
    for i in range(n):
        r, b = reduce(monoid, val[ptr[i]:ptr[i + 1]])
        w[i] = r
        if bound is not None:
            bound[i] = b if b is not None else 0.0
    return (w if bound is not None else w.astype(F32)), bound


# ---- conversions ---------------------------------------------------------------------

def dense2sparse(x, identity):
    """Entries != identity, in index order (value source and, for identity 0,
    the bitmap source: bit i == x[i] != 0)."""
    x = _f(x)
    ind = np.nonzero(x != F32(identity))[0]
    return ind.astype(np.int32), x[ind]


def sparse2dense(n, ind, val, identity, struconly=False):
    """identity everywhere, then the stored values (1 in struct-only mode)."""
    return densify(n, ind, np.ones(len(ind), F32) if struconly else val, identity)


def convert(sparse_now, entries, length, switchpoint, ratio):
    """Vector::convert's direction switch.  Returns (sparse_after, ratio_after):
    fill = entries / length; sparse -> dense when fill > switchpoint and fill >
    ratio (growing), dense -> sparse when fill <= switchpoint and fill < ratio
    (shrinking), otherwise the storage stays and ratio becomes fill."""
    fill = np.float32(entries)/np.float32(length)
    sp, seen = np.float32(switchpoint), np.float32(ratio)
    if sparse_now and fill > sp and fill > seen:
        return False, ratio
    if not sparse_now and fill <= sp and fill < seen:
        return True, ratio
    return sparse_now, float(fill)
