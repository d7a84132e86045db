"""assign into a matrix on the CPU (test infrastructure only): the submatrix
C(I, J) = accum(C(I, J), op(A)), the column C(I, j) = u, the row C(i, J) = u and the
constant C(I, J) = val, restated in numpy.

C is an m x n CSR (ptr, ind, val).  I = None (GrB_ALL) means every row of C, J = None
every column; lists repeat no index.  Each form places a source at (I[p], J[q]):
op(A)(p, q) (op(A) = A' with tran), u's stored entries, or val everywhere.  Without
accum, C's entries in I x J go and the placed entries take their place; with accum
(an operator name of mxm_reference.OPS, pinned to the C oracle) the two are united and
a position both hold becomes accum(c, a), C's value first.  C comes out as a sorted
CSR (rowptr, colind, val) with C's value type.
"""
import numpy as np

from extract_reference import transpose
from mxm_reference import OPS


def _list(L, extent):
    return np.arange(extent, dtype=np.int64) if L is None else np.asarray(L, np.int64)


def _triples(ptr, ind, val, nrows):
    ptr = np.asarray(ptr, np.int64)
    rows = np.repeat(np.arange(nrows, dtype=np.int64), np.diff(ptr))
    return rows, np.asarray(ind, np.int64), np.asarray(val)


def place(C, m, n, er, ec, ev, I, J, accum=None):
    """C with the entries (er, ec, ev) (C's coordinates, no position twice) placed in
    the region I x J."""
    ptr, ind, val = C
    cr, cc, cv = _triples(ptr, ind, val, m)
    ev = np.asarray(ev).astype(cv.dtype)
    ck, ek = cr*n + cc, np.asarray(er, np.int64)*n + np.asarray(ec, np.int64)
    order = np.argsort(ek, kind="stable")
    ek, ev = ek[order], ev[order]
    if accum is None:
        in_i = np.zeros(m, bool)
        in_i[_list(I, m)] = True
        in_j = np.zeros(n, bool)
        in_j[_list(J, n)] = True
        keep = ~(in_i[cr] & in_j[cc])
        ck, cv = ck[keep], cv[keep]
        only_e = np.ones(len(ek), bool)
    else:
        at = np.searchsorted(ck, ek)
        hit = at < len(ck)
        hit[hit] = ck[at[hit]] == ek[hit]
        cv = cv.copy()
        cv[at[hit]] = np.asarray(OPS[accum](cv[at[hit]], ev[hit])).astype(cv.dtype)
        only_e = ~hit
    # both key lists ascend and share no key: E's entry k lands after the C entries
    # below it and the k E entries before it
    ek, ev = ek[only_e], ev[only_e]
    e_at = np.searchsorted(ck, ek) + np.arange(len(ek))
    keys = np.empty(len(ck) + len(ek), np.int64)
    vals = np.empty(len(keys), cv.dtype)
    from_c = np.ones(len(keys), bool)
    from_c[e_at] = False
    keys[e_at], vals[e_at] = ek, ev
    keys[from_c], vals[from_c] = ck, cv
    rowptr = np.zeros(m + 1, np.int64)
    np.cumsum(np.bincount(keys//n, minlength=m), out=rowptr[1:])
    return rowptr.astype(np.int32), (keys % n).astype(np.int32), vals


def assign_matrix(C, m, n, A, I, J, accum=None, tran=False):
    """C(I, J) = accum(C(I, J), op(A)); A = (ptr, ind, val, nrows, ncols)."""
    a_ptr, a_ind, a_val, a_m, a_n = A
    if tran:
        a_ptr, a_ind, a_val = transpose(a_m, a_n, a_ptr, a_ind, a_val)
        a_m, a_n = a_n, a_m
    p, q, v = _triples(a_ptr, a_ind, a_val, a_m)
    return place(C, m, n, _list(I, m)[p], _list(J, n)[q], v, I, J, accum)


def assign_constant(C, m, n, val, I, J, accum=None):
    """C(I, J) = accum(C(I, J), val): every position of I x J stored."""
    ii, jj = _list(I, m), _list(J, n)
    er, ec = np.repeat(ii, len(jj)), np.tile(jj, len(ii))
    ev = np.full(len(er), val).astype(np.asarray(C[2]).dtype)
    return place(C, m, n, er, ec, ev, I, J, accum)


def assign_column(C, m, n, u_ind, u_val, I, j, accum=None):
    """C(I, j) = accum(C(I, j), u); u's stored entries (u_ind into I)."""
    er = _list(I, m)[np.asarray(u_ind, np.int64)]
    return place(C, m, n, er, np.full(len(er), j, np.int64), u_val, I, [j], accum)


def assign_row(C, m, n, u_ind, u_val, i, J, accum=None):
    """C(i, J) = accum(C(i, J), u); u's stored entries (u_ind into J)."""
    ec = _list(J, n)[np.asarray(u_ind, np.int64)]
    return place(C, m, n, np.full(len(ec), i, np.int64), ec, u_val, [i], J, accum)
