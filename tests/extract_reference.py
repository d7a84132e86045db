"""extract on the CPU (test infrastructure only): submatrices C = op(A)(I, J),
columns w = op(A)(I, j) and subvectors w = u(I), restated in numpy.

op(A) is A, or its transpose.  I = None (GrB_ALL) means every row of op(A), J =
None every column.  C(i, p) = op(A)(I[i], J[p]) wherever that entry is stored:
duplicates in I or J repeat rows or columns, stored zeros stay stored, and C comes
out as a sorted CSR (rowptr, colind, val) with the values of A's type.
"""
import numpy as np


def transpose(nrows, ncols, ptr, ind, val):
    """(ptr, ind, val) of the transpose, rows sorted inside every column."""
    ptr = np.asarray(ptr, np.int64)
    rows = np.repeat(np.arange(nrows, dtype=np.int64), np.diff(ptr))
    order = np.lexsort((rows, np.asarray(ind, np.int64)))
    t_ptr = np.zeros(ncols + 1, np.int64)
    np.cumsum(np.bincount(np.asarray(ind, np.int64), minlength=ncols), out=t_ptr[1:])
    return t_ptr, rows[order].astype(np.int32), np.asarray(val)[order]


def cut(ptr, ind, val, nrows, ncols, I, J):
    """C = S(I, J) of the CSR S (nrows x ncols); (rowptr, colind, val)."""
    ptr = np.asarray(ptr, np.int64)
    ind = np.asarray(ind, np.int64)
    val = np.asarray(val)
    I = np.arange(nrows, dtype=np.int64) if I is None else np.asarray(I, np.int64)
    lens = ptr[I + 1] - ptr[I]
    sel_rows = np.repeat(np.arange(len(I), dtype=np.int64), lens)
    starts = np.repeat(ptr[I], lens)
    offs = np.arange(len(sel_rows), dtype=np.int64) - np.repeat(np.cumsum(lens) - lens, lens)
    slots = starts + offs
    k = ind[slots]
    if J is None:
        c_rows, c_cols, c_slots = sel_rows, k, slots
    else:
        J = np.asarray(J, np.int64)
        jpos = np.argsort(J, kind="stable")
        jptr = np.searchsorted(J[jpos], np.arange(ncols + 1), side="left")
        mult = jptr[k + 1] - jptr[k]
        c_rows = np.repeat(sel_rows, mult)
        c_slots = np.repeat(slots, mult)
        base = np.repeat(jptr[k], mult)
        off = np.arange(len(c_rows), dtype=np.int64) - np.repeat(np.cumsum(mult) - mult, mult)
        c_cols = jpos[base + off]
        order = np.lexsort((c_cols, c_rows))
        c_rows, c_cols, c_slots = c_rows[order], c_cols[order], c_slots[order]
    rowptr = np.zeros(len(I) + 1, np.int64)
    np.cumsum(np.bincount(c_rows, minlength=len(I)), out=rowptr[1:])
    return rowptr.astype(np.int32), c_cols.astype(np.int32), val[c_slots]


def extract_matrix(ptr, ind, val, nrows, ncols, I, J, tran=False):
    """C = op(A)(I, J), A an nrows x ncols CSR; op(A) = A' with tran."""
    if tran:
        ptr, ind, val = transpose(nrows, ncols, ptr, ind, val)
        nrows, ncols = ncols, nrows
    return cut(ptr, ind, val, nrows, ncols, I, J)


def extract_column(ptr, ind, val, nrows, ncols, I, j, tran=False):
    """w = op(A)(I, j) as (indices, values): row j of op(A)' with column list I."""
    if not tran:
        ptr, ind, val = transpose(nrows, ncols, ptr, ind, val)
        nrows, ncols = ncols, nrows
    _, w_ind, w_val = cut(ptr, ind, val, nrows, ncols, [j], I)
    return w_ind, w_val


def extract_dense_vector(u, I):
    """w = u(I) of a dense u."""
    u = np.asarray(u)
    return u.copy() if I is None else u[np.asarray(I, np.int64)]


def extract_sparse_vector(u_ind, u_val, size, I):
    """w = u(I) of a sparse u (ascending indices) as (indices, values)."""
    ptr = np.array([0, len(u_ind)], np.int64)
    _, w_ind, w_val = cut(ptr, u_ind, u_val, 1, size, None, I)
    return w_ind, w_val
