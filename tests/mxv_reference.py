"""mxv / vxm on the CPU, one function per device route (test infrastructure only).

Every function takes the TRAVERSED structure as CSR arrays (ptr, ind, val): for
the pull that is A's CSR under mxv and A's CSC under vxm, for the push it is A's
CSC under mxv and A's CSR under vxm.  The scalar operations are the OPS /
SEMIRINGS tables of mxm_reference.py (numpy float32, checked against the C
oracle's orc_add / orc_mul there); test_mxv_reference_cpu.py checks these
functions against the oracle's orc_vxm where the two define the same thing.

  pull       generic semiring pull (spmv.hpp: merge-path and hub-cached kernels)
  push       sparse-frontier push (spmspv.hpp, kernels/spmspv_push.cuh)
  bool_pull  fused masked Boolean pull, bit-map and value forms
             (spmv.hpp, kernels/spmv_pull.cuh)
"""
import numpy as np

from mxm_reference import F32, OPS, SEMIRINGS

ASSOCIATIVE_ADDS = ("or", "plus", "min", "max")


def _kept(mask, scmp):
    """Rows a dense mask keeps: nonzero ones, or zero ones under GrB_SCMP.
    -0.0 counts as zero."""
    nz = np.asarray(mask, F32) != 0
    return ~nz if scmp else nz


def _fold_rows(add, ident, ptr, prods):
    """w[i] = add(...add(add(ident, p0), p1)..., pL-1) over row i, in order."""
    n = len(ptr) - 1
    lens = np.diff(ptr)
    acc = np.full(n, ident, F32)
    for k in range(int(lens.max()) if n else 0):
        rows = np.nonzero(lens > k)[0]
        acc[rows] = add(acc[rows], prods[ptr[rows] + k])
    return acc


def pull(semiring, ptr, ind, val, u, mask=None, scmp=False, w_old=None):
    """w = A' (+.x) u for a dense u (every u[col] takes part).

    Returns (w, bound).  For a plus add w is the float64 sum and bound the
    per-row error bound of a float32 fold, (L + 1) 2^-24 sum |p_k| (L = row
    length); the device result must lie within it.  For every other add w is
    float32 and bound None: min / max / or folds are exact in any order.
    """
    add_name, mul_name, ident = SEMIRINGS[semiring]
    add, mul = OPS[add_name], OPS[mul_name]
    ptr = np.asarray(ptr, np.int64)
    ind = np.asarray(ind, np.int64)
    val = np.asarray(val, F32)
    u = np.asarray(u, F32)
    n = len(ptr) - 1
    with np.errstate(all="ignore"):
        # products in float32, as the kernel forms them; no identity short-circuit
        prods = mul(val, u[ind]) if len(ind) else np.zeros(0, F32)
        nonempty = np.diff(ptr) > 0
        bound = None
        if add_name == "plus":
            p64 = prods.astype(np.float64)
            w = np.zeros(n, np.float64)
            mag = np.zeros(n, np.float64)
            if nonempty.any():
                starts = ptr[:-1][nonempty]
                w[nonempty] = np.add.reduceat(p64, starts)
                mag[nonempty] = np.add.reduceat(np.abs(p64), starts)
            bound = (np.diff(ptr) + 1)*2.0**-24*mag
        elif add_name in ("min", "max"):
            red = add                 # np.fmin / np.fmax: NaN products are ignored
            w = np.full(n, ident, F32)
            if nonempty.any():
                part = red.reduceat(prods, ptr[:-1][nonempty])
                w[nonempty] = add(w[nonempty], part)      # fold starts at identity
        else:
            w = _fold_rows(add, ident, ptr, prods)
        if mask is not None:
            # masked-out rows get the IDENTITY (assignDenseDenseMaskKernel), not 0
            out = ~_kept(mask, scmp)
            w[out] = ident
            if bound is not None:
                bound[out] = 0
        if w_old is not None:
            # accum combines with the SEMIRING's add; the accum functor is ignored
            # (reference spmv.hpp:213-219)
            w_old = np.asarray(w_old, F32)
            if add_name == "plus":
                w = w_old.astype(np.float64) + w
                bound = bound + 2.0**-24*np.abs(w)
            else:
                w = add(w_old, w)
    return w, bound


def push(semiring, ptr, ind, val, f_ind, f_val, nout, mask=None, scmp=False,
         struconly=False):
    """Sparse w from the sparse frontier (f_ind, f_val): row f_ind[j] of the
    traversed structure is spread over its columns.  Returns sorted, duplicate
    free (w_ind, w_val).

    Per kept edge (c, a) of frontier entry (r, x):
      prod = identity if a == identity or x == identity else mul(a, x)
          (identity short-circuit, reference kernels/ewisemult.hpp:22-25);
      the mask is read per edge with the reference's inverted flag
          (spmspv.hpp:33-37): keep c where mask[c] != 0, where == 0 under SCMP.
    An entry is present iff it received at least one kept edge: the first
    combine into a cell always finds the identity there and sets its touched
    bit, whatever the product.  Its value is the fold of its products from the
    identity.  accum is ignored (reference spmspv.hpp "TODO: add accum").
    Masked key-value mode drops entries whose value is 0 (-0.0 included); in
    struct-only mode every present entry holds 1.
    """
    add_name, mul_name, ident = SEMIRINGS[semiring]
    add, mul = OPS[add_name], OPS[mul_name]
    ptr = np.asarray(ptr, np.int64)
    ind = np.asarray(ind, np.int64)
    val = np.asarray(val, F32)
    f_ind = np.asarray(f_ind, np.int64)
    f_val = np.asarray(f_val, F32)
    lens = ptr[f_ind + 1] - ptr[f_ind]
    src = np.repeat(np.arange(len(f_ind)), lens)
    edge = (np.arange(len(src)) - np.repeat(np.cumsum(lens) - lens, lens)
            + np.repeat(ptr[f_ind], lens)).astype(np.int64)
    cols = ind[edge]
    keep = np.ones(len(cols), bool) if mask is None else _kept(mask, scmp)[cols]
    cols, edge, src = cols[keep], edge[keep], src[keep]
    present = np.zeros(nout, bool)
    present[cols] = True
    w_ind = np.nonzero(present)[0]
    if struconly:
        return w_ind.astype(np.int32), np.ones(len(w_ind), F32)
    a, x = val[edge], f_val[src]
    with np.errstate(all="ignore"):
        prods = np.where((a == ident) | (x == ident), ident, mul(a, x)).astype(F32)
        # fold per column in frontier order, then edge order
        order = np.argsort(cols, kind="stable")
        c_sorted = cols[order]
        cptr = np.searchsorted(c_sorted, np.arange(nout + 1))
        w = _fold_rows(add, ident, cptr, prods[order]) if len(cols) else \
            np.full(nout, ident, F32)
    w_val = w[w_ind]
    if mask is not None:
        nz = w_val != 0
        w_ind, w_val = w_ind[nz], w_val[nz]
    return w_ind.astype(np.int32), w_val.astype(F32)


def bool_pull(ptr, ind, mask, u, identity=0.0, scmp=False, opreuse=False):
    """Fused masked Boolean pull: w[i] = 1 iff row i is kept by the mask and some
    neighbour c has probe[c] set, 0 otherwise.  probe is the mask under opreuse
    (set: mask[c] != 0) and u otherwise (set: u[c] != identity; the bit-map form
    is the identity-0 case, one bit per u[c] != 0).  Early exit stops a row at
    its first hit and cannot change the result."""
    ptr = np.asarray(ptr, np.int64)
    ind = np.asarray(ind, np.int64)
    mask = np.asarray(mask, F32)
    probe = (mask != 0) if opreuse else (np.asarray(u, F32) != F32(identity))
    n = len(ptr) - 1
    hits = np.zeros(n, np.int64)
    rows = np.repeat(np.arange(n), np.diff(ptr))
    np.add.at(hits, rows, probe[ind].astype(np.int64))
    return ((hits > 0) & _kept(mask, scmp)).astype(F32)
