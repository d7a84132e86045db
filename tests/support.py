"""Helpers shared by more than one test module: the device fixture, host CSR matrices
and their device copies, graph inputs and checkers.  Test infrastructure only; the
suites and tools/bench_cc.py import what they use from here."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

import oracle_binding as orc

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def gb():
    import graphblast_b200 as g
    g.init(0)
    return g


# ---------------------------------------------------------------------------
# host-side sparse matrices
# ---------------------------------------------------------------------------

def transpose(rp, ci, ncols=None):
    """(ptr, ind, order) of the transpose of the pattern (rp, ci) with ncols columns
    (default: square): order takes the values along, val[order]."""
    n = len(rp) - 1
    ncols = n if ncols is None else ncols
    rows = np.repeat(np.arange(n, dtype=np.int32), np.diff(rp))
    order = np.lexsort((rows, ci))
    t_rp = np.concatenate([[0], np.cumsum(np.bincount(ci, minlength=ncols))]).astype(np.int32)
    return t_rp, rows[order], order


class Csr(object):
    """nrows x ncols CSR on the host: int32 ptr and ind, values as given."""

    def __init__(self, nrows, ncols, ptr, ind, val):
        self.nrows, self.ncols = nrows, ncols
        self.ptr = np.asarray(ptr, np.int32)
        self.ind = np.asarray(ind, np.int32)
        self.val = np.asarray(val)

    @property
    def nnz(self):
        return len(self.ind)

    def rows(self):
        return np.repeat(np.arange(self.nrows, dtype=np.int32), np.diff(self.ptr))

    @property
    def T(self):
        """CSR of the transpose (= this matrix's CSC)."""
        t_ptr, t_ind, order = transpose(self.ptr, self.ind, self.ncols)
        return Csr(self.ncols, self.nrows, t_ptr, t_ind, self.val[order])

    def astype(self, dt):
        return Csr(self.nrows, self.ncols, self.ptr, self.ind, self.val.astype(dt))

    def with_values(self, val):
        return Csr(self.nrows, self.ncols, self.ptr, self.ind, val)

    def scipy(self, dtype=np.float64):
        import scipy.sparse as sp
        return sp.csr_matrix((self.val.astype(dtype), self.ind, self.ptr),
                             shape=(self.nrows, self.ncols))


def csr(nrows, ncols, rows, cols, vals, dtype):
    """Csr of the (rows, cols, vals) triples, values as dtype; no entry twice."""
    rows = np.asarray(rows, np.int64)
    cols = np.asarray(cols, np.int64)
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    assert not np.any((np.diff(rows) == 0) & (np.diff(cols) == 0)), "duplicate entry"
    ptr = np.zeros(nrows + 1, np.int64)
    np.add.at(ptr, rows + 1, 1)
    return Csr(nrows, ncols, np.cumsum(ptr), cols, np.asarray(vals, dtype)[order])


def random_csr(rng, nrows, ncols, density, values, zeros=0.1, empty=0.1):
    """Mixed row lengths (a few rows 10x denser), some empty rows and columns,
    about `zeros` of the stored values 0."""
    d = np.full(nrows, density)
    d[rng.rand(nrows) < 0.05] *= 10
    d[rng.rand(nrows) < empty] = 0
    dead_cols = rng.rand(ncols) < empty
    rows, cols = [], []
    for i in range(nrows):
        c = np.nonzero((rng.rand(ncols) < d[i]) & ~dead_cols)[0]
        rows.append(np.full(len(c), i))
        cols.append(c)
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    vals = rng.choice(values, len(cols)).astype(values.dtype)
    vals[rng.rand(len(vals)) < zeros] = 0
    return csr(nrows, ncols, rows, cols, vals, values.dtype)


# ---------------------------------------------------------------------------
# device matrices
# ---------------------------------------------------------------------------

def _dev(a, dt, offset=0):
    """Device copy of a, `offset` elements past an aligned allocation."""
    import torch
    a = torch.from_numpy(np.ascontiguousarray(a, dt))
    t = torch.zeros(len(a) + offset + 1, dtype=a.dtype, device="cuda")
    view = t[offset:offset + len(a)]
    view.copy_(a)
    return view


def device_matrix(gb, S, csc=True, symmetric=False, integer=False, offset=0, into=None):
    """A Matrix adopting device copies of S's CSR and, with csc, of its CSC (without
    it the matrix has no column side).  symmetric: the CSR alone, marked symmetric so
    that the CSC aliases it (graphs.matrix_from_csr).  integer: INT32 values, FP32
    otherwise.  offset: colind and val that many elements past a 32-byte aligned
    address.  into: an existing Matrix to adopt them.  A matrix without stored
    entries is built through the ingest entry, since adopting takes stored entries."""
    vt = np.int32 if integer else np.float32
    dtype = gb.api.INT32 if integer else gb.api.FP32
    if symmetric:
        from graphblast_b200.graphs import matrix_from_csr
        return matrix_from_csr(S.nrows, _dev(S.ptr, np.int32), _dev(S.ind, np.int32),
                               _dev(S.val, vt), dtype=dtype)
    M = gb.Matrix(S.nrows, S.ncols, dtype=dtype) if into is None else into
    if S.nnz == 0:
        gb.api._check(M._lib.gb200_matrix_build_coo_device(M._h, None, None, None,
                                                           0, 0), "empty matrix")
        return M

    def arrays(X):
        return (_dev(X.ptr, np.int32), _dev(X.ind, np.int32, offset),
                _dev(X.val, vt, offset))
    M.build_device_csr(*arrays(S), S.nnz, *(arrays(S.T) if csc else ()))
    return M


def make_matrix(gb, rp, ci, val=None, symmetric=True, csc=True, integer=False):
    """device_matrix of the square pattern (rp, ci), values val or all 1."""
    n = len(rp) - 1
    if val is None:
        val = np.ones(len(ci), np.int32 if integer else np.float32)
    return device_matrix(gb, Csr(n, n, rp, ci, val), csc=csc, symmetric=symmetric,
                         integer=integer)


# ---------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------

def symmetric_csr(n, src, dst):
    return orc.build_csr(n, np.asarray(src, np.int32), np.asarray(dst, np.int32), True)


def directed_csr(n, src, dst):
    return orc.build_csr(n, np.asarray(src, np.int32), np.asarray(dst, np.int32), False)


def mtx_graph(name):
    n, src, dst, _ = orc.read_mtx_edges(os.path.join(HERE, "golden", name + ".mtx"))
    return orc.build_csr(n, src, dst, True)


def graphs():
    """(name, rp, ci) of the golden graphs and three R-MATs."""
    out = [("chesapeake",) + mtx_graph("chesapeake"), ("test_cc",) + mtx_graph("test_cc"),
           ("test_bc",) + mtx_graph("test_bc"), ("test_sgm",) + mtx_graph("test_sgm")]
    for scale in (10, 11, 12):
        out.append(("rmat%d" % scale,) + orc.rmat_csr(scale))
    return out


def star_graph(nleaves):
    """Vertex 0 adjacent to all others: one row of nleaves entries (spans many
    merge-path tiles) plus nleaves rows of one entry."""
    src = np.zeros(nleaves, dtype=np.int32)
    dst = np.arange(1, nleaves + 1, dtype=np.int32)
    return orc.build_csr(nleaves + 1, src, dst, True)


def path_graph(n):
    src = np.arange(n - 1, dtype=np.int32)
    return orc.build_csr(n, src, src + 1, True)


def ragged_graph():
    """Empty rows at the start, middle and end; isolated vertices; n % 32 != 0."""
    n = 1003
    rng = np.random.RandomState(5)
    src = rng.randint(100, 600, 4000).astype(np.int32)
    dst = rng.randint(300, 900, 4000).astype(np.int32)
    return orc.build_csr(n, src, dst, True)


# ---------------------------------------------------------------------------
# checkers
# ---------------------------------------------------------------------------

def same(x, y):
    """Equal entry by entry, NaN equal to NaN."""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    return x.shape == y.shape and bool(np.all((x == y) | (np.isnan(x) & np.isnan(y))))


def check_csr(C, want):
    """C's row offsets, column indices and values equal want's (a Csr), bit for bit
    (NaN equal to NaN, -0 equal to +0)."""
    rp, ci, val = C.extract_csr()
    assert np.array_equal(rp, want.ptr), "row offsets differ"
    assert np.array_equal(ci, want.ind), "column indices differ"
    if val.dtype == np.float32:
        ok = np.array_equal(val, want.val.astype(np.float32), equal_nan=True)
    else:
        ok = np.array_equal(val.astype(np.int64), want.val.astype(np.int64))
    if not ok:
        bad = np.nonzero(~((val == want.val) | (np.isnan(val) & np.isnan(want.val))))[0]
        pytest.fail("%d of %d values differ, first at %d: got %r want %r" % (
            len(bad), len(val), bad[0], val[bad[0]], want.val[bad[0]]))


def components(n, rp, ci):
    """(label, count): scipy's weakly connected components of the pattern (rp, ci),
    each label mapped to its component's minimum vertex id."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    if n == 0:
        return np.zeros(0, np.int64), 0
    A = sp.csr_matrix((np.ones(len(ci), np.int8), np.asarray(ci, np.int64),
                       np.asarray(rp, np.int64)), shape=(n, n))
    k, lab = connected_components(A, directed=True, connection="weak")
    low = np.full(k, n, np.int64)
    np.minimum.at(low, lab, np.arange(n, dtype=np.int64))
    return low[lab], int(k)


def check_structure(rp, ci, label):
    """Without scipy: every stored entry joins equal labels, and each label is a
    vertex no larger than i that labels itself."""
    n = len(rp) - 1
    label = np.asarray(label, np.int64)
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(rp))
    assert np.array_equal(label[rows], label[np.asarray(ci, np.int64)]), "an edge spans two labels"
    assert np.all((label >= 0) & (label <= np.arange(n))), "a label above its vertex"
    assert np.array_equal(label[label], label), "a label that does not label itself"


def bfs_levels(rp, ci, s, max_niter=None):
    """The oracle's BFS levels; with a cut-off after max_niter iterations only levels
    1..max_niter are assigned (reference algorithm/bfs.hpp: the frontier found in
    the last iteration is not), the rest are unreached."""
    want = orc.bfs(rp, ci, s)
    if max_niter is not None:
        want = np.where(want <= max_niter, want, 0).astype(want.dtype)
    return want


# ---------------------------------------------------------------------------
# counters and the CPU model of the fused BFS
# ---------------------------------------------------------------------------

def fused_stats(desc, n):
    """levels, entries inspected pulling, pull levels, vertices pushed, edges
    pushed, vertices discovered pushing — of the last fused traversal."""
    from graphblast_b200 import _lib
    st = (C.c_ulonglong * 6)()
    _lib.load().gb200_bfs_stats(desc._h, n, st)
    return [int(x) for x in st]


def launch_count(gb):
    out = C.c_ulonglong(0)
    gb.api._lib.load().gb200_launch_count(C.byref(out))
    return out.value


def launches_per_call(gb, call):
    """The kernel launches of call(), after one call that lets its vectors take their
    storage and fills its caches."""
    call()
    before = launch_count(gb)
    call()
    return launch_count(gb) - before


def bfs_pull_model():
    """tools/bfs_pull_model.py, loaded as a module."""
    spec = importlib.util.spec_from_file_location(
        "bfs_pull_model", os.path.join(os.path.dirname(HERE), "tools", "bfs_pull_model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod
