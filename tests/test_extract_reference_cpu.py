"""The CPU restatement of extract (extract_reference) against numpy indexing of a dense
copy with its stored-entry mask (which keeps stored zeros) and against scipy's fancy
indexing (which keeps the same entries where no stored value is 0), on seeded random
matrices: unsorted and repeated I and J, GrB_ALL, a single index, the transpose and
stored zeros.  Also the companion header include/graphblast_b200_extract.h: every
declared symbol is exported and bound, it compiles as C99, and the refusals that
come before the device check."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import extract_reference as X
from support import random_csr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HEADER = open(os.path.join(ROOT, "include", "graphblast_b200_extract.h")).read()
VALUES = np.array([-3, -1, 0.5, 1, 2, 7], np.float32)


def dense_of(S):
    """(stored mask, values) of a Csr as dense arrays."""
    mask = np.zeros((S.nrows, S.ncols), bool)
    dense = np.zeros((S.nrows, S.ncols), S.val.dtype)
    rows = S.rows()
    mask[rows, S.ind] = True
    dense[rows, S.ind] = S.val
    return mask, dense


def index_sets(rng, n):
    """(name, list) pairs: ALL, sorted, unsorted, repeated, single."""
    return [
        ("all", None),
        ("sorted", np.sort(rng.choice(n, max(1, n//3), replace=False))),
        ("shuffled", rng.permutation(n)[:max(1, n//2)]),
        ("repeated", rng.randint(0, n, n + 5)),
        ("sorted_repeated", np.sort(rng.randint(0, n, n))),
        ("single", np.array([rng.randint(n)])),
    ]


def want_dense(mask, dense, I, J):
    I = np.arange(mask.shape[0]) if I is None else np.asarray(I)
    J = np.arange(mask.shape[1]) if J is None else np.asarray(J)
    return mask[np.ix_(I, J)], dense[np.ix_(I, J)]


def check_against_dense(rp, ci, val, m_want, d_want):
    nrows, ncols = m_want.shape
    assert len(rp) == nrows + 1 and rp[0] == 0
    for i in range(nrows):
        cols = ci[rp[i]:rp[i + 1]]
        assert np.all(np.diff(cols) > 0), "row %d not sorted and duplicate-free" % i
        assert np.array_equal(cols, np.nonzero(m_want[i])[0]), "row %d pattern" % i
        assert np.array_equal(val[rp[i]:rp[i + 1]], d_want[i, cols]), "row %d values" % i


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("tran", [False, True])
def test_matrix_against_dense_indexing(seed, tran):
    rng = np.random.RandomState(seed)
    S = random_csr(rng, 23, 31, 0.15, VALUES, zeros=0.2)
    mask, dense = dense_of(S)
    if tran:
        mask, dense = mask.T, dense.T
    for iname, I in index_sets(rng, mask.shape[0]):
        for jname, J in index_sets(rng, mask.shape[1]):
            rp, ci, val = X.extract_matrix(S.ptr, S.ind, S.val, S.nrows, S.ncols, I, J,
                                           tran=tran)
            m_want, d_want = want_dense(mask, dense, I, J)
            check_against_dense(rp, ci, val, m_want, d_want)


@pytest.mark.parametrize("seed", [3, 4])
def test_matrix_against_scipy(seed):
    rng = np.random.RandomState(seed)
    S = random_csr(rng, 40, 35, 0.2, VALUES, zeros=0.0)
    A = S.scipy(np.float32)
    for _, I in index_sets(rng, 40):
        for _, J in index_sets(rng, 35):
            rp, ci, val = X.extract_matrix(S.ptr, S.ind, S.val, S.nrows, S.ncols, I, J)
            ii = np.arange(40) if I is None else I
            jj = np.arange(35) if J is None else J
            want = A[ii][:, jj].tocsr()
            want.sort_indices()
            assert np.array_equal(rp, want.indptr)
            assert np.array_equal(ci, want.indices)
            assert np.array_equal(val, want.data)


@pytest.mark.parametrize("tran", [False, True])
def test_column_and_vectors(tran):
    rng = np.random.RandomState(7)
    S = random_csr(rng, 19, 26, 0.25, VALUES, zeros=0.2)
    mask, dense = dense_of(S)
    if tran:
        mask, dense = mask.T, dense.T
    for _, I in index_sets(rng, mask.shape[0]):
        for j in (0, mask.shape[1] - 1, rng.randint(mask.shape[1])):
            w_ind, w_val = X.extract_column(S.ptr, S.ind, S.val, S.nrows, S.ncols, I, j,
                                            tran=tran)
            m_want, d_want = want_dense(mask, dense, I, [j])
            assert np.array_equal(w_ind, np.nonzero(m_want[:, 0])[0])
            assert np.array_equal(w_val, d_want[w_ind, 0])
    u = rng.choice(VALUES, 30)
    u_ind = np.sort(rng.choice(30, 12, replace=False))
    stored = np.zeros(30, bool)
    stored[u_ind] = True
    for _, I in index_sets(rng, 30):
        assert np.array_equal(X.extract_dense_vector(u, I), u if I is None else u[I])
        w_ind, w_val = X.extract_sparse_vector(u_ind, u[u_ind], 30, I)
        ii = np.arange(30) if I is None else I
        assert np.array_equal(w_ind, np.nonzero(stored[ii])[0])
        assert np.array_equal(w_val, u[ii][w_ind])


# ---------------------------------------------------------------------------
# the companion header's contract
# ---------------------------------------------------------------------------

def test_header_symbols_exported_and_bound():
    from graphblast_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    names = sorted(set(re.findall(r"\b(gb200_[a-z0-9_]+)\s*\(", HEADER)))
    assert names == ["gb200_extract_column", "gb200_extract_matrix", "gb200_extract_vector"]
    for name in names:
        assert hasattr(lib, name), "missing export: " + name
    assert {s[0] for s in _lib.EXTRACT_SIGNATURES} == set(names)


def test_header_is_plain_c(tmp_path):
    src = str(tmp_path / "extract_header_check.c")
    with open(src, "w") as f:
        f.write('#include "graphblast_b200_extract.h"\nint main(void) { return 0; }\n')
    out = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror",
                          "-I", os.path.join(ROOT, "include"), "-fsyntax-only", src],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


def test_refusals_before_the_device_check():
    """NULL handles, then counts < 1, then element types: none reads a device."""
    import graphblast_b200 as gb
    from graphblast_b200 import _lib
    lib = _lib.load()
    UNINIT = int(gb.Info.GrB_UNINITIALIZED_OBJECT)
    INVALID = int(gb.Info.GrB_INVALID_VALUE)
    DOMAIN = int(gb.Info.GrB_DOMAIN_MISMATCH)
    zero = (C.c_ubyte*64)()
    Z = C.cast(zero, C.c_void_p)        # a handle of neither element type, never read
    idx = (C.c_int*2)(0, 1)
    cases = [
        ("gb200_extract_matrix", [None, None, Z, idx, 2, idx, 2, Z], UNINIT),
        ("gb200_extract_matrix", [Z, None, None, idx, 2, idx, 2, Z], UNINIT),
        ("gb200_extract_matrix", [Z, None, Z, idx, 2, idx, 2, None], UNINIT),
        ("gb200_extract_matrix", [Z, None, Z, idx, 0, idx, 2, Z], INVALID),
        ("gb200_extract_matrix", [Z, None, Z, idx, 2, idx, -1, Z], INVALID),
        ("gb200_extract_matrix", [Z, None, Z, idx, 2, idx, 2, Z], DOMAIN),
        ("gb200_extract_column", [None, None, Z, idx, 2, 0, Z], UNINIT),
        ("gb200_extract_column", [Z, None, None, idx, 2, 0, Z], UNINIT),
        ("gb200_extract_column", [Z, None, Z, idx, 2, 0, None], UNINIT),
        ("gb200_extract_column", [Z, None, Z, idx, 0, 0, Z], INVALID),
        ("gb200_extract_column", [Z, None, Z, idx, 2, 0, Z], DOMAIN),
        ("gb200_extract_vector", [None, None, Z, idx, 2, Z], UNINIT),
        ("gb200_extract_vector", [Z, None, None, idx, 2, Z], UNINIT),
        ("gb200_extract_vector", [Z, None, Z, idx, 2, None], UNINIT),
        ("gb200_extract_vector", [Z, None, Z, idx, 0, Z], INVALID),
    ]
    for name, args, want in cases:
        got = getattr(lib, name)(*args)
        assert got == want, "%s%r: %d, expected %d" % (name, tuple(args), got, want)
