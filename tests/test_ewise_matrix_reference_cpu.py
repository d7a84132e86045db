"""The CPU reference of the matrix eWiseAdd / eWiseMult (ewise_matrix_reference)
against a dict-of-keys restatement on every semiring, and against scipy for
plus-times."""
import numpy as np
import pytest

import ewise_matrix_reference as ref
from mxm_reference import OPS, SEMIRINGS
from support import same

VALUES = np.array([-4, -2, -1, -0.5, 0, 0.5, 1, 2, 4], np.float32)


def random_csr(rng, nrows, ncols, density, values):
    dense = (rng.rand(nrows, ncols) < density)
    dense[rng.rand(nrows) < 0.1, :] = False            # empty rows
    dense[:, rng.rand(ncols) < 0.1] = False            # empty columns
    rows, cols = np.nonzero(dense)
    ptr = np.zeros(nrows + 1, np.int64)
    np.cumsum(np.bincount(rows, minlength=nrows), out=ptr[1:])
    return ptr, cols.astype(np.int32), rng.choice(values, len(cols)).astype(values.dtype)


def as_dict(ptr, ind, val):
    return {(i, int(ind[e])): val[e] for i in range(len(ptr) - 1)
            for e in range(ptr[i], ptr[i + 1])}


def dok(add, semiring, A, B):
    name = SEMIRINGS[semiring][0 if add else 1]
    f = OPS[name]
    da, db = as_dict(*A), as_dict(*B)
    keys = sorted(set(da) | set(db)) if add else sorted(set(da) & set(db))
    out = {}
    with np.errstate(all="ignore"):
        for k in keys:
            if k in da and k in db:
                out[k] = f(np.array([da[k]], np.float32), np.array([db[k]], np.float32))[0]
            else:
                out[k] = da[k] if k in da else db[k]
    return out


@pytest.mark.parametrize("add", [True, False])
@pytest.mark.parametrize("semiring", range(17))
def test_against_dict_of_keys(add, semiring):
    rng = np.random.RandomState(semiring)
    m, n = 37, 53
    A = random_csr(rng, m, n, 0.2, VALUES)
    B = random_csr(rng, m, n, 0.2, VALUES)
    rp, ci, val = ref.ewise(add, semiring, *A, *B, n)
    want = dok(add, semiring, A, B)
    got = as_dict(rp, ci, val)
    assert list(got) == list(want)                    # same keys, row-major sorted
    assert all(same(got[k], want[k]) for k in want)
    assert np.all(np.diff(rp) >= 0) and rp[-1] == len(ci)


@pytest.mark.parametrize("add", [True, False])
def test_plus_times_against_scipy(add):
    import scipy.sparse as sp
    rng = np.random.RandomState(7)
    m, n = 120, 90
    A = random_csr(rng, m, n, 0.1, VALUES)
    B = random_csr(rng, m, n, 0.1, VALUES)
    rp, ci, val = ref.ewise(add, 1, *A, *B, n)
    SA = sp.csr_matrix((A[2].astype(np.float64), A[1], A[0]), shape=(m, n))
    SB = sp.csr_matrix((B[2].astype(np.float64), B[1], B[0]), shape=(m, n))
    S = (SA + SB) if add else SA.multiply(SB).tocsr()
    S = sp.csr_matrix(S)
    S.sort_indices()
    got = as_dict(rp, ci, val)
    want = as_dict(S.indptr, S.indices, S.data)
    # scipy prunes zeros: compare where no result is 0
    nonzero = {k: v for k, v in got.items() if v != 0}
    assert set(nonzero) == {k for k, v in want.items() if v != 0}
    assert all(nonzero[k] == want[k] for k in nonzero)


def test_int_plus_times():
    rng = np.random.RandomState(3)
    ivals = np.array([-3, -1, 0, 2, 5], np.int32)
    A = random_csr(rng, 30, 40, 0.2, ivals)
    B = random_csr(rng, 30, 40, 0.2, ivals)
    for add in (True, False):
        rp, ci, val = ref.ewise(add, 1, *A, *B, 40, integer=True)
        got = as_dict(rp, ci, val)
        da, db = as_dict(*A), as_dict(*B)
        keys = sorted(set(da) | set(db)) if add else sorted(set(da) & set(db))
        for k in keys:
            if k in da and k in db:
                assert got[k] == (int(da[k]) + int(db[k]) if add else int(da[k])*int(db[k]))
            else:
                assert got[k] == (da[k] if k in da else db[k])
        assert list(got) == keys


def test_empty_and_edge_shapes():
    e = (np.zeros(4, np.int64), np.zeros(0, np.int32), np.zeros(0, np.float32))
    A = (np.array([0, 1, 1, 2]), np.array([0, 2], np.int32), np.float32([1, 2]))
    for add in (True, False):
        rp, ci, val = ref.ewise(add, 1, *A, *e, 3)
        assert list(rp) == ([0, 1, 1, 2] if add else [0, 0, 0, 0])
        rp, ci, val = ref.ewise(add, 1, *e, *e, 3)
        assert list(rp) == [0, 0, 0, 0] and len(ci) == 0
