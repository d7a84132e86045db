"""The CPU reference of the unmasked product (mxm_reference.mxm) against scipy
and against a plain dict-of-rows restatement over the C oracle's own scalar
operations; and the bin constants of the GPU test against the kernels."""
import os
import re

import numpy as np
import pytest

import mxm_reference as ref
import oracle_binding as orc
from support import same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = os.path.join(ROOT, "graphblast_b200", "csrc", "graphblas", "backend",
                       "cuda", "kernels")


def random_int_csr(rng, nrows, ncols, density):
    """Integer-valued, with empty rows and columns and stored zeros."""
    mask = rng.rand(nrows, ncols) < density
    mask[rng.rand(nrows) < 0.15, :] = False
    mask[:, rng.rand(ncols) < 0.15] = False
    rows, cols = np.nonzero(mask)
    vals = rng.randint(-3, 4, len(rows)).astype(np.float32)
    ptr = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=nrows))])
    return ptr, cols.astype(np.int32), vals


def dict_rows_product(semiring, A, B):
    """{i: {j: value}} through orc_add / orc_mul / orc_identity, ascending k."""
    lib = orc.lib()
    (ap, ai, av), (bp, bi, bv) = A, B
    out = {}
    for i in range(len(ap) - 1):
        row = {}
        for e in range(ap[i], ap[i + 1]):
            k = ai[e]
            for f in range(bp[k], bp[k + 1]):
                j = int(bi[f])
                prod = lib.orc_mul(semiring, float(av[e]), float(bv[f]))
                acc = row.get(j, lib.orc_identity(semiring))
                row[j] = lib.orc_add(semiring, acc, prod)
        if row:
            out[i] = row
    return out


def as_dict(rp, ci, val):
    out = {}
    for i in range(len(rp) - 1):
        if rp[i + 1] > rp[i]:
            out[i] = {int(ci[e]): float(val[e]) for e in range(rp[i], rp[i + 1])}
    return out


@pytest.mark.parametrize("shape", [(1, 1, 1), (7, 13, 5), (40, 30, 60), (120, 90, 70)])
def test_plus_times_against_scipy(shape):
    import scipy.sparse as sp
    m, k, n = shape
    rng = np.random.RandomState(m + k + n)
    A = random_int_csr(rng, m, k, 0.2)
    B = random_int_csr(rng, k, n, 0.2)
    rp, ci, val = ref.mxm(1, *A, *B, n)
    SA = sp.csr_matrix((A[2].astype(np.float64), A[1], A[0]), shape=(m, k))
    SB = sp.csr_matrix((B[2].astype(np.float64), B[1], B[0]), shape=(k, n))
    got = np.zeros((m, n))
    got[np.repeat(np.arange(m), np.diff(rp)), ci] = val
    assert np.array_equal(got, (SA @ SB).toarray())
    # pattern: every (i, j) that some k joins, cancelled or zero products included
    PA = sp.csr_matrix((np.ones(len(A[1])), A[1], A[0]), shape=(m, k))
    PB = sp.csr_matrix((np.ones(len(B[1])), B[1], B[0]), shape=(k, n))
    P = (PA @ PB).tocsr()
    P.sort_indices()
    assert np.array_equal(rp, P.indptr) and np.array_equal(ci, P.indices)
    irp, ici, ival = ref.mxm(1, *A, *B, n, integer=True)
    assert np.array_equal(irp, rp) and np.array_equal(ici, ci)
    assert np.array_equal(ival, val.astype(np.int64))


@pytest.mark.parametrize("semiring", range(17))
def test_every_semiring_against_dict_rows(semiring):
    rng = np.random.RandomState(semiring)
    vals = np.float32([-4, -2, -1, -0.5, 0, 0.5, 1, 2, 4])
    for m, k, n in ((1, 1, 1), (6, 5, 7), (12, 9, 10)):
        A = random_int_csr(rng, m, k, 0.5)
        B = random_int_csr(rng, k, n, 0.5)
        A = (A[0], A[1], rng.choice(vals, len(A[1])))
        B = (B[0], B[1], rng.choice(vals, len(B[1])))
        rp, ci, val = ref.mxm(semiring, *A, *B, n)
        got, want = as_dict(rp, ci, val), dict_rows_product(semiring, A, B)
        assert got.keys() == want.keys()
        for i in want:
            assert got[i].keys() == want[i].keys()
            for j in want[i]:
                assert same(got[i][j], want[i][j]), (semiring, i, j)


def test_cancellation_and_identity_quirk():
    # row 0 of A*B: 1*1 + (-1)*1 = 0, stored; MaximumMultiplies folds from its
    # identity 0, so all-negative products give 0
    A = (np.array([0, 2]), np.array([0, 1], np.int32), np.float32([1, -1]))
    B = (np.array([0, 1, 2]), np.array([0, 0], np.int32), np.float32([1, 1]))
    rp, ci, val = ref.mxm(1, *A, *B, 1)
    assert list(rp) == [0, 1] and list(ci) == [0] and val[0] == 0
    A2 = (A[0], A[1], np.float32([-1, -2]))
    rp, ci, val = ref.mxm(3, *A2, *B, 1)
    assert list(ci) == [0] and val[0] == 0
    assert dict_rows_product(3, A2, B) == {0: {0: 0.0}}


def test_kernel_constants_match_the_gpu_test():
    """A change to a bin limit must come with a change to the designed rows of
    test_mxm_unmasked_gpu.py; this fails first."""
    import test_mxm_unmasked_gpu as g
    src = open(os.path.join(KERNELS, "spgemm_unmasked.cuh")).read()
    got = {k: int(v) for k, v in re.findall(r"#define\s+(GB_MXM_\w+)\s+(\d+)", src)}
    want = {"GB_MXM_SYM_S": g.SYM[0], "GB_MXM_SYM_M": g.SYM[1], "GB_MXM_SYM_L": g.SYM[2],
            "GB_MXM_NUM_S": g.NUM[0], "GB_MXM_NUM_M": g.NUM[1], "GB_MXM_NUM_L": g.NUM[2]}
    assert {k: got[k] for k in want} == want
    for lim in g.SYM + g.NUM:
        assert str(lim) in g.__doc__
