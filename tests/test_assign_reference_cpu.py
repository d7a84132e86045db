"""The CPU restatement of assign into a matrix (assign_reference) against a brute force
over a dict of entries, on seeded small matrices: the submatrix, constant, column and
row forms, with and without every accum operator, GrB_ALL, sorted, shuffled and single
lists, the transpose and stored zeros; and against extract_reference for the round
trip (after C(I,J) = A, C(I,J) is A and C outside the region is unchanged).  Also the
companion header include/graphblast_b200_assign.h: every declared symbol is exported
and bound, it compiles as C99, and the refusals that come before the device check."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import assign_reference as R
import extract_reference as X
from mxm_reference import OPS
from support import random_csr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HEADER = open(os.path.join(ROOT, "include", "graphblast_b200_assign.h")).read()
VALUES = np.array([-3, -1, 0.5, 1, 2, 7], np.float32)
# the accum of each monoid, in graphblast_b200.api.Monoid order
ACCUMS = [None, "plus", "mul", "min", "max", "or", "and", "gt", "lt", "ne"]


def index_sets(rng, n):
    """(name, list) pairs: ALL, sorted, shuffled, single; no index twice."""
    return [
        ("all", None),
        ("sorted", np.sort(rng.choice(n, max(1, n//3), replace=False))),
        ("shuffled", rng.permutation(n)[:max(1, n//2)]),
        ("single", np.array([rng.randint(n)])),
    ]


def entries(ptr, ind, val):
    out = {}
    for r in range(len(ptr) - 1):
        for k in range(ptr[r], ptr[r + 1]):
            out[(r, int(ind[k]))] = val[k]
    return out


def brute(C, m, n, placed, I, J, accum):
    """placed: {(row, col): value} in C's coordinates."""
    d = entries(*C)
    ii = range(m) if I is None else [int(i) for i in I]
    jj = set(range(n)) if J is None else {int(j) for j in J}
    if accum is None:
        for i in ii:
            for j in jj:
                d.pop((i, j), None)
        d.update(placed)
    else:
        for k, v in placed.items():
            d[k] = OPS[accum](d[k], v) if k in d else v
    keys = sorted(d)
    ptr = np.zeros(m + 1, np.int64)
    for r, _ in keys:
        ptr[r + 1] += 1
    return np.cumsum(ptr), np.array([c for _, c in keys]), np.array([d[k] for k in keys])


def same(got, want):
    assert np.array_equal(got[0], want[0]), "row offsets differ"
    assert np.array_equal(got[1], want[1]), "columns differ"
    assert np.array_equal(np.asarray(got[2], np.float64), np.asarray(want[2], np.float64)), \
        "values differ"


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("tran", [False, True])
def test_submatrix_against_brute_force(seed, tran):
    rng = np.random.RandomState(seed)
    m, n = 17, 23
    Cs = random_csr(rng, m, n, 0.2, VALUES, zeros=0.2)
    C = (Cs.ptr, Cs.ind, Cs.val)
    for _, I in index_sets(rng, m):
        for _, J in index_sets(rng, n):
            nI = m if I is None else len(I)
            nJ = n if J is None else len(J)
            ar, ac = (nJ, nI) if tran else (nI, nJ)
            As = random_csr(rng, ar, ac, 0.3, VALUES, zeros=0.2)
            ii = np.arange(m) if I is None else I
            jj = np.arange(n) if J is None else J
            op = entries(As.ptr, As.ind, As.val)
            placed = {(int(ii[c if tran else r]), int(jj[r if tran else c])): v
                      for (r, c), v in op.items()}
            for accum in ACCUMS:
                got = R.assign_matrix(C, m, n, (As.ptr, As.ind, As.val, ar, ac), I, J,
                                      accum=accum, tran=tran)
                same(got, brute(C, m, n, placed, I, J, accum))


def test_constant_column_row_against_brute_force():
    rng = np.random.RandomState(5)
    m, n = 19, 14
    Cs = random_csr(rng, m, n, 0.25, VALUES, zeros=0.2)
    C = (Cs.ptr, Cs.ind, Cs.val)
    for _, I in index_sets(rng, m):
        for _, J in index_sets(rng, n):
            ii = np.arange(m) if I is None else I
            jj = np.arange(n) if J is None else J
            for accum in ACCUMS:
                placed = {(int(i), int(j)): np.float32(2) for i in ii for j in jj}
                same(R.assign_constant(C, m, n, 2.0, I, J, accum),
                     brute(C, m, n, placed, I, J, accum))
        for accum in ACCUMS:
            for u_ind in (np.arange(len(ii)), np.sort(rng.choice(len(ii), len(ii)//2,
                                                                  replace=False)), []):
                u_ind = np.asarray(u_ind, np.int64)
                u_val = rng.choice(VALUES, len(u_ind))
                j = int(rng.randint(n))
                placed = {(int(ii[k]), j): v for k, v in zip(u_ind, u_val)}
                same(R.assign_column(C, m, n, u_ind, u_val, I, j, accum),
                     brute(C, m, n, placed, I, [j], accum))
    for _, J in index_sets(rng, n):
        jj = np.arange(n) if J is None else J
        for accum in ACCUMS:
            u_ind = np.sort(rng.choice(len(jj), max(1, len(jj)//2), replace=False))
            u_val = rng.choice(VALUES, len(u_ind))
            i = int(rng.randint(m))
            placed = {(i, int(jj[k])): v for k, v in zip(u_ind, u_val)}
            same(R.assign_row(C, m, n, u_ind, u_val, i, J, accum),
                 brute(C, m, n, placed, [i], J, accum))


def test_round_trip_through_extract():
    rng = np.random.RandomState(9)
    m, n = 40, 31
    Cs = random_csr(rng, m, n, 0.15, VALUES, zeros=0.2)
    C = (Cs.ptr, Cs.ind, Cs.val)
    for _, I in index_sets(rng, m):
        for _, J in index_sets(rng, n):
            nI = m if I is None else len(I)
            nJ = n if J is None else len(J)
            As = random_csr(rng, nI, nJ, 0.3, VALUES, zeros=0.2)
            out = R.assign_matrix(C, m, n, (As.ptr, As.ind, As.val, nI, nJ), I, J)
            back = X.extract_matrix(*out, m, n, I, J)
            same(back, (As.ptr, As.ind, As.val))
            # outside the region: C's entries, unchanged
            keep_r = np.setdiff1d(np.arange(m), [] if I is None else I)
            if I is not None:
                same(X.extract_matrix(*out, m, n, keep_r, None),
                     X.extract_matrix(*C, m, n, keep_r, None))
            if J is not None:
                keep_c = np.setdiff1d(np.arange(n), J)
                same(X.extract_matrix(*out, m, n, None, keep_c),
                     X.extract_matrix(*C, m, n, None, keep_c))


def test_integer_plus_keeps_stored_zeros():
    rng = np.random.RandomState(4)
    Cs = random_csr(rng, 12, 12, 0.4, np.array([-2, 0, 1, 3], np.int32), zeros=0.3)
    As = random_csr(rng, 5, 6, 0.5, np.array([-1, 0, 2], np.int32), zeros=0.3)
    I, J = np.array([3, 0, 7, 11, 5]), np.array([1, 2, 9, 4, 10, 6])
    got = R.assign_matrix((Cs.ptr, Cs.ind, Cs.val), 12, 12, (As.ptr, As.ind, As.val, 5, 6),
                          I, J, accum="plus")
    assert got[2].dtype == np.int32
    placed = {(int(I[r]), int(J[c])): v for (r, c), v in
              entries(As.ptr, As.ind, As.val).items()}
    same(got, brute((Cs.ptr, Cs.ind, Cs.val), 12, 12, placed, I, J, "plus"))
    assert np.any(got[2] == 0)


# ---------------------------------------------------------------------------
# the companion header's contract
# ---------------------------------------------------------------------------

def test_header_symbols_exported_and_bound():
    from graphblast_b200 import _lib
    lib = C.CDLL(_lib.LIB_PATH)
    names = sorted(set(re.findall(r"\b(gb200_[a-z0-9_]+)\s*\(", HEADER)))
    assert names == ["gb200_assign_column", "gb200_assign_matrix",
                     "gb200_assign_matrix_scalar", "gb200_assign_row"]
    for name in names:
        assert hasattr(lib, name), "missing export: " + name
    assert {s[0] for s in _lib.ASSIGN_SIGNATURES} == set(names)
    assert "#define GB200_NO_ACCUM (-1)" in HEADER


def test_header_is_plain_c(tmp_path):
    src = str(tmp_path / "assign_header_check.c")
    with open(src, "w") as f:
        f.write('#include "graphblast_b200_assign.h"\n'
                'int main(void) { return GB200_NO_ACCUM + 1; }\n')
    out = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror",
                          "-I", os.path.join(ROOT, "include"), "-fsyntax-only", src],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr


def test_refusals_before_the_device_check():
    """NULL handles, then counts < 1 and unknown accums, then element types: none
    reads a device."""
    import graphblast_b200 as gb
    from graphblast_b200 import _lib
    lib = _lib.load()
    UNINIT = int(gb.Info.GrB_UNINITIALIZED_OBJECT)
    INVALID = int(gb.Info.GrB_INVALID_VALUE)
    DOMAIN = int(gb.Info.GrB_DOMAIN_MISMATCH)
    zero = (C.c_ubyte*64)()
    Z = C.cast(zero, C.c_void_p)        # a handle of neither element type, never read
    idx = (C.c_int*2)(0, 1)
    N = -1
    cases = [
        ("gb200_assign_matrix", [None, None, N, Z, idx, 2, idx, 2, Z], UNINIT),
        ("gb200_assign_matrix", [Z, None, N, None, idx, 2, idx, 2, Z], UNINIT),
        ("gb200_assign_matrix", [Z, None, N, Z, idx, 2, idx, 2, None], UNINIT),
        ("gb200_assign_matrix", [Z, None, N, Z, idx, 0, idx, 2, Z], INVALID),
        ("gb200_assign_matrix", [Z, None, N, Z, idx, 2, idx, -1, Z], INVALID),
        ("gb200_assign_matrix", [Z, None, 9, Z, idx, 2, idx, 2, Z], INVALID),
        ("gb200_assign_matrix", [Z, None, -2, Z, idx, 2, idx, 2, Z], INVALID),
        ("gb200_assign_matrix", [Z, None, N, Z, idx, 2, idx, 2, Z], DOMAIN),
        ("gb200_assign_matrix", [Z, None, 0, Z, idx, 2, idx, 2, Z], DOMAIN),
        ("gb200_assign_matrix_scalar", [None, None, N, 1.0, idx, 2, idx, 2, Z], UNINIT),
        ("gb200_assign_matrix_scalar", [Z, None, N, 1.0, idx, 2, idx, 2, None], UNINIT),
        ("gb200_assign_matrix_scalar", [Z, None, N, 1.0, idx, 0, idx, 2, Z], INVALID),
        ("gb200_assign_matrix_scalar", [Z, None, N, 1.0, idx, 2, idx, 0, Z], INVALID),
        ("gb200_assign_matrix_scalar", [Z, None, 9, 1.0, idx, 2, idx, 2, Z], INVALID),
        ("gb200_assign_column", [None, None, N, Z, idx, 2, 0, Z], UNINIT),
        ("gb200_assign_column", [Z, None, N, None, idx, 2, 0, Z], UNINIT),
        ("gb200_assign_column", [Z, None, N, Z, idx, 2, 0, None], UNINIT),
        ("gb200_assign_column", [Z, None, N, Z, idx, 0, 0, Z], INVALID),
        ("gb200_assign_column", [Z, None, 12, Z, idx, 2, 0, Z], INVALID),
        ("gb200_assign_column", [Z, None, N, Z, idx, 2, 0, Z], DOMAIN),
        ("gb200_assign_row", [None, None, N, Z, 0, idx, 2, Z], UNINIT),
        ("gb200_assign_row", [Z, None, N, None, 0, idx, 2, Z], UNINIT),
        ("gb200_assign_row", [Z, None, N, Z, 0, idx, 2, None], UNINIT),
        ("gb200_assign_row", [Z, None, N, Z, 0, idx, 0, Z], INVALID),
        ("gb200_assign_row", [Z, None, 9, Z, 0, idx, 2, Z], INVALID),
        ("gb200_assign_row", [Z, None, N, Z, 0, idx, 2, Z], DOMAIN),
    ]
    for name, args, want in cases:
        got = getattr(lib, name)(*args)
        assert got == want, "%s%r: %d, expected %d" % (name, tuple(args), got, want)
