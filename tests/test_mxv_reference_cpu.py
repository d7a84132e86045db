"""The CPU reference of mxv / vxm (mxv_reference.py) against the C oracle's
orc_vxm wherever the two define the same result (no mask on the generic pull,
no identity-valued operands), on every semiring; and the kernel constants the
designed shapes of test_mxv_gpu.py depend on, against the #defines."""
import os
import re

import numpy as np
import pytest

import mxm_reference as mref
import mxv_reference as ref
import oracle_binding as orc
from support import same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.path.join(ROOT, "graphblast_b200", "csrc", "graphblas", "backend", "cuda")


def random_coo(rng, nrows, ncols, density):
    mask = rng.rand(nrows, ncols) < density
    mask[rng.rand(nrows) < 0.15, :] = False
    mask[:, rng.rand(ncols) < 0.15] = False
    return np.nonzero(mask)


def to_csr(nrows, rows, cols, vals):
    order = np.lexsort((cols, rows))
    ptr = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=nrows))])
    return ptr.astype(np.int32), cols[order].astype(np.int32), vals[order]


def values_for(semiring, rng, n):
    """No value equals the semiring's identity (0, 1, FLT_MAX or FLT_MIN)."""
    pool = np.float32([-4, -3, -2, -0.5, 0.5, 2, 3, 4])
    if semiring != 11:
        pool = np.concatenate([pool, np.float32([-1, 1])])
    return rng.choice(pool, n).astype(np.float32)


SHAPES = [(1, 1), (7, 13), (40, 30), (90, 120)]


@pytest.mark.parametrize("semiring", range(17))
def test_pull_and_push_against_orc_vxm(semiring):
    rng = np.random.RandomState(100 + semiring)
    for m, n in SHAPES:
        rows, cols = random_coo(rng, m, n, 0.3)
        vals = values_for(semiring, rng, len(rows))
        rp, ci, rv = to_csr(m, rows, cols, vals)          # A, m x n
        cp, ri, cv = to_csr(n, cols, rows, vals)          # A's CSC
        u = values_for(semiring, rng, m)
        want, wp = orc.vxm(semiring, rp, ci, rv, u, ncols=n)
        # vxm pulls over the CSC: w = u^T A, column by column in row order
        got, bound = ref.pull(semiring, cp, ri, cv, u)
        if bound is None:
            assert same(got, want), (m, n)
        else:
            assert np.all(np.abs(got - want) <= bound + 2.0**-24*np.abs(got))
        # vxm pushes over the CSR from a sparse frontier; the present entries are
        # the columns some frontier row reaches
        f = np.sort(rng.choice(m, max(1, m//2), replace=False))
        up = np.zeros(m, np.uint8)
        up[f] = 1
        want, wp = orc.vxm(semiring, rp, ci, rv, u, ncols=n, u_present=up)
        w_ind, w_val = ref.push(semiring, rp, ci, rv, f, u[f], n)
        assert np.array_equal(w_ind, np.nonzero(wp)[0])
        assert same(w_val, want[wp != 0])


@pytest.mark.parametrize("scmp", [False, True])
@pytest.mark.parametrize("opreuse", [False, True])
def test_bool_pull_against_orc_vxm(scmp, opreuse):
    rng = np.random.RandomState(7)
    for m, n in SHAPES + [(50, 50)]:
        if opreuse and m != n:
            continue                  # the mask is the probe: square only
        rows, cols = random_coo(rng, m, n, 0.2)
        cp, ri, _ = to_csr(n, cols, rows, np.ones(len(rows), np.float32))
        rp, ci, rv = to_csr(m, rows, cols, np.ones(len(rows), np.float32))
        u = rng.choice(np.float32([0, 0, -0.0, 1, 2.5]), m)
        mask = rng.choice(np.float32([0, -0.0, 1, -3]), n)
        probe = mask if opreuse else u
        want, _ = orc.vxm(0, rp, ci, rv, probe, ncols=n, mask=mask, scmp=scmp)
        got = ref.bool_pull(cp, ri, mask, u, scmp=scmp, opreuse=opreuse)
        assert np.array_equal(got, (want != 0).astype(np.float32))


def test_quirks_the_oracle_does_not_define():
    # one row [a=-4 on column 0, a=2 on column 1]; MinimumPlus, identity FLT_MAX
    ptr, ind, val = np.array([0, 2]), np.array([0, 1]), np.float32([-4, 2])
    FM = mref.FLT_MAX
    # pull: masked-out rows hold the identity, accum folds with the semiring add
    w, _ = ref.pull(2, ptr, ind, val, np.float32([1, 1]), mask=np.float32([0]))
    assert w[0] == FM
    w, _ = ref.pull(2, ptr, ind, val, np.float32([1, 1]), mask=np.float32([0]),
                    w_old=np.float32([5]))
    assert w[0] == 5
    # pull has no identity short-circuit, push has one: u = FLT_MAX
    w, _ = ref.pull(2, ptr, ind, val, np.float32([FM, FM]))
    assert w[0] == np.float32(FM) + np.float32(-4)
    pi, pv = ref.push(2, np.array([0, 2]), np.array([0, 1]), val, [0], [FM], 2)
    assert list(pi) == [0, 1] and list(pv) == [FM, FM]
    # masked key-value push drops zero values, -0.0 included
    pi, pv = ref.push(1, np.array([0, 2]), np.array([0, 1]), np.float32([-1, 2]),
                      [0], [np.float32(0)], 2, mask=np.float32([1, 1]))
    assert len(pi) == 0
    pi, pv = ref.push(1, np.array([0, 2]), np.array([0, 1]), np.float32([-1, 2]),
                      [0], [np.float32(0)], 2)
    assert list(pi) == [0, 1]
    # min over -4 and -0.0 is -4, in either order
    pi, pv = ref.push(10, np.array([0, 1, 2]), np.array([0, 0]), np.float32([-4, -1]),
                      [0, 1], np.float32([1, 0]), 1)
    assert pv[0] == -4
    pi, pv = ref.push(10, np.array([0, 1, 2]), np.array([0, 0]), np.float32([-1, -4]),
                      [0, 1], np.float32([0, 1]), 1)
    assert pv[0] == -4


def _defines(*names):
    out = {}
    for name in names:
        text = open(os.path.join(CUDA, name)).read()
        for k, v in re.findall(r"^#define\s+(\w+)\s+(.+?)\s*(?://.*)?$", text, re.M):
            out[k] = v
    return out


def _int(d, key):
    expr = d[key]
    for k in sorted(d, key=len, reverse=True):
        if k in expr and k != key:
            expr = expr.replace(k, "(%s)" % d[k])
    return int(eval(expr, {}, {}))


def test_kernel_constants_match_the_gpu_test():
    """A change to a tile or class limit must come with a change to the designed
    shapes of test_mxv_gpu.py; this fails first."""
    import test_mxv_gpu as g
    d = _defines("kernels/spmv_pull.cuh", "kernels/spmv_hub.cuh", "spmv_hub.hpp",
                 "kernels/spmspv_push.cuh", "kernels/util.cuh")
    assert _int(d, "GB_SPMV_NT") == g.SPMV_NT
    assert _int(d, "GB_SPMV_IPT") == g.SPMV_IPT
    assert _int(d, "GB_SPMV_TILE") == g.TILE == 1152
    assert _int(d, "GB_HUB_RW") == g.HUB_RW
    assert _int(d, "GB_HUB_TILE") == g.HUB_TILE
    assert _int(d, "GB_HUB_CAPACITY") == g.HUB_CAPACITY
    assert _int(d, "GB_HUB_GROUPS") == g.HUB_GROUPS
    assert _int(d, "GB_PUSH_TILE") == g.PUSH_TILE
    assert _int(d, "GB_PUSH_SEG") == g.PUSH_SEG
    assert _int(d, "GB_DEGSCAN_MAX") == g.DEGSCAN_MAX
    assert _int(d, "GB_PULL_WPI") == g.PULL_WPI
    # a hub tile holds at most HUB_TILE / HUB_RW row ends: chunk_rel is one byte
    assert g.HUB_TILE // g.HUB_RW == g.HUB_ROWEND_LIMIT <= 255
