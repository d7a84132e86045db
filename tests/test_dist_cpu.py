"""CPU tests of the multi-GPU host logic in graphblast_b200/dist.py: the
nnz-balanced partition and the slice extraction (the traversals need a GPU and are
covered by the gpu-marked tests and bench.py --gpus N)."""
import numpy as np
import torch

import oracle_binding as orc
from graphblast_b200 import dist as gdist


def test_partition_bounds_properties():
    rp, ci = orc.rmat_csr(12)
    n = len(rp) - 1
    for world in (1, 2, 4, 8):
        b = gdist.partition_bounds(rp, world, align=32)
        assert b[0] == 0 and b[-1] == n and len(b) == world + 1
        assert all(x % 32 == 0 for x in b)
        assert all(b[i] <= b[i + 1] for i in range(world))
        if world > 1:
            share = np.diff(rp[np.array(b)]) / float(rp[-1])
            # RMAT rows are heavily skewed towards low ids; equal vertex ranges
            # would give rank 0 ~40% of the entries at world 8
            assert share.max() < 2.0 / world + 0.05


def test_local_slice_permutation_carries_values():
    """local_slice(return_order=True): val[order] are the CSC values of the owned
    rows, i.e. the (colptr, rowind, val[order]) triple is the transpose of
    (rp_local, ci_local, val) — what weighted_local_matrix hands to the library — on
    hand-picked slices and on the partition_bounds slices of 2 and 3 ranks."""
    rp, ci = orc.rmat_csr(9)
    n = len(rp) - 1
    rowptr = torch.from_numpy(rp)
    colind = torch.from_numpy(ci)
    rng = np.random.RandomState(3)
    val = torch.from_numpy(rng.randint(1, 65, size=len(ci)).astype(np.float32))
    slices = [(0, n), (64, 320), (n - 128, n)]
    for world in (2, 3):
        b = gdist.partition_bounds(rowptr, world, align=64)
        slices += [(b[p], b[p + 1]) for p in range(world)]
    for lo, hi in slices:
        rp_l, ci_l, colptr, rowind, order = gdist.local_slice(
            rowptr, colind, lo, hi, n, return_order=True)
        e0, e1 = int(rp[lo]), int(rp[hi])
        val_l = val[e0:e1]
        cval = val_l[order]
        dense = np.zeros((hi - lo, n), dtype=np.float32)
        rp_n, ci_n = rp_l.numpy(), ci_l.numpy()
        for r in range(hi - lo):
            dense[r, ci_n[rp_n[r]:rp_n[r + 1]]] = val_l.numpy()[rp_n[r]:rp_n[r + 1]]
        cp, ri, cv = colptr.numpy(), rowind.numpy(), cval.numpy()
        assert cp[-1] == e1 - e0
        for c in range(n):
            rows = ri[cp[c]:cp[c + 1]]
            assert np.all(np.diff(rows) > 0)                 # sorted, unique
            assert np.array_equal(dense[rows, c], cv[cp[c]:cp[c + 1]])
        assert np.count_nonzero(dense) == e1 - e0
