"""sssp_pr_reference.py on the CPU: sssp_rounds against the oracle's lazy Dijkstra,
pagerank64 against the oracle's float32 PageRank within pagerank_bound, and the
bound tight enough that one dropped edge or one halved value leaves it."""
import numpy as np
import pytest

import oracle_binding as orc
import sssp_pr_reference as ref
import support

FLT_MAX = ref.FLT_MAX


def _graphs():
    out = {"rmat12": orc.rmat_csr(12), "star": support.star_graph(500),
           "path": support.path_graph(300), "ragged": support.ragged_graph()}
    src, dst = orc.rmat_edges(10)
    out["rmat10dir"] = orc.build_csr(1 << 10, src, dst, False)
    return out


GRAPHS = _graphs()


@pytest.mark.parametrize("kind", ["int", "real", "zero10", "spread", "overflow"])
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_sssp_rounds_at_convergence_is_the_oracle(name, kind):
    rp, ci = GRAPHS[name]
    w = ref.sssp_weights(kind, len(ci))
    deg = np.diff(rp)
    for s in (int(np.argmax(deg)), len(rp) - 2):
        want = orc.sssp(rp, ci, w, s)
        got, rounds = ref.sssp_rounds(rp, ci, w, s)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (s, kind)
        assert np.all(np.isfinite(got))
        if kind == "overflow" and name == "path":
            # the far end of the path is reached only by sums that overflow
            far, near = (-1, s + 1) if s < 150 else (0, s - 1)
            assert got[far] == FLT_MAX and 0 < got[near] < FLT_MAX


def test_sssp_rounds_cut():
    """k rounds reach exactly the vertices within k hops, each at its shortest
    distance over at most k edges."""
    rp, ci = GRAPHS["path"]
    w = ref.sssp_weights("real", len(ci))
    full, rounds = ref.sssp_rounds(rp, ci, w, 0)
    assert rounds == len(rp) - 1            # the last round improves nothing
    for k in (1, 2, 3):
        got, r = ref.sssp_rounds(rp, ci, w, 0, k)
        assert r == k
        assert np.array_equal(got[:k + 1], full[:k + 1])
        assert np.all(got[k + 1:] == FLT_MAX)


def normalised(rp, ci, val, alpha):
    """The device's pr_normalize in float32: fl(fl(alpha * a) / rowsum)."""
    f = np.float32
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    rowsum = np.zeros(len(rp) - 1, np.float64)
    np.add.at(rowsum, rows, val.astype(np.float64))
    return (f(alpha)*val.astype(f)) / rowsum.astype(f)[rows]


@pytest.mark.parametrize("alpha", [0.85, 0.1])
@pytest.mark.parametrize("name", ["rmat12", "star", "path", "ragged"])
def test_pagerank64_is_the_oracle_within_the_bound(name, alpha):
    rp, ci = GRAPHS[name]
    n = len(rp) - 1
    val = normalised(rp, ci, np.ones(len(ci), np.float32), alpha)
    jump, p0 = ref.jump_and_start(alpha, n)
    ps = ref.pagerank64(rp, ci, val, jump, p0, 10)
    bs = ref.pagerank_bound(rp, ci, val, ps, jump, order="oracle")
    for k in (1, 2, 10):
        got = orc.pr(rp, ci, alpha=alpha, eps=0.0, max_niter=k)
        assert ref.within(got, ps[k], bs[k]), k
    # the device-order bound is no looser than the oracle-order one
    db = ref.pagerank_bound(rp, ci, val, ps, jump)
    assert np.all(db[10] <= bs[10])


def _edge_into(ci, j, nth):
    """Position of the nth stored entry in column j."""
    return int(np.nonzero(ci == j)[0][nth])


@pytest.mark.parametrize("mutation", ["drop", "halve"])
@pytest.mark.parametrize("name", ["rmat12", "rmat10dir", "ragged"])
def test_bound_catches_one_wrong_entry(name, mutation):
    """For three vertices of in-degree <= 8: one dropped entry into the vertex, or
    one of its normalised values halved, moves the reference out of the bound there,
    at iteration 1 and at 10."""
    rp, ci = GRAPHS[name]
    n = len(rp) - 1
    val = normalised(rp, ci, ref.sssp_weights("real", len(ci)), 0.85)
    jump, p0 = ref.jump_and_start(0.85, n)
    ps = ref.pagerank64(rp, ci, val, jump, p0, 10)
    bs = ref.pagerank_bound(rp, ci, val, ps, jump)
    indeg = np.bincount(ci, minlength=n)
    targets = np.nonzero((indeg >= 1) & (indeg <= 8))[0]
    assert len(targets) >= 3
    for j in targets[[0, len(targets)//2, -1]]:
        e = _edge_into(ci, j, int(indeg[j]) - 1)
        mval = val.copy()
        if mutation == "drop":
            mval[e] = 0             # the same as removing the entry
        else:
            mval[e] = mval[e] / 2
        wrong = ref.pagerank64(rp, ci, mval, jump, p0, 10)
        for k in (1, 10):
            assert ref.outside(wrong[k], ps[k], bs[k])[j], (j, k)
