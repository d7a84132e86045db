"""The pull levels of the fused BFS (kernels/bfs_fused.cuh): the highest-degree
neighbour each open row probes (pullMaxDegreeNeighbourKernel), the walk that starts
at entry 0, and the scan that takes a chunk's open rows 32 at a time.  Levels are
compared bit-exactly with the oracle's BFS in all three mxvmodes; in pull-only
traversals the kernel's count of inspected entries must equal the CPU model of
tools/bfs_pull_model.py."""
import numpy as np
import pytest

import oracle_binding as orc
from support import bfs_pull_model, fused_stats, gb, make_matrix, symmetric_csr, transpose

pytestmark = pytest.mark.gpu

FUSED = dict(struconly=1, opreuse=1, earlyexit=1)
model = bfs_pull_model()


def model_inspected(rp, ci, s, directed=False):
    """entries_inspected_pulling of a pull-only traversal, by the CPU model."""
    if not directed:
        _, insp = model.replay(rp.astype(np.int64), ci, s, mode=2)
        return insp["maxdeg"]
    t_rp, t_ci, _ = transpose(rp, ci)
    isolated = (np.diff(t_rp) == 0) & (np.diff(rp) == 0)
    _, insp = model.replay(t_rp.astype(np.int64), t_ci, s, mode=2, isolated=isolated)
    return insp["maxdeg"]


def check(gb, rp, ci, sources, directed=False, count=True):
    """Levels in all three modes against the oracle; in pull-only mode the
    inspected entries against the model."""
    from graphblast_b200 import algorithm
    n = len(rp) - 1
    A = make_matrix(gb, rp, ci, symmetric=not directed)
    for mode in (0, 1, 2):
        desc = gb.Descriptor(mxvmode=mode, **FUSED)
        for s in sources:
            v = gb.Vector(n)
            algorithm.bfs(v, A, s, desc)
            got = v.extractTuples().astype(np.int32)
            assert np.array_equal(got, orc.bfs(rp, ci, s)), (mode, s)
            stats = fused_stats(desc, n)
            assert stats[0] > 0
            if mode == 2 and count:
                assert stats[2] == stats[0]
                assert stats[1] == model_inspected(rp, ci, s, directed), s


def test_summary_is_the_highest_degree_neighbour():
    """The CPU model's summary on a hand-checked graph: ties take the earliest
    entry, empty rows are -1."""
    # 0: {1, 2, 3}; 1: {0}; 2: {0, 4, 5}; 3: {0, 6, 7}; 4..7 leaves of 2 and 3; 8 alone
    rp, ci = symmetric_csr(9, [0, 0, 0, 2, 2, 3, 3], [1, 2, 3, 4, 5, 6, 7])
    probe = model.probe_summary(rp.astype(np.int64), ci, "maxdeg")
    assert list(probe) == [2, 0, 0, 0, 2, 2, 3, 3, -1]
    assert list(model.probe_summary(rp.astype(np.int64), ci, "first")) == \
        [1, 0, 0, 0, 2, 2, 3, 3, -1]


def test_highest_degree_neighbour_not_first(gb):
    """Every row of the middle layer has a low-degree first neighbour and a
    high-degree later one."""
    src, dst = [], []
    hubs = list(range(100, 110))
    for h in hubs:                                  # hubs of degree 40 + middle rows
        for k in range(40):
            src.append(h); dst.append(1000 + 40 * (h - 100) + k)
    for r in range(10, 90):                         # middle rows: [r - 10, hub]
        src.append(r); dst.append(r - 10)
        src.append(r); dst.append(hubs[r % 10])
    n = 1500
    rp, ci = symmetric_csr(n, src, dst)
    check(gb, rp, ci, [100, 0, 15, 1005])


def test_degree_ties(gb):
    """Rows whose neighbours all have the same degree: the earliest one is probed."""
    rng = np.random.default_rng(5)
    n = 4096
    # a 4-regular circulant graph: every neighbour ties
    v = np.arange(n)
    src = np.concatenate([v, v])
    dst = np.concatenate([(v + 1) % n, (v + 7) % n])
    rp, ci = symmetric_csr(n, src, dst)
    check(gb, rp, ci, [0, int(rng.integers(n))])


def test_single_entry_rows(gb):
    """Stars and chains: most rows have one entry (bit 31 of the summary)."""
    src = [0] * 300 + list(range(300, 2000))
    dst = list(range(1, 301)) + list(range(301, 2001))
    rp, ci = symmetric_csr(2100, src, dst)
    check(gb, rp, ci, [0, 5, 2000, 1200])


def test_only_visited_neighbour_is_entry_zero(gb):
    """Row 1's list is [0, 2]: 2 has the higher degree and is probed, but only 0
    is visited at the first pull level.  A walk that started at entry 1 would miss
    it and give row 1 the wrong level."""
    src = [1, 1] + [2] * 50 + [10] * 60
    dst = [0, 2] + list(range(100, 150)) + list(range(200, 260))
    n = 300
    rp, ci = symmetric_csr(n, src, dst)
    assert list(ci[rp[1]:rp[2]]) == [0, 2]
    assert model.probe_summary(rp.astype(np.int64), ci, "maxdeg")[1] == 2
    from graphblast_b200 import algorithm
    A = make_matrix(gb, rp, ci)
    desc = gb.Descriptor(mxvmode=2, **FUSED)
    v = gb.Vector(n)
    algorithm.bfs(v, A, 0, desc)
    got = v.extractTuples().astype(np.int32)
    assert got[1] == 2 and got[2] == 3
    assert np.array_equal(got, orc.bfs(rp, ci, 0))
    check(gb, rp, ci, [0, 2, 100])


def test_directed_in_and_out_degree_rank_differently(gb):
    """Row r's in-neighbours are a (many out-edges, one in-edge) and b (many
    in-edges, one out-edge to r): the summary ranks by in-degree and probes b."""
    src, dst = [], []
    a, b = 10, 20
    for r in range(100, 140):
        src += [a, b]; dst += [r, r]
    for k in range(200, 260):                       # in-edges of b
        src.append(k); dst.append(b)
    for k in range(300, 320):                       # out-edges of a
        src.append(a); dst.append(k)
    src += [0, 0, 1]; dst += [a, 1, 200]            # 0 -> a, 0 -> 1 -> 200 -> b
    n = 400
    rp, ci = orc.build_csr(n, np.asarray(src, np.int32), np.asarray(dst, np.int32), False)
    t_rp, t_ci, _ = transpose(rp, ci)
    probe = model.probe_summary(t_rp.astype(np.int64), t_ci, "maxdeg")
    assert probe[100] == b
    check(gb, rp, ci, [0, a, 1, 250], directed=True)


@pytest.mark.parametrize("scale", [8, 11, 13])
def test_rmat_inspected_count(gb, scale):
    rp, ci = orc.rmat_csr(scale)
    deg = np.diff(rp)
    check(gb, rp, ci, [int(np.argmax(deg)), int(np.nonzero(deg)[0][-1])])


def test_directed_rmat_inspected_count(gb):
    n = 1 << 12
    src, dst = orc.rmat_edges(12, 8, seed=7)
    rp, ci = orc.build_csr(n, src, dst, False)
    check(gb, rp, ci, [int(np.argmax(np.diff(rp))), 0], directed=True)


def test_chunks_with_few_and_many_open_rows(gb):
    """Chunks of 1024 rows with 0, 1, 31, 32, 33, 128, 129 and 1024 non-isolated
    rows spread over their words, 32 in one word, then a last chunk of 517 rows (n
    is not a multiple of 32).  Sparse chunks take their open rows 32 at a time, 4
    rounds per batch; dense ones a word at a time."""
    rng = np.random.default_rng(11)
    layouts = [0, 1, 31, 32, 33, 128, 129, 1024, "word"]
    rows = []
    for c, k in enumerate(layouts):
        if k == "word":
            pos = np.arange(64, 96)
        else:
            pos = np.sort(rng.choice(1024, k, replace=False))
        rows.append(c * 1024 + pos)
    tail = 517
    n = len(layouts) * 1024 + tail
    rows.append(np.arange(len(layouts) * 1024, n))
    live = rng.permutation(np.concatenate(rows))
    # a random tree over the live rows (depth ~ log) plus as many random edges
    parent = live[(rng.random(len(live) - 1) * np.arange(1, len(live))).astype(np.int64)]
    src = np.concatenate([live[1:], live[rng.integers(len(live), size=len(live))]])
    dst = np.concatenate([parent, live[rng.integers(len(live), size=len(live))]])
    keep = src != dst
    rp, ci = symmetric_csr(n, src[keep], dst[keep])
    assert (np.diff(rp)[:1024] == 0).all() and np.diff(rp)[n - 1] > 0
    deg = np.diff(rp)
    check(gb, rp, ci, [int(live[0]), int(np.argmax(deg)), n - 1, int(rows[1][0])])
