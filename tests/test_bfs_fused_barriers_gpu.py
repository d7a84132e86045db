"""The grid barriers of the fused BFS (kernels/bfs_fused.cuh): one after the set-up,
one per level, and one more after each second phase, which a level runs only when
its main phase left work for the whole grid (a heavy vertex listed pushing, a chunk
listed pulling).  Level 1 of a push expands the source's list grid-wide, at any
degree, without scanning the frontier bitmap.

GB200_BFS_TRACE=1 prints the second phases of each traversal (each level marks in
its clock cell whether it ran one) and the barrier count they give on a `bfs
barriers:` line, and a walk time of 0 for a pull level without a second phase; the
switch is read once per process, so the traversals run in one subprocess.  Every
traversal is checked bit-exactly against the oracle's BFS in all three mxvmodes; the
second phases against the CPU model of tools/bfs_pull_model.py (listed chunks
pulling) and the oracle's levels (heavy vertices pushing); the work counters against
the values of the kernel before this barrier scheme."""
import functools
import json
import re

import numpy as np
import pytest

import oracle_binding as orc
from support import bfs_pull_model, star_graph
from test_bfs_fused_trace_gpu import run_traced
from test_bfs_fused_walk_gpu import H, S, layered

FUSED = dict(struconly=1, opreuse=1, earlyexit=1, switchpoint=0.01)
HEAVY = 2048              # GB_BFS_HEAVY
WALK_INLINE = 64          # GB_BFS_WALK_INLINE

model = bfs_pull_model()


# ---- graphs --------------------------------------------------------------------------

def listed_design():
    """The walk test's skeleton with 65 spread walk rows in chunk 2: the first pull
    level (level 2) lists that chunk, a second phase."""
    return layered(4200, walk_rows=2048 + 15 * np.arange(65))


def heavy_design():
    """S -> 200 mid rows -> 100 rows Q spread over four chunks -> P -> V -> 2100
    leaves.  Levels 2 and 3 pull (200 and 100 of 8192 rows); level 4 pushes P, which
    finds V; level 5 pushes V, whose 2101 neighbours go to the grid in a second
    phase."""
    mid, q, p, v = np.arange(100, 300), 3200 + 32 * np.arange(100), 400, 500
    leaves = 1024 + np.arange(2100)
    src = np.concatenate([np.full(len(mid), S), mid, q, [p], np.full(len(leaves), v)])
    dst = np.concatenate([mid, q[np.arange(len(mid)) % len(q)], np.full(len(q), p), [v],
                          leaves])
    return orc.build_csr(8192, src.astype(np.int32), dst.astype(np.int32), True)


def both_design():
    """The listed design with 1500 more leaves on H (2165 neighbours): level 2 lists
    chunk 2, level 3 pulls and finds H, level 4 pushes H in a second phase."""
    extra = [(H, 4200 + k) for k in range(1500)]
    return layered(5800, walk_rows=2048 + 15 * np.arange(65), extra=extra)


def self_loop_csr(width):
    """Hand-built, symmetric as a multiset: vertex 0 lists itself once and each of
    1..width twice, which list 0 twice back; vertex width+1 hangs off vertex 1, and
    the last 5 vertices are isolated.  width 5: a light source, 1100: a heavy one."""
    n = width + 7
    rows = [[0] + [i for i in range(1, width + 1) for _ in (0, 1)], [0, 0, width + 1]]
    rows += [[0, 0] for _ in range(2, width + 1)] + [[1]] + [[] for _ in range(5)]
    assert len(rows) == n
    rp = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    ci = np.concatenate([np.asarray(r, np.int32) for r in rows]).astype(np.int32)
    return rp, ci


@functools.lru_cache(maxsize=None)
def graph(name):
    """(rp, ci, {source name: vertex}) of a test graph."""
    if name == "rmat13":
        rp, ci = orc.rmat_csr(13)
        deg = np.diff(rp)
        light = int(np.nonzero((deg > 0) & (deg <= 4))[0][0])
        return rp, ci, {"hub": int(np.argmax(deg)), "light": light}
    if name == "star":
        rp, ci = star_graph(2100)
        return rp, ci, {"centre": 0, "leaf": 7}
    rp, ci = {"listed": listed_design, "heavy": heavy_design, "both": both_design,
              "loop5": lambda: self_loop_csr(5),
              "loop1100": lambda: self_loop_csr(1100)}[name]()
    return rp, ci, {"s": S}


MODES = (0, 1, 2)
# (graph, source, mode, max_niter or None)
CASES = ([("rmat13", s, m, cut) for s in ("hub", "light") for m in MODES
          for cut in (None, 1, 2)] +
         [(g, "s", m, None) for g in ("listed", "heavy", "both") for m in MODES] +
         [(g, "s", m, cut) for g in ("loop5", "loop1100") for m in MODES
          for cut in (None, 1)] +
         [("star", s, m, cut) for s in ("centre", "leaf") for m in MODES
          for cut in (None, 1, 2)])


def expected_second_phases(name, src, mode, cut):
    """Pull levels the model lists chunks at, and push levels after the first whose
    frontier holds a vertex of more than HEAVY neighbours, among the levels run."""
    rp, ci, sources = graph(name)
    s = sources[src]
    lv = orc.bfs(rp, ci, s)
    ran = int(lv.max()) if cut is None else min(cut, int(lv.max()))
    iters, _ = model.replay(rp.astype(np.int64), ci, s, mode=mode,
                            switchpoint=np.float32(0.01), walk_inline=WALK_INLINE)
    listed = {it["level"]: it["listed_chunks"] for it in iters}
    deg = np.diff(rp)
    phases = 0
    for level in range(1, ran + 1):
        if level in listed:
            phases += listed[level] > 0
        elif level > 1:
            phases += bool((deg[lv == level] > HEAVY).any())
    return phases


# The six work counters of each case (levels, entries inspected pulling, pull levels,
# vertices pushed, edges pushed, vertices discovered pushing), fixed from the kernel
# with two barriers per level and a frontier scan at level 1: SCRIPT below run on an
# NVIDIA H100 80GB HBM3 with GB200_LIB naming a library built from that kernel.  Every
# case's levels equalled the oracle's there.  The counters do not depend on the
# barriers or on which threads expand the source.
PARENT_STATS = {
    ('rmat13', 'hub', 0, None): [4, 4466, 3, 1, 2174, 2174],
    ('rmat13', 'hub', 0, 1): [1, 0, 0, 1, 2174, 2174],
    ('rmat13', 'hub', 0, 2): [2, 4334, 1, 1, 2174, 2174],
    ('rmat13', 'hub', 1, None): [4, 0, 0, 6478, 203876, 6477],
    ('rmat13', 'hub', 1, 1): [1, 0, 0, 1, 2174, 2174],
    ('rmat13', 'hub', 1, 2): [2, 0, 0, 2175, 169824, 6345],
    ('rmat13', 'hub', 2, None): [4, 44037, 4, 0, 0, 0],
    ('rmat13', 'hub', 2, 1): [1, 39571, 1, 0, 0, 0],
    ('rmat13', 'hub', 2, 2): [2, 43905, 2, 0, 0, 0],
    ('rmat13', 'light', 0, None): [6, 7561, 3, 9, 613, 498],
    ('rmat13', 'light', 0, 1): [1, 0, 0, 1, 4, 4],
    ('rmat13', 'light', 0, 2): [2, 0, 0, 5, 609, 498],
    ('rmat13', 'light', 1, None): [6, 0, 0, 6478, 203876, 6477],
    ('rmat13', 'light', 1, 1): [1, 0, 0, 1, 4, 4],
    ('rmat13', 'light', 1, 2): [2, 0, 0, 5, 609, 498],
    ('rmat13', 'light', 2, None): [6, 365351, 6, 0, 0, 0],
    ('rmat13', 'light', 2, 1): [1, 208851, 1, 0, 0, 0],
    ('rmat13', 'light', 2, 2): [2, 357790, 2, 0, 0, 0],
    ('listed', 's', 0, None): [5, 1997, 3, 2, 865, 800],
    ('listed', 's', 1, None): [5, 0, 0, 867, 1860, 866],
    ('listed', 's', 2, None): [5, 4258, 5, 0, 0, 0],
    ('heavy', 's', 0, None): [6, 8709, 3, 3, 2402, 2301],
    ('heavy', 's', 1, None): [6, 0, 0, 2403, 5202, 2402],
    ('heavy', 's', 2, None): [6, 17814, 6, 0, 0, 0],
    ('both', 's', 0, None): [5, 6497, 3, 2, 2365, 2300],
    ('both', 's', 1, None): [5, 0, 0, 2367, 4860, 2366],
    ('both', 's', 2, None): [5, 13258, 5, 0, 0, 0],
    ('loop5', 's', 0, None): [3, 7, 3, 0, 0, 0],
    ('loop5', 's', 0, 1): [1, 6, 1, 0, 0, 0],
    ('loop5', 's', 1, None): [3, 0, 0, 7, 23, 6],
    ('loop5', 's', 1, 1): [1, 0, 0, 1, 11, 5],
    ('loop5', 's', 2, None): [3, 7, 3, 0, 0, 0],
    ('loop5', 's', 2, 1): [1, 6, 1, 0, 0, 0],
    ('loop1100', 's', 0, None): [3, 1, 2, 1, 2201, 1100],
    ('loop1100', 's', 0, 1): [1, 0, 0, 1, 2201, 1100],
    ('loop1100', 's', 1, None): [3, 0, 0, 1102, 4403, 1101],
    ('loop1100', 's', 1, 1): [1, 0, 0, 1, 2201, 1100],
    ('loop1100', 's', 2, None): [3, 1102, 3, 0, 0, 0],
    ('loop1100', 's', 2, 1): [1, 1101, 1, 0, 0, 0],
    ('star', 'centre', 0, None): [2, 0, 1, 1, 2100, 2100],
    ('star', 'centre', 0, 1): [1, 0, 0, 1, 2100, 2100],
    ('star', 'centre', 0, 2): [2, 0, 1, 1, 2100, 2100],
    ('star', 'centre', 1, None): [2, 0, 0, 2101, 4200, 2100],
    ('star', 'centre', 1, 1): [1, 0, 0, 1, 2100, 2100],
    ('star', 'centre', 1, 2): [2, 0, 0, 2101, 4200, 2100],
    ('star', 'centre', 2, None): [2, 2100, 2, 0, 0, 0],
    ('star', 'centre', 2, 1): [1, 2100, 1, 0, 0, 0],
    ('star', 'centre', 2, 2): [2, 2100, 2, 0, 0, 0],
    ('star', 'leaf', 0, None): [3, 0, 1, 2, 2101, 2100],
    ('star', 'leaf', 0, 1): [1, 0, 0, 1, 1, 1],
    ('star', 'leaf', 0, 2): [2, 0, 0, 2, 2101, 2100],
    ('star', 'leaf', 1, None): [3, 0, 0, 2101, 4200, 2100],
    ('star', 'leaf', 1, 1): [1, 0, 0, 1, 1, 1],
    ('star', 'leaf', 1, 2): [2, 0, 0, 2, 2101, 2100],
    ('star', 'leaf', 2, None): [3, 4206, 3, 0, 0, 0],
    ('star', 'leaf', 2, 1): [1, 2107, 1, 0, 0, 0],
    ('star', 'leaf', 2, 2): [2, 4206, 2, 0, 0, 0],
}


# ---- the designs do what they say (CPU) ----------------------------------------------

def test_designs_second_phases():
    assert expected_second_phases("listed", "s", 0, None) == 1
    assert expected_second_phases("heavy", "s", 0, None) == 1
    assert expected_second_phases("both", "s", 0, None) == 2
    # the heavy vertex enters the frontier at a push level that follows a pull level
    for name, v in (("heavy", 500), ("both", H)):
        rp, ci, _ = graph(name)
        lv = orc.bfs(rp, ci, S)
        iters, _ = model.replay(rp.astype(np.int64), ci, S, mode=0,
                                switchpoint=np.float32(0.01), walk_inline=WALK_INLINE)
        pulls = {it["level"] for it in iters}
        assert np.diff(rp)[v] > HEAVY and lv[v] not in pulls and min(pulls) < lv[v], name
    rp, ci, _ = graph("listed")
    iters, _ = model.replay(rp.astype(np.int64), ci, S, mode=0,
                            switchpoint=np.float32(0.01), walk_inline=WALK_INLINE)
    assert [it["listed_chunks"] for it in iters][0] == 1
    rp, _, sources = graph("rmat13")
    assert np.diff(rp)[sources["light"]] <= HEAVY
    assert expected_second_phases("rmat13", "hub", 0, None) == 0
    for width in (5, 1100):
        rp, ci = self_loop_csr(width)
        row0 = ci[rp[0]:rp[1]]
        assert 0 in row0 and len(np.unique(row0)) < len(row0)
        assert (len(row0) > HEAVY) == (width == 1100)


# ---- the kernel (GPU) ---------------------------------------------------------------

SCRIPT = """
import json
import numpy as np
import graphblast_b200 as gb
from graphblast_b200 import algorithm
from support import bfs_levels, fused_stats, make_matrix
from test_bfs_fused_barriers_gpu import CASES, FUSED, graph
gb.init(0)
mats = {}
for name, src, mode, cut in CASES:
    rp, ci, sources = graph(name)
    if name not in mats:
        mats[name] = make_matrix(gb, rp, ci)
    s, n = sources[src], len(rp) - 1
    knobs = dict(FUSED, mxvmode=mode)
    if cut is not None:
        knobs["max_niter"] = cut
    desc = gb.Descriptor(**knobs)
    v = gb.Vector(n)
    algorithm.bfs(v, mats[name], s, desc)
    gb.sync()
    got = v.extractTuples().astype(np.int32)
    ok = bool(np.array_equal(got, bfs_levels(rp, ci, s, cut)))
    print(json.dumps([name, src, mode, cut, ok, fused_stats(desc, n)]), flush=True)
"""

BARRIERS_RE = re.compile(r"bfs barriers: (\d+) \(second phases (\d+)\)")
PULL_WALK_RE = re.compile(r" L\d+ pull [\d.]+us \(scan [\d.]+ walk ([\d.]+),")


@pytest.fixture(scope="module")
def traced():
    """{case: (levels equal the oracle's, stats, barriers, second phases, trace line)}"""
    stdout, stderr = run_traced(SCRIPT)
    rows = [json.loads(l) for l in stdout.splitlines()]
    lines = stderr.splitlines()
    traces = [l for l in lines if l.startswith("bfs trace:")]
    counts = [BARRIERS_RE.fullmatch(l) for l in lines if l.startswith("bfs barriers:")]
    assert len(rows) == len(traces) == len(counts) == len(CASES), stderr[-4000:]
    assert all(m is not None for m in counts), stderr[-4000:]
    out = {}
    for row, trace, m in zip(rows, traces, counts):
        out[tuple(row[:4])] = (row[4], row[5], int(m.group(1)), int(m.group(2)), trace)
    assert sorted(out, key=str) == sorted(CASES, key=str)
    return out


@pytest.mark.gpu
def test_levels_equal_the_oracle(traced):
    bad = [case for case, r in traced.items() if not r[0]]
    assert not bad, bad


@pytest.mark.gpu
def test_rmat13_hub_one_barrier_per_level(traced):
    _, stats, barriers, phases, trace = traced[("rmat13", "hub", 0, None)]
    assert stats[2] > 0 and phases == 0 and barriers == 1 + stats[0], (stats, barriers)
    # a pull level without a second phase reports a walk of 0
    walks = PULL_WALK_RE.findall(trace)
    assert len(walks) == stats[2] and all(float(w) == 0.0 for w in walks), trace


@pytest.mark.gpu
def test_second_phases_where_predicted(traced):
    for case, (_, stats, barriers, phases, trace) in traced.items():
        assert phases == expected_second_phases(*case), (case, trace)
        assert barriers == 1 + stats[0] + phases, (case, stats, barriers, phases)
        # a pull level's walk time is 0 exactly when it ran no second phase
        walks = PULL_WALK_RE.findall(trace)
        assert len(walks) == stats[2], trace
        assert sum(float(w) > 0.0 for w in walks) <= phases, trace
    assert traced[("listed", "s", 0, None)][3] == 1
    assert traced[("heavy", "s", 0, None)][3] == 1
    assert traced[("both", "s", 0, None)][3] == 2


@pytest.mark.gpu
def test_level_one_from_the_source(traced):
    """Cut after level 1 in the push modes: one vertex pushed, its whole list (self
    loop and duplicates included) as the edges pushed."""
    for case, (_, stats, _, _, _) in traced.items():
        name, src, mode, cut = case
        rp, ci, sources = graph(name)
        s = sources[src]
        if cut == 1 and mode == 1:
            deg = int(rp[s + 1] - rp[s])
            lv = orc.bfs(rp, ci, s)
            assert stats[3] == 1 and stats[4] == deg, (case, stats)
            assert stats[5] == int((lv == 2).sum()), (case, stats)


@pytest.mark.gpu
def test_work_counters_equal_the_parents(traced):
    for case, (_, stats, _, _, _) in traced.items():
        assert stats == PARENT_STATS[case], (case, stats, PARENT_STATS[case])
