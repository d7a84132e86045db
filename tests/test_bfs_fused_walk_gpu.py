"""The walk of the fused BFS's pull levels (kernels/bfs_fused.cuh): a chunk of 1024
rows with at most GB_BFS_WALK_INLINE rows to walk is walked by the warp that scanned
it, its discoveries going out with the owners' stores of the chunk's words; a chunk
with more is listed and walked grid-wide after the scan barrier.  Designed graphs put
chunks on both sides of the threshold, inline discoveries in the same bitmap words as
the scan's, a long inline walk through the warp-wide loop and a partial last chunk.
Levels are compared bit-exactly with the oracle's BFS in all three mxvmodes, and in
modes 0 and 2 the kernel's count of inspected entries with the CPU model of
tools/bfs_pull_model.py."""
import numpy as np
import pytest

import oracle_binding as orc
from support import bfs_pull_model, fused_stats, gb, make_matrix, transpose

FUSED = dict(struconly=1, opreuse=1, earlyexit=1, switchpoint=0.01)
WALK_INLINE = 64          # GB_BFS_WALK_INLINE


model = bfs_pull_model()

# The designed graphs share one skeleton.  S reaches the mid rows at the first level;
# H has the highest degree (its leaves), so a row whose entries are a mid row and H
# probes H, which is not visited, and is walked; its walk finds the mid row once that
# is visited.  A row whose only entry is a mid row is found by the scan's probe.
S, H = 0, 500
MID = np.arange(100, 300)
LEAVES = np.arange(3072, 3672)


def layered(n, walk_rows=(), hit_rows=(), late_rows=(), extra=()):
    """walk_rows: walked, found a level after the mid rows; hit_rows: found by the
    probe at the same level; late_rows: walked at that level without a find (their
    entries are a leaf of H and H).  extra: more (src, dst) pairs."""
    walk_rows, hit_rows, late_rows = (np.asarray(x, np.int64)
                                      for x in (walk_rows, hit_rows, late_rows))
    src = [np.full(len(MID), S), np.full(len(LEAVES), H), walk_rows, walk_rows,
           hit_rows, late_rows, late_rows]
    dst = [MID, LEAVES, MID[np.arange(len(walk_rows)) % len(MID)],
           np.full(len(walk_rows), H), MID[np.arange(len(hit_rows)) % len(MID)],
           LEAVES[np.arange(len(late_rows)) % len(LEAVES)], np.full(len(late_rows), H)]
    for s_, d_ in extra:
        src.append(np.asarray([s_])); dst.append(np.asarray([d_]))
    src = np.concatenate(src).astype(np.int32)
    dst = np.concatenate(dst).astype(np.int32)
    return orc.build_csr(n, src, dst, True)


def both_paths():
    """Chunk 1: 64 walk rows in two full words (word path, inline); chunk 2: 65
    spread rows (row path, listed); chunk 4: 65 rows in three words (word path,
    listed); chunk 5: 64 spread rows (row path, inline)."""
    rows = np.concatenate([1024 + np.arange(64), 2048 + 15 * np.arange(65),
                           4096 + np.arange(65), 5120 + 15 * np.arange(64)])
    return layered(6400, walk_rows=rows)


def shared_words():
    """Walked rows found inline, walked rows not found and rows the probe finds,
    interleaved in the same bitmap words: chunk 1 on the word path (two full words),
    chunk 2 on the row path (four open rows in each of 24 words)."""
    dense = 1024 + np.arange(64)
    sparse = 2048 + 8 * np.arange(96)
    walk = np.concatenate([dense[0::3], sparse[0::3]])
    hit = np.concatenate([dense[1::3], sparse[1::3]])
    late = np.concatenate([dense[2::3], sparse[2::3]])
    return layered(4200, walk_rows=walk, hit_rows=hit, late_rows=late)


def long_row():
    """Row 1500, alone in its chunk with three short walk rows, lists H, 40 leaves of
    its own and, last, 5100, which S reaches: the walk takes four entries, then the
    warp walks the other 38, and only the last one is visited."""
    extra = [(1500, H)] + [(1500, 5000 + k) for k in range(40)] + [(1500, 5100),
                                                                    (S, 5100)]
    return layered(5200, walk_rows=[1501, 1530, 1990], extra=extra)


def partial_last_chunk():
    """n = 5 * 1024 + 517 (not a multiple of 32): 40 walk rows and 20 probe hits in
    the last chunk, row n - 1 among the walked, and a listed chunk of 100 rows."""
    n = 5 * 1024 + 517
    walk = np.concatenate([n - 1 - 13 * np.arange(40), 1024 + 7 * np.arange(100)])
    hit = n - 2 - 13 * np.arange(20)
    return layered(n, walk_rows=walk, hit_rows=hit)


DESIGNS = {"both_paths": both_paths, "shared_words": shared_words,
           "long_row": long_row, "partial_last_chunk": partial_last_chunk}


def model_levels(rp, ci, s, mode, directed=False):
    """Per-pull-level dicts and the entries inspected pulling, by the CPU model."""
    if not directed:
        iters, insp = model.replay(rp.astype(np.int64), ci, s, mode=mode,
                                   switchpoint=np.float32(0.01), walk_inline=WALK_INLINE)
        return iters, insp["maxdeg"]
    t_rp, t_ci, _ = transpose(rp, ci)
    isolated = (np.diff(t_rp) == 0) & (np.diff(rp) == 0)
    iters, insp = model.replay(t_rp.astype(np.int64), t_ci, s, mode=mode,
                               switchpoint=np.float32(0.01), isolated=isolated,
                               walk_inline=WALK_INLINE)
    return iters, insp["maxdeg"]


# ---- the designs do what they say (CPU) -----------------------------------------------

@pytest.mark.parametrize("mode", [0, 2])
def test_designs_put_chunks_on_both_sides(mode):
    rp, ci = both_paths()
    iters, _ = model_levels(rp, ci, S, mode)
    levels = [it for it in iters
              if WALK_INLINE in it["walk_counts"] and WALK_INLINE + 1 in it["walk_counts"]]
    assert levels, [list(it["walk_counts"]) for it in iters]
    assert all(it["listed_chunks"] == 2 for it in levels)

    rp, ci = partial_last_chunk()
    n = len(rp) - 1
    iters, _ = model_levels(rp, ci, S, mode)
    assert any(it["listed_chunks"] == 1 and 40 in it["walk_counts"] for it in iters)
    assert n % 32 != 0 and n % 1024 != 0

    rp, ci = long_row()
    assert ci[rp[1501] - 1] == 5100 and rp[1501] - rp[1500] == 42
    # row 1500 probes H, and when it is found its last entry is its only visited one
    assert model.probe_summary(rp.astype(np.int64), ci, "maxdeg")[1500] == H
    lv = orc.bfs(rp, ci, S)
    nbrs = ci[rp[1500]:rp[1501]]
    assert lv[1500] == lv[5100] + 1 and (lv[nbrs[:-1]] > lv[5100]).all()
    iters, _ = model_levels(rp, ci, S, mode)
    assert all(it["listed_chunks"] == 0 for it in iters)

    rp, ci = shared_words()
    iters, _ = model_levels(rp, ci, S, mode)
    assert all(it["listed_chunks"] == 0 for it in iters)
    assert any(it["walked_found_maxdeg"] > 0 and it["walked_not_found_maxdeg"] > 0
               for it in iters)


# ---- the kernel (GPU) ---------------------------------------------------------------

def check(gb, rp, ci, sources, directed=False):
    """Levels in all three modes against the oracle, one descriptor per mode for
    all the sources (traversals back to back); in modes 0 and 2 the inspected
    entries against the model."""
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
            if mode != 1:
                _, want = model_levels(rp, ci, s, mode, directed)
                assert stats[1] == want, (mode, s)


@pytest.mark.gpu
@pytest.mark.parametrize("design", sorted(DESIGNS))
def test_designed_walks(gb, design):
    rp, ci = DESIGNS[design]()
    n = len(rp) - 1
    check(gb, rp, ci, [S, int(MID[3]), n - 1])


@pytest.mark.gpu
def test_back_to_back_listed_then_inline(gb):
    """One descriptor: a traversal that lists chunks, one from a leaf of H whose pull
    levels walk other chunks, then the first again and one from a listed chunk's
    row: stale walk lists or counts would show in the levels or the counts."""
    rp, ci = both_paths()
    check(gb, rp, ci, [S, int(LEAVES[7]), S, 2048 + 15 * 10, S])


@pytest.mark.gpu
def test_directed_both_paths(gb):
    """The both-paths layout directed: S -> mid rows, H <-> its leaves, a mid row
    and H -> each walk row, every fourth walk row -> H.  Rows are pulled over their
    in-neighbours, and H has the most."""
    n = 6400
    rows = np.concatenate([1024 + np.arange(64), 2048 + 15 * np.arange(65),
                           4096 + np.arange(65), 5120 + 15 * np.arange(64)])
    mids = MID[np.arange(len(rows)) % len(MID)]
    src = np.concatenate([np.full(len(MID), S), np.full(len(LEAVES), H), LEAVES,
                          mids, np.full(len(rows), H), rows[::4]]).astype(np.int32)
    dst = np.concatenate([MID, LEAVES, np.full(len(LEAVES), H), rows, rows,
                          np.full(len(rows[::4]), H)]).astype(np.int32)
    rp, ci = orc.build_csr(n, src, dst, False)
    iters, _ = model_levels(rp, ci, S, 2, directed=True)
    assert any(it["listed_chunks"] == 2 and WALK_INLINE in it["walk_counts"]
               for it in iters)
    check(gb, rp, ci, [S, H, int(rows[4]), int(MID[0])], directed=True)
