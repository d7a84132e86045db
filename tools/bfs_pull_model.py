"""CPU model of the pull levels of the fused BFS (kernels/bfs_fused.cuh).

Replays the kernel's decisions level by level on a CSR structure and counts, for
every pull iteration, the open rows (unvisited, not isolated), the open bitmap
words, the scan's batches (on the word path, on the row path, and with the
kernel's choice per chunk), and the rows the scan leaves to the walk under a probe
summary: a row is walked when it has more than one entry and its probed neighbour
is not visited as of the level's start.  Two summaries are compared: `first` (the
smallest-id neighbour) and `maxdeg` (the neighbour with the longest row, earliest
entry on a tie: the one the fused kernel probes).  It also gives entries_inspected_pulling as
the kernel counts it under `maxdeg`: one per probed open row, plus, per walked row,
its entries from entry 0 up to and including the first visited one (all of them
when none is).  Per pull level it gives the walk's shape: rows to walk per chunk of
1024 rows (p50, p99, max), the entries those walks inspect, and the chunks and rows
above GB_BFS_WALK_INLINE, which the kernel lists and walks grid-wide after the scan
instead of in the warp that scanned them.  And per pull level the floor of the
scan's summary stream: every open word needs its 32 `pull_probe` entries, one
128-byte line, so the scan reads at least 128 bytes per open word; those bytes
over the H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth are a floor computed
from the data sheet, not a measurement.

    python tools/bfs_pull_model.py [--scale 24] [--seed 1] [--mxvmode 0]
                                   [--walk-inline 64]

uses the oracle's R-MAT (tests/oracle_binding.py, symmetric) and the highest-degree
vertex as the source, as bench.py does.
"""
import argparse
import os
import sys

import numpy as np

BLOCK = 1 << 21          # rows per block of the entry-wise passes (bounds memory)
WALK_INLINE = 64         # GB_BFS_WALK_INLINE: a chunk with more rows to walk is listed
LINE = 128               # bytes of the summary line of one bitmap word (32 entries)
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet, HBM3


def probe_summary(rp, ci, rule, lengths=None):
    """probe[i]: the column row i probes, -1 for an empty row.  rule 'first' or
    'maxdeg'; lengths: the row lengths maxdeg ranks by (default: those of rp)."""
    n = len(rp) - 1
    if lengths is None:
        lengths = np.diff(rp)
    lengths = lengths.astype(np.int64)
    probe = np.full(n, -1, dtype=np.int64)
    for r0 in range(0, n, BLOCK):
        r1 = min(n, r0 + BLOCK)
        beg, end = int(rp[r0]), int(rp[r1])
        lens = np.diff(rp[r0:r1 + 1]).astype(np.int64)
        rows = np.nonzero(lens)[0]
        if len(rows) == 0:
            continue
        starts = (rp[r0:r1][rows] - beg).astype(np.int64)
        cols = ci[beg:end].astype(np.int64)
        if rule == "first":
            probe[r0 + rows] = cols[starts]
            continue
        pos = np.arange(end - beg, dtype=np.int64) - np.repeat(rp[r0:r1] - beg, lens)
        key = (lengths[cols] << 32) | (0xffffffff - pos)
        best = np.maximum.reduceat(key, starts)
        probe[r0 + rows] = cols[starts + (0xffffffff - (best & 0xffffffff))]
    return probe


def first_visited(rp, ci, rows, visited):
    """For each row in rows: position of its first visited entry, or its length."""
    out = (rp[rows + 1] - rp[rows]).astype(np.int64)
    rows_all = rows
    for k0 in range(0, len(rows_all), BLOCK):
        part = np.arange(k0, min(len(rows_all), k0 + BLOCK))
        part = part[out[part] > 0]
        if len(part) == 0:
            continue
        sel = rows_all[part]
        beg = rp[sel].astype(np.int64)
        lens = out[part]
        idx = np.repeat(beg - np.cumsum(lens) + lens, lens) + np.arange(lens.sum())
        pos = idx - np.repeat(beg, lens)
        hit = visited[ci[idx]]
        starts = np.cumsum(lens) - lens
        big = np.iinfo(np.int64).max
        first = np.minimum.reduceat(np.where(hit, pos, big), starts)
        out[part] = np.where(first == big, lens, first)
    return out


def has_visited_neighbour(rp, ci, rows, visited):
    return first_visited(rp, ci, rows, visited) < (rp[rows + 1] - rp[rows])


def replay(rp, ci, source, mode=0, switchpoint=0.01, isolated=None, probes=None,
           walk_inline=WALK_INLINE):
    """Level loop of the fused kernel on the pulled structure (rp, ci): row i's
    entries are the vertices it is discovered from.  isolated: rows visited from
    the start (default: the empty rows, as for a symmetric structure).  probes:
    {name: probe array}.  walk_inline: the kernel's GB_BFS_WALK_INLINE.  Returns a
    list of per-pull-iteration dicts and the total entries inspected pulling for
    each probe summary."""
    n = len(rp) - 1
    lens = np.diff(rp).astype(np.int64)
    if isolated is None:
        isolated = lens == 0
    if probes is None:
        probes = {"first": probe_summary(rp, ci, "first"),
                  "maxdeg": probe_summary(rp, ci, "maxdeg")}
    visited = isolated.copy()
    visited[source] = True
    fcount, dense, prev = 1, mode == 2, 0.0
    iters, inspected = [], {k: 0 for k in probes}
    level = 1
    while fcount > 0:
        if mode == 0:
            ratio = np.float32(fcount) / np.float32(n)
            if not dense:
                if ratio > switchpoint and ratio > prev:
                    dense = True
                else:
                    prev = ratio
            else:
                if ratio <= switchpoint and ratio < prev:
                    dense = False
                else:
                    prev = ratio
        open_rows = np.nonzero(~visited)[0]
        found = has_visited_neighbour(rp, ci, open_rows, visited)
        new = open_rows[found]
        if dense:
            words = np.unique(open_rows >> 5)
            it = {"level": level, "open_rows": len(open_rows), "open_words": len(words)}
            # scan batches (4 rounds) per chunk of 1024 rows: a round is an open word
            # on the word path, 32 open rows on the row path; a chunk takes the row
            # path when it needs fewer than half the batches
            wb = (np.bincount(words >> 5) + 3) // 4
            rb = (np.bincount(open_rows >> 10, minlength=len(wb)) + 127) // 128
            it["batches_word"] = int(wb.sum())
            it["batches_row"] = int(rb.sum())
            it["batches_chosen"] = int(np.where(2 * rb < wb, rb, wb).sum())
            for name, probe in probes.items():
                p = probe[open_rows]
                nonempty = p >= 0
                probed_hit = np.zeros(len(open_rows), dtype=bool)
                probed_hit[nonempty] = visited[p[nonempty]]
                walk = nonempty & ~probed_hit & (lens[open_rows] > 1)
                it["walked_" + name] = int(walk.sum())
                it["walked_found_" + name] = int((walk & found).sum())
                it["walked_not_found_" + name] = int((walk & ~found).sum())
                if name == "maxdeg":
                    fv = first_visited(rp, ci, open_rows[walk], visited)
                    wl = lens[open_rows[walk]]
                    walked = np.where(fv < wl, fv + 1, wl)
                    inspected[name] += int(nonempty.sum()) + int(walked.sum())
                    # the walk's split: chunks with at most walk_inline rows to
                    # walk are walked inline by the warp that scanned them, the
                    # others listed and walked grid-wide after the barrier
                    per_chunk = np.bincount(open_rows[walk] >> 10)
                    per_chunk = per_chunk[per_chunk > 0]
                    heavy = per_chunk > walk_inline
                    it["walk_counts"] = per_chunk
                    it["walk_chunks"] = len(per_chunk)
                    it["walk_per_chunk"] = (
                        tuple(int(np.percentile(per_chunk, q, method="lower"))
                              for q in (50, 99)) + (int(per_chunk.max()),)
                        if len(per_chunk) else (0, 0, 0))
                    it["walk_entries"] = int(walked.sum())
                    it["walk_entries_row_max"] = int(walked.max()) if len(wl) else 0
                    it["listed_chunks"] = int(heavy.sum())
                    it["listed_rows"] = int(per_chunk[heavy].sum())
            iters.append(it)
        visited[new] = True
        fcount = len(new)
        level += 1
    return iters, inspected


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--edgefactor", type=int, default=16)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--mxvmode", type=int, default=0, choices=[0, 2])
    ap.add_argument("--switchpoint", type=float, default=0.01)
    ap.add_argument("--walk-inline", type=int, default=WALK_INLINE,
                    help="rows to walk per chunk above which a chunk is listed")
    args = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                    "..", "tests"))
    import oracle_binding as orc
    rp, ci = orc.rmat_csr(args.scale, args.edgefactor, args.seed)
    rp = rp.astype(np.int64)
    source = int(np.argmax(np.diff(rp)))
    iters, inspected = replay(rp, ci, source, args.mxvmode, np.float32(args.switchpoint),
                              walk_inline=args.walk_inline)
    print("R-MAT-%d, edge factor %d, seed %d, source %d, mxvmode %d"
          % (args.scale, args.edgefactor, args.seed, source, args.mxvmode))
    print("%-5s %10s %10s %24s %24s" % ("level", "open rows", "open words",
                                        "walked first (found/not)",
                                        "walked maxdeg (found/not)"))
    for it in iters:
        print("L%-4d %10d %10d %10d (%d/%d) %10d (%d/%d)" % (
            it["level"], it["open_rows"], it["open_words"],
            it["walked_first"], it["walked_found_first"], it["walked_not_found_first"],
            it["walked_maxdeg"], it["walked_found_maxdeg"],
            it["walked_not_found_maxdeg"]))
    for it in iters:
        print("L%d scan batches: word path %d, row path %d, chosen per chunk %d" % (
            it["level"], it["batches_word"], it["batches_row"], it["batches_chosen"]))
    for it in iters:
        p50, p99, top = it["walk_per_chunk"]
        print("L%d walk (maxdeg): %d rows in %d chunks, per chunk p50 %d p99 %d max %d; "
              "%d entries inspected, at most %d per row; above %d per chunk: "
              "%d chunks, %d rows" % (
                  it["level"], it["walked_maxdeg"], it["walk_chunks"], p50, p99, top,
                  it["walk_entries"], it["walk_entries_row_max"], args.walk_inline,
                  it["listed_chunks"], it["listed_rows"]))
    for it in iters:
        nbytes = LINE*it["open_words"]
        print("L%d summary floor: %d open words, %d bytes of pull_probe lines, "
              "%.1f us at the data sheet's 3.35 TB/s (not a measurement)" % (
                  it["level"], it["open_words"], nbytes, 1e6*nbytes/HBM_BYTES_PER_S))
    print("entries inspected pulling (maxdeg probe, walk from entry 0): %d"
          % inspected["maxdeg"])


if __name__ == "__main__":
    main()
