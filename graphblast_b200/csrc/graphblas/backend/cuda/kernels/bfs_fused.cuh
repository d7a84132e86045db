// graphblast_b200 backend — the whole direction-optimised BFS as ONE persistent
// cooperative kernel (SURVEY.md §8 f2, loop fusion behind the same API).
//
// The operation sequence of reference graphblas/algorithm/bfs.hpp:46-79 per level —
//   assign(v<f> = level); vxm(f' <!v> = f (||.&&) A); swap; succ = reduce(+, f') —
// with --struconly 1 --opreuse 1 --earlyexit 1 --fusedmask 1 costs 2 launches on a
// pull level and 6 on a push level through the generic operations, plus a host
// read of the frontier size; a traversal of R-MAT scale 24 (6 levels, 0.47 ms) is
// then half launch latency.  Here the level loop, the direction decision, the
// level assignment and the frontier count all live in the kernel; levels are
// separated by grid-wide barriers (cooperative launch, one CTA set resident for
// the whole traversal).
//
// State: visited bitmap (two copies, ping-pong on pull levels), frontier bitmap F,
// next-frontier bitmap N, a byte per row holding its level while the traversal runs,
// float levels v (the result, 1-based, 0 = unreached).
//   A level is a main phase and one grid barrier.  A second phase, and a second
//   barrier, follow only when the main phase left work for the whole grid (heavy
//   vertices pushing, listed chunks pulling); the count of that work is complete at
//   the barrier, so every thread takes the same branch.
//   push level (frontier small): warps scan F; a vertex of moderate degree is
//     expanded by its warp, lanes striding the adjacency; vertices with more than
//     GB_BFS_HEAVY neighbours go to a list that the WHOLE grid expands in the second
//     phase (an R-MAT source has 10^5..10^6 neighbours).  Level 1 scans nothing: its
//     frontier is the source, whose list the grid expands in the main phase.
//     Discoveries set the visited bit with atomicOr immediately (same level either
//     way), the winner writes v and the N bit.
//   pull level (frontier large): the fused Boolean pull of kernels/spmv_pull.cuh,
//     probing the visited bitmap AS OF THE LEVEL'S START (operand reuse, reference
//     kernels/spmv.hpp:35-41), a scan and, when it listed chunks, a walk of them:
//     scan  — warps take chunks of 32 bitmap words (1024 rows) round-robin; a
//             lane per word, fully visited words only move their bitmap words on.
//             Every open row probes one neighbour, its highest-degree one (the
//             one most likely to be visited; pullMaxDegreeNeighbourKernel), in
//             batches of GB_BFS_BATCH rounds of 32 rows (all their summary loads,
//             then all their probes, in flight together).  A dense chunk takes
//             its open words a lane per row of the word; a sparse one takes its
//             open rows 32 at a time, a lane per open row.  Rows whose probed
//             neighbour is not visited and that have more entries are written to
//             the chunk's slice of the walk list.  A chunk with at most
//             GB_BFS_WALK_INLINE of them is walked right there by the warp that
//             scanned it (bfsWalkRows), discoveries going into the chunk's words;
//             a chunk with more goes to a list of such chunks.
//             The owner of a word writes N, the merged visited word of the other
//             copy, the level bytes of the discovered rows and clears F.
//     walk  — (second phase) warps claim listed chunks from a counter and walk their
//             rows by the same rules; discoveries are ORed into N and the other
//             visited copy.
//   The walk (bfsWalkRows): a lane walks its row's list from entry 0 (the probed
//   entry is looked at again), GB_BFS_WALK_STEP entries per step, a list still
//   longer than GB_BFS_WALK_WARP after the first step is walked by the whole warp,
//   32 entries and one ballot per step.
//   v is written once per row, after the last level, in one pass of full-line
//   stores: the level byte of every reached row, 0 for the others (and, when
//   max_levels cuts the traversal off, for the rows found at the last level: only
//   levels 1..max_levels are assigned, as in the operation-by-operation loop).  A
//   row reached at level 255 or deeper keeps byte 255 and gets v when discovered.
// Direction: the reference's ratio rule with hysteresis (vector.hpp:318-342):
// sparse -> dense when |f|/n > switchpoint and growing, dense -> sparse when
// <= switchpoint and shrinking; results do not depend on it.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_BFS_FUSED_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_BFS_FUSED_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/cooperative.cuh"

namespace graphblas {
namespace backend {

// CTA shape and register bound, chosen on an H100 (DESIGN.md §4.5, §9)
// Traversals that may pull: 512 x 2 per SM, the most warps the pull runs at without
// spilling (64 registers).  Push-only traversals (mode 1) compile the pull out and
// keep the 768 x 2 shape: the push levels are latency-bound and want the warps.
#ifndef GB_BFS_NT
#define GB_BFS_NT     512
#endif
#ifndef GB_BFS_MINB
#define GB_BFS_MINB   2               // resident CTAs per SM the register budget allows
#endif
#ifndef GB_BFS_PUSH_NT
#define GB_BFS_PUSH_NT   768
#endif
#ifndef GB_BFS_PUSH_MINB
#define GB_BFS_PUSH_MINB 2
#endif
#ifndef GB_BFS_BATCH
#define GB_BFS_BATCH  4               // rounds of 32 rows whose summaries a warp loads together
#endif
#ifndef GB_BFS_WALK_STEP
#define GB_BFS_WALK_STEP 4            // entries a lane requests at once walking a list
#endif
#ifndef GB_BFS_WALK_WARP
#define GB_BFS_WALK_WARP 32           // list remainder longer than this: walked by a warp
#endif
#ifndef GB_BFS_WALK_INLINE
#define GB_BFS_WALK_INLINE 64         // chunk with at most this many rows to walk: walked
#endif                                // by the warp that scanned it (DESIGN.md §4.5)
#define GB_BFS_HEAVY  2048            // adjacency longer than this: grid-wide expansion
#define GB_BFS_HEAVY_CAP 4096         // heavy vertices per level kept in the list
#define GB_BFS_CHUNK  1024            // rows of a pull chunk (32 bitmap words)

struct BfsFusedArgs {
  // structure: rows to expand when pushing, rows to inspect when pulling
  const Index* push_ptr;   const Index* push_ind;     // out-neighbours of a vertex
  const Index* pull_ptr;   const Index* pull_ind;     // in-neighbours of a vertex
  const Index* pull_probe;                            // neighbour each pulled row probes
                                                      // first: its highest-degree one
  const unsigned int* pull_empty;                     // bitmap of rows without in-neighbours
  const unsigned int* push_empty;                     // ... without out-neighbours; NULL
                                                      // when the structure is symmetric
  int   trace;               // count the rows walked per level (GB200_BFS_TRACE)
  unsigned long long* prof_bytes;  // profiler cell the traversal's algorithmic bytes
                                   // are added to; NULL when profiling is off
  Index n;
  Index source;
  int   max_levels;
  float switchpoint;
  int   mode;                // 0 push-pull, 1 push only, 2 pull only (reference --mxvmode)
  // state (device memory, sized for n)
  float*        levels;      // result
  unsigned char* level8;     // [n] level of each row reached so far, 255: level >= 255
  unsigned int* visited[2];
  unsigned int* frontier;    // F
  unsigned int* next;        // N
  // small cells, indexed by BfsCell
  unsigned long long* counters;   // [GB_BFS_NCOUNTERS]
  Index*        heavy;            // [GB_BFS_HEAVY_CAP]
  Index*        walk;             // [nchunks * GB_BFS_CHUNK] rows to walk, by chunk
  int*          walk_count;       // [nchunks] rows to walk per chunk
  Index*        walk_chunks;      // [nchunks] the chunks with rows to walk, listed
};

// Levels whose clocks and trace counts have a cell: levels 0..15.
#define GB_BFS_TIMED_LEVELS 16

// The cells of BfsFusedArgs::counters.  A rotating cell is a triple used by level L
// as cell L % 3 (bfsLevelCell): thread 0 zeroes it at the start of level L-1, it is
// added to during L and read after L's first barrier (heavy, listed: their counts
// come from the main phase) or its last (the frontier count).  One barrier per level
// is enough to keep the triples race-free.  Level L zeroes cell L+1, which is cell
// L-2: every read of L-2's cells happens after L-2's last barrier and before the
// reading thread arrives at L-1's first barrier, which thread 0 has passed when it
// starts level L.  The first add to cell L+1 comes after L's first barrier, when the
// zero store of level L is ordered before it.  With two cells a thread still reading
// level L-1's count after L-1's barrier would meet level L+1's zeroing.
// Clocks are %globaltimer nanoseconds.
enum BfsCell {
  // zeroed at the start of a traversal
  GB_BFS_CELL_FOUND = 0,                              // rotating: next-frontier size
  GB_BFS_CELL_HEAVY = GB_BFS_CELL_FOUND + 3,          // rotating: heavy-list length
  // results, read by bfsFusedStats in this order
  GB_BFS_CELL_LEVELS = GB_BFS_CELL_HEAVY + 3,         // levels executed
  GB_BFS_CELL_INSPECTED,                              // entries inspected pulling
  GB_BFS_CELL_PULL_LEVELS,                            // pull levels
  GB_BFS_CELL_PUSHED_VERTICES,                        // vertices pushed
  GB_BFS_CELL_PUSHED_EDGES,                           // edges pushed
  GB_BFS_CELL_FOUND_PUSHING,                          // vertices discovered pushing
  // clocks
  GB_BFS_CELL_LEVEL_CLOCK,                            // per level: end of the set-up
                                                      // (0) and of every level, ns << 2
                                                      // | second phase << 1 | pulled
  GB_BFS_CELL_START_CLOCK = GB_BFS_CELL_LEVEL_CLOCK + GB_BFS_TIMED_LEVELS,
  GB_BFS_CELL_END_PASS_CLOCK,                         // end of the pass that writes v
                                                      // (GB200_BFS_TRACE only)
  GB_BFS_CELL_LAST_LEVEL_CLOCK,                       // end of the last level
  // pull levels, zeroed at the start of a traversal
  GB_BFS_CELL_WALK_CLAIM = 35,                        // rotating: walk-chunk claims
  GB_BFS_CELL_LISTED = GB_BFS_CELL_WALK_CLAIM + 3,    // rotating: chunks in walk_chunks
  GB_BFS_CELL_SCAN_CLOCK = 44,                        // per pull level: the scan barrier
  // per level, GB200_BFS_TRACE only: rows the scan left to walk (inline and listed,
  // zeroed at the start of a traversal) and chunks it listed
  GB_BFS_CELL_WALKED = GB_BFS_CELL_SCAN_CLOCK + GB_BFS_TIMED_LEVELS,
  GB_BFS_CELL_LISTED_CHUNKS = GB_BFS_CELL_WALKED + GB_BFS_TIMED_LEVELS,
  GB_BFS_NCOUNTERS = 128
};
static_assert(GB_BFS_CELL_LISTED_CHUNKS + GB_BFS_TIMED_LEVELS <= GB_BFS_NCOUNTERS,
              "the per-level cells of the last timed level are past the counters");

// Level's cell of the rotating triple that starts at cell `first`, and the next
// level's, zeroed.
__device__ __forceinline__ unsigned long long* bfsLevelCell(unsigned long long* cells,
                                                            int first, int level) {
  return cells + first + level % 3;
}
__device__ __forceinline__ void bfsZeroNextCell(unsigned long long* cells, int first,
                                                int level) {
  cells[first + (level + 1) % 3] = 0ull;
}

// Sets vertex vtx's bit in visited; true for the one thread that set it.  V: the
// vertex-id type (Index, or long long for the global ids of the multi-GPU kernel).
template <typename V>
__device__ __forceinline__ bool bfsClaim(unsigned int* visited, V vtx) {
  const unsigned int bit = 1u << (vtx & 31);
  unsigned int* word = visited + (vtx >> 5);
  if (*reinterpret_cast<volatile unsigned int*>(word) & bit) return false;
  return (atomicOr(word, bit) & bit) == 0;
}

// Row `row` is reached at level lv.  Levels are kept as one byte per row during the
// traversal (16.8 MB at RMAT-24: it stays in L2 beside the bitmaps) and v is written
// after the last level, in full lines.  From level 255 on the byte is 255 and v is
// written here; the pass at the end leaves those rows alone.
__device__ __forceinline__ void bfsSetLevel(const BfsFusedArgs& a, Index row, int lv) {
  if (lv < 255) {
    a.level8[row] = static_cast<unsigned char>(lv);
  } else {
    a.level8[row] = 255;
    a.levels[row] = static_cast<float>(lv);
  }
}

// The next chunk for this warp from a claim counter (warp-uniform result).
__device__ __forceinline__ Index bfsClaimChunk(unsigned long long* cell, int lane) {
  unsigned long long c = 0ull;
  if (lane == 0) c = atomicAdd(cell, 1ull);
  return static_cast<Index>(__shfl_sync(GB_FULL_MASK, c, 0));
}

// The bitmap copies in use: visited[vsel] is the visited set as of the level's
// start, fsel says whether frontier/next have swapped roles.  Two bits instead of
// four live pointers (registers are what bounds the CTAs per SM); the pointers are
// re-read from the kernel parameters.
__device__ __forceinline__ unsigned int* bfsVis(const BfsFusedArgs& a, int vsel) {
  return vsel ? a.visited[1] : a.visited[0];
}
__device__ __forceinline__ unsigned int* bfsVisOther(const BfsFusedArgs& a, int vsel) {
  return vsel ? a.visited[0] : a.visited[1];
}
__device__ __forceinline__ unsigned int* bfsF(const BfsFusedArgs& a, int fsel) {
  return fsel ? a.next : a.frontier;
}
__device__ __forceinline__ unsigned int* bfsN(const BfsFusedArgs& a, int fsel) {
  return fsel ? a.frontier : a.next;
}

// Rows of word w no level can discover and nothing can be discovered from: no
// in-neighbours, and (in a directed structure) no out-neighbours either.  They count
// as visited from the start and are unreached unless one is the source.
__device__ __forceinline__ unsigned int bfsIsolated(const BfsFusedArgs& a, Index w) {
  return a.pull_empty[w] & (a.push_empty != NULL ? a.push_empty[w] : 0xffffffffu);
}

// Adds a phase's discoveries to the level's count (and, pushing, to the vertices
// discovered pushing), one atomic per CTA.
template <int NT>
__device__ __forceinline__ void bfsAddFound(const BfsFusedArgs& a,
                                            unsigned long long* count_cell, int found_here,
                                            bool pushing, int* s_red) {
  const int block_found = blockSum<NT>(found_here, s_red);
  if (threadIdx.x == 0 && block_found) {
    atomicAdd(count_cell, static_cast<unsigned long long>(block_found));
    if (pushing)
      atomicAdd(a.counters + GB_BFS_CELL_FOUND_PUSHING,
                static_cast<unsigned long long>(block_found));
  }
}

// The whole grid expands vertex u's list, a thread per entry; returns its length.
__device__ __forceinline__ Index bfsExpandGrid(const BfsFusedArgs& a, int vsel, int fsel,
                                               int level, Index u, Index gtid,
                                               Index gthreads, int& found_here) {
  const Index beg = __ldg(a.push_ptr + u);
  const Index deg = __ldg(a.push_ptr + u + 1) - beg;
  for (Index k = gtid; k < deg; k += gthreads) {
    const Index nbr = __ldg(a.push_ind + beg + k);
    if (bfsClaim(bfsVis(a, vsel), nbr)) {
      bfsSetLevel(a, nbr, level + 1);
      atomicOr(bfsN(a, fsel) + (nbr >> 5), 1u << (nbr & 31));
      ++found_here;
    }
  }
  return deg;
}

// The pull walk of one row per lane (warp-collective; a lane without a row passes
// active = false).  True when the row has an entry visited as of the level's start.
// The scan's inline walk and the grid-wide walk both come here, so the rules and the
// count of inspected entries are the same whichever walks a row.  The list is walked
// from entry 0: the probed entry, wherever it is in the list, is looked at again (and
// counted again in inspected).  It reads only visited[vsel], which no thread writes
// during a pull level, so it sees the same bits during the scan as after it.
__device__ __forceinline__ bool bfsWalkRows(const BfsFusedArgs& a, int vsel, Index row,
                                            bool active, int lane, int& inspected) {
  Index k = 0, end = 0;
  if (active) {
    k = __ldg(a.pull_ptr + row);
    end = __ldg(a.pull_ptr + row + 1);
  }
  // most walks end after a few entries: every lane starts on its own list
  const Index stop = (end - k > GB_BFS_WALK_WARP + GB_BFS_WALK_STEP)
                     ? k + GB_BFS_WALK_STEP : end;
  bool found = false;
  // GB_BFS_WALK_STEP entries per step: their bitmap words are fetched together, then
  // examined in list order (the count stops at the first visited one)
  while (k < stop && !found) {
    Index col[GB_BFS_WALK_STEP];
    unsigned int wv[GB_BFS_WALK_STEP];
#pragma unroll
    for (int u = 0; u < GB_BFS_WALK_STEP; ++u)
      col[u] = (k + u < stop) ? __ldg(a.pull_ind + k + u) : static_cast<Index>(-1);
#pragma unroll
    for (int u = 0; u < GB_BFS_WALK_STEP; ++u)
      wv[u] = (col[u] >= 0) ? bfsVis(a, vsel)[col[u] >> 5] : 0u;
#pragma unroll
    for (int u = 0; u < GB_BFS_WALK_STEP; ++u) {
      if (found || col[u] < 0) continue;
      ++inspected;
      found = (wv[u] >> (col[u] & 31)) & 1u;
    }
    k += GB_BFS_WALK_STEP;
  }
  // a list with more than GB_BFS_WALK_WARP entries left: the whole warp walks it,
  // 32 entries and one ballot per step
  unsigned int longs = __ballot_sync(GB_FULL_MASK, !found && k < end);
  while (longs != 0u) {
    const int src = __ffs(longs) - 1;
    longs &= longs - 1u;
    const Index lend = __shfl_sync(GB_FULL_MASK, end, src);
    bool hit = false;
    for (Index lk = __shfl_sync(GB_FULL_MASK, k, src); lk < lend && !hit; lk += 32) {
      bool v = false;
      if (lk + lane < lend) {
        const Index col = __ldg(a.pull_ind + lk + lane);
        v = (bfsVis(a, vsel)[col >> 5] >> (col & 31)) & 1u;
      }
      const unsigned int b = __ballot_sync(GB_FULL_MASK, v);
      hit = (b != 0u);
      if (lane == 0)
        inspected += hit ? __ffs(b) : (lend - lk < 32 ? lend - lk : 32);
    }
    if (lane == src) found = hit;
  }
  return found;
}

// NT x MINB: the CTA shape; PULL = false compiles the pull level out (push-only
// traversals, a.mode == 1).
template <int NT, int MINB, bool PULL>
__global__ void __launch_bounds__(NT, MINB)
bfsFusedKernel(BfsFusedArgs a) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  __shared__ int s_red[NT/32];
  // pull scan, per warp: the discovery words of its chunk (row path)
  __shared__ unsigned int s_found[PULL ? NT/32 : 1][PULL ? 32 : 1];

  const Index n = a.n;
  const Index nwords = (n + 31) >> 5;
  const int lane = threadIdx.x & 31;
  // The kernel is launched with NT threads per CTA.  The constant instead of
  // blockDim.x lets the compiler rebuild gthreads from gridDim.x where it needs it
  // instead of keeping it in a register: at 768 x 2 (40 registers) that is what keeps
  // spill reloads out of the push expansion loops.
  const Index gtid = blockIdx.x*NT + threadIdx.x;                 // grid << 2^31 threads
  const Index gthreads = gridDim.x*NT;
  const Index gwarp = gtid >> 5;
  const Index gwarps = gthreads >> 5;
  const Index nchunks = (nwords + 31) >> 5;               // pull chunks of 32 words

  if (gtid == 0) a.counters[GB_BFS_CELL_START_CLOCK] = globalTimerNs();
  // ---- level 0: clear the bitmaps, mark the source visited (v is written once per
  // row, after the last level) ------------------------------------------------------------
  // F is not seeded: a push at level 1 expands the source without reading F, a pull
  // only clears it, and the end pass adds the source back to what it reaches.
  // visited[1] is not cleared: it is read (as visited[vsel], and by the end pass)
  // only once vsel is 1, after a pull level whose owners' stores wrote every word of
  // it, and it is never read in a push-only traversal.
  if (gtid == 0) a.level8[a.source] = 1;
  for (Index w = gtid; w < nwords; w += gthreads) {
    const unsigned int seed = (w == (a.source >> 5)) ? (1u << (a.source & 31)) : 0u;
    // rows nothing points at count as visited from the start: no level can discover
    // them, and the pull levels would look at them every time
    a.visited[0][w] = seed | bfsIsolated(a, w);
    a.frontier[w] = 0u; a.next[w] = 0u;
  }
  if (gtid <= GB_BFS_CELL_FOUND_PUSHING) a.counters[gtid] = 0ull;
  if (gtid >= GB_BFS_CELL_WALK_CLAIM && gtid < GB_BFS_CELL_LISTED + 3) a.counters[gtid] = 0ull;
  if (gtid >= GB_BFS_CELL_WALKED && gtid < GB_BFS_CELL_WALKED + GB_BFS_TIMED_LEVELS)
    a.counters[gtid] = 0ull;
  grid.sync();
  if (gtid == 0) a.counters[GB_BFS_CELL_LEVEL_CLOCK] = globalTimerNs() << 2;

  int vsel = 0;                           // bfsVis / bfsVisOther
  int fsel = 0;                           // bfsF / bfsN
  unsigned int fcount = 1u;               // frontier size (<= n)
  bool dense = PULL && (a.mode == 2);             // direction state (storage of the frontier)
  float prev_ratio = 0.f;
  int inspected = 0;                      // colind entries looked at by this thread
  int pushed_vertices = 0;                // frontier entries expanded (lane 0 counts,
                                          // thread 0 the source at level 1)
  unsigned int pushed_edges = 0u;         // their adjacency lengths (a vertex is pushed
                                          // once: at most nnz < 2^31 per thread)
  int pull_levels = 0;
  int level = 1;

  for (; level <= a.max_levels && fcount > 0u; ++level) {
    // direction for this level (reference Vector::convert)
    if (PULL && a.mode == 0) {
      const float ratio = static_cast<float>(fcount)/static_cast<float>(n);
      if (!dense) {
        if (ratio > a.switchpoint && ratio > prev_ratio) dense = true; else prev_ratio = ratio;
      } else {
        if (ratio <= a.switchpoint && ratio < prev_ratio) dense = false; else prev_ratio = ratio;
      }
    }
    unsigned long long* const count_cell = bfsLevelCell(a.counters, GB_BFS_CELL_FOUND, level);
    unsigned long long* const heavy_cell = bfsLevelCell(a.counters, GB_BFS_CELL_HEAVY, level);
    if (gtid == 0) {
      bfsZeroNextCell(a.counters, GB_BFS_CELL_FOUND, level);
      bfsZeroNextCell(a.counters, GB_BFS_CELL_HEAVY, level);
      bfsZeroNextCell(a.counters, GB_BFS_CELL_WALK_CLAIM, level);
      bfsZeroNextCell(a.counters, GB_BFS_CELL_LISTED, level);
    }
    int found_here = 0;

    if (!dense && level == 1) {
      // ---------------- push from the source: the grid expands its list ----------
      // (no scan of F for its one vertex, no barrier before a heavy source's list)
      const Index deg = bfsExpandGrid(a, vsel, fsel, level, a.source, gtid, gthreads,
                                      found_here);
      if (gtid == 0) { ++pushed_vertices; pushed_edges += deg; }
    } else if (!dense) {
      // ---------------- push: expand the frontier --------------------------------
      // A warp reads 32 frontier words at once (the frontier is sparse here: most
      // words are zero and a word-at-a-time scan is a chain of dependent loads),
      // then walks the non-empty ones.
      for (Index w0 = gwarp*32; w0 < nwords; w0 += gwarps*32) {
        const Index mine = w0 + lane;
        unsigned int my_bits = (mine < nwords) ? bfsF(a, fsel)[mine] : 0u;
        if (my_bits != 0u) bfsF(a, fsel)[mine] = 0u;   // this buffer is the next level's N
        unsigned int pending = __ballot_sync(GB_FULL_MASK, my_bits != 0u);
        while (pending != 0u) {
          const int src_lane = __ffs(pending) - 1;
          pending &= pending - 1u;
          unsigned int bits = __shfl_sync(GB_FULL_MASK, my_bits, src_lane);
          const Index w = w0 + src_lane;
          while (bits != 0u) {
            const int b = __ffs(bits) - 1;
            bits &= bits - 1u;
            const Index u = w*32 + b;
            const Index beg = __ldg(a.push_ptr + u);
            const Index deg = __ldg(a.push_ptr + u + 1) - beg;
            if (lane == 0) { ++pushed_vertices; pushed_edges += deg; }
            if (deg > GB_BFS_HEAVY) {
              // the whole grid expands it in the second phase; a full list falls
              // back to this warp (slow, still correct)
              unsigned long long slot = 0ull;
              if (lane == 0) slot = atomicAdd(heavy_cell, 1ull);
              slot = __shfl_sync(GB_FULL_MASK, slot, 0);
              if (slot < GB_BFS_HEAVY_CAP) {
                if (lane == 0) a.heavy[slot] = u;
                continue;
              }
            }
            for (Index k = lane; k < deg; k += 32) {
              const Index nbr = __ldg(a.push_ind + beg + k);
              if (bfsClaim(bfsVis(a, vsel), nbr)) {
                bfsSetLevel(a, nbr, level + 1);
                atomicOr(bfsN(a, fsel) + (nbr >> 5), 1u << (nbr & 31));
                ++found_here;
              }
            }
          }
        }
      }
    } else if (PULL) {
      ++pull_levels;
      // ---------------- pull: every unvisited row looks for a visited neighbour ----
      unsigned long long* const list_cell = bfsLevelCell(a.counters, GB_BFS_CELL_LISTED, level);
      // scan: a lane per bitmap word of the chunk, chunks dealt round-robin (the
      // grid has ~4 chunks per warp at RMAT-24 and they cost about the same); the
      // next chunk's words are requested before this one is worked on
      Index c = gwarp;
      unsigned int next_vis = (c < nchunks && c*32 + lane < nwords)
                              ? bfsVis(a, vsel)[c*32 + lane] : 0xffffffffu;
      while (c < nchunks) {
        const Index word = c*32 + lane;
        const unsigned int my_vis = next_vis;
        const Index c_next = c + gwarps;
        next_vis = (c_next < nchunks && c_next*32 + lane < nwords)
                   ? bfsVis(a, vsel)[c_next*32 + lane] : 0xffffffffu;
        Index* const walk = a.walk + c*GB_BFS_CHUNK;
        int nwalk = 0;                        // rows of this chunk left to walk
        unsigned int my_out = 0u;             // discoveries in this lane's word
        unsigned int open = __ballot_sync(GB_FULL_MASK, my_vis != 0xffffffffu);
        // Row path: the chunk's open rows (rows past n are not), numbered in word
        // order by a prefix of the per-word counts and taken 32 at a time, a lane
        // per row; the lane of open row r finds the word holding it (binary search
        // on the prefix) and its bit (binary search on bit counts).  Word path
        // (below): the open words, a lane per row of the word.  A row batch costs
        // about twice a word batch (the searches; DESIGN.md §6), so a chunk takes
        // the row path when that needs fewer than half the batches: at RMAT-24 the
        // second pull level (2.3 open rows per open word) takes it in nearly every
        // chunk, the first (17) in some.
        unsigned int my_open = ~my_vis;
        if (word == nwords - 1 && (n & 31) != 0) my_open &= (1u << (n & 31)) - 1u;
        const int nopen = __popc(my_open);
        int first = nopen;                    // inclusive prefix, then exclusive
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          const int t = __shfl_up_sync(GB_FULL_MASK, first, off);
          if (lane >= off) first += t;
        }
        const int total = __shfl_sync(GB_FULL_MASK, first, 31);
        first -= nopen;
        const int word_batches = (__popc(open) + GB_BFS_BATCH - 1)/GB_BFS_BATCH;
        const int row_batches = (total + 32*GB_BFS_BATCH - 1)/(32*GB_BFS_BATCH);
        if (2*row_batches < word_batches) {
          open = 0u;
          unsigned int* const found_bits = s_found[threadIdx.x >> 5];
          found_bits[lane] = 0u;
          __syncwarp();
          for (int r0 = 0; r0 < total; r0 += 32*GB_BFS_BATCH) {
            // GB_BFS_BATCH rounds of 32 open rows: all summary loads, then all
            // probes, then the decisions.  The summary is read once per level, so
            // its loads bypass L1 (ldStream32) and leave it to the probes' bitmap
            // lines (DESIGN.md §4.5)
            int local[GB_BFS_BATCH];          // offset of the row in the chunk
            Index f[GB_BFS_BATCH];
#pragma unroll
            for (int j = 0; j < GB_BFS_BATCH; ++j) {
              const int r = r0 + 32*j + lane;
              int wl = 0, base = 0;           // the last word whose prefix is <= r
#pragma unroll
              for (int step = 16; step > 0; step >>= 1) {
                const int fs = __shfl_sync(GB_FULL_MASK, first, wl + step);
                if (fs <= r) { wl += step; base = fs; }
              }
              unsigned int m = __shfl_sync(GB_FULL_MASK, my_open, wl);
              int k = r - base, b = 0;        // bit of the k-th open row of the word
#pragma unroll
              for (int width = 16; width > 0; width >>= 1) {
                const int lo = __popc(m & ((1u << width) - 1u));
                if (k >= lo) { k -= lo; b += width; m >>= width; }
              }
              local[j] = wl*32 + b;
              f[j] = (r < total) ? ldStream32(a.pull_probe + c*GB_BFS_CHUNK + local[j])
                                 : static_cast<Index>(-1);
            }
            unsigned int pword[GB_BFS_BATCH];
#pragma unroll
            for (int j = 0; j < GB_BFS_BATCH; ++j)
              pword[j] = (f[j] != static_cast<Index>(-1))
                         ? bfsVis(a, vsel)[(f[j] & 0x7fffffff) >> 5] : 0u;
#pragma unroll
            for (int j = 0; j < GB_BFS_BATCH; ++j) {
              if (r0 + 32*j >= total) break;  // warp-uniform
              const bool found = (pword[j] >> (f[j] & 31)) & 1u;
              // the probed entry is looked at (-1: past the open rows, or a row
              // without entries)
              inspected += (f[j] != static_cast<Index>(-1)) ? 1 : 0;
              // more entries and the probed one not visited: the row goes into the
              // chunk's slice of the walk list
              const bool walk_row = f[j] >= 0 && !found;
              const Index row = c*GB_BFS_CHUNK + local[j];
              const unsigned int walkers = __ballot_sync(GB_FULL_MASK, walk_row);
              if (walk_row) walk[nwalk + __popc(walkers & ((1u << lane) - 1u))] = row;
              nwalk += __popc(walkers);
              if (found) {
                atomicOr(found_bits + (local[j] >> 5), 1u << (local[j] & 31));
                bfsSetLevel(a, row, level + 1);
                ++found_here;
              }
            }
          }
          __syncwarp();
          my_out = found_bits[lane];
        }
        while (open != 0u) {
          // up to GB_BFS_BATCH open words: all summary loads (bypassing L1, as on
          // the row path), then all probes, then the decisions
          const unsigned int batch = open;
          Index f[GB_BFS_BATCH];
#pragma unroll
          for (int j = 0; j < GB_BFS_BATCH; ++j) {
            const int wl = __ffs(open) - 1;   // -1 when none is left
            open &= open - 1u;
            f[j] = static_cast<Index>(-1);
            if (wl >= 0) {
              const unsigned int m = __shfl_sync(GB_FULL_MASK, my_vis, wl);
              const Index row = c*GB_BFS_CHUNK + wl*32 + lane;
              if (row < n && !((m >> lane) & 1u)) f[j] = ldStream32(a.pull_probe + row);
            }
          }
          unsigned int pword[GB_BFS_BATCH];
#pragma unroll
          for (int j = 0; j < GB_BFS_BATCH; ++j)
            pword[j] = (f[j] != static_cast<Index>(-1))
                       ? bfsVis(a, vsel)[(f[j] & 0x7fffffff) >> 5] : 0u;
          unsigned int hit = 0u, more = 0u;   // bit j: row of batch word j
#pragma unroll
          for (int j = 0; j < GB_BFS_BATCH; ++j) {
            const bool found = (pword[j] >> (f[j] & 31)) & 1u;
            // the probed entry is looked at (-1: not open, or a row without entries)
            inspected += (f[j] != static_cast<Index>(-1)) ? 1 : 0;
            hit |= static_cast<unsigned int>(found) << j;
            // more entries and the probed one not visited: the row goes into the
            // chunk's slice of the walk list
            more |= static_cast<unsigned int>(f[j] >= 0 && !found) << j;
          }
          unsigned int rest = batch;
#pragma unroll
          for (int j = 0; j < GB_BFS_BATCH && rest != 0u; ++j) {
            const int wl = __ffs(rest) - 1;
            rest &= rest - 1u;
            const Index row = c*GB_BFS_CHUNK + wl*32 + lane;
            const bool found = (hit >> j) & 1u, walk_row = (more >> j) & 1u;
            const unsigned int walkers = __ballot_sync(GB_FULL_MASK, walk_row);
            if (walk_row) walk[nwalk + __popc(walkers & ((1u << lane) - 1u))] = row;
            nwalk += __popc(walkers);
            const unsigned int out = __ballot_sync(GB_FULL_MASK, found);
            if (found) { bfsSetLevel(a, row, level + 1); ++found_here; }
            if (lane == wl) my_out = out;
          }
        }
        if (nwalk > 0 && nwalk <= GB_BFS_WALK_INLINE) {
          // A light chunk's rows are walked here, by this warp, instead of after the
          // barrier: at RMAT-24 the first pull level leaves at most a few dozen
          // short rows per chunk, and listing them for the grid costs more than
          // walking them (DESIGN.md §4.5).  The rows are the ones the lanes just
          // stored in the chunk's slice of a.walk; the __syncwarp orders those
          // stores for the warp.  Discoveries are ORed into the chunk's shared words
          // (seeded with the scan's) and go out with the owners' stores below, so
          // no global atomics.  The walk reads visited[vsel] only, which no thread
          // writes during a pull level: it finds what the walk after the barrier
          // would, and counts the same entries.
          unsigned int* const found_bits = s_found[threadIdx.x >> 5];
          found_bits[lane] = my_out;
          __syncwarp();
          for (int i0 = 0; i0 < nwalk; i0 += 32) {
            const bool active = i0 + lane < nwalk;
            const Index row = active ? walk[i0 + lane] : 0;
            if (bfsWalkRows(a, vsel, row, active, lane, inspected)) {
              const int local = row & (GB_BFS_CHUNK - 1);
              atomicOr(found_bits + (local >> 5), 1u << (local & 31));
              bfsSetLevel(a, row, level + 1);
              ++found_here;
            }
          }
          __syncwarp();
          my_out = found_bits[lane];
        }
        if (word < nwords) {
          bfsN(a, fsel)[word] = my_out;
          bfsVisOther(a, vsel)[word] = my_vis | my_out;
          bfsF(a, fsel)[word] = 0u;
        }
        if (lane == 0 && nwalk > 0) {
          if (nwalk > GB_BFS_WALK_INLINE) {
            a.walk_count[c] = nwalk;
            a.walk_chunks[atomicAdd(list_cell, 1ull)] = c;
          }
          if (a.trace && level < GB_BFS_TIMED_LEVELS)
            atomicAdd(a.counters + GB_BFS_CELL_WALKED + level,
                      static_cast<unsigned long long>(nwalk));
        }
        c = c_next;
      }
    }
    // ---- the level's barrier, then the second phase when there is one ---------------
    // One barrier and one count for each phase, from one place in the code: written
    // twice, the push-only instantiation reloads more spilled values after them.
    for (int phase = 0; ; ++phase) {
      bfsAddFound<NT>(a, count_cell, found_here, !dense, s_red);
      grid.sync();
      // After the main phase: heavy vertices listed pushing, chunks listed pulling.
      // Every add to the cell came before the barrier, so every thread reads the
      // same value and takes the same branch.
      const unsigned long long listed = phase ? 0ull : loadCell(
          bfsLevelCell(a.counters, dense ? GB_BFS_CELL_LISTED : GB_BFS_CELL_HEAVY, level));
      if (gtid == 0 && level < GB_BFS_TIMED_LEVELS) {
        const unsigned long long t = globalTimerNs();
        if (dense && phase == 0) {
          a.counters[GB_BFS_CELL_SCAN_CLOCK + level] = t;
          if (a.trace) a.counters[GB_BFS_CELL_LISTED_CHUNKS + level] = listed;
        }
        if (listed == 0ull)
          a.counters[GB_BFS_CELL_LEVEL_CLOCK + level] =
              (t << 2) | (static_cast<unsigned long long>(phase) << 1) | (dense ? 1ull : 0ull);
      }
      if (listed == 0ull) break;
      found_here = 0;                       // the main phase's are counted
      if (!dense) {
        // the heavy vertices' lists, each by the whole grid
        const int nheavy = (listed > GB_BFS_HEAVY_CAP) ? GB_BFS_HEAVY_CAP
                                                       : static_cast<int>(listed);
        for (int h = 0; h < nheavy; ++h)
          bfsExpandGrid(a, vsel, fsel, level, a.heavy[h], gtid, gthreads, found_here);
      } else if (PULL) {
        // walk: the heavy chunks' rows, chunks claimed from a counter, a lane per row
        unsigned long long* const walk_cell =
            bfsLevelCell(a.counters, GB_BFS_CELL_WALK_CLAIM, level);
        const Index nlisted = static_cast<Index>(listed);
        for (Index i = gwarp; i < nlisted; ) {
          const Index i_next = gwarps + bfsClaimChunk(walk_cell, lane);
          const Index c = a.walk_chunks[i];
          const int nwalk = a.walk_count[c];
          for (int i0 = 0; i0 < nwalk; i0 += 32) {
            const bool active = i0 + lane < nwalk;
            const Index row = active ? a.walk[c*GB_BFS_CHUNK + i0 + lane] : 0;
            if (bfsWalkRows(a, vsel, row, active, lane, inspected)) {
              const unsigned int bit = 1u << (row & 31);
              atomicOr(bfsN(a, fsel) + (row >> 5), bit);
              atomicOr(bfsVisOther(a, vsel) + (row >> 5), bit);
              bfsSetLevel(a, row, level + 1);
              ++found_here;
            }
          }
          i = i_next;
        }
      }
    }
    // ---- frontier size of the next level ------------------------------------------
    fcount = static_cast<unsigned int>(loadCell(count_cell));
    if (dense) vsel ^= 1;
    fsel ^= 1;
  }
  if (gtid == 0) a.counters[GB_BFS_CELL_LAST_LEVEL_CLOCK] = globalTimerNs();
  // ---- v, every row once, in full lines ----------------------------------------
  // A row is reached when it is visited now and not only because nothing points at
  // it (the source is reached).  A traversal cut off after max_levels (the frontier
  // is not empty): the rows found at the last level, now the frontier, get no level
  // either, as in the operation-by-operation loop, which assigns levels 1..max_niter.
  // Reached rows get their byte, the others 0; a byte is only read for a row reached
  // in this traversal, which wrote it.
  const unsigned int* const cut_rows = (fcount > 0u) ? bfsF(a, fsel) : NULL;
  // An adopted array need not be 16-byte aligned: then every row is stored alone.
  const bool lines = (reinterpret_cast<uintptr_t>(a.levels) & 15u) == 0u;
  // A warp takes 512 rows (16 bitmap words, 512 bytes): lanes 0..15 build the reach
  // masks, then each lane writes 4 rows per step, a warp 512 contiguous bytes per
  // 16-byte store.  4 rows holding a level of 255 or more, or past n, or not aligned,
  // are written row by row.  The loop counts blocks of 16 words, not rows, so that
  // stepping past the last block cannot overflow (rows stay below n + 512, as the
  // pull scan's stay below n + 1024).  The 4-byte load also takes the bytes of rows
  // not reached, which this traversal never wrote; their values are not used.  The
  // 16-byte stores are streaming (st.global.cs, evict-first): nothing reads the 4n
  // bytes of v again in the kernel, and marked so they do not push the level bytes
  // and bitmaps the pass still reads out of L2.
  const Index nblocks = (nwords + 15) >> 4;
  if (PULL) {
    // The loads of a block go out before the stores of the block before it: the warp
    // requests block blk + gwarps's reach masks and level bytes, then stores block
    // blk's floats, so the loads' latency sits under the stores instead of between
    // one block's stores and the next (RMAT-24: end pass 36-38 -> 30-32 us, DESIGN.md
    // §6).  A block past the last loads nothing, and a group of 4 rows gets its
    // 4-byte load only when it can be stored as a line.  Not in the push-only
    // instantiation: the 5 more live registers spill there at 768 x 2.  The two
    // loops share no lambda: one gave the pull instantiation another register
    // allocation throughout and a slower scan (DESIGN.md §4.5).
    auto load_block = [&](Index blk, unsigned int& reached, unsigned int (&b)[4]) {
      reached = 0u;
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = 0u;
      if (blk >= nblocks) return;
      const Index w = blk*16 + (lane & 15);
      if (lane < 16 && w < nwords) {
        reached = bfsVis(a, vsel)[w] & ~bfsIsolated(a, w);
        if (cut_rows != NULL) reached &= ~cut_rows[w];
        if (w == (a.source >> 5)) reached |= 1u << (a.source & 31);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const Index row = blk*512 + 128*j + 4*lane;
        if (lines && row + 4 <= n) b[j] = *reinterpret_cast<const unsigned int*>(a.level8 + row);
      }
    };
    unsigned int next_reached, next_b[4];
    load_block(gwarp, next_reached, next_b);
    for (Index blk = gwarp; blk < nblocks; blk += gwarps) {
      const Index r0 = blk*512;
      const unsigned int reached = next_reached;
      unsigned int lb[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) lb[j] = next_b[j];
      load_block(blk + gwarps, next_reached, next_b);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const unsigned int bits =
            (__shfl_sync(GB_FULL_MASK, reached, 4*j + (lane >> 3)) >> (4*(lane & 7))) & 0xfu;
        const Index row = r0 + 128*j + 4*lane;
        if (row >= n) continue;
        if (lines && row + 4 <= n) {
          const unsigned int b = lb[j];
          float f[4];
          bool escape = false;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const unsigned int byte = (b >> (8*k)) & 0xffu;
            const bool r = (bits >> k) & 1u;
            escape |= r && byte == 255u;
            f[k] = r ? static_cast<float>(byte) : 0.f;
          }
          if (!escape) {
            __stcs(reinterpret_cast<float4*>(a.levels + row), make_float4(f[0], f[1], f[2], f[3]));
            continue;
          }
        }
        for (int k = 0; k < 4 && row + k < n; ++k) {
          if (!((bits >> k) & 1u)) {
            a.levels[row + k] = 0.f;
          } else {
            const unsigned int byte = a.level8[row + k];
            if (byte != 255u) a.levels[row + k] = static_cast<float>(byte);
          }
        }
      }
    }
  } else {
    for (Index blk = gwarp; blk < nblocks; blk += gwarps) {
      const Index r0 = blk*512;
      const Index w = blk*16 + (lane & 15);
      unsigned int reached = 0u;
      if (lane < 16 && w < nwords) {
        reached = bfsVis(a, vsel)[w] & ~bfsIsolated(a, w);
        if (cut_rows != NULL) reached &= ~cut_rows[w];
        if (w == (a.source >> 5)) reached |= 1u << (a.source & 31);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const unsigned int bits =
            (__shfl_sync(GB_FULL_MASK, reached, 4*j + (lane >> 3)) >> (4*(lane & 7))) & 0xfu;
        const Index row = r0 + 128*j + 4*lane;
        if (row >= n) continue;
        if (lines && row + 4 <= n) {
          const unsigned int b = *reinterpret_cast<const unsigned int*>(a.level8 + row);
          float f[4];
          bool escape = false;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const unsigned int byte = (b >> (8*k)) & 0xffu;
            const bool r = (bits >> k) & 1u;
            escape |= r && byte == 255u;
            f[k] = r ? static_cast<float>(byte) : 0.f;
          }
          if (!escape) {
            __stcs(reinterpret_cast<float4*>(a.levels + row), make_float4(f[0], f[1], f[2], f[3]));
            continue;
          }
        }
        for (int k = 0; k < 4 && row + k < n; ++k) {
          if (!((bits >> k) & 1u)) {
            a.levels[row + k] = 0.f;
          } else {
            const unsigned int byte = a.level8[row + k];
            if (byte != 255u) a.levels[row + k] = static_cast<float>(byte);
          }
        }
      }
    }
  }
  if (a.trace) {
    grid.sync();                  // only to time the end pass: not counted in the barriers
    if (gtid == 0) a.counters[GB_BFS_CELL_END_PASS_CLOCK] = globalTimerNs();
  }
  // ---- results: the work counters, the algorithmic bytes of SURVEY.md §8d --------
  const int block_insp = blockSum<NT>(inspected, s_red);
  const int block_pv = blockSum<NT>(pushed_vertices, s_red);
  if (threadIdx.x == 0) {
    if (block_insp)
      atomicAdd(a.counters + GB_BFS_CELL_INSPECTED, static_cast<unsigned long long>(block_insp));
    if (block_pv)
      atomicAdd(a.counters + GB_BFS_CELL_PUSHED_VERTICES,
                static_cast<unsigned long long>(block_pv));
  }
  if (pushed_edges)
    atomicAdd(a.counters + GB_BFS_CELL_PUSHED_EDGES,
              static_cast<unsigned long long>(pushed_edges));
  if (gtid == 0) {
    a.counters[GB_BFS_CELL_LEVELS] = static_cast<unsigned long long>(level - 1);
    a.counters[GB_BFS_CELL_PULL_LEVELS] = static_cast<unsigned long long>(pull_levels);
  }
  if (a.prof_bytes != NULL) {
    // The traversal's algorithmic bytes (SURVEY.md §8d): per pull level 4(n+1) + 4n
    // + 4n, 4 per inspected entry; per push 12 per frontier entry, 8 per expanded
    // edge (colind + visited lookup), 8 per discovered vertex.  The sum is linear in
    // the work counters, so every CTA adds its own share and CTA 0 the per-level
    // terms (the count of vertices discovered pushing is complete: the last level
    // ended with a grid barrier).  A last-CTA ticket would need a device-scope
    // fence, and with one in the kernel ptxas turns
    // every fire-and-forget reduction (REDG) into an atomic that waits (ATOMG),
    // the push levels' visited and next-frontier ORs included: push-only BFS
    // 156.7-157.5 ms per launch against 149.7-150.7 (DESIGN.md §9).
    if (pushed_edges) atomicAdd(a.prof_bytes, 8ull*pushed_edges);
    if (threadIdx.x == 0) {
      unsigned long long bytes = 4ull*static_cast<unsigned long long>(block_insp) +
                                 12ull*static_cast<unsigned long long>(block_pv);
      if (blockIdx.x == 0)
        bytes += static_cast<unsigned long long>(pull_levels)*
                     (12ull*static_cast<unsigned long long>(n) + 4ull) +
                 8ull*loadCell(a.counters + GB_BFS_CELL_FOUND_PUSHING);
      if (bytes) atomicAdd(a.prof_bytes, bytes);
    }
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_BFS_FUSED_CUH_
