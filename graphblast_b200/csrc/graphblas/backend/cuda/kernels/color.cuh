// graphblast_b200 backend — greedy Jones–Plassmann graph colouring as ONE persistent
// cooperative kernel (backend::graphColor, algorithm::gc; host side color.hpp).
//
// Semantics.  Vertices i != j conflict when A(i,j) or A(j,i) is stored; self-loops are
// ignored.  A vertex's list is its CSR row followed, when the matrix is not symmetric,
// by its CSC column, so the graph coloured is the undirected graph of the pattern.
// Every vertex has the priority
//     p(v) = (gcHash(seed, v), v), compared lexicographically,
//     gcHash(seed, v) = fmix32(v ^ (seed * 0x9E3779B9)),
//     fmix32(x): x ^= x >> 16; x *= 0x85EBCA6B; x ^= x >> 13; x *= 0xC2B2AE35; x ^= x >> 16
// (32-bit unsigned arithmetic; fmix32 is the murmur3 finaliser).  A vertex is coloured
// once every higher-priority neighbour is, with the smallest colour c >= 1 none of them
// holds.  The result is sequential greedy first-fit colouring in decreasing p order
// (tests/gc_oracle.c restates it), whatever the launch shape or timing.
//
// Determinism.  colour[v] goes from 0 to its final value in one 32-bit store, and v is
// stored only after v has seen every higher-priority neighbour non-zero.  A
// lower-priority neighbour u of v cannot be coloured before v (u waits for v), so when
// v picks its colour the non-zero colours among its neighbours are exactly the final
// colours of its higher-priority neighbours.  Scheduling decides only when v is
// coloured, never with what.  Progress: the highest-priority uncoloured vertex is never
// blocked, and no warp waits on another warp; a blocked vertex is put back.
//
// Schedule.
//   sweeps — while more than 32 vertices per resident warp are uncoloured, the grid
//     sweeps the list of uncoloured vertices (the first sweep: all vertices), one lane
//     per vertex whose list has at most GB_GC_LANE_MAX entries and one warp per longer
//     list.  An attempt at v (gcTry): if v is known to wait on a neighbour that is still
//     uncoloured, nothing else is read; otherwise v's list is scanned from where the
//     last scan stopped for the first uncoloured higher-priority neighbour, which
//     becomes waiting_on[v]; with none left, the colour pass.  Vertices still
//     uncoloured are appended to the next list (one atomic per warp); a grid barrier
//     separates sweeps.
//   tail — with at most 32 per resident warp left, lane l of warp w owns list entry
//     w + l * (warps): no more barriers.  A warp tests the waiting_on colour of all its
//     vertices at once (a lane each), and attempts the ones whose blocker is coloured
//     together, one at a time, until all its vertices are coloured.
//   out — after one more barrier, out[i] = colour[i] and ncolors = max colour.
// Colour pass: colours up to degree + 1, taken 64 at a time: a 64-bit mask of the
// window's colours held by the neighbours (warp OR-reduced when a warp has the vertex);
// the next window is looked at only when all 64 are held.  The pass also checks that no
// higher-priority neighbour reads 0; if one does the attempt is given up (it never
// happens when loads are coherent, and keeps the colour correct if it does).
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_COLOR_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_COLOR_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/common.cuh"

namespace graphblas {
namespace backend {

#define GB_GC_NT        512            // CTA shape of the colouring kernel
#define GB_GC_MINB      2              // resident CTAs per SM the register budget allows
#define GB_GC_LANE_MAX  32             // longest list a single lane takes in a sweep

struct GcArgs {
  const Index* row_ptr;  const Index* row_ind;        // CSR
  const Index* col_ptr;  const Index* col_ind;        // CSC; NULL when it is the CSR
  Index n;
  unsigned int seed;
  unsigned int* colour;          // [n] 0 = uncoloured
  Index* waiting_on;             // [n] uncoloured higher-priority neighbour last seen
  Index* resume;                 // [n] list position where the blocker scan goes on
  Index* list[2];                // [n] uncoloured vertices, ping-pong between sweeps
  unsigned long long* counters;  // [0..2] list length (rotating with the sweep % 3: the
                                 // cell of sweep s + 1 is zeroed during s), [3] ncolors
};

// The priority hash, host and device (the oracle restates it).
__host__ __device__ __forceinline__ unsigned int gcHash(unsigned int seed, unsigned int v) {
  unsigned int x = v ^ (seed*0x9E3779B9u);
  x ^= x >> 16; x *= 0x85EBCA6Bu;
  x ^= x >> 13; x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

// p(u) > p(v)
__device__ __forceinline__ bool gcAbove(unsigned int hu, Index u, unsigned int hv, Index v) {
  return hu > hv || (hu == hv && u > v);
}

// Colour loads MUST NOT go through the non-coherent path (__ldg, ld.global.nc): a
// vertex re-reads colours that other SMs store while the kernel runs, and a
// non-coherent load may keep returning a stale 0 from L1 for as long as the line
// stays there, so a blocked vertex would never see its blocker coloured.
// ld.relaxed.gpu reads at GPU scope (L2); volatile keeps every re-read in the loop.
__device__ __forceinline__ unsigned int gcLoadColour(const unsigned int* p) {
  unsigned int c;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(c) : "l"(p));
  return c;
}

__device__ __forceinline__ void gcStoreColour(unsigned int* p, unsigned int c) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(c) : "memory");
}

// A vertex's list: its CSR row, then its CSC column (dc = 0 when symmetric).  Args is
// any kernel argument struct with GcArgs's row_ptr / row_ind / col_ptr / col_ind
// (GcArgs here, MisArgs in kernels/mis.cuh).
struct GcList {
  Index r0, dr, c0, dc;
};

template <typename Args>
__device__ __forceinline__ GcList gcListOf(const Args a, Index v) {
  GcList l;
  l.r0 = a.row_ptr[v];
  l.dr = a.row_ptr[v + 1] - l.r0;
  l.c0 = 0; l.dc = 0;
  if (a.col_ptr != NULL) {
    l.c0 = a.col_ptr[v];
    l.dc = a.col_ptr[v + 1] - l.c0;
  }
  return l;
}

template <typename Args>
__device__ __forceinline__ Index gcEntry(const Args a, const GcList& l, Index k) {
  return k < l.dr ? __ldg(a.row_ind + l.r0 + k) : __ldg(a.col_ind + l.c0 + (k - l.dr));
}

// One attempt at colouring v by G lanes (G = 1: the calling lane alone; G = 32: the
// whole warp, every lane with the same arguments).  waiting < 0: no blocker known yet.
// Returns true when v got its colour; otherwise waiting / resume hold where to look
// next time (the same in every lane).
template <int G>
__device__ __forceinline__ bool gcTry(const GcArgs a, Index v, const GcList& l,
                                      Index& waiting, Index& resume, int lane) {
  if (waiting >= 0 && gcLoadColour(a.colour + waiting) == 0u) return false;
  const unsigned int hv = gcHash(a.seed, static_cast<unsigned int>(v));
  const Index len = l.dr + l.dc;
  const int me = (G == 1) ? 0 : lane;
  // the first uncoloured higher-priority neighbour at or after `resume`: entries before
  // it are lower-priority or coloured, and a colour never goes back to 0
  for (Index k0 = resume; k0 < len; k0 += G) {
    const Index k = k0 + me;
    Index u = -1;
    if (k < len) {
      const Index x = gcEntry(a, l, k);
      if (gcAbove(gcHash(a.seed, static_cast<unsigned int>(x)), x, hv, v) &&
          gcLoadColour(a.colour + x) == 0u)
        u = x;
    }
    int src = 0;
    if (G == 32) {
      const unsigned int m = __ballot_sync(GB_FULL_MASK, u >= 0);
      if (m == 0u) continue;
      src = __ffs(m) - 1;
      u = __shfl_sync(GB_FULL_MASK, u, src);
    } else if (u < 0) {
      continue;
    }
    waiting = u;
    resume = k0 + src;
    return false;
  }
  // the colour pass: 64 colours per window
  for (unsigned int base = 0u;; base += 64u) {
    unsigned long long used = 0ull;
    Index stale = -1;
#pragma unroll 4
    for (Index k = me; k < len; k += G) {
      const Index x = gcEntry(a, l, k);
      const unsigned int c = gcLoadColour(a.colour + x);
      if (c == 0u && base == 0u &&
          gcAbove(gcHash(a.seed, static_cast<unsigned int>(x)), x, hv, v))
        stale = x;
      const unsigned int d = c - 1u - base;           // wraps for 0 and for c <= base
      if (d < 64u) used |= 1ull << d;
    }
    if (base == 0u) {
      if (G == 32) {
        const unsigned int m = __ballot_sync(GB_FULL_MASK, stale >= 0);
        if (m != 0u) stale = __shfl_sync(GB_FULL_MASK, stale, __ffs(m) - 1);
      }
      if (stale >= 0) {
        waiting = stale;
        resume = 0;
        return false;
      }
    }
    if (G == 32) {
      const unsigned int lo = __reduce_or_sync(GB_FULL_MASK, static_cast<unsigned int>(used));
      const unsigned int hi = __reduce_or_sync(GB_FULL_MASK,
                                               static_cast<unsigned int>(used >> 32));
      used = (static_cast<unsigned long long>(hi) << 32) | lo;
    }
    if (~used != 0ull) {
      if (me == 0)
        gcStoreColour(a.colour + v, base + static_cast<unsigned int>(
                                               __ffsll(static_cast<long long>(~used))));
      return true;
    }
  }
}

template <typename W>
__global__ void __launch_bounds__(GB_GC_NT, GB_GC_MINB)
graphColorKernel(GcArgs a, W* out) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31;
  const Index gtid = blockIdx.x*GB_GC_NT + threadIdx.x;
  const Index gwarp = gtid >> 5;
  const Index gwarps = (gridDim.x*GB_GC_NT) >> 5;
  const Index tail_max = gwarps*32;

  // ---- sweeps ------------------------------------------------------------------------
  Index m = a.n;                     // vertices left
  const Index* in = NULL;            // the list of sweep s >= 1; the first is 0..n-1
  int s = 0;
  while (m > tail_max) {
    Index* next = (s & 1) ? a.list[1] : a.list[0];   // no dynamic index into the params
    unsigned long long* count = a.counters + (s % 3);
    if (gtid == 0) a.counters[(s + 1) % 3] = 0ull;
    for (Index i0 = gwarp*32; i0 < m; i0 += gwarps*32) {
      const Index i = i0 + lane;
      Index v = -1, waiting = -1, resume = 0;
      GcList l = {0, 0, 0, 0};
      bool done = true;
      if (i < m) {
        v = (s == 0) ? i : in[i];
        if (s > 0) { waiting = a.waiting_on[v]; resume = a.resume[v]; }
        l = gcListOf(a, v);
        if (l.dr + l.dc <= GB_GC_LANE_MAX) done = gcTry<1>(a, v, l, waiting, resume, lane);
      }
      unsigned int heavy = __ballot_sync(GB_FULL_MASK, i < m && l.dr + l.dc > GB_GC_LANE_MAX);
      while (heavy != 0u) {
        const int src = __ffs(heavy) - 1;
        heavy &= heavy - 1u;
        const Index hv = __shfl_sync(GB_FULL_MASK, v, src);
        Index hw = __shfl_sync(GB_FULL_MASK, waiting, src);
        Index hr = __shfl_sync(GB_FULL_MASK, resume, src);
        const bool ok = gcTry<32>(a, hv, gcListOf(a, hv), hw, hr, lane);
        if (lane == src) { done = ok; waiting = hw; resume = hr; }
      }
      if (!done) { a.waiting_on[v] = waiting; a.resume[v] = resume; }
      const unsigned int left = __ballot_sync(GB_FULL_MASK, !done);
      if (left != 0u) {
        Index at = 0;
        if (lane == 0) at = static_cast<Index>(atomicAdd(count, __popc(left)));
        at = __shfl_sync(GB_FULL_MASK, at, 0);
        if (!done) next[at + __popc(left & ((1u << lane) - 1u))] = v;
      }
    }
    grid.sync();
    m = static_cast<Index>(*reinterpret_cast<volatile unsigned long long*>(count));
    in = next;
    ++s;
  }

  // ---- tail: a warp owns up to 32 vertices and works on them until all are coloured ---
  {
    const Index i = gwarp + static_cast<Index>(lane)*gwarps;
    Index v = -1, waiting = -1, resume = 0;
    if (i < m) {
      v = (s == 0) ? i : in[i];
      if (s > 0) { waiting = a.waiting_on[v]; resume = a.resume[v]; }
    }
    unsigned int pending = __ballot_sync(GB_FULL_MASK, i < m);
    while (pending != 0u) {
      const bool ready = ((pending >> lane) & 1u) &&
                         (waiting < 0 || gcLoadColour(a.colour + waiting) != 0u);
      unsigned int go = __ballot_sync(GB_FULL_MASK, ready);
      if (go == 0u) __nanosleep(200);
      while (go != 0u) {
        const int src = __ffs(go) - 1;
        go &= go - 1u;
        const Index hv = __shfl_sync(GB_FULL_MASK, v, src);
        Index hw = __shfl_sync(GB_FULL_MASK, waiting, src);
        Index hr = __shfl_sync(GB_FULL_MASK, resume, src);
        const bool ok = gcTry<32>(a, hv, gcListOf(a, hv), hw, hr, lane);
        if (lane == src) { waiting = hw; resume = hr; }
        if (ok) pending &= ~(1u << src);
      }
    }
  }
  grid.sync();

  // ---- out ---------------------------------------------------------------------------
  unsigned int top = 0u;
  for (Index i = gtid; i < a.n; i += gwarps*32) {
    const unsigned int c = __ldcg(a.colour + i);
    out[i] = static_cast<W>(c);
    top = c > top ? c : top;
  }
  top = __reduce_max_sync(GB_FULL_MASK, top);
  if (lane == 0 && top != 0u) atomicMax(a.counters + 3, static_cast<unsigned long long>(top));
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_COLOR_CUH_
