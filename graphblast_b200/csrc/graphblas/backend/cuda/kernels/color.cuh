// graphblast_b200 backend — greedy Jones–Plassmann graph colouring as ONE persistent
// cooperative kernel (backend::graphColor, algorithm::gc; host side color.hpp): the
// greedy schedule (kernels/greedy_schedule.cuh, which defines the graph and the
// priority p) with the colouring's step.
//
// Semantics.  A vertex is coloured once every higher-priority neighbour is, with the
// smallest colour c >= 1 none of them holds.  The result is sequential greedy first-fit
// colouring in decreasing p order (tests/gc_oracle.c restates it), whatever the launch
// shape or timing.
//
// Determinism.  colour[v] goes from 0 to its final value in one 32-bit store, and v is
// stored only after v has seen every higher-priority neighbour non-zero.  A
// lower-priority neighbour u of v cannot be coloured before v (u waits for v), so when
// v picks its colour the non-zero colours among its neighbours are exactly the final
// colours of its higher-priority neighbours.  Scheduling decides only when v is
// coloured, never with what.  Progress: the highest-priority uncoloured vertex is never
// blocked.
//
// Step.  poll: v is BLOCKED while the neighbour it is known to wait on reads colour 0,
// otherwise it is attempted (the colouring is never DONE at a poll).  An attempt scans
// v's list from where the last scan stopped for the first uncoloured higher-priority
// neighbour, which becomes waiting_on[v]; with none left, the colour pass.  Out:
// out[i] = colour[i] and ncolors = max colour.
// Colour pass: colours up to degree + 1, taken 64 at a time: a 64-bit mask of the
// window's colours held by the neighbours (warp OR-reduced when a warp has the vertex);
// the next window is looked at only when all 64 are held.  The pass also checks that no
// higher-priority neighbour reads 0; if one does the attempt is given up (it never
// happens when loads are coherent, and keeps the colour correct if it does).
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_COLOR_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_COLOR_CUH_

#include "graphblas/backend/cuda/kernels/greedy_schedule.cuh"

namespace graphblas {
namespace backend {

struct ColorStep {
  static __device__ __forceinline__ int poll(const GreedyArgs a, Index v, Index waiting) {
    return waiting >= 0 && ldRelaxed(a.state + waiting) == 0u ? GREEDY_BLOCKED
                                                                 : GREEDY_ATTEMPT;
  }

  template <int G>
  static __device__ __forceinline__ bool attempt(const GreedyArgs a, Index v,
                                                 const GcList& l, Index& waiting,
                                                 Index& resume, int lane) {
    const unsigned int hv = gcHash(a.seed, static_cast<unsigned int>(v));
    const Index len = l.dr + l.dc;
    const int me = (G == 1) ? 0 : lane;
    // the first uncoloured higher-priority neighbour at or after `resume`: entries
    // before it are lower-priority or coloured, and a colour never goes back to 0
    for (Index k0 = resume; k0 < len; k0 += G) {
      const Index k = k0 + me;
      Index u = -1;
      if (k < len) {
        const Index x = gcEntry(a, l, k);
        if (gcAbove(gcHash(a.seed, static_cast<unsigned int>(x)), x, hv, v) &&
            ldRelaxed(a.state + x) == 0u)
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
        const unsigned int c = ldRelaxed(a.state + x);
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
        const unsigned int lo = __reduce_or_sync(GB_FULL_MASK,
                                                 static_cast<unsigned int>(used));
        const unsigned int hi = __reduce_or_sync(GB_FULL_MASK,
                                                 static_cast<unsigned int>(used >> 32));
        used = (static_cast<unsigned long long>(hi) << 32) | lo;
      }
      if (~used != 0ull) {
        if (me == 0)
          stRelaxed(a.state + v, base + static_cast<unsigned int>(
                                               __ffsll(static_cast<long long>(~used))));
        return true;
      }
    }
  }

  template <typename W>
  static __device__ __forceinline__ void out(const GreedyArgs a, W* out, Index first,
                                             Index stride, int lane) {
    unsigned int top = 0u;
    for (Index i = first; i < a.n; i += stride) {
      const unsigned int c = __ldcg(a.state + i);
      out[i] = static_cast<W>(c);
      top = c > top ? c : top;
    }
    top = __reduce_max_sync(GB_FULL_MASK, top);
    if (lane == 0 && top != 0u) atomicMax(a.counters + GREEDY_COUNT,
                                          static_cast<unsigned long long>(top));
  }
};

template <typename W>
__global__ void __launch_bounds__(GB_GC_NT, GB_GC_MINB)
graphColorKernel(GreedyArgs a, W* out) { greedySchedule<ColorStep>(a, out); }

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_COLOR_CUH_
