// graphblast_b200 backend — the greedy schedule: ONE persistent cooperative kernel body
// that decides every vertex in decreasing priority order among its neighbours, shared
// by the graph colouring (kernels/color.cuh) and the maximal independent set
// (kernels/mis.cuh); host side greedy_schedule.hpp.
//
// Graph and priority.  Vertices i != j conflict when A(i,j) or A(j,i) is stored;
// self-loops are ignored.  A vertex's list is its CSR row followed, when the matrix is
// not symmetric, by its CSC column, so the graph is the undirected graph of the
// pattern.  Every vertex has the priority
//     p(v) = (gcHash(seed, v), v), compared lexicographically,
//     gcHash(seed, v) = fmix32(v ^ (seed * 0x9E3779B9)),
//     fmix32(x): x ^= x >> 16; x *= 0x85EBCA6B; x ^= x >> 13; x *= 0xC2B2AE35; x ^= x >> 16
// (32-bit unsigned arithmetic; fmix32 is the murmur3 finaliser).
//
// Step.  What deciding a vertex means is the step type's; the schedule never branches
// on which algorithm it serves.  A step supplies
//   poll(a, v, waiting) — GREEDY_DONE (v is decided), GREEDY_BLOCKED (v still waits on
//     its known blocker `waiting`; nothing else is read) or GREEDY_ATTEMPT, by one lane;
//   attempt<G>(a, v, list, waiting, resume, lane) — by G lanes (G = 1: the calling lane
//     alone; G = 32: the whole warp, every lane with the same arguments): true when v
//     is decided, otherwise waiting / resume hold where to look next time (the same in
//     every lane);
//   out(a, out, first, stride, lane) — the out pass over all n vertices, and its count
//     into counters[3].
// A step keeps progress: the highest-priority undecided vertex is never blocked, and
// no warp waits on another warp; a blocked vertex is put back.
//
// Schedule.
//   sweeps — while more than 32 vertices per resident warp are undecided, the grid
//     sweeps the list of undecided vertices (the first sweep: all vertices).  A lane
//     polls each vertex; one that polls ATTEMPT loads its list bounds and is attempted
//     by its lane when the list has at most GB_GC_LANE_MAX entries, by the whole warp
//     otherwise.  Vertices still undecided are appended to the next list (one atomic
//     per warp); a grid barrier separates sweeps.
//   tail — with at most 32 per resident warp left, lane l of warp w owns list entry
//     w + l * (warps): no more barriers.  A warp polls all its vertices at once (a lane
//     each), and attempts the ones that poll ATTEMPT together, one at a time, until all
//     its vertices are decided; it sleeps briefly only when none is ready.
//   out — after one more barrier, the step's out pass.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_GREEDY_SCHEDULE_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_GREEDY_SCHEDULE_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/common.cuh"

namespace graphblas {
namespace backend {

#define GB_GC_NT        512            // CTA shape of the greedy kernels
#define GB_GC_MINB      2              // resident CTAs per SM the register budget allows
#define GB_GC_LANE_MAX  32             // longest list a single lane takes in a sweep

struct GreedyArgs {
  const Index* row_ptr;  const Index* row_ind;        // CSR
  const Index* col_ptr;  const Index* col_ind;        // CSC; NULL when it is the CSR
  Index n;
  unsigned int seed;
  unsigned int* state;           // [n] the step's per-vertex word: colour or MIS state
  Index* waiting_on;             // [n] undecided higher-priority neighbour last seen
  Index* resume;                 // [n] list position where the blocker scan goes on
  Index* list[2];                // [n] undecided vertices, ping-pong between sweeps
  unsigned long long* counters;  // [0..2] list length (rotating with the sweep % 3: the
                                 // cell of sweep s + 1 is zeroed during s), [3] the count
};

enum GreedyPoll { GREEDY_DONE, GREEDY_BLOCKED, GREEDY_ATTEMPT };

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

// State loads MUST NOT go through the non-coherent path (__ldg, ld.global.nc): a
// vertex re-reads states that other SMs store while the kernel runs, and a
// non-coherent load may keep returning a stale 0 from L1 for as long as the line
// stays there, so a blocked vertex would never see its blocker decided.
// ld.relaxed.gpu reads at GPU scope (L2); volatile keeps every re-read in the loop.
__device__ __forceinline__ unsigned int gcLoadState(const unsigned int* p) {
  unsigned int c;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(c) : "l"(p));
  return c;
}

__device__ __forceinline__ void gcStoreState(unsigned int* p, unsigned int c) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(c) : "memory");
}

// A vertex's list: its CSR row, then its CSC column (dc = 0 when symmetric).
struct GcList {
  Index r0, dr, c0, dc;
};

__device__ __forceinline__ GcList gcListOf(const GreedyArgs a, Index v) {
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

__device__ __forceinline__ Index gcEntry(const GreedyArgs a, const GcList& l, Index k) {
  return k < l.dr ? __ldg(a.row_ind + l.r0 + k) : __ldg(a.col_ind + l.c0 + (k - l.dr));
}

// The kernel body; the __global__ entry points call it with their step.
template <typename Step, typename W>
__device__ __forceinline__ void greedySchedule(const GreedyArgs a, W* out) {
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
      bool done = true, heavy_v = false;
      if (i < m) {
        v = (s == 0) ? i : in[i];
        if (s > 0) { waiting = a.waiting_on[v]; resume = a.resume[v]; }
        const int p = Step::poll(a, v, waiting);
        done = p == GREEDY_DONE;
        if (p == GREEDY_ATTEMPT) {
          const GcList l = gcListOf(a, v);
          heavy_v = l.dr + l.dc > GB_GC_LANE_MAX;
          if (!heavy_v) done = Step::template attempt<1>(a, v, l, waiting, resume, lane);
        }
      }
      unsigned int heavy = __ballot_sync(GB_FULL_MASK, heavy_v);
      while (heavy != 0u) {
        const int src = __ffs(heavy) - 1;
        heavy &= heavy - 1u;
        const Index hv = __shfl_sync(GB_FULL_MASK, v, src);
        Index hw = __shfl_sync(GB_FULL_MASK, waiting, src);
        Index hr = __shfl_sync(GB_FULL_MASK, resume, src);
        const bool ok = Step::template attempt<32>(a, hv, gcListOf(a, hv), hw, hr, lane);
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

  // ---- tail: a warp owns up to 32 vertices and works on them until all are decided ---
  {
    const Index i = gwarp + static_cast<Index>(lane)*gwarps;
    Index v = -1, waiting = -1, resume = 0;
    if (i < m) {
      v = (s == 0) ? i : in[i];
      if (s > 0) { waiting = a.waiting_on[v]; resume = a.resume[v]; }
    }
    unsigned int pending = __ballot_sync(GB_FULL_MASK, i < m);
    while (pending != 0u) {
      const int p = ((pending >> lane) & 1u) ? Step::poll(a, v, waiting) : GREEDY_BLOCKED;
      pending &= ~__ballot_sync(GB_FULL_MASK, p == GREEDY_DONE);
      unsigned int go = __ballot_sync(GB_FULL_MASK, p == GREEDY_ATTEMPT);
      if (go == 0u && pending != 0u) __nanosleep(200);
      while (go != 0u) {
        const int src = __ffs(go) - 1;
        go &= go - 1u;
        const Index hv = __shfl_sync(GB_FULL_MASK, v, src);
        Index hw = __shfl_sync(GB_FULL_MASK, waiting, src);
        Index hr = __shfl_sync(GB_FULL_MASK, resume, src);
        const bool ok = Step::template attempt<32>(a, hv, gcListOf(a, hv), hw, hr, lane);
        if (lane == src) { waiting = hw; resume = hr; }
        if (ok) pending &= ~(1u << src);
      }
    }
  }
  grid.sync();

  // ---- out ---------------------------------------------------------------------------
  Step::out(a, out, gtid, gwarps*32, lane);
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_GREEDY_SCHEDULE_CUH_
