// graphblast_b200 backend — maximal independent set as ONE persistent cooperative
// kernel (algorithm::mis; host side mis.hpp).  It uses the colouring's priority, lists
// and schedule (kernels/color.cuh) without its colour pass.
//
// Semantics.  The graph is the colouring's: i != j conflict when A(i,j) or A(j,i) is
// stored, self-loops are ignored, and v's list is its CSR row followed, when the matrix
// is not symmetric, by its CSC column.  The priority is the colouring's
// p(v) = (gcHash(seed, v), v).  Only candidates take part.  The set is the sequential
// greedy MIS in decreasing p order over the candidates: v joins iff no higher-priority
// candidate neighbour joined (tests/mis_oracle.c orc_mis restates it), whatever the
// launch shape or timing.
//
// State.  One word per vertex: MIS_UNDECIDED, MIS_IN or MIS_OUT.  The init pass sets
// non-candidates OUT, so they are never tried and never block anyone.  A vertex goes
// IN once every higher-priority neighbour is OUT, and OUT once one of them is IN.
//
// Determinism.  Every store writes the vertex's final value, so no store ever
// overwrites another with a different value:
//   - v stores IN only after it has read every higher-priority neighbour OUT, and goes
//     OUT as soon as it reads one IN;
//   - an IN vertex marks its lower-priority neighbours OUT (its higher-priority ones are
//     OUT already: it read them so), and a neighbour of a member is never a member;
//   - a lower-priority neighbour u of v cannot be IN while v is UNDECIDED (u would have
//     to read v OUT first), so no OUT can land on an IN.
// By induction over the stores in the order they happen, each writes the greedy
// answer.  Scheduling decides only when a vertex is decided, never how.  Progress: the
// highest-priority UNDECIDED vertex is never blocked, and no warp waits on another.
//
// Schedule: the colouring's (kernels/color.cuh).  Sweeps over the undecided list while
// more than 32 vertices per resident warp remain, a lane per list of at most
// GB_GC_LANE_MAX entries and a warp per longer list, a grid barrier between sweeps;
// then the tail, where a warp owns up to 32 vertices and runs without barriers; then
// the out pass, out[i] = (state[i] == IN) and nmembers.  An attempt at v:
//   1. misPoll: state[v] OUT (marked by a member): done.  v waits on a blocker: only the
//      blocker is read; UNDECIDED keeps v blocked, IN makes v OUT, OUT lets the scan
//      go on from resume[v].
//   2. misScan: v's higher-priority neighbours from resume[v]: one IN makes v OUT; the
//      first UNDECIDED one becomes waiting_on[v]; with neither, v stores IN and marks
//      its lower-priority neighbours OUT (a lane or a warp, as v was attempted).
// State loads and stores are gcLoadColour / gcStoreColour (ld/st.relaxed.gpu), for the
// reason written there.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_MIS_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_MIS_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/color.cuh"

namespace graphblas {
namespace backend {

#define MIS_UNDECIDED 0u
#define MIS_IN        1u
#define MIS_OUT       2u

struct MisArgs {
  const Index* row_ptr;  const Index* row_ind;        // CSR
  const Index* col_ptr;  const Index* col_ind;        // CSC; NULL when it is the CSR
  Index n;
  unsigned int seed;
  unsigned int* state;           // [n] MIS_UNDECIDED / MIS_IN / MIS_OUT
  Index* waiting_on;             // [n] UNDECIDED higher-priority neighbour last seen
  Index* resume;                 // [n] list position where the blocker scan goes on
  Index* list[2];                // [n] undecided vertices, ping-pong between sweeps
  unsigned long long* counters;  // [0..2] list length (rotating as in GcArgs), [3] nmembers
};

// Init pass, dense candidates: a vertex takes part when its value is non-zero.
template <typename C>
__global__ void misInitDenseKernel(unsigned int* __restrict__ state,
                                   const C* __restrict__ cand, Index n) {
  const Index stride = gridDim.x*blockDim.x;
  for (Index i = blockIdx.x*blockDim.x + threadIdx.x; i < n; i += stride)
    state[i] = cand[i] != static_cast<C>(0) ? MIS_UNDECIDED : MIS_OUT;
}

// Init pass, sparse candidates (state already all MIS_OUT): a stored non-zero value
// makes its index a candidate.
template <typename C>
__global__ void misInitSparseKernel(unsigned int* __restrict__ state,
                                    const Index* __restrict__ ind,
                                    const C* __restrict__ val, Index nvals, Index n) {
  const Index stride = gridDim.x*blockDim.x;
  for (Index k = blockIdx.x*blockDim.x + threadIdx.x; k < nvals; k += stride) {
    const Index i = ind[k];
    if (val[k] != static_cast<C>(0) && i >= 0 && i < n) state[i] = MIS_UNDECIDED;
  }
}

#define MIS_DONE    0
#define MIS_BLOCKED 1
#define MIS_SCAN    2

// Step 1 of an attempt at v by one lane.  waiting < 0: no blocker known yet.
__device__ __forceinline__ int misPoll(const MisArgs a, Index v, Index waiting) {
  if (gcLoadColour(a.state + v) != MIS_UNDECIDED) return MIS_DONE;
  if (waiting >= 0) {
    const unsigned int b = gcLoadColour(a.state + waiting);
    if (b == MIS_UNDECIDED) return MIS_BLOCKED;
    if (b == MIS_IN) {
      gcStoreColour(a.state + v, MIS_OUT);
      return MIS_DONE;
    }
  }
  return MIS_SCAN;
}

// Step 2 by G lanes (G = 1: the calling lane alone; G = 32: the whole warp, every lane
// with the same arguments).  Returns true when v is decided; otherwise waiting / resume
// hold where to look next time (the same in every lane).
template <int G>
__device__ __forceinline__ bool misScan(const MisArgs a, Index v, const GcList& l,
                                        Index& waiting, Index& resume, int lane) {
  const unsigned int hv = gcHash(a.seed, static_cast<unsigned int>(v));
  const Index len = l.dr + l.dc;
  const int me = (G == 1) ? 0 : lane;
  // entries before `resume` are lower-priority or were read OUT, and OUT is final
  for (Index k0 = resume; k0 < len; k0 += G) {
    const Index k = k0 + me;
    Index x = -1;
    unsigned int s = MIS_OUT;
    if (k < len) {
      x = gcEntry(a, l, k);
      if (gcAbove(gcHash(a.seed, static_cast<unsigned int>(x)), x, hv, v))
        s = gcLoadColour(a.state + x);
    }
    int src = 0;
    if (G == 32) {
      if (__ballot_sync(GB_FULL_MASK, s == MIS_IN) != 0u) {
        if (me == 0) gcStoreColour(a.state + v, MIS_OUT);
        return true;
      }
      const unsigned int m = __ballot_sync(GB_FULL_MASK, s == MIS_UNDECIDED);
      if (m == 0u) continue;
      src = __ffs(m) - 1;
      x = __shfl_sync(GB_FULL_MASK, x, src);
    } else if (s == MIS_IN) {
      gcStoreColour(a.state + v, MIS_OUT);
      return true;
    } else if (s != MIS_UNDECIDED) {
      continue;
    }
    waiting = x;
    resume = k0 + src;
    return false;
  }
  if (me == 0) gcStoreColour(a.state + v, MIS_IN);
  for (Index k = me; k < len; k += G) {
    const Index x = gcEntry(a, l, k);
    if (gcAbove(hv, v, gcHash(a.seed, static_cast<unsigned int>(x)), x))
      gcStoreColour(a.state + x, MIS_OUT);
  }
  return true;
}

template <typename W>
__global__ void __launch_bounds__(GB_GC_NT, GB_GC_MINB)
misKernel(MisArgs a, W* out) {
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
      bool done = true, heavy_v = false;
      if (i < m) {
        v = (s == 0) ? i : in[i];
        if (s > 0) { waiting = a.waiting_on[v]; resume = a.resume[v]; }
        const int p = misPoll(a, v, waiting);
        done = p == MIS_DONE;
        if (p == MIS_SCAN) {
          l = gcListOf(a, v);
          heavy_v = l.dr + l.dc > GB_GC_LANE_MAX;
          if (!heavy_v) done = misScan<1>(a, v, l, waiting, resume, lane);
        }
      }
      unsigned int heavy = __ballot_sync(GB_FULL_MASK, heavy_v);
      while (heavy != 0u) {
        const int src = __ffs(heavy) - 1;
        heavy &= heavy - 1u;
        const Index hv = __shfl_sync(GB_FULL_MASK, v, src);
        Index hw = __shfl_sync(GB_FULL_MASK, waiting, src);
        Index hr = __shfl_sync(GB_FULL_MASK, resume, src);
        const bool ok = misScan<32>(a, hv, gcListOf(a, hv), hw, hr, lane);
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
      const int p = ((pending >> lane) & 1u) ? misPoll(a, v, waiting) : MIS_BLOCKED;
      pending &= ~__ballot_sync(GB_FULL_MASK, p == MIS_DONE);
      unsigned int go = __ballot_sync(GB_FULL_MASK, p == MIS_SCAN);
      if (go == 0u && pending != 0u) __nanosleep(200);
      while (go != 0u) {
        const int src = __ffs(go) - 1;
        go &= go - 1u;
        const Index hv = __shfl_sync(GB_FULL_MASK, v, src);
        Index hw = __shfl_sync(GB_FULL_MASK, waiting, src);
        Index hr = __shfl_sync(GB_FULL_MASK, resume, src);
        const bool ok = misScan<32>(a, hv, gcListOf(a, hv), hw, hr, lane);
        if (lane == src) { waiting = hw; resume = hr; }
        if (ok) pending &= ~(1u << src);
      }
    }
  }
  grid.sync();

  // ---- out ---------------------------------------------------------------------------
  unsigned int members = 0u;
  for (Index i = gtid; i < a.n; i += gwarps*32) {
    const bool member = __ldcg(a.state + i) == MIS_IN;
    out[i] = static_cast<W>(member ? 1 : 0);
    members += member ? 1u : 0u;
  }
  members = __reduce_add_sync(GB_FULL_MASK, members);
  if (lane == 0 && members != 0u)
    atomicAdd(a.counters + 3, static_cast<unsigned long long>(members));
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_MIS_CUH_
