// graphblast_b200 backend — maximal independent set as ONE persistent cooperative
// kernel (algorithm::mis; host side mis.hpp): the greedy schedule
// (kernels/greedy_schedule.cuh, which defines the graph and the priority p) with the
// MIS step, after an init pass over the candidates.
//
// Semantics.  Only candidates take part.  The set is the sequential greedy MIS in
// decreasing p order over the candidates: v joins iff no higher-priority candidate
// neighbour joined (tests/mis_oracle.c orc_mis restates it), whatever the launch shape
// or timing.
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
// highest-priority UNDECIDED vertex is never blocked.
//
// Step.
//   poll: state[v] OUT (marked by a member): done.  v waits on a blocker: only the
//     blocker is read; UNDECIDED keeps v blocked, IN makes v OUT, OUT lets the scan go
//     on from resume[v].
//   attempt: v's higher-priority neighbours from resume[v]: one IN makes v OUT; the
//     first UNDECIDED one becomes waiting_on[v]; with neither, v stores IN and marks
//     its lower-priority neighbours OUT (a lane or a warp, as v was attempted).
//   out: out[i] = (state[i] == IN) and nmembers.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_MIS_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_MIS_CUH_

#include "graphblas/backend/cuda/kernels/greedy_schedule.cuh"

namespace graphblas {
namespace backend {

#define MIS_UNDECIDED 0u
#define MIS_IN        1u
#define MIS_OUT       2u

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

struct MisStep {
  static __device__ __forceinline__ int poll(const GreedyArgs a, Index v, Index waiting) {
    if (gcLoadState(a.state + v) != MIS_UNDECIDED) return GREEDY_DONE;
    if (waiting >= 0) {
      const unsigned int b = gcLoadState(a.state + waiting);
      if (b == MIS_UNDECIDED) return GREEDY_BLOCKED;
      if (b == MIS_IN) {
        gcStoreState(a.state + v, MIS_OUT);
        return GREEDY_DONE;
      }
    }
    return GREEDY_ATTEMPT;
  }

  template <int G>
  static __device__ __forceinline__ bool attempt(const GreedyArgs a, Index v,
                                                 const GcList& l, Index& waiting,
                                                 Index& resume, int lane) {
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
          s = gcLoadState(a.state + x);
      }
      int src = 0;
      if (G == 32) {
        if (__ballot_sync(GB_FULL_MASK, s == MIS_IN) != 0u) {
          if (me == 0) gcStoreState(a.state + v, MIS_OUT);
          return true;
        }
        const unsigned int m = __ballot_sync(GB_FULL_MASK, s == MIS_UNDECIDED);
        if (m == 0u) continue;
        src = __ffs(m) - 1;
        x = __shfl_sync(GB_FULL_MASK, x, src);
      } else if (s == MIS_IN) {
        gcStoreState(a.state + v, MIS_OUT);
        return true;
      } else if (s != MIS_UNDECIDED) {
        continue;
      }
      waiting = x;
      resume = k0 + src;
      return false;
    }
    if (me == 0) gcStoreState(a.state + v, MIS_IN);
    for (Index k = me; k < len; k += G) {
      const Index x = gcEntry(a, l, k);
      if (gcAbove(hv, v, gcHash(a.seed, static_cast<unsigned int>(x)), x))
        gcStoreState(a.state + x, MIS_OUT);
    }
    return true;
  }

  template <typename W>
  static __device__ __forceinline__ void out(const GreedyArgs a, W* out, Index first,
                                             Index stride, int lane) {
    unsigned int members = 0u;
    for (Index i = first; i < a.n; i += stride) {
      const bool member = __ldcg(a.state + i) == MIS_IN;
      out[i] = static_cast<W>(member ? 1 : 0);
      members += member ? 1u : 0u;
    }
    members = __reduce_add_sync(GB_FULL_MASK, members);
    if (lane == 0 && members != 0u)
      atomicAdd(a.counters + 3, static_cast<unsigned long long>(members));
  }
};

template <typename W>
__global__ void __launch_bounds__(GB_GC_NT, GB_GC_MINB)
misKernel(GreedyArgs a, W* out) { greedySchedule<MisStep>(a, out); }

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_MIS_CUH_
