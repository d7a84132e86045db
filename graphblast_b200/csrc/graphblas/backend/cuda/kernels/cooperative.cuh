// graphblast_b200 backend — device primitives the persistent cooperative kernels share:
// coherent loads and stores, counter-cell reads, the global timer, a warp-aggregated append.
//
// Memory model.  A word other SMs write while the kernel runs is read with ldRelaxed
// (ld.relaxed.gpu, from L2), never through the non-coherent path (__ldg, ld.global.nc)
// or L1: a stale line may stay in L1 for as long as it is there, so a blocked vertex
// would never see its blocker decided.  The asm is volatile: every re-read in a loop is
// issued.  Writes before a grid barrier are visible to every thread after it.  Arrays
// nothing writes during the kernel, such as the CSR and CSC, take the non-coherent path.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_COOPERATIVE_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_COOPERATIVE_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/common.cuh"

namespace graphblas {
namespace backend {

__device__ __forceinline__ int ldRelaxed(const int* p) {
  int x;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(x) : "l"(p));
  return x;
}

__device__ __forceinline__ unsigned int ldRelaxed(const unsigned int* p) {
  unsigned int x;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(x) : "l"(p));
  return x;
}

__device__ __forceinline__ void stRelaxed(int* p, int x) {
  asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" :: "l"(p), "r"(x) : "memory");
}

__device__ __forceinline__ void stRelaxed(unsigned int* p, unsigned int x) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(x) : "memory");
}

// A counter cell, read after the barrier that ends its updates (volatile: re-read on
// every call, not kept in a register across the barrier).
template <typename T>
__device__ __forceinline__ T loadCell(const T* p) {
  return *reinterpret_cast<const volatile T*>(p);
}

// %globaltimer, nanoseconds.
__device__ __forceinline__ unsigned long long globalTimerNs() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Appends y at q[base + the cell's count], one atomic for the lanes that append together.
__device__ __forceinline__ void warpAppend(Index* q, Index base, unsigned long long* cell,
                                           Index y) {
  namespace cg = cooperative_groups;
  cg::coalesced_group g = cg::coalesced_threads();
  unsigned long long at = 0ull;
  if (g.thread_rank() == 0) at = atomicAdd(cell, static_cast<unsigned long long>(g.size()));
  at = g.shfl(at, 0);
  q[base + static_cast<Index>(at) + static_cast<Index>(g.thread_rank())] = y;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_COOPERATIVE_CUH_
