// graphblast_b200 backend — the element-wise tail of one SSSP / PageRank iteration
// as a single pass (backend/cuda/loop_steps.hpp).  Both kernels fold their
// reduction with the indexing of reducePartialKernel (same grid, same per-thread
// order), so the scalar they produce is the one the separate reduce would give.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_LOOP_STEPS_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_LOOP_STEPS_CUH_

#include "graphblas/backend/cuda/kernels/reduce.cuh"

namespace graphblas {
namespace backend {

// SSSP, after relaxed = frontier (min.+) A:
//   improved = relaxed < dist ; dist = min(dist, relaxed) ;
//   relaxed<!improved> = inf ; partials = sum(improved)
template <typename T>
__global__ void __launch_bounds__(GB_REDUCE_NT)
ssspRelaxKernel(T* __restrict__ dist, T* __restrict__ relaxed, Index n, T inf,
                T* __restrict__ partials) {
  __shared__ T s_red[GB_REDUCE_NT/32];
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  PlusMonoid<T> add;
  T improved = static_cast<T>(0);
  for (; i < n; i += stride) {
    const T w = relaxed[i];
    const T d = dist[i];
    if (w < d) {
      dist[i] = w;
      improved = add(improved, static_cast<T>(1));
    } else {
      relaxed[i] = inf;
      improved = add(improved, static_cast<T>(0));
    }
  }
  const T total = blockReduce(improved, add, static_cast<T>(0), s_red);
  if (threadIdx.x == 0) partials[blockIdx.x] = total;
}

// PageRank, after contrib = rank_before (+.*) A:
//   rank = contrib + jump ; partials = sum(diff^2), where diff is what the dense
//   eWiseMult PlusMinus of the separate route gives: rank - rank_before, or its
//   identity 0 where either rank is 0 (ewiseMultDenseKernel)
template <typename T>
__global__ void __launch_bounds__(GB_REDUCE_NT)
prUpdateKernel(T* __restrict__ rank, const T* __restrict__ contrib,
               const T* __restrict__ rank_before, Index n, T jump,
               T* __restrict__ partials) {
  __shared__ T s_red[GB_REDUCE_NT/32];
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  PlusMonoid<T> add;
  T acc = static_cast<T>(0);
  for (; i < n; i += stride) {
    const T now    = contrib[i] + jump;
    const T before = rank_before[i];
    const T diff   = (now == static_cast<T>(0) || before == static_cast<T>(0))
                         ? static_cast<T>(0) : now - before;
    rank[i] = now;
    // the separate operations round the square before it is added: no fma here
    const T square = static_cast<T>(__fmul_rn(static_cast<float>(diff),
                                              static_cast<float>(diff)));
    acc = add(acc, square);
  }
  const T total = blockReduce(acc, add, static_cast<T>(0), s_red);
  if (threadIdx.x == 0) partials[blockIdx.x] = total;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_LOOP_STEPS_CUH_
