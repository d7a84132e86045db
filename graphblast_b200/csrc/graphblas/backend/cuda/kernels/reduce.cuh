// graphblast_b200 backend — monoid reductions.  Two launches with a fixed grid
// (deterministic combination order for a given n): grid-stride partials per
// CTA, then one CTA folds the partials.  Replaces the cub::DeviceReduce /
// cub::DeviceSegmentedReduce calls of reference reduce.hpp:13-50, :131-139.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_REDUCE_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_REDUCE_CUH_

#include "graphblas/backend/cuda/kernels/common.cuh"
#include "graphblas/backend/cuda/kernels/util.cuh"

namespace graphblas {
namespace backend {

#define GB_REDUCE_NT 256

template <typename T, typename Op>
__device__ __forceinline__ T blockReduce(T v, Op op, T identity, T* s_red) {
  const int lane = threadIdx.x & 31;
  const int wid  = threadIdx.x >> 5;
  v = warpReduce(v, op);
  if (lane == 0) s_red[wid] = v;
  __syncthreads();
  if (wid == 0) {
    T x = (lane < GB_REDUCE_NT/32) ? s_red[lane] : identity;
    x = warpReduce(x, op);
    if (lane == 0) s_red[0] = x;
  }
  __syncthreads();
  T out = s_red[0];
  __syncthreads();
  return out;
}

// partials[cta] = fold of in[cta*NT + t + k*stride]
template <typename T, typename U, typename Op>
__global__ void __launch_bounds__(GB_REDUCE_NT)
reducePartialKernel(T* __restrict__ partials, const U* __restrict__ in,
                    Index n, Op op, T identity) {
  __shared__ T s_red[GB_REDUCE_NT/32];
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  T acc = identity;
  for (; i < n; i += stride) acc = op(acc, static_cast<T>(in[i]));
  T total = blockReduce(acc, op, identity, s_red);
  if (threadIdx.x == 0) partials[blockIdx.x] = total;
}

template <typename T, typename Op>
__global__ void __launch_bounds__(GB_REDUCE_NT)
reduceFinalKernel(T* __restrict__ out, const T* __restrict__ partials,
                  int nparts, Op op, T identity,
                  unsigned long long* mail, unsigned long long ticket) {
  __shared__ T s_red[GB_REDUCE_NT/32];
  T acc = identity;
  for (int i = threadIdx.x; i < nparts; i += GB_REDUCE_NT)
    acc = op(acc, partials[i]);
  T total = blockReduce(acc, op, identity, s_red);
  if (threadIdx.x == 0) {
    *out = total;
    if (mail != NULL && sizeof(T) == 4) {   // post to the host (util.hpp mailbox)
      unsigned int bits;
      memcpy(&bits, &total, 4);
      mailPost(mail, ticket, bits);
    }
  }
}

// w[row] = fold of A_val[rowptr[row] .. rowptr[row+1]) ; warp per row.
// Used once per PageRank run (out-degrees, reference example/gpr.cu:77-79),
// not on the per-iteration path.
template <typename W, typename a, typename Op>
__global__ void reduceRowsKernel(W* __restrict__ w,
                                 const Index* __restrict__ rowptr,
                                 const a* __restrict__ A_val, Index nrows,
                                 Op op, W identity) {
  const int lane = threadIdx.x & 31;
  Index row = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
  const Index nwarps = (gridDim.x*blockDim.x) >> 5;
  for (; row < nrows; row += nwarps) {
    Index beg = rowptr[row], end = rowptr[row+1];
    W acc = identity;
    for (Index k = beg + lane; k < end; k += 32)
      acc = op(acc, static_cast<W>(A_val[k]));
    acc = warpReduce(acc, op);
    if (lane == 0) w[row] = acc;
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_REDUCE_CUH_
