// graphblast_b200 backend — small utility kernels: fill, scatter, nnz count,
// bitmap maintenance.  Functional counterparts of reference
// graphblas/backend/cuda/kernels/util.hpp:26-220 (zeroKernel, scatter,
// countZero, ...) written as grid-stride kernels sized to the SM count.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_UTIL_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_UTIL_CUH_

#include "graphblas/backend/cuda/kernels/common.cuh"

namespace graphblas {
namespace backend {

// w[i] = val for i in [0, n).  (reference zeroKernel, kernels/util.hpp:26-32;
// the reference fills dense vectors on the HOST and copies 4n bytes H2D,
// dense_vector.hpp:312-318.)
template <typename T>
__global__ void fillKernel(T* __restrict__ w, T val, Index n) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < n; i += stride) w[i] = val;
}

// w[i] = i
template <typename T>
__global__ void iotaKernel(T* __restrict__ w, Index n) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < n; i += stride) w[i] = static_cast<T>(i);
}

// w[ind[i]] = val          (reference scatter, kernels/util.hpp:181-192)
template <typename T>
__global__ void scatterConstKernel(T* __restrict__ w,
                                   const Index* __restrict__ ind,
                                   T val, Index nvals) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < nvals; i += stride) w[ind[i]] = val;
}

// w[ind[i]] = vals[i]      (reference scatter, kernels/util.hpp:194-206)
template <typename T>
__global__ void scatterValsKernel(T* __restrict__ w,
                                  const Index* __restrict__ ind,
                                  const T* __restrict__ vals, Index nvals) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < nvals; i += stride) w[ind[i]] = vals[i];
}

// *counter += #{i : u[i] != identity}.  One atomic per CTA.
// (reference countZero + cub::DeviceReduce, dense_vector.hpp:138-186)
template <int NT, typename T>
__global__ void countNonIdentityKernel(unsigned long long* counter,
                                       const T* __restrict__ u, T identity,
                                       Index n) {
  __shared__ int s_red[NT/32];
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  int local = 0;
  for (; i < n; i += stride) local += (u[i] != identity) ? 1 : 0;
  int total = blockSum<NT>(local, s_red);
  if (threadIdx.x == 0 && total)
    atomicAdd(counter, static_cast<unsigned long long>(total));
}

// Bitmap of a constant vector of n elements: every word all-zero, or all-one with
// the bits past n in the last word CLEAR (whole-word consumers — popcount,
// ordered compaction — rely on the tail being zero).
__global__ void fillBitmapKernel(unsigned int* __restrict__ bits, Index n,
                                 bool ones) {
  Index w = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  const Index nwords = (n + 31) >> 5;
  for (; w < nwords; w += stride) {
    unsigned int word = ones ? 0xffffffffu : 0u;
    if (ones && w == nwords - 1 && (n & 31) != 0) word = (1u << (n & 31)) - 1u;
    bits[w] = word;
  }
}

// bits = bitmap of {i : u[i] != 0}; one 32-bit word per warp-iteration.
template <typename T>
__global__ void denseToBitmapKernel(unsigned int* __restrict__ bits,
                                    const T* __restrict__ u, Index n) {
  // Each warp converts 32 consecutive elements into one word with a ballot.
  const int lane = threadIdx.x & 31;
  Index warp = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
  const Index nwarps = (gridDim.x*blockDim.x) >> 5;
  const Index nwords = (n + 31) >> 5;
  for (; warp < nwords; warp += nwarps) {
    Index i = warp*32 + lane;
    bool set = (i < n) && (u[i] != static_cast<T>(0));
    unsigned int word = __ballot_sync(GB_FULL_MASK, set);
    if (lane == 0) bits[warp] = word;
  }
}

// u[i] = bit i of bits ? 1 : 0   (inverse of denseToBitmapKernel for 0/1 data)
template <typename T>
__global__ void bitmapToDenseKernel(T* __restrict__ u,
                                    const unsigned int* __restrict__ bits,
                                    Index n) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < n; i += stride)
    u[i] = ((bits[i >> 5] >> (i & 31)) & 1u) ? static_cast<T>(1)
                                             : static_cast<T>(0);
}

// *counter += popcount of the first nwords words
__global__ void popcountKernel(unsigned long long* counter,
                               const unsigned int* __restrict__ bits,
                               Index nwords) {
  __shared__ int s_red[256/32];
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  int local = 0;
  for (; i < nwords; i += stride) local += __popc(bits[i]);
  int total = blockSum<256>(local, s_red);
  if (threadIdx.x == 0 && total)
    atomicAdd(counter, static_cast<unsigned long long>(total));
}

// deg[i] = rowptr[f[i]+1] - rowptr[f[i]] for i < nf, deg[nf] = 0.
// (reference indirectScanKernel, kernels/util.hpp:150-165)
__global__ void frontierDegreeKernel(Index* __restrict__ deg,
                                     const Index* __restrict__ rowptr,
                                     const Index* __restrict__ f_ind,
                                     Index nf) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i <= nf; i += stride) {
    Index d = 0;
    if (i < nf) {
      Index r = f_ind[i];
      d = rowptr[r+1] - rowptr[r];
    }
    deg[i] = d;
  }
}

// Single-launch form of frontierDegreeKernel + exclusive scan for short frontiers
// (the first and last levels of a traversal): offs[i] = sum_{j<i} deg(f[j]) for
// i in [0, nf], computed by one CTA in chunks of 1024.
#define GB_DEGSCAN_NT  1024
#define GB_DEGSCAN_MAX (GB_DEGSCAN_NT*8)
__global__ void __launch_bounds__(GB_DEGSCAN_NT)
frontierDegreeScanKernel(Index* __restrict__ offs,
                         const Index* __restrict__ rowptr,
                         const Index* __restrict__ f_ind, Index nf) {
  __shared__ int s_scan[GB_DEGSCAN_NT/32 + 1];
  __shared__ int s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (Index base = 0; base <= nf; base += GB_DEGSCAN_NT) {
    const Index i = base + threadIdx.x;
    int d = 0;
    if (i < nf) {
      const Index r = f_ind[i];
      d = rowptr[r+1] - rowptr[r];
    }
    int total;
    const int excl = blockExclusiveScan<GB_DEGSCAN_NT>(d, s_scan, &total);
    const int carry = s_carry;
    if (i <= nf) offs[i] = carry + excl;
    __syncthreads();
    if (threadIdx.x == 0) s_carry = carry + total;
    __syncthreads();
  }
}

// Posts a value of at most 40 bits to a host mailbox slot (backend/cuda/util.hpp).
__device__ __forceinline__ void mailPost(unsigned long long* mail, unsigned long long ticket,
                                         unsigned long long value) {
  *reinterpret_cast<volatile unsigned long long*>(mail) = (ticket << 40) | value;
  __threadfence_system();
}

// Posts one device-side Index to the host mailbox.
__global__ void postIndexKernel(const Index* __restrict__ value,
                                unsigned long long* mail,
                                unsigned long long ticket) {
  mailPost(mail, ticket, static_cast<unsigned int>(*value));
}

// Binary search helper kept for API parity with reference kernels/util.hpp:8-24.
__device__ __forceinline__ Index binarySearch(const Index* array, Index target,
                                              Index begin, Index end) {
  while (begin < end) {
    Index mid = begin + ((end - begin) >> 1);
    Index item = __ldg(array + mid);
    if (item == target) return mid;
    if (item > target) end = mid; else begin = mid + 1;
  }
  return -1;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_UTIL_CUH_
