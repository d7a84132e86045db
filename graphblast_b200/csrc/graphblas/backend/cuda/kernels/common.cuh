// graphblast_b200 backend — device-side building blocks shared by all kernels:
// cache-hinted loads for sm_90a, warp/CTA reductions, semiring atomics,
// bitmap helpers.  No reference counterpart (the reference delegates these to
// moderngpu/cub, see SURVEY.md §2b).
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_COMMON_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_COMMON_CUH_

#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

namespace graphblas {
namespace backend {

#define GB_FULL_MASK 0xffffffffu

// ---------------------------------------------------------------------------
// Streaming loads.  CSR colind/val are read exactly once per mxv: keep them out
// of L1 (L1::no_allocate) and, on the 8-word path, evict-first in L2 so the
// gathered dense vector (which IS reused) keeps its L2 residency (50 MB L2).
// sm_90a has no 256-bit global load: 8 words are two 128-bit loads, each with
// an L2::cache_hint carrying an evict-first policy.
// ---------------------------------------------------------------------------
struct Word8 { int w[8]; };

// Not volatile: the policy is a pure value, so the compiler creates it once per
// kernel instead of once per load.
__device__ __forceinline__ uint64_t streamPolicy() {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

__device__ __forceinline__ Word8 ldStream256(const void* p /* 32B aligned */) {
  const uint64_t pol = streamPolicy();
  const int* q = static_cast<const int*>(p);
  Word8 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.b32 "
               "{%0, %1, %2, %3}, [%4], %5;"
               : "=r"(r.w[0]), "=r"(r.w[1]), "=r"(r.w[2]), "=r"(r.w[3])
               : "l"(q), "l"(pol));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.b32 "
               "{%0, %1, %2, %3}, [%4], %5;"
               : "=r"(r.w[4]), "=r"(r.w[5]), "=r"(r.w[6]), "=r"(r.w[7])
               : "l"(q + 4), "l"(pol));
  return r;
}

__device__ __forceinline__ int4 ldStream128(const void* p /* 16B aligned */) {
  int4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

__device__ __forceinline__ int ldStream32(const void* p) {
  int v;
  asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];"
               : "=r"(v) : "l"(p));
  return v;
}

template <typename T>
__device__ __forceinline__ T ldStream(const T* p) {
  static_assert(sizeof(T) == 4, "32-bit element expected");
  int bits = ldStream32(p);
  T v;
  memcpy(&v, &bits, 4);
  return v;
}

// L2 eviction policy for the gathered operand (evict-last).  createpolicy is a
// uniform-datapath instruction; call once per kernel.
__device__ __forceinline__ uint64_t makeEvictLastPolicy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;"
               : "=l"(pol));
  return pol;
}

__device__ __forceinline__ int ldGather32(const void* p, uint64_t pol) {
  int v;
  asm volatile("ld.global.nc.L2::cache_hint.s32 %0, [%1], %2;"
               : "=r"(v) : "l"(p), "l"(pol));
  return v;
}

template <typename T>
__device__ __forceinline__ T ldGather(const T* p, uint64_t pol) {
  static_assert(sizeof(T) == 4, "32-bit element expected");
  int bits = ldGather32(p, pol);
  T v;
  memcpy(&v, &bits, 4);
  return v;
}

// ---------------------------------------------------------------------------
// Warp reductions with an arbitrary binary functor.
// ---------------------------------------------------------------------------
template <typename T, typename Op>
__device__ __forceinline__ T warpReduce(T v, Op op) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1)
    v = op(v, __shfl_xor_sync(GB_FULL_MASK, v, off));
  return v;
}

__device__ __forceinline__ int warpSum(int v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1)
    v += __shfl_xor_sync(GB_FULL_MASK, v, off);
  return v;
}

// CTA-wide sum of an int; result valid in every thread.  NT multiple of 32.
template <int NT>
__device__ __forceinline__ int blockSum(int v, int* smem /* NT/32 ints */) {
  const int lane = threadIdx.x & 31;
  const int wid  = threadIdx.x >> 5;
  v = warpSum(v);
  if (lane == 0) smem[wid] = v;
  __syncthreads();
  int total = 0;
#pragma unroll
  for (int i = 0; i < NT/32; ++i) total += smem[i];
  __syncthreads();
  return total;
}

// CTA-wide exclusive scan of one int per thread; returns the exclusive prefix,
// *total receives the CTA sum.  NT multiple of 32, NT <= 1024.
template <int NT>
__device__ __forceinline__ int blockExclusiveScan(int v, int* smem, int* total) {
  const int lane = threadIdx.x & 31;
  const int wid  = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    int t = __shfl_up_sync(GB_FULL_MASK, incl, off);
    if (lane >= off) incl += t;
  }
  if (lane == 31) smem[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int w = (lane < NT/32) ? smem[lane] : 0;
    int wi = w;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      int t = __shfl_up_sync(GB_FULL_MASK, wi, off);
      if (lane >= off) wi += t;
    }
    if (lane < NT/32) smem[lane] = wi - w;      // exclusive warp offsets
    if (lane == NT/32 - 1) smem[NT/32] = wi;    // total
  }
  __syncthreads();
  int result = smem[wid] + incl - v;
  *total = smem[NT/32];
  __syncthreads();
  return result;
}

// ---------------------------------------------------------------------------
// Semiring "add" applied atomically to a 32-bit cell.  Generic CAS loop with an
// early-out when the combine would not change the cell (monotone monoids such
// as min/max/or stop issuing atomics once the cell has converged).
// ---------------------------------------------------------------------------
template <typename T, typename AddOp>
__device__ __forceinline__ void atomicCombine(T* addr, T val, AddOp add_op) {
  static_assert(sizeof(T) == 4, "atomicCombine handles 32-bit values");
  unsigned int* a = reinterpret_cast<unsigned int*>(addr);
  unsigned int old = *a;
  while (true) {
    T cur;
    memcpy(&cur, &old, 4);
    T next = add_op(cur, val);
    unsigned int next_bits;
    memcpy(&next_bits, &next, 4);
    if (next_bits == old) return;
    unsigned int prev = atomicCAS(a, old, next_bits);
    if (prev == old) return;
    old = prev;
  }
}

// Same combine, returning the cell's value BEFORE this update.  `kind` is what
// the semiring's add answers for add(3, 5) — the reference's own way of telling
// monoids apart (spmv.hpp:76-85): 3 = minimum, 5 = maximum, 8 = plus.  For float
// cells those three map to one native atomic (ordered-int trick for min/max:
// floats with a clear sign bit order like signed ints, floats with the sign bit
// set like reversed unsigned ints); everything else takes the CAS loop.  The
// branch goes by the sign bit, not by `>= 0`: -0.0 compares equal to 0 but is
// INT_MIN as a signed int, so atomicMin(int) would overwrite a negative cell.
template <typename T, typename AddOp>
__device__ __forceinline__ T atomicCombineFetch(T* addr, T val, AddOp add_op,
                                                int kind) {
  static_assert(sizeof(T) == 4, "atomicCombineFetch handles 32-bit values");
  if (std::is_same<T, float>::value && (kind == 3 || kind == 5 || kind == 8)) {
    float* fa = reinterpret_cast<float*>(addr);
    float fv;
    memcpy(&fv, &val, 4);
    float old;
    if (kind == 8) {
      old = atomicAdd(fa, fv);
    } else {
      const bool neg = (__float_as_uint(fv) >> 31) != 0u;
      const bool as_signed = (kind == 3) ? !neg : neg;
      if (kind == 3) {
        old = as_signed
            ? __int_as_float(atomicMin(reinterpret_cast<int*>(fa),
                                       __float_as_int(fv)))
            : __uint_as_float(atomicMax(reinterpret_cast<unsigned int*>(fa),
                                        __float_as_uint(fv)));
      } else {
        old = !as_signed
            ? __int_as_float(atomicMax(reinterpret_cast<int*>(fa),
                                       __float_as_int(fv)))
            : __uint_as_float(atomicMin(reinterpret_cast<unsigned int*>(fa),
                                        __float_as_uint(fv)));
      }
    }
    T out;
    memcpy(&out, &old, 4);
    return out;
  }
  unsigned int* a = reinterpret_cast<unsigned int*>(addr);
  unsigned int old = *a;
  while (true) {
    T cur;
    memcpy(&cur, &old, 4);
    T next = add_op(cur, val);
    unsigned int next_bits;
    memcpy(&next_bits, &next, 4);
    if (next_bits == old) return cur;
    unsigned int prev = atomicCAS(a, old, next_bits);
    if (prev == old) return cur;
    old = prev;
  }
}

// ---------------------------------------------------------------------------
// Bitmap helpers (one bit per vertex, 32-bit words).
// ---------------------------------------------------------------------------
__device__ __forceinline__ bool bitTest(const unsigned int* bits, int i) {
  return (bits[i >> 5] >> (i & 31)) & 1u;
}

// Returns true if this call set the bit (it was clear before).
__device__ __forceinline__ bool bitSetAtomic(unsigned int* bits, int i) {
  const unsigned int m = 1u << (i & 31);
  unsigned int* w = bits + (i >> 5);
  if (*w & m) return false;
  return (atomicOr(w, m) & m) == 0;
}

// fmix32, the murmur3 finaliser: the vertex hash of the components sample and of the
// greedy priority (host and device; the colouring oracle restates it).
__host__ __device__ __forceinline__ unsigned int fmix32(unsigned int x) {
  x ^= x >> 16; x *= 0x85EBCA6Bu;
  x ^= x >> 13; x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

// upper_bound over a sorted int array: first index with a[idx] > key.
__device__ __forceinline__ int upperBound(const int* a, int n, int key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] <= key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// upper_bound executed by a whole warp as a 32-ary search: every step probes 32
// evenly spaced positions at once, so a search over n elements costs
// ceil(log32 n) dependent loads instead of log2 n.  All 32 lanes must call it
// with the same arguments; all lanes return the result.
__device__ __forceinline__ int warpUpperBound(const int* a, int n, int key) {
  const int lane = threadIdx.x & 31;
  int lo = 0, hi = n;
  while (hi > lo) {
    const int step = (hi - lo + 31) >> 5;
    const int idx  = lo + lane*step;
    const bool gt  = (idx < hi) ? (__ldg(a + idx) > key) : true;
    const unsigned m = __ballot_sync(GB_FULL_MASK, gt);
    const int first = m ? (__ffs(m) - 1) : 32;
    const int cand   = lo + first*step;
    const int new_hi = (first == 0) ? lo : (cand < hi ? cand : hi);
    const int new_lo = (first == 0) ? lo : lo + (first - 1)*step + 1;
    lo = new_lo;
    hi = new_hi;
  }
  return lo;
}

// Exact-match binary search in a sorted int array segment [lo, hi); -1 if absent.
__device__ __forceinline__ int findSorted(const int* a, int lo, int hi, int key) {
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    int v = __ldg(a + mid);
    if (v < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_COMMON_CUH_
