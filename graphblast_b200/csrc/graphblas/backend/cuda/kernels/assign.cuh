// graphblast_b200 backend — assign: C(I, J) = accum(C(I, J), op(A)), the kernels
// behind assign_matrix.hpp.
//
// All four forms build one EMBEDDED SOURCE E, an m x n CSR holding op(A) (nI x nJ)
// placed at (I[p], J[q]), and then merge C with E on the merged-stream tiles of
// ewise_matrix.cuh, C on the A side so that its value comes first under accum:
//   E's row offsets: op(A)'s row lengths scattered through I (zero for rows outside
//     I), then scanned (assignRowLengthsKernel);
//   E's entries: op(A)'s entry t of row p goes to slot Eptr[I[p]] + t - ptr[p] with
//     column J[col] (assignEmbedKernel).  J increasing keeps every row sorted as it
//     is written; otherwise (row p << cbits | J[col], t) pairs are sorted with
//     radixSortPairs and assignSortedEmbedKernel writes them.  p is the high part of
//     the key, so a row's entries keep the slots of op(A)'s row;
//   the constant form fills each selected row with the sorted J (assignConstKernel).
// Without accum, C's entries in I x J are dropped by the merge's keep test, a
// bitmap of I over C's rows and one of J over its columns (AssignKeep); a matched
// pair takes E's value.  With accum nothing is dropped and a match writes
// accum(c, e).  Lists hold no repeated index (the host refuses them), so E is
// duplicate-free and the bitmaps are set with plain atomicOr.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_ASSIGN_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_ASSIGN_CUH_

#include "graphblas/backend/cuda/kernels/common.cuh"

namespace graphblas {
namespace backend {

// Element p of a list (list == NULL: GrB_ALL, p itself).
__device__ __forceinline__ Index asgAt(const Index* __restrict__ list, Index p) {
  return list != NULL ? __ldg(list + p) : p;
}

// Bit i of a bitmap (bits == NULL: every bit set).
__device__ __forceinline__ bool asgInSet(const unsigned int* __restrict__ bits, Index i) {
  return bits == NULL || ((__ldg(bits + (i >> 5)) >> (i & 31)) & 1u);
}

// The merge's keep test without accum: C's entry (r, c) stays unless r is in I
// and c in J.
struct AssignKeep {
  const unsigned int* rows;     // bitmap of I over C's rows, NULL = GrB_ALL
  const unsigned int* cols;     // bitmap of J over C's columns, NULL = GrB_ALL
  __device__ __forceinline__ bool operator()(Index r, Index c) const {
    return !(asgInSet(rows, r) && asgInSet(cols, c));
  }
};

// The combine step without accum: the assigned value replaces C's.
struct AssignTakeNew {
  template <typename X>
  __device__ __forceinline__ X operator()(X, X e) const { return e; }
};

// Largest p in [0, nrows) with ptr[p] <= t: the row of op(A) holding entry t.
__device__ __forceinline__ Index asgRowOf(long long t, const Index* __restrict__ ptr,
                                          Index nrows) {
  Index lo = 0, hi = nrows - 1;
  while (lo < hi) {
    const Index mid = lo + (hi - lo + 1)/2;
    if (__ldg(ptr + mid) <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// bits |= 1 << list[p] for every p < n (bits zeroed by the caller).
__global__ void assignMarkKernel(unsigned int* __restrict__ bits,
                                 const Index* __restrict__ list, Index n) {
  for (Index p = blockIdx.x*blockDim.x + threadIdx.x; p < n; p += gridDim.x*blockDim.x) {
    const Index i = __ldg(list + p);
    atomicOr(bits + (i >> 5), 1u << (i & 31));
  }
}

// out[p] = how many of u's nnz ascending indices lie below p, for p <= n (dense:
// every index is stored, out[p] = p).  With n = size(u) this is the row offsets of
// u as an n x 1 matrix; read up to nnz it is u's index list.
__global__ void assignStoredBelowKernel(Index* __restrict__ out,
                                        const Index* __restrict__ ind, Index nnz,
                                        Index n, bool dense) {
  for (Index p = blockIdx.x*blockDim.x + threadIdx.x; p <= n; p += gridDim.x*blockDim.x) {
    if (dense) {
      out[p] = p;
      continue;
    }
    Index lo = 0, hi = nnz;
    while (lo < hi) {
      const Index mid = (lo + hi) >> 1;
      if (__ldg(ind + mid) < p) lo = mid + 1; else hi = mid;
    }
    out[p] = lo;
  }
}

// Eptr[I[p]] = length of op(A)'s row p (ptr == NULL: len, the constant form), for
// p < nI; Eptr zeroed by the caller, scanned after.
__global__ void assignRowLengthsKernel(Index* __restrict__ Eptr,
                                       const Index* __restrict__ rows,
                                       const Index* __restrict__ ptr, Index nI, Index len) {
  for (Index p = blockIdx.x*blockDim.x + threadIdx.x; p < nI; p += gridDim.x*blockDim.x)
    Eptr[asgAt(rows, p)] = ptr != NULL ? __ldg(ptr + p + 1) - __ldg(ptr + p) : len;
}

// op(A)'s entries into E.  Keys: (p << cbits | J[col], t) pairs to be sorted;
// otherwise E's column and value (and, with Eoval, the other orientation's value
// at the same slot) at their place.
template <typename T, bool Keys>
__global__ void assignEmbedKernel(Index* __restrict__ Eind, T* __restrict__ Eval,
                                  T* __restrict__ Eoval, const Index* __restrict__ Eptr,
                                  const Index* __restrict__ rows,
                                  const Index* __restrict__ cols,
                                  const Index* __restrict__ ptr,
                                  const Index* __restrict__ ind, const T* __restrict__ val,
                                  const T* __restrict__ oval, Index nI, Index nnz,
                                  int cbits, unsigned long long* __restrict__ keys,
                                  unsigned int* __restrict__ pay) {
  for (Index t = blockIdx.x*blockDim.x + threadIdx.x; t < nnz; t += gridDim.x*blockDim.x) {
    const Index p = asgRowOf(t, ptr, nI);
    const Index col = asgAt(cols, __ldg(ind + t));
    if (Keys) {
      keys[t] = (static_cast<unsigned long long>(p) << cbits) |
                static_cast<unsigned long long>(col);
      pay[t] = static_cast<unsigned int>(t);
    } else {
      const Index at = __ldg(Eptr + asgAt(rows, p)) + (t - __ldg(ptr + p));
      Eind[at] = col;
      Eval[at] = val[t];
      if (Eoval != NULL) Eoval[at] = oval[t];
    }
  }
}

// After the sort of the embed pairs: sorted pair t (of row p) lands at
// Eptr[I[p]] + t - ptr[p].
template <typename T>
__global__ void assignSortedEmbedKernel(Index* __restrict__ Eind, T* __restrict__ Eval,
                                        T* __restrict__ Eoval, const Index* __restrict__ Eptr,
                                        const Index* __restrict__ rows,
                                        const Index* __restrict__ ptr,
                                        const T* __restrict__ val, const T* __restrict__ oval,
                                        const unsigned long long* __restrict__ keys,
                                        const unsigned int* __restrict__ pay, Index nnz,
                                        int cbits) {
  const unsigned long long cmask = (1ull << cbits) - 1ull;
  for (Index t = blockIdx.x*blockDim.x + threadIdx.x; t < nnz; t += gridDim.x*blockDim.x) {
    const unsigned long long key = __ldg(keys + t);
    const Index p = static_cast<Index>(key >> cbits);
    const unsigned int s = __ldg(pay + t);
    const Index at = __ldg(Eptr + asgAt(rows, p)) + (t - __ldg(ptr + p));
    Eind[at] = static_cast<Index>(key & cmask);
    Eval[at] = val[s];
    if (Eoval != NULL) Eoval[at] = oval[s];
  }
}

// The constant form: selected row p holds the nJ columns of the sorted J (jsorted
// == NULL: 0 .. nJ-1), every value val (and Eoval's too, when given).
template <typename T, typename JT>
__global__ void assignConstKernel(Index* __restrict__ Eind, T* __restrict__ Eval,
                                  T* __restrict__ Eoval, const Index* __restrict__ Eptr,
                                  const Index* __restrict__ rows,
                                  const JT* __restrict__ jsorted, Index nI, Index nJ,
                                  T val) {
  const long long total = static_cast<long long>(nI)*nJ;
  for (long long e = static_cast<long long>(blockIdx.x)*blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x)*blockDim.x) {
    const Index p = static_cast<Index>(e/nJ);
    const Index q = static_cast<Index>(e - static_cast<long long>(p)*nJ);
    const Index at = __ldg(Eptr + asgAt(rows, p)) + q;
    Eind[at] = jsorted != NULL ? static_cast<Index>(jsorted[q]) : q;
    Eval[at] = val;
    if (Eoval != NULL) Eoval[at] = val;
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_ASSIGN_CUH_
