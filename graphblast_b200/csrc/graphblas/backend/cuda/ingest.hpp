// graphblast_b200 backend — graph ingest on the device: edge tuples -> CSR / CSC
// with the semantics of the reference's HOST loader (graphblas/util.hpp:264-329
// removeSelfloop + customSort, :502-600 coo2csr / coo2csc / csr2csc):
//   * optionally add the reverse of every non-loop tuple (undirected graphs);
//     the reverse copies follow ALL forward tuples in input order, as in the
//     reference, so "first duplicate wins" picks the same tuple;
//   * sort by (row, col) — here a stable LSD radix sort of packed 64-bit keys
//     (kernels/radix_sort.cuh) instead of std::sort over a vector of tuples;
//   * optionally drop self-loops and repeated (row, col) pairs;
//   * rows of the CSR sorted by column, values follow their tuple.
// SURVEY.md §8 row f1.  Everything runs on the backend stream; the only host
// round trips are the two totals (valid tuples, stored entries).
#ifndef GRAPHBLAS_BACKEND_CUDA_INGEST_HPP_
#define GRAPHBLAS_BACKEND_CUDA_INGEST_HPP_

#include "graphblas/backend/cuda/util.hpp"
#include "graphblas/backend/cuda/kernels/radix_sort.cuh"

namespace graphblas {
namespace backend {

enum IngestFlags {
  GB_INGEST_SYMMETRIZE = 1,     // add (col, row) for every tuple with row != col
  GB_INGEST_DROP_LOOPS = 2,     // drop tuples with row == col
  GB_INGEST_DEDUP      = 4      // keep the first of equal (row, col) tuples
};

inline int ingestBitsFor(Index extent) {        // bits that hold 0 .. extent-1
  int b = 1;
  while (b < 31 && (static_cast<long long>(1) << b) < static_cast<long long>(extent)) ++b;
  return b;
}

// ---- scan / sort drivers -------------------------------------------------------

// In-place exclusive scan of n ints, stream-ordered, no host read; *grand (device,
// may be NULL) receives the total.
inline void scanExclusiveAsync(int* data, long long n, unsigned long long* grand) {
  if (n <= 0) return;
  cudaStream_t s = gbStream();
  const int ntiles = static_cast<int>((n + GB_SCAN_TILE - 1)/GB_SCAN_TILE);
  int* totals = reinterpret_cast<int*>(gbMalloc((static_cast<size_t>(ntiles) + 1)*sizeof(int)));
  scanTileKernel<<<ntiles, GB_SCAN_NT, 0, s>>>(data, totals, n);
  GB_KERNEL_CHECK();
  scanTotalsKernel<<<1, GB_SCAN_NT, 0, s>>>(totals, ntiles, grand);
  GB_KERNEL_CHECK();
  if (ntiles > 1) {
    scanAddKernel<<<ntiles, GB_SCAN_NT, 0, s>>>(data, totals, n);
    GB_KERNEL_CHECK();
  }
  gbFree(totals);
}

// In-place exclusive scan of n ints; returns the grand total (one host read).
inline unsigned long long scanExclusiveInPlace(int* data, long long n) {
  if (n <= 0) return 0ull;
  unsigned long long* grand = reinterpret_cast<unsigned long long*>(
      gbMalloc(sizeof(unsigned long long)));
  scanExclusiveAsync(data, n, grand);
  const unsigned long long total = runtime().fetch(grand);
  gbFree(grand);
  return total;
}

// Stable sort of (key, payload) pairs by the low `bits` bits of the key.  The
// result ends up in (*keys, *pay); the buffers may have been swapped with the
// temporaries.  pay == NULL sorts keys only.
inline void radixSortPairs(unsigned long long** keys, unsigned int** pay,
                           unsigned long long** keys_tmp, unsigned int** pay_tmp,
                           long long n, int bits) {
  if (n <= 1) return;
  cudaStream_t s = gbStream();
  const int ntiles = static_cast<int>((n + GB_RADIX_TILE - 1)/GB_RADIX_TILE);
  const long long nhist = static_cast<long long>(GB_RADIX_BINS)*ntiles;
  int* hist = reinterpret_cast<int*>(gbMalloc(static_cast<size_t>(nhist)*sizeof(int)));
  const bool has_pay = (pay != NULL && *pay != NULL);
  for (int pos = 0; pos < bits; pos += 8) {
    const int width = bits - pos < 8 ? bits - pos : 8;
    const int shift = pos | (width << 8);        // see radixDigit
    radixHistogramKernel<<<ntiles, GB_RADIX_NT, 0, s>>>(hist, *keys, n, shift, ntiles);
    GB_KERNEL_CHECK();
    scanExclusiveInPlace(hist, nhist);
    if (has_pay)
      radixScatterKernel<true><<<ntiles, GB_RADIX_NT, 0, s>>>(*keys_tmp, *pay_tmp,
          *keys, *pay, hist, n, shift, ntiles);
    else
      radixScatterKernel<false><<<ntiles, GB_RADIX_NT, 0, s>>>(*keys_tmp, NULL,
          *keys, NULL, hist, n, shift, ntiles);
    GB_KERNEL_CHECK();
    std::swap(*keys, *keys_tmp);
    if (has_pay) std::swap(*pay, *pay_tmp);
  }
  gbFree(hist);
}

// ---- ingest kernels --------------------------------------------------------------

// flags[e] = forward tuple kept, flags[m + e] = reverse tuple generated
__global__ void ingestFlagKernel(int* __restrict__ flags,
                                 const Index* __restrict__ src,
                                 const Index* __restrict__ dst, long long m,
                                 Index nrows, Index ncols, int mode) {
  long long e = static_cast<long long>(blockIdx.x)*blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x)*blockDim.x;
  for (; e < m; e += stride) {
    const Index r = src[e], c = dst[e];
    const bool inside = r >= 0 && r < nrows && c >= 0 && c < ncols;
    const bool loop = (r == c);
    flags[e] = (inside && !(loop && (mode & GB_INGEST_DROP_LOOPS))) ? 1 : 0;
    if (mode & GB_INGEST_SYMMETRIZE)
      flags[m + e] = (inside && !loop && c < nrows && r < ncols) ? 1 : 0;
  }
}

// keys[slot] = row << cbits | col, pay[slot] = tuple index, at the scanned slots
__global__ void ingestEmitKernel(unsigned long long* __restrict__ keys,
                                 unsigned int* __restrict__ pay,
                                 const int* __restrict__ slots,
                                 const Index* __restrict__ src,
                                 const Index* __restrict__ dst, long long m,
                                 Index nrows, Index ncols, int mode, int cbits,
                                 long long nvalid) {
  long long e = static_cast<long long>(blockIdx.x)*blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x)*blockDim.x;
  for (; e < m; e += stride) {
    const Index r = src[e], c = dst[e];
    const bool inside = r >= 0 && r < nrows && c >= 0 && c < ncols;
    const bool loop = (r == c);
    if (inside && !(loop && (mode & GB_INGEST_DROP_LOOPS))) {
      const int at = slots[e];
      keys[at] = (static_cast<unsigned long long>(r) << cbits) |
                 static_cast<unsigned long long>(c);
      pay[at] = static_cast<unsigned int>(e);
    }
    if ((mode & GB_INGEST_SYMMETRIZE) && inside && !loop && c < nrows && r < ncols) {
      const int at = slots[m + e];
      keys[at] = (static_cast<unsigned long long>(c) << cbits) |
                 static_cast<unsigned long long>(r);
      pay[at] = static_cast<unsigned int>(e);
    }
  }
}

// flags[i] = 1 for the first of every run of equal keys (all ones without dedup)
__global__ void ingestUniqueFlagKernel(int* __restrict__ flags,
                                       const unsigned long long* __restrict__ keys,
                                       long long n, bool dedup) {
  long long i = static_cast<long long>(blockIdx.x)*blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x)*blockDim.x;
  for (; i < n; i += stride)
    flags[i] = (!dedup || i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

// Kept tuple i goes to position slots[i]: column, value, and (through its row and
// the row of the kept tuple before it) the row offsets of every row that starts at
// or before it.  last[0] = key of the last kept tuple, for the trailing rows.
template <typename T>
__global__ void ingestStoreKernel(Index* __restrict__ rowptr,
                                  Index* __restrict__ colind, T* __restrict__ val,
                                  const unsigned long long* __restrict__ keys,
                                  const unsigned int* __restrict__ pay,
                                  const int* __restrict__ slots,
                                  const T* __restrict__ tuple_val,
                                  long long n, bool dedup, int cbits,
                                  Index nrows, Index nnz) {
  long long i = static_cast<long long>(blockIdx.x)*blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x)*blockDim.x;
  const unsigned long long cmask = (1ull << cbits) - 1ull;
  for (; i < n; i += stride) {
    const unsigned long long k = keys[i];
    const bool first = (i == 0) || keys[i - 1] != k;
    const Index row = static_cast<Index>(k >> cbits);
    if (i == n - 1)                          // rows behind the last tuple are empty
      for (Index r = row + 1; r <= nrows; ++r) rowptr[r] = nnz;
    if (dedup && !first) continue;
    const Index at = slots[i];
    colind[at] = static_cast<Index>(k & cmask);
    val[at] = (tuple_val != NULL) ? tuple_val[pay[i]] : static_cast<T>(1);
    // rows (prev_row, row] start at `at`
    const Index prev_row = (i == 0) ? -1 : static_cast<Index>(keys[i - 1] >> cbits);
    for (Index r = prev_row + 1; r <= row; ++r) rowptr[r] = at;
  }
}

// keys[k] = col << rbits | row of stored entry k (row found by upper_bound), pay = k
__global__ void ingestTransposeKeysKernel(unsigned long long* __restrict__ keys,
                                          unsigned int* __restrict__ pay,
                                          const Index* __restrict__ rowptr,
                                          const Index* __restrict__ colind,
                                          Index nrows, Index nnz, int rbits) {
  Index k = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; k < nnz; k += stride) {
    Index lo = 0, hi = nrows - 1;            // smallest r with rowptr[r+1] > k
    while (lo < hi) {
      const Index mid = (lo + hi) >> 1;
      if (__ldg(rowptr + mid + 1) <= k) lo = mid + 1; else hi = mid;
    }
    keys[k] = (static_cast<unsigned long long>(colind[k]) << rbits) |
              static_cast<unsigned long long>(lo);
    pay[k] = static_cast<unsigned int>(k);
  }
}

template <typename T>
__global__ void ingestFillRowptrKernel(Index* __restrict__ rowptr, Index count, T v) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < count; i += stride) rowptr[i] = v;
}

// ---- drivers ---------------------------------------------------------------------

// Sorted (row-major) CSR from device-resident tuples.  Allocates rowptr
// [nrows+1], colind / val [max(nnz,1)] from the pool; returns nnz.
template <typename T>
Index ingestCooToCsr(Index nrows, Index ncols, const Index* d_src, const Index* d_dst,
                     const T* d_val, long long m, int mode,
                     Index** rowptr_out, Index** colind_out, T** val_out) {
  cudaStream_t s = gbStream();
  const bool sym = (mode & GB_INGEST_SYMMETRIZE) != 0;
  const long long cap = sym ? 2*m : m;
  Index* rowptr = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(nrows) + 1)*sizeof(Index)));
  *rowptr_out = rowptr;
  if (cap <= 0) {
    ingestFillRowptrKernel<<<gridFor(nrows + 1, 256), 256, 0, s>>>(rowptr, nrows + 1, 0);
    GB_KERNEL_CHECK();
    *colind_out = reinterpret_cast<Index*>(gbMalloc(sizeof(Index)));
    *val_out = reinterpret_cast<T*>(gbMalloc(sizeof(T)));
    return 0;
  }
  const int cbits = ingestBitsFor(ncols);
  const int rbits = ingestBitsFor(nrows);
  int* flags = reinterpret_cast<int*>(gbMalloc(static_cast<size_t>(cap)*sizeof(int)));
  ingestFlagKernel<<<gridFor(m, 256, 8), 256, 0, s>>>(flags, d_src, d_dst, m, nrows,
      ncols, mode);
  GB_KERNEL_CHECK();
  const long long nvalid = static_cast<long long>(scanExclusiveInPlace(flags, cap));
  const size_t nv = nvalid > 0 ? static_cast<size_t>(nvalid) : 1;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(gbMalloc(nv*8));
  unsigned long long* keys_tmp = reinterpret_cast<unsigned long long*>(gbMalloc(nv*8));
  unsigned int* pay = reinterpret_cast<unsigned int*>(gbMalloc(nv*4));
  unsigned int* pay_tmp = reinterpret_cast<unsigned int*>(gbMalloc(nv*4));
  ingestEmitKernel<<<gridFor(m, 256, 8), 256, 0, s>>>(keys, pay, flags, d_src, d_dst,
      m, nrows, ncols, mode, cbits, nvalid);
  GB_KERNEL_CHECK();
  gbFree(flags);
  radixSortPairs(&keys, &pay, &keys_tmp, &pay_tmp, nvalid, cbits + rbits);
  gbFree(keys_tmp);
  gbFree(pay_tmp);

  const bool dedup = (mode & GB_INGEST_DEDUP) != 0;
  int* slots = reinterpret_cast<int*>(gbMalloc(nv*sizeof(int)));
  Index nnz = 0;
  if (nvalid > 0) {
    ingestUniqueFlagKernel<<<gridFor(nvalid, 256, 8), 256, 0, s>>>(slots, keys, nvalid,
        dedup);
    GB_KERNEL_CHECK();
    nnz = static_cast<Index>(scanExclusiveInPlace(slots, nvalid));
  }
  const size_t nz = nnz > 0 ? static_cast<size_t>(nnz) : 1;
  Index* colind = reinterpret_cast<Index*>(gbMalloc(nz*sizeof(Index)));
  T* val = reinterpret_cast<T*>(gbMalloc(nz*sizeof(T)));
  if (nvalid > 0) {
    ingestStoreKernel<<<gridFor(nvalid, 256, 8), 256, 0, s>>>(rowptr, colind, val,
        keys, pay, slots, d_val, nvalid, dedup, cbits, nrows, nnz);
    GB_KERNEL_CHECK();
  } else {
    ingestFillRowptrKernel<<<gridFor(nrows + 1, 256), 256, 0, s>>>(rowptr, nrows + 1, 0);
    GB_KERNEL_CHECK();
  }
  gbFree(slots);
  gbFree(pay);
  gbFree(keys);
  *colind_out = colind;
  *val_out = val;
  return nnz;
}

// CSC of a CSR (a stable sort of the stored entries by column): colptr [ncols+1],
// rowind / cval [max(nnz,1)], rows sorted inside every column.  Any output
// pointer may be NULL when the caller does not need that array.
template <typename T>
void ingestCsrToCsc(Index nrows, Index ncols, Index nnz, const Index* rowptr,
                    const Index* colind, const T* val, Index** colptr_out,
                    Index** rowind_out, T** cval_out) {
  cudaStream_t s = gbStream();
  const size_t nz = nnz > 0 ? static_cast<size_t>(nnz) : 1;
  // Sort keys col << rbits | row with the entry index as payload, then store
  // through the tuple path's kernel (no dedup: the CSR has none).
  const int rbits = ingestBitsFor(nrows);
  const int cbits = ingestBitsFor(ncols);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(gbMalloc(nz*8));
  unsigned long long* keys_tmp = reinterpret_cast<unsigned long long*>(gbMalloc(nz*8));
  unsigned int* pay = reinterpret_cast<unsigned int*>(gbMalloc(nz*4));
  unsigned int* pay_tmp = reinterpret_cast<unsigned int*>(gbMalloc(nz*4));
  Index* colptr = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(ncols) + 1)*sizeof(Index)));
  Index* rowind = reinterpret_cast<Index*>(gbMalloc(nz*sizeof(Index)));
  T* cval = reinterpret_cast<T*>(gbMalloc(nz*sizeof(T)));
  if (nnz > 0) {
    ingestTransposeKeysKernel<<<gridFor(nnz, 256, 8), 256, 0, s>>>(keys, pay, rowptr,
        colind, nrows, nnz, rbits);
    GB_KERNEL_CHECK();
    radixSortPairs(&keys, &pay, &keys_tmp, &pay_tmp, nnz, rbits + cbits);
    int* slots = reinterpret_cast<int*>(gbMalloc(nz*sizeof(int)));
    ingestUniqueFlagKernel<<<gridFor(nnz, 256, 8), 256, 0, s>>>(slots, keys, nnz, false);
    GB_KERNEL_CHECK();
    scanExclusiveInPlace(slots, nnz);
    ingestStoreKernel<<<gridFor(nnz, 256, 8), 256, 0, s>>>(colptr, rowind, cval, keys,
        pay, slots, val, nnz, false, rbits, ncols, nnz);
    GB_KERNEL_CHECK();
    gbFree(slots);
  } else {
    ingestFillRowptrKernel<<<gridFor(ncols + 1, 256), 256, 0, s>>>(colptr, ncols + 1, 0);
    GB_KERNEL_CHECK();
  }
  gbFree(pay_tmp); gbFree(pay); gbFree(keys_tmp); gbFree(keys);
  if (colptr_out != NULL) *colptr_out = colptr; else gbFree(colptr);
  if (rowind_out != NULL) *rowind_out = rowind; else gbFree(rowind);
  if (cval_out != NULL) *cval_out = cval; else gbFree(cval);
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_INGEST_HPP_
