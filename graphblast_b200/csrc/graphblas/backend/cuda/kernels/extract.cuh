// graphblast_b200 backend — extract: C = S(I, J) of one stored orientation S
// (A's CSR, or its CSC for Aᵀ), the kernels behind extract.hpp.
//
// The selected rows I[0..nsel) form a VIRTUAL CSR over S's entries: selected row
// i holds S's row I[i], and sel[i] (an exclusive scan of the selected lengths) is
// where it starts in the stream of selected entries.  Rows are skewed on graphs
// (R-MAT hubs), so the work is cut over that stream, not over rows: a CTA takes a
// tile of GB_EXT_TILE consecutive selected entries and each thread GB_EXT_IPT of
// them, whatever the row lengths; a thread finds its first row with one binary
// search over sel (between the rows its CTA spans).
//
// Column map (J given): jptr[k]..jptr[k+1] are the positions of S's column k in
// J, ascending, listed in jpos.  An entry in column k becomes jptr[k+1] - jptr[k]
// entries of C, at C columns jpos[jptr[k]..jptr[k+1]).  Two passes, as in
// ewise_matrix.cuh:
//   extractCountKernel: C entries per tile, per selected row (integer atomics on
//     C's row pointer array, scanned into C's row offsets) and in all (64-bit,
//     the one value the host reads);
//   extractFillKernel : after a scan of the tile counts, writes each tile's
//     entries from its base, in stream order.
// Without a map (J = ALL) every entry is one entry of C at its own stream
// position: no count pass, and the fill is a segmented copy.
//
// Stream order is S's column order inside a row, then the map's positions.  When
// J is non-decreasing that is ascending C column order.  Otherwise the fill writes
// (row << pbits | column, source slot) pairs instead, the caller sorts them with
// radixSortPairs and extractSortedStoreKernel writes C's columns and values.
// No value goes through an atomic, so two calls give identical bytes.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_EXTRACT_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_EXTRACT_CUH_

#include "graphblas/backend/cuda/kernels/common.cuh"

namespace graphblas {
namespace backend {

#define GB_EXT_NT   128                       // threads per CTA
#define GB_EXT_IPT  8                         // selected entries per thread
#define GB_EXT_TILE (GB_EXT_NT*GB_EXT_IPT)    // selected entries per CTA

// Source row of selected row i (rows == NULL: every row, in order).
__device__ __forceinline__ Index extSource(const Index* __restrict__ rows, Index i) {
  return rows != NULL ? __ldg(rows + i) : i;
}

// Largest i in [lo, hi] with sel[i] <= e (sel[lo] <= e): the selected row holding e.
__device__ __forceinline__ Index extRowOf(long long e, const Index* __restrict__ sel,
                                          Index lo, Index hi) {
  while (lo < hi) {
    const Index mid = lo + (hi - lo + 1)/2;
    if (__ldg(sel + mid) <= e) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Cursor of one thread: the selected row, where it ends in the stream, and the
// slot in S of the next entry.
struct ExtCursor {
  Index i, end, slot;
};

__device__ __forceinline__ void extSeek(ExtCursor& q, long long e, Index i,
    const Index* __restrict__ sel, const Index* __restrict__ rows,
    const Index* __restrict__ ptr) {
  q.i = i;
  q.end = __ldg(sel + i + 1);
  q.slot = __ldg(ptr + extSource(rows, i)) + static_cast<Index>(e - __ldg(sel + i));
}

// Before taking entry e: if the row is used up, move to the row holding e
// (usually the next one; a run of empty rows costs one binary search).
__device__ __forceinline__ bool extNextRowIfDone(ExtCursor& q, long long e, Index r_hi,
    const Index* __restrict__ sel, const Index* __restrict__ rows,
    const Index* __restrict__ ptr) {
  if (e < q.end) return false;
  Index i = q.i + 1;
  if (__ldg(sel + i + 1) <= e) i = extRowOf(e, sel, i + 1, r_hi);
  extSeek(q, e, i, sel, rows, ptr);
  return true;
}

// Row span of the CTA's tile [e0, e1) into shared memory.
__device__ __forceinline__ void extTileRows(long long e0, long long e1, Index nsel,
    const Index* __restrict__ sel, Index* s_rows) {
  if (threadIdx.x == 0) {
    const Index lo = extRowOf(e0, sel, 0, nsel - 1);
    s_rows[0] = lo;
    s_rows[1] = extRowOf(e1 - 1, sel, lo, nsel - 1);
  }
  __syncthreads();
}

// CTA sum of a 64-bit count, valid in thread 0.  NT multiple of 32.
template <int NT>
__device__ __forceinline__ unsigned long long extBlockSum64(unsigned long long v,
                                                            unsigned long long* smem) {
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(GB_FULL_MASK, v, off);
  if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned long long total = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < NT/32; ++w) total += smem[w];
  return total;
}

// sel[i] = length of S's row I[i] (i < nsel), sel[nsel] = 0; *total += their sum
// (64-bit: duplicates in I can select more entries than S holds).
__global__ void __launch_bounds__(256)
extractRowLengthsKernel(Index* __restrict__ sel, const Index* __restrict__ rows,
                        const Index* __restrict__ ptr, Index nsel,
                        unsigned long long* __restrict__ total) {
  __shared__ unsigned long long s_sum[256/32];
  unsigned long long mine = 0;
  for (Index i = blockIdx.x*blockDim.x + threadIdx.x; i <= nsel; i += gridDim.x*blockDim.x) {
    Index len = 0;
    if (i < nsel) {
      const Index r = extSource(rows, i);
      len = __ldg(ptr + r + 1) - __ldg(ptr + r);
    }
    sel[i] = len;
    mine += static_cast<unsigned long long>(len);
  }
  const unsigned long long cta = extBlockSum64<256>(mine, s_sum);
  if (threadIdx.x == 0 && cta > 0) atomicAdd(total, cta);
}

// jptr[k] = first position of column k in the sorted keys (k <= ncols): the
// bucket bounds of the column map.
__global__ void extractMapBoundsKernel(Index* __restrict__ jptr,
                                       const unsigned long long* __restrict__ keys,
                                       Index nkeys, Index ncols) {
  for (Index k = blockIdx.x*blockDim.x + threadIdx.x; k <= ncols; k += gridDim.x*blockDim.x) {
    Index lo = 0, hi = nkeys;
    while (lo < hi) {
      const Index mid = (lo + hi) >> 1;
      if (__ldg(keys + mid) < static_cast<unsigned long long>(k)) lo = mid + 1; else hi = mid;
    }
    jptr[k] = lo;
  }
}

// keys[p] = J[p], pay[p] = p: the pairs whose stable sort by key gives jpos.
__global__ void extractMapKeysKernel(unsigned long long* __restrict__ keys,
                                     unsigned int* __restrict__ pay,
                                     const Index* __restrict__ cols, Index ncut) {
  for (Index p = blockIdx.x*blockDim.x + threadIdx.x; p < ncut; p += gridDim.x*blockDim.x) {
    keys[p] = static_cast<unsigned long long>(__ldg(cols + p));
    pay[p] = static_cast<unsigned int>(p);
  }
}

// C entries per tile (tile_count[t]), per selected row (atomics into row_count,
// zeroed by the caller) and in all (*total_count, 64-bit).
__global__ void __launch_bounds__(GB_EXT_NT)
extractCountKernel(const Index* __restrict__ sel, const Index* __restrict__ rows,
                   const Index* __restrict__ ptr, const Index* __restrict__ ind,
                   const Index* __restrict__ jptr, Index nsel, long long total,
                   int* __restrict__ tile_count, int* __restrict__ row_count,
                   unsigned long long* __restrict__ total_count) {
  __shared__ Index s_rows[2];
  __shared__ unsigned long long s_sum[GB_EXT_NT/32];
  const long long e0 = static_cast<long long>(blockIdx.x)*GB_EXT_TILE;
  const long long e1 = e0 + GB_EXT_TILE < total ? e0 + GB_EXT_TILE : total;
  extTileRows(e0, e1, nsel, sel, s_rows);
  const Index r_lo = s_rows[0], r_hi = s_rows[1];

  long long e = e0 + static_cast<long long>(threadIdx.x)*GB_EXT_IPT;
  const long long e_end = e + GB_EXT_IPT < e1 ? e + GB_EXT_IPT : e1;
  unsigned long long mine = 0;
  if (e < e_end) {
    ExtCursor q;
    extSeek(q, e, extRowOf(e, sel, r_lo, r_hi), sel, rows, ptr);
    long long in_row = 0;                         // C entries of row q.i so far
    for (; e < e_end; ++e) {
      const Index i = q.i;
      if (extNextRowIfDone(q, e, r_hi, sel, rows, ptr) && in_row > 0) {
        atomicAdd(row_count + i, static_cast<int>(in_row));
        mine += in_row;
        in_row = 0;
      }
      const Index k = __ldg(ind + q.slot);
      in_row += __ldg(jptr + k + 1) - __ldg(jptr + k);
      ++q.slot;
    }
    if (in_row > 0) atomicAdd(row_count + q.i, static_cast<int>(in_row));
    mine += in_row;
  }
  // CTA sum in 64 bits: one entry can stand for every position of J
  const unsigned long long tile = extBlockSum64<GB_EXT_NT>(mine, s_sum);
  if (threadIdx.x == 0) {
    // a tile past 2^31 - 1 entries means C is too; the caller refuses it
    tile_count[blockIdx.x] = static_cast<int>(tile);
    if (tile > 0) atomicAdd(total_count, tile);
  }
}

// C's entries of one tile, in stream order.  Map: tile_base[t] (the scanned tile
// counts) is where the tile's entries start, and each thread's share follows from
// a CTA scan; without a map entry e is C's entry e.  Keys: (row << pbits | column,
// slot in S) pairs to be sorted; otherwise C's column, its value and, with
// C_oval, the value of the other orientation at the same slot.
template <bool Map, bool Keys, typename T>
__global__ void __launch_bounds__(GB_EXT_NT)
extractFillKernel(const Index* __restrict__ sel, const Index* __restrict__ rows,
                  const Index* __restrict__ ptr, const Index* __restrict__ ind,
                  const T* __restrict__ val, const T* __restrict__ oval,
                  const Index* __restrict__ jptr, const Index* __restrict__ jpos,
                  Index nsel, long long total, const int* __restrict__ tile_base,
                  int pbits, Index* __restrict__ C_ind, T* __restrict__ C_val,
                  T* __restrict__ C_oval, unsigned long long* __restrict__ keys,
                  unsigned int* __restrict__ pay) {
  __shared__ Index s_rows[2];
  __shared__ int s_scan[GB_EXT_NT/32 + 1];
  const long long e0 = static_cast<long long>(blockIdx.x)*GB_EXT_TILE;
  const long long e1 = e0 + GB_EXT_TILE < total ? e0 + GB_EXT_TILE : total;
  extTileRows(e0, e1, nsel, sel, s_rows);
  const Index r_lo = s_rows[0], r_hi = s_rows[1];

  const long long p0 = e0 + static_cast<long long>(threadIdx.x)*GB_EXT_IPT;
  const int n = p0 < e1 ? static_cast<int>(e1 - p0 < GB_EXT_IPT ? e1 - p0 : GB_EXT_IPT) : 0;
  // every thread's ranges start empty: one past the tile's end writes nothing
  Index slot[GB_EXT_IPT], row[GB_EXT_IPT], lo[GB_EXT_IPT], hi[GB_EXT_IPT];
#pragma unroll
  for (int j = 0; j < GB_EXT_IPT; ++j) lo[j] = hi[j] = 0;
  int mine = 0;
  if (n > 0) {
    ExtCursor q;
    extSeek(q, p0, extRowOf(p0, sel, r_lo, r_hi), sel, rows, ptr);
#pragma unroll
    for (int j = 0; j < GB_EXT_IPT; ++j) {
      if (j < n) {
        extNextRowIfDone(q, p0 + j, r_hi, sel, rows, ptr);
        slot[j] = q.slot++;
        row[j] = q.i;
        const Index k = __ldg(ind + slot[j]);
        if (Map) {
          lo[j] = __ldg(jptr + k);
          hi[j] = __ldg(jptr + k + 1);
        } else {
          lo[j] = k;                              // the column itself
          hi[j] = k + 1;
        }
        mine += hi[j] - lo[j];
      }
    }
  }
  long long at = p0;
  if (Map) {
    int tile;
    at = tile_base[blockIdx.x] + blockExclusiveScan<GB_EXT_NT>(mine, s_scan, &tile);
  }
#pragma unroll
  for (int j = 0; j < GB_EXT_IPT; ++j) {
    for (Index m = lo[j]; m < hi[j]; ++m, ++at) {
      const Index p = Map ? __ldg(jpos + m) : m;
      if (Keys) {
        keys[at] = (static_cast<unsigned long long>(row[j]) << pbits) |
                   static_cast<unsigned long long>(p);
        pay[at] = static_cast<unsigned int>(slot[j]);
      } else {
        C_ind[at] = p;
        C_val[at] = val[slot[j]];
        if (C_oval != NULL) C_oval[at] = oval[slot[j]];
      }
    }
  }
}

// After the sort of the fill's pairs: C's column, value and other-orientation
// value of entry t.
template <typename T>
__global__ void extractSortedStoreKernel(Index* __restrict__ C_ind, T* __restrict__ C_val,
                                         T* __restrict__ C_oval,
                                         const unsigned long long* __restrict__ keys,
                                         const unsigned int* __restrict__ pay,
                                         const T* __restrict__ val,
                                         const T* __restrict__ oval, Index nnz, int pbits) {
  const unsigned long long pmask = (1ull << pbits) - 1ull;
  for (Index t = blockIdx.x*blockDim.x + threadIdx.x; t < nnz; t += gridDim.x*blockDim.x) {
    const unsigned int s = __ldg(pay + t);
    C_ind[t] = static_cast<Index>(__ldg(keys + t) & pmask);
    C_val[t] = val[s];
    if (C_oval != NULL) C_oval[t] = oval[s];
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_EXTRACT_CUH_
