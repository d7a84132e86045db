// graphblast_b200 backend — element-wise union (eWiseAdd) and intersection
// (eWiseMult) of two sparse matrices, C = op(A) ⊕ op(B) / op(A) ⊗ op(B).
//
// Row i of C merges the sorted column lists of row i of A and of B.  Rows are
// power-law on graphs (a hub row holds hundreds of thousands of entries), so the
// work is cut over the MERGED ITEM STREAM, not over rows: item d of the stream
// lies in the row i with S(i) <= d < S(i+1), S(i) = A_ptr[i] + B_ptr[i] (S is
// monotone), at offset d - S(i) of that row's merge.  A CTA takes a tile of
// GB_EWM_TILE consecutive items and each of its threads GB_EWM_IPT of them,
// whatever the row lengths; a thread finds its start with one binary search over
// S (between the rows its CTA spans) and one merge-path search of the two column
// lists of its row.  The merge takes A's entry first on equal columns, so a
// matched pair (equal column, same row) is always an A item directly followed by
// its B item, and each side sees the match locally:
//   A item: matched iff the head of B's list has its column (already loaded);
//   B item: matched iff the last A entry taken in this row has its column.
// A pair split by a tile or thread boundary is therefore seen once on each side.
//
// An item is EMITTED (becomes an entry of C) when
//   eWiseAdd : it is not a matched A item; a matched B item writes add(a, b),
//              with A's value first, any other item its own value unchanged;
//   eWiseMult: it is a matched B item, and writes mul(a, b).
// An unmatched A item is emitted only where keep(row, column) holds: eWiseAdd
// passes EwmKeepAll; assign (assign.cuh) drops C's entries inside the region it
// replaces, and passes its accum (or "take B's value") as add.
// C's entries are the emitted items in stream order, so an entry's position is
// the number of items emitted before it.  Two passes over the same tiles:
//   ewiseMatrixCountKernel: emitted items per tile (and their 64-bit total, the
//     one value the host reads), and per row (integer atomics on C's row
//     pointer array, which an exclusive scan turns into C's row offsets);
//   ewiseMatrixFillKernel : after a scan of the tile counts, re-merges each tile,
//     stages its entries in shared memory in order and stores them as one
//     coalesced run at the tile's base.
// No value is combined through an atomic, so two calls give identical bytes.
//
// Algorithmic bytes: count 4(m+1)·2 + 4(nnzA + nnzB); fill the same plus
// 4(nnzA + nnzB) values, 4(m+1) row offsets and 8·nnz(C) written.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_EWISE_MATRIX_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_EWISE_MATRIX_CUH_

#include "graphblas/backend/cuda/kernels/common.cuh"

namespace graphblas {
namespace backend {

#define GB_EWM_NT   128                       // threads per CTA
#define GB_EWM_IPT  16                        // merged items per thread
#define GB_EWM_TILE (GB_EWM_NT*GB_EWM_IPT)    // merged items per CTA
#define GB_EWM_END  0x7fffffff                // column past the end of a row's list

// S(i): merged items in the rows before i.
__device__ __forceinline__ long long ewmStart(const Index* __restrict__ A_ptr,
                                              const Index* __restrict__ B_ptr, Index i) {
  return static_cast<long long>(__ldg(A_ptr + i)) + __ldg(B_ptr + i);
}

// Largest i in [lo, hi] with S(i) <= d (S(lo) <= d): the row holding item d.
__device__ __forceinline__ Index ewmRowOf(long long d, const Index* __restrict__ A_ptr,
                                          const Index* __restrict__ B_ptr, Index lo,
                                          Index hi) {
  while (lo < hi) {
    const Index mid = lo + (hi - lo + 1)/2;
    if (ewmStart(A_ptr, B_ptr, mid) <= d) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Merge state of one thread: the row, the next entry of each list and its
// column (GB_EWM_END past the row's end), and the column of the last A entry
// taken in this row (-1 when none).
struct EwmCursor {
  Index r;
  Index a, a_end, ca;
  Index b, b_end, cb;
  Index last_a;
};

__device__ __forceinline__ void ewmEnterRow(EwmCursor& q, Index r,
    const Index* __restrict__ A_ptr, const Index* __restrict__ A_ind,
    const Index* __restrict__ B_ptr, const Index* __restrict__ B_ind) {
  q.r = r;
  q.a = __ldg(A_ptr + r);  q.a_end = __ldg(A_ptr + r + 1);
  q.b = __ldg(B_ptr + r);  q.b_end = __ldg(B_ptr + r + 1);
  q.ca = q.a < q.a_end ? __ldg(A_ind + q.a) : GB_EWM_END;
  q.cb = q.b < q.b_end ? __ldg(B_ind + q.b) : GB_EWM_END;
  q.last_a = -1;
}

// Cursor on merged item d (< total) of row r.
__device__ __forceinline__ void ewmSeek(EwmCursor& q, long long d, Index r,
    const Index* __restrict__ A_ptr, const Index* __restrict__ A_ind,
    const Index* __restrict__ B_ptr, const Index* __restrict__ B_ind) {
  const Index a0 = __ldg(A_ptr + r), b0 = __ldg(B_ptr + r);
  const Index a1 = __ldg(A_ptr + r + 1), b1 = __ldg(B_ptr + r + 1);
  const Index k = static_cast<Index>(d - (static_cast<long long>(a0) + b0));
  // x = A entries among the row's first k merged items (A first on ties)
  Index lo = k - (b1 - b0) > 0 ? k - (b1 - b0) : 0;
  Index hi = k < a1 - a0 ? k : a1 - a0;
  while (lo < hi) {
    const Index mid = (lo + hi) >> 1;
    if (__ldg(A_ind + a0 + mid) <= __ldg(B_ind + b0 + k - 1 - mid)) lo = mid + 1;
    else hi = mid;
  }
  q.r = r;
  q.a = a0 + lo;      q.a_end = a1;
  q.b = b0 + k - lo;  q.b_end = b1;
  q.ca = q.a < a1 ? __ldg(A_ind + q.a) : GB_EWM_END;
  q.cb = q.b < b1 ? __ldg(B_ind + q.b) : GB_EWM_END;
  q.last_a = q.a > a0 ? __ldg(A_ind + q.a - 1) : -1;
}

// Before taking item p: if the row is used up, move to the row holding p
// (usually the next one; a run of empty rows costs one binary search).
__device__ __forceinline__ bool ewmNextRowIfDone(EwmCursor& q, long long p, Index r_hi,
    const Index* __restrict__ A_ptr, const Index* __restrict__ A_ind,
    const Index* __restrict__ B_ptr, const Index* __restrict__ B_ind) {
  if (q.a < q.a_end || q.b < q.b_end) return false;
  Index r = q.r + 1;
  if (ewmStart(A_ptr, B_ptr, r + 1) <= p) r = ewmRowOf(p, A_ptr, B_ptr, r + 1, r_hi);
  ewmEnterRow(q, r, A_ptr, A_ind, B_ptr, B_ind);
  return true;
}

// Row span of the CTA's tile [d0, d1) into shared memory.
__device__ __forceinline__ void ewmTileRows(long long d0, long long d1, Index nrows,
    const Index* __restrict__ A_ptr, const Index* __restrict__ B_ptr, Index* s_rows) {
  if (threadIdx.x == 0) {
    const Index lo = ewmRowOf(d0, A_ptr, B_ptr, 0, nrows - 1);
    s_rows[0] = lo;
    s_rows[1] = ewmRowOf(d1 - 1, A_ptr, B_ptr, lo, nrows - 1);
  }
  __syncthreads();
}

// The keep test of the eWise operations: every unmatched A item is emitted.
struct EwmKeepAll {
  __device__ __forceinline__ bool operator()(Index, Index) const { return true; }
};

// Emitted items per tile (tile_count[t]), per row (atomics into row_count, zeroed
// by the caller) and in all (*total, 64-bit).
template <bool IsAdd, typename Keep>
__global__ void __launch_bounds__(GB_EWM_NT)
ewiseMatrixCountKernel(const Index* __restrict__ A_ptr, const Index* __restrict__ A_ind,
                       const Index* __restrict__ B_ptr, const Index* __restrict__ B_ind,
                       Index nrows, long long total, int* __restrict__ tile_count,
                       int* __restrict__ row_count,
                       unsigned long long* __restrict__ total_count, Keep keep) {
  __shared__ Index s_rows[2];
  __shared__ int s_sum[GB_EWM_NT/32];
  const long long d0 = static_cast<long long>(blockIdx.x)*GB_EWM_TILE;
  const long long d1 = d0 + GB_EWM_TILE < total ? d0 + GB_EWM_TILE : total;
  ewmTileRows(d0, d1, nrows, A_ptr, B_ptr, s_rows);
  const Index r_lo = s_rows[0], r_hi = s_rows[1];

  long long p = d0 + static_cast<long long>(threadIdx.x)*GB_EWM_IPT;
  const long long p_end = p + GB_EWM_IPT < d1 ? p + GB_EWM_IPT : d1;
  int mine = 0;
  if (p < p_end) {
    EwmCursor q;
    ewmSeek(q, p, ewmRowOf(p, A_ptr, B_ptr, r_lo, r_hi), A_ptr, A_ind, B_ptr, B_ind);
    int in_row = 0;                               // emitted in row q.r so far
    for (; p < p_end; ++p) {
      const Index r = q.r;
      if (ewmNextRowIfDone(q, p, r_hi, A_ptr, A_ind, B_ptr, B_ind) && in_row > 0) {
        atomicAdd(row_count + r, in_row);
        mine += in_row;
        in_row = 0;
      }
      if (q.ca <= q.cb) {                         // A item
        if (IsAdd && q.cb != q.ca && keep(q.r, q.ca)) ++in_row;
        q.last_a = q.ca;
        ++q.a;
        q.ca = q.a < q.a_end ? __ldg(A_ind + q.a) : GB_EWM_END;
      } else {                                    // B item
        if (IsAdd || q.last_a == q.cb) ++in_row;
        ++q.b;
        q.cb = q.b < q.b_end ? __ldg(B_ind + q.b) : GB_EWM_END;
      }
    }
    if (in_row > 0) atomicAdd(row_count + q.r, in_row);
    mine += in_row;
  }
  const int tile = blockSum<GB_EWM_NT>(mine, s_sum);
  if (threadIdx.x == 0) {
    tile_count[blockIdx.x] = tile;
    if (tile > 0) atomicAdd(total_count, static_cast<unsigned long long>(tile));
  }
}

// C's colind / val: every tile re-merged, its emitted items written from
// tile_base[t] on (exclusive scan of the count pass's tile counts).  An item's
// column and value stay in registers between the merge and the staging.
template <bool IsAdd, typename c, typename a, typename b, typename MulOp,
          typename AddOp, typename Keep>
__global__ void __launch_bounds__(GB_EWM_NT)
ewiseMatrixFillKernel(const Index* __restrict__ A_ptr, const Index* __restrict__ A_ind,
                      const a* __restrict__ A_val, const Index* __restrict__ B_ptr,
                      const Index* __restrict__ B_ind, const b* __restrict__ B_val,
                      Index nrows, long long total, const int* __restrict__ tile_base,
                      Index* __restrict__ C_ind, c* __restrict__ C_val, MulOp mul_op,
                      AddOp add_op, Keep keep) {
  __shared__ Index s_rows[2];
  __shared__ int s_scan[GB_EWM_NT/32 + 1];
  const long long d0 = static_cast<long long>(blockIdx.x)*GB_EWM_TILE;
  const long long d1 = d0 + GB_EWM_TILE < total ? d0 + GB_EWM_TILE : total;
  ewmTileRows(d0, d1, nrows, A_ptr, B_ptr, s_rows);
  const Index r_lo = s_rows[0], r_hi = s_rows[1];

  const long long p0 = d0 + static_cast<long long>(threadIdx.x)*GB_EWM_IPT;
  const int n = p0 < d1 ? static_cast<int>(d1 - p0 < GB_EWM_IPT ? d1 - p0 : GB_EWM_IPT) : 0;
  Index col[GB_EWM_IPT];
  c val[GB_EWM_IPT];
  unsigned int emit = 0;
  if (n > 0) {
    EwmCursor q;
    ewmSeek(q, p0, ewmRowOf(p0, A_ptr, B_ptr, r_lo, r_hi), A_ptr, A_ind, B_ptr, B_ind);
#pragma unroll
    for (int j = 0; j < GB_EWM_IPT; ++j) {
      if (j < n) {
        ewmNextRowIfDone(q, p0 + j, r_hi, A_ptr, A_ind, B_ptr, B_ind);
        if (q.ca <= q.cb) {                       // A item
          if (IsAdd && q.cb != q.ca && keep(q.r, q.ca)) {
            col[j] = q.ca;
            val[j] = static_cast<c>(A_val[q.a]);
            emit |= 1u << j;
          }
          q.last_a = q.ca;
          ++q.a;
          q.ca = q.a < q.a_end ? __ldg(A_ind + q.a) : GB_EWM_END;
        } else {                                  // B item
          const bool matched = q.last_a == q.cb;
          if (IsAdd || matched) {
            col[j] = q.cb;
            if (IsAdd && !matched)
              val[j] = static_cast<c>(B_val[q.b]);
            else if (IsAdd)
              val[j] = static_cast<c>(add_op(static_cast<c>(A_val[q.a - 1]),
                                             static_cast<c>(B_val[q.b])));
            else
              val[j] = static_cast<c>(mul_op(static_cast<c>(A_val[q.a - 1]),
                                             static_cast<c>(B_val[q.b])));
            emit |= 1u << j;
          }
          ++q.b;
          q.cb = q.b < q.b_end ? __ldg(B_ind + q.b) : GB_EWM_END;
        }
      }
    }
  }
  // the tile's entries are one contiguous run of C: staged in shared memory in
  // order, then stored by consecutive threads
  __shared__ Index s_ind[GB_EWM_TILE];
  __shared__ c s_val[GB_EWM_TILE];
  int tile;
  int at = blockExclusiveScan<GB_EWM_NT>(__popc(emit), s_scan, &tile);
#pragma unroll
  for (int j = 0; j < GB_EWM_IPT; ++j) {
    if (emit & (1u << j)) {
      s_ind[at] = col[j];
      s_val[at] = val[j];
      ++at;
    }
  }
  __syncthreads();
  const long long base = tile_base[blockIdx.x];
  for (int k = threadIdx.x; k < tile; k += GB_EWM_NT) {
    C_ind[base + k] = s_ind[k];
    C_val[base + k] = s_val[k];
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_EWISE_MATRIX_CUH_
