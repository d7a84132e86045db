// graphblast_b200 backend — SpMM C = op(A) (+.x) B: A sparse (CSR rows, or the
// CSC under GrB_INP0 = GrB_TRAN), B (k x N) and C (m x N) dense, row-major, fp32.
//
// Load balance follows the merge-path SpMV (spmv_pull.cuh): the rows and entries
// of A are cut into tiles of GB_SPMV_TILE merge items by the same cached partition
// (spmvMergePartitionKernel), so a hub row spreads over as many tiles as its length
// asks for.  One CTA takes one tile and one slice of at most GB_SPMM_COL_TILE
// columns (gridDim.y).  Inside the CTA, groups of L lanes split the tile's items
// evenly; each lane of a group holds 4 columns of the slice in registers:
//   N <= GB_SPMM_GROUP_N    L = the power of two >= ceil(N/4): several groups, and
//                           so several rows or segments, per warp;
//   N <= GB_SPMM_COL_TILE   L = 32: a warp per segment, one column slice;
//   N >  GB_SPMM_COL_TILE   L = 32, the columns tiled over gridDim.y.
// With N % 4 == 0 a lane's 4 columns are adjacent and go through 16-byte loads and
// stores when B and C are 16-byte aligned (scalar loads of the same columns
// otherwise); with any other N they are 4 columns L apart.  The group layout, and
// with it every fold order, depends on N alone, never on alignment.
//
// Folds: a group folds each row piece in ascending entry order from the identity.
// A row that ends inside a group but started in an earlier one (its "head") is
// folded after the tails of the earlier groups of the CTA, left to right; the open
// row at the end of the tile leaves a carry of N values per tile, and
// spmmCarryFixupKernel folds runs of carries of one row, in tile order, on the left
// of that row's stored value.  No atomics: each output's order depends only on
// (A's structure, N), and two calls give identical bytes.
//
// Bytes of one call (compulsory): 4(m+1) rowptr + 8 nnz colind/val + 4 k N read
// of B + 4 m N written; the gathers move 4 nnz N, served mostly from L2.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_SPMM_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_SPMM_CUH_

#include "graphblas/backend/cuda/kernels/common.cuh"
#include "graphblas/backend/cuda/kernels/spmv_pull.cuh"

namespace graphblas {
namespace backend {

#define GB_SPMM_NT       128   // threads per CTA
#define GB_SPMM_GROUP_N  64    // widest N that still shares a warp between groups
#define GB_SPMM_COL_TILE 128   // columns per CTA (32 lanes x 4)
#define GB_SPMM_UNROLL   4     // entries whose B rows are loaded together
// Resident CTAs per SM the registers must allow (64 per thread).  Left to itself
// ptxas stays under 64 anyway but spills a few values to do so.
#define GB_SPMM_MINB     8

static_assert(GB_SPMV_TILE % GB_SPMM_NT == 0, "every group count divides the tile");

// Lanes per group for N columns (host and tests agree on this rule).
inline int spmmLanes(long long ncols) {
  if (ncols > GB_SPMM_GROUP_N) return 32;
  const long long chunks = (ncols + 3)/4;
  int lanes = 1;
  while (lanes < chunks) lanes <<= 1;
  return lanes;
}

// Column layout of one lane: ADJ = the 4 columns are adjacent (N % 4 == 0),
// otherwise `lanes` apart.
template <bool ADJ>
struct SpmmCols {
  int first, lanes, end;
  __device__ __forceinline__ int off(int q) const { return ADJ ? first + q : first + q*lanes; }
  __device__ __forceinline__ bool ok(int q) const { return off(q) < end; }
};

template <bool ADJ, bool VEC, typename W>
__device__ __forceinline__ void spmmLoad(W (&x)[4], const W* __restrict__ row,
                                         const SpmmCols<ADJ>& cols, W fill) {
  if (VEC) {
    if (cols.ok(0)) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(row + cols.off(0)));
      x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w;
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) x[q] = fill;
    }
  } else {
#pragma unroll
    for (int q = 0; q < 4; ++q) x[q] = cols.ok(q) ? __ldg(row + cols.off(q)) : fill;
  }
}

template <bool ADJ, bool VEC, typename W>
__device__ __forceinline__ void spmmStore(W* __restrict__ row, const SpmmCols<ADJ>& cols,
                                          const W (&x)[4]) {
  if (VEC) {
    if (cols.ok(0))
      *reinterpret_cast<float4*>(row + cols.off(0)) = make_float4(x[0], x[1], x[2], x[3]);
  } else {
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (cols.ok(q)) row[cols.off(q)] = x[q];
  }
}

// acc (+)= A(k) (x) B(col(k), cols) for k in [k, stop), ascending.
template <bool ADJ, bool VEC, typename W, typename a, typename MulOp, typename AddOp>
__device__ __forceinline__ void spmmFold(W (&acc)[4], Index k, Index stop,
    const Index* __restrict__ colind, const a* __restrict__ val,
    const W* __restrict__ B, int ncols, const SpmmCols<ADJ>& cols, W identity,
    MulOp mul_op, AddOp add_op) {
  for (; k + GB_SPMM_UNROLL <= stop; k += GB_SPMM_UNROLL) {
    Index col[GB_SPMM_UNROLL];
    a     av[GB_SPMM_UNROLL];
    W     bv[GB_SPMM_UNROLL][4];
#pragma unroll
    for (int u = 0; u < GB_SPMM_UNROLL; ++u) {
      col[u] = __ldg(colind + k + u);
      av[u]  = __ldg(val + k + u);
    }
#pragma unroll
    for (int u = 0; u < GB_SPMM_UNROLL; ++u)
      spmmLoad<ADJ, VEC>(bv[u], B + static_cast<long long>(col[u])*ncols, cols, identity);
#pragma unroll
    for (int u = 0; u < GB_SPMM_UNROLL; ++u)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = add_op(acc[q], mul_op(av[u], bv[u][q]));
  }
  for (; k < stop; ++k) {
    W bv[4];
    const Index col = __ldg(colind + k);
    const a av = __ldg(val + k);
    spmmLoad<ADJ, VEC>(bv, B + static_cast<long long>(col)*ncols, cols, identity);
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[q] = add_op(acc[q], mul_op(av, bv[q]));
  }
}

// Row ends of a tile consumed before its merge item p (row end i is item
// i + rowend[i] - k0, increasing in i).
__device__ __forceinline__ int spmmRowsBefore(const Index* rowend, int nr, Index k0,
                                              int p) {
  int lo = 0, hi = nr;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (mid + (rowend[mid] - k0) < p) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// One CTA per (merge tile, column slice); see the top of the file.
template <bool ADJ, bool VEC, typename W, typename a, typename MulOp, typename AddOp>
__global__ void __launch_bounds__(GB_SPMM_NT, GB_SPMM_MINB)
spmmMergeKernel(W* __restrict__           C,
                const Index* __restrict__ tile_rows,
                Index* __restrict__       carry_row,
                W* __restrict__           carry_val,
                const Index* __restrict__ rowptr,
                const Index* __restrict__ colind,
                const a* __restrict__     val,
                const W* __restrict__     B,
                Index                     nrows,
                Index                     nnz,
                int                       ncols,
                int                       lanes,
                int                       nslices,
                W                         identity,
                MulOp                     mul_op,
                AddOp                     add_op) {
  static_assert(sizeof(W) == 4 && sizeof(Index) == 4, "32-bit values and indices");
  __shared__ Index s_rowend[GB_SPMV_TILE + 1];
  __shared__ Index s_key[GB_SPMM_NT];             // open row of each group
  __shared__ W     s_tail[GB_SPMM_NT*4];          // its partial, per lane and column

  const int t = threadIdx.x;
  const int g = t / lanes;                         // group
  const int l = t % lanes;                         // lane in the group
  const int ngroups = GB_SPMM_NT/lanes;
  const int items_per_group = GB_SPMV_TILE/ngroups;

  const long long total = static_cast<long long>(nrows) + nnz;
  const long long d0 = static_cast<long long>(blockIdx.x)*GB_SPMV_TILE;
  long long d1 = d0 + GB_SPMV_TILE; if (d1 > total) d1 = total;
  const int tile_items = static_cast<int>(d1 - d0);
  const Index r0 = __ldg(tile_rows + blockIdx.x);
  const Index r1 = __ldg(tile_rows + blockIdx.x + 1);
  const Index k0 = static_cast<Index>(d0 - r0);
  const int   nr = r1 - r0;                        // rows that end in this tile

  for (int i = t; i <= nr; i += GB_SPMM_NT) {
    const Index r = r0 + i;
    s_rowend[i] = (r < nrows) ? __ldg(rowptr + r + 1) : nnz;
  }
  __syncthreads();

  int p_begin = g*items_per_group;
  if (p_begin > tile_items) p_begin = tile_items;
  int p_end = p_begin + items_per_group;
  if (p_end > tile_items) p_end = tile_items;
  const int start_i = spmmRowsBefore(s_rowend, nr, k0, p_begin);
  const int end_i = spmmRowsBefore(s_rowend, nr, k0, p_end);
  const Index k_begin = k0 + (p_begin - start_i);
  const Index k_end = k0 + (p_end - end_i);

  for (int slice = blockIdx.y; slice < nslices; slice += gridDim.y) {
    // N <= INT32_MAX: a slice's last column + 1 still fits an int
    const int base = slice*GB_SPMM_COL_TILE;
    const int end = (ncols - base > GB_SPMM_COL_TILE) ? base + GB_SPMM_COL_TILE : ncols;
    const SpmmCols<ADJ> cols = {base + (ADJ ? 4*l : l), lanes, end};

    // ---- each group: its row pieces in order ------------------------------------
    W head[4];
    Index k = k_begin;
    for (int i = start_i; i <= end_i; ++i) {
      const Index stop = (i < end_i) ? s_rowend[i] : k_end;
      W acc[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = identity;
      spmmFold<ADJ, VEC>(acc, k, stop, colind, val, B, ncols, cols, identity, mul_op,
                         add_op);
      k = stop;
      if (i == end_i) {
#pragma unroll
        for (int q = 0; q < 4; ++q) s_tail[4*t + q] = acc[q];
      } else if (i == start_i) {
#pragma unroll
        for (int q = 0; q < 4; ++q) head[q] = acc[q];
      } else {
        spmmStore<ADJ, VEC>(C + static_cast<long long>(r0 + i)*ncols, cols, acc);
      }
    }
    if (l == 0) s_key[g] = end_i;
    __syncthreads();

    // ---- heads: the tails of the earlier groups on the same row, then the head --
    if (end_i > start_i) {
      int gs = g;
      while (gs > 0 && s_key[gs - 1] == start_i) --gs;
      W out[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) out[q] = identity;
      for (int g2 = gs; g2 < g; ++g2)
#pragma unroll
        for (int q = 0; q < 4; ++q)
          out[q] = add_op(out[q], s_tail[4*(g2*lanes + l) + q]);
#pragma unroll
      for (int q = 0; q < 4; ++q) out[q] = add_op(out[q], head[q]);
      spmmStore<ADJ, VEC>(C + static_cast<long long>(r0 + start_i)*ncols, cols, out);
    }
    // ---- the tile's carry: the run of tails on its open row ----------------------
    if (g == ngroups - 1) {
      const Index row = r0 + end_i;
      if (l == 0 && slice == 0) carry_row[blockIdx.x] = (row < nrows) ? row : -1;
      if (row < nrows) {
        int gs = g;
        while (gs > 0 && s_key[gs - 1] == end_i) --gs;
        W out[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) out[q] = identity;
        for (int g2 = gs; g2 <= g; ++g2)
#pragma unroll
          for (int q = 0; q < 4; ++q)
            out[q] = add_op(out[q], s_tail[4*(g2*lanes + l) + q]);
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (cols.ok(q))
            carry_val[static_cast<long long>(blockIdx.x)*ncols + cols.off(q)] = out[q];
      }
    }
    __syncthreads();                   // s_tail / s_key are reused by the next slice
  }
}

// One thread per (carry, column): the first carry of a run of equal rows folds the
// run in tile order and adds it on the left of the row's stored value.
template <typename W, typename AddOp>
__global__ void spmmCarryFixupKernel(W* __restrict__ C,
                                     const Index* __restrict__ carry_row,
                                     const W* __restrict__ carry_val,
                                     int ncarry, long long ncols, AddOp add_op) {
  const long long id = static_cast<long long>(blockIdx.x)*blockDim.x + threadIdx.x;
  if (id >= ncarry*ncols) return;
  const int c = static_cast<int>(id/ncols);
  const long long j = id - c*ncols;
  const Index row = carry_row[c];
  if (row < 0) return;
  if (c > 0 && carry_row[c - 1] == row) return;
  W total = carry_val[c*ncols + j];
  for (int c2 = c + 1; c2 < ncarry && carry_row[c2] == row; ++c2)
    total = add_op(total, carry_val[c2*ncols + j]);
  C[row*ncols + j] = add_op(total, C[row*ncols + j]);
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_SPMM_CUH_
