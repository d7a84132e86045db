// graphblast_b200 backend — unmasked SpGEMM C = A (+.x) B, row by row (Gustavson).
//
// Row i of C gathers the products A(i,k)*B(k,j) over the entries k of row i of A.
// The driver (spgemm.hpp, spgemmUnmasked) runs four steps on the backend stream:
//   1. mxmRowBoundKernel: ub_i = sum_k |B(k,:)| (64-bit), stored clamped to ncols as
//      the row's bound on |C(i,:)|; mxmClassifyKernel bins the rows by it.  A row of
//      A with one entry k needs no counting (|C(i,:)| = |B(k,:)|).
//   2. symbolic: one group per row counts the distinct columns in a shared-memory
//      hash table of keys (load <= 0.5); a row whose bound exceeds the largest table
//      counts in a bitmap over ncols that its CTA owns in global memory.
//   3. the counts are scanned into C's row offsets (after a 64-bit check of their
//      total) and binned again by the exact count.
//   4. numeric: the same groups with key/value tables; products are combined with the
//      semiring's add (native atomicAdd for plus, a CAS loop otherwise), the table is
//      sorted by column (bitonic sort in shared memory, empty slots sort last) and the
//      first count entries are the row.  Rows beyond the largest table accumulate in
//      a dense value array plus bitmap over ncols per CTA, which comes out sorted.
//
// Products of a row are enumerated by warps in chunks of 32 entries of A: each lane
// loads one |B(k,:)|, a warp scan lays the chunk's products end to end, and each
// lane finds the entry its product belongs to by a five-step search over the scan.
// A row whose B rows are short keeps all 32 lanes busy all the same.
//
// Bins (bound in step 2, exact count in step 4):
//   bin  group              symbolic: bound   table          numeric: count  table
//   S    one warp (8/CTA)   1 .. 1024         <= 2048 slots  1 .. 256        <= 512
//   M    256-thread CTA     .. 4096           <= 8192        .. 2048         <= 4096
//   L    1024-thread CTA    .. 16384          <= 32768       .. 8192         <= 16384
//   D    1024-thread CTA    beyond            bitmap         beyond          dense
// Each table is a power of two of at least twice the bound / count.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_SPGEMM_UNMASKED_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_SPGEMM_UNMASKED_CUH_

#include "graphblas/backend/cuda/kernels/common.cuh"
#include "graphblas/backend/cuda/kernels/spgemm_hash.cuh"   // hashSlot

namespace graphblas {
namespace backend {

#define GB_MXM_EMPTY   0x7fffffff  // empty slot: above every column index, sorts last
#define GB_MXM_SYM_S   1024        // symbolic bins: largest bound per bin
#define GB_MXM_SYM_M   4096
#define GB_MXM_SYM_L   16384
#define GB_MXM_NUM_S   256         // numeric bins: largest count per bin
#define GB_MXM_NUM_M   2048
#define GB_MXM_NUM_L   8192
#define GB_MXM_NBIN    4           // S, M, L, D
#define GB_MXM_WARPS   8           // warps per CTA of the warp-table kernels

// Device cells of one classification: rows per bin, the grab counters of the CTA
// kernels, the 64-bit sum of the classified values and (symbolic pass) the sum of
// the exact counts of the rows that skip counting.
struct MxmCells {
  unsigned int       count[GB_MXM_NBIN];
  unsigned int       grab[GB_MXM_NBIN];
  unsigned long long total;
  unsigned long long exact;
};

// bound[i] = min(sum over k in A(i,:) of |B(k,:)|, ncols); one warp per 32 rows.
__global__ void mxmRowBoundKernel(const Index* __restrict__ A_ptr,
                                  const Index* __restrict__ A_ind,
                                  const Index* __restrict__ B_ptr,
                                  Index nrows, Index ncols, Index* __restrict__ bound) {
  const int lane = threadIdx.x & 31;
  const long long warp = (static_cast<long long>(blockIdx.x)*blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x)*blockDim.x) >> 5;
  for (long long base = 32*warp; base < nrows; base += 32*nwarps) {
    const int nr = (nrows - base < 32) ? static_cast<int>(nrows - base) : 32;
    long long mine = 0;
    for (int r = 0; r < nr; ++r) {
      const Index i = static_cast<Index>(base) + r;
      const Index a_end = __ldg(A_ptr + i + 1);
      long long ub = 0;
      for (Index e = __ldg(A_ptr + i) + lane; e < a_end; e += 32) {
        const Index k = __ldg(A_ind + e);
        ub += __ldg(B_ptr + k + 1) - __ldg(B_ptr + k);
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) ub += __shfl_xor_sync(GB_FULL_MASK, ub, off);
      if (lane == r) mine = ub;
    }
    if (lane < nr) bound[base + lane] = static_cast<Index>(mine < ncols ? mine : ncols);
  }
}

// Rows with value > 0 go to bin S / M / L (value <= cap_s / cap_m / cap_l) or D;
// lists: GB_MXM_NBIN arrays of `stride` rows.  With A_ptr, rows of A with at most
// one entry stay out of the lists: their value is already exact (cells->exact).
__global__ void mxmClassifyKernel(const Index* __restrict__ val, Index nrows,
                                  const Index* __restrict__ A_ptr,
                                  int cap_s, int cap_m, int cap_l,
                                  Index* __restrict__ lists, size_t stride,
                                  MxmCells* cells) {
  const int lane = threadIdx.x & 31;
  const Index step = gridDim.x*blockDim.x;
  // whole warps iterate together (the ballots below need every lane)
  for (Index base = blockIdx.x*blockDim.x + threadIdx.x - lane; base < nrows; base += step) {
    const Index v = base + lane;
    Index x = 0;
    bool exact = false;
    int cls = -1;
    if (v < nrows) {
      x = val[v];
      exact = A_ptr != NULL && __ldg(A_ptr + v + 1) - __ldg(A_ptr + v) <= 1;
      if (x > 0 && !exact)
        cls = x <= cap_s ? 0 : x <= cap_m ? 1 : x <= cap_l ? 2 : 3;
    }
    unsigned long long sum = exact ? 0ull : static_cast<unsigned long long>(x);
    unsigned long long ex  = exact ? static_cast<unsigned long long>(x) : 0ull;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      sum += __shfl_xor_sync(GB_FULL_MASK, sum, off);
      ex  += __shfl_xor_sync(GB_FULL_MASK, ex, off);
    }
    if (lane == 0 && sum) atomicAdd(&cells->total, sum);
    if (lane == 0 && ex) atomicAdd(&cells->exact, ex);
#pragma unroll
    for (int k = 0; k < GB_MXM_NBIN; ++k) {
      const unsigned int in = __ballot_sync(GB_FULL_MASK, cls == k);
      if (in == 0) continue;
      unsigned int first = 0;
      if (lane == 0) first = atomicAdd(cells->count + k, __popc(in));
      first = __shfl_sync(GB_FULL_MASK, first, 0);
      if (cls == k) lists[k*stride + first + __popc(in & ((1u << lane) - 1u))] = v;
    }
  }
}

// f(position in A, position in B) for every product of row entries [a_beg, a_end)
// of A that this warp takes: chunks of 32 entries, first_chunk, first_chunk + step,
// ...  Cnt holds a chunk's product count (int where the bins bound it).
template <typename Cnt, typename F>
__device__ __forceinline__ void mxmRowProducts(Index a_beg, Index a_end, int first_chunk,
    int chunk_step, const Index* __restrict__ A_ind, const Index* __restrict__ B_ptr,
    F f) {
  const int lane = threadIdx.x & 31;
  for (long long base = a_beg + 32ll*first_chunk; base < a_end; base += 32ll*chunk_step) {
    const long long e = base + lane;
    Index b_beg = 0;
    Cnt b_len = 0;
    if (e < a_end) {
      const Index k = __ldg(A_ind + e);
      b_beg = __ldg(B_ptr + k);
      b_len = __ldg(B_ptr + k + 1) - b_beg;
    }
    Cnt incl = b_len;                                   // inclusive warp scan
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const Cnt up = __shfl_up_sync(GB_FULL_MASK, incl, d);
      if (lane >= d) incl += up;
    }
    const Cnt total = __shfl_sync(GB_FULL_MASK, incl, 31);
    for (Cnt p0 = 0; p0 < total; p0 += 32) {
      const Cnt p = p0 + lane;
      int j = 0;                                        // lanes whose products end <= p
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) {
        const Cnt at = __shfl_sync(GB_FULL_MASK, incl, j + s - 1);
        if (at <= p) j += s;
      }
      const Cnt j_incl = __shfl_sync(GB_FULL_MASK, incl, j);
      const Cnt j_len = __shfl_sync(GB_FULL_MASK, b_len, j);
      const Index j_beg = __shfl_sync(GB_FULL_MASK, b_beg, j);
      if (p < total) f(base + j, j_beg + static_cast<Index>(p - (j_incl - j_len)));
    }
  }
}

// Slot of `key` in a table of keys with linear probing, inserted when absent;
// *fresh tells whether this call inserted it.
__device__ __forceinline__ unsigned int mxmTableSlot(int* keys, int key, int shift,
                                                     unsigned int smask, bool* fresh) {
  unsigned int s = hashSlot(key, shift);
  while (true) {
    const int k = keys[s];
    if (k == key) { *fresh = false; return s; }
    if (k == GB_MXM_EMPTY) {
      const int prev = atomicCAS(keys + s, GB_MXM_EMPTY, key);
      if (prev == GB_MXM_EMPTY) { *fresh = true; return s; }
      if (prev == key) { *fresh = false; return s; }
    }
    s = (s + 1) & smask;
  }
}

// log2 of the table for `n` keys: a power of two >= 2n (load <= 0.5), >= 32 slots.
__device__ __forceinline__ int mxmTableLog(Index n, int slots) {
  int lg = 5;
  while ((1 << lg) < 2*n && (1 << lg) < slots) ++lg;
  return lg;
}

template <bool WARP>
__device__ __forceinline__ void mxmGroupSync() {
  if (WARP) __syncwarp(); else __syncthreads();
}

// Next row of the bin for this group: warp tables walk the list with a fixed stride
// (their rows cost about the same), CTAs take rows one at a time.
template <bool WARP>
__device__ __forceinline__ unsigned int mxmNextItem(unsigned int prev, unsigned int* grab,
                                                    unsigned int* s_item) {
  if (WARP) return prev == ~0u ? blockIdx.x*GB_MXM_WARPS + (threadIdx.x >> 5)
                               : prev + gridDim.x*GB_MXM_WARPS;
  __syncthreads();                       // the previous row is done with the table
  if (threadIdx.x == 0) *s_item = atomicAdd(grab, 1u);
  __syncthreads();
  return *s_item;
}

// Symbolic: row_val[row] (the bound on entry) becomes the row's distinct column count.
template <int CT, bool WARP, int SLOTS>
__global__ void __launch_bounds__(CT)
mxmSymbolicKernel(const Index* __restrict__ rows, const MxmCells* cells, int bin,
                  unsigned int* grab,
                  const Index* __restrict__ A_ptr, const Index* __restrict__ A_ind,
                  const Index* __restrict__ B_ptr, const Index* __restrict__ B_ind,
                  Index* __restrict__ row_val) {
  constexpr int GT = WARP ? 32 : CT;
  extern __shared__ __align__(16) int mxm_smem[];
  __shared__ unsigned int s_item;
  __shared__ int s_count;
  const int lane = threadIdx.x & 31;
  const int gtid = WARP ? lane : threadIdx.x;
  int* keys = mxm_smem + (WARP ? (threadIdx.x >> 5)*SLOTS : 0);
  const unsigned int nitems = cells->count[bin];
  unsigned int idx = ~0u;
  while (true) {
    idx = mxmNextItem<WARP>(idx, grab, &s_item);
    if (idx >= nitems) break;
    const Index row = rows[idx];
    const int lg = mxmTableLog(row_val[row], SLOTS);
    const int nslots = 1 << lg;
    for (int s = gtid; s < nslots; s += GT) keys[s] = GB_MXM_EMPTY;
    if (!WARP && threadIdx.x == 0) s_count = 0;
    mxmGroupSync<WARP>();
    int mine = 0;
    mxmRowProducts<int>(__ldg(A_ptr + row), __ldg(A_ptr + row + 1),
        WARP ? 0 : threadIdx.x >> 5, WARP ? 1 : CT/32, A_ind, B_ptr,
        [&](long long, Index b) {
          bool fresh;
          mxmTableSlot(keys, __ldg(B_ind + b), 32 - lg, nslots - 1, &fresh);
          mine += fresh;
        });
    mine = warpSum(mine);
    if (WARP) {
      if (lane == 0) row_val[row] = mine;
      __syncwarp();
    } else {
      if (lane == 0 && mine) atomicAdd(&s_count, mine);
      __syncthreads();
      if (threadIdx.x == 0) row_val[row] = s_count;
    }
  }
}

// Symbolic, rows beyond the largest table: a bitmap over ncols per CTA (`words`
// 32-bit words each, zero on entry and left zero).
template <int CT>
__global__ void __launch_bounds__(CT)
mxmSymbolicDenseKernel(const Index* __restrict__ rows, const MxmCells* cells, int bin,
                       unsigned int* grab,
                       const Index* __restrict__ A_ptr, const Index* __restrict__ A_ind,
                       const Index* __restrict__ B_ptr, const Index* __restrict__ B_ind,
                       Index* __restrict__ row_val, unsigned int* bits_all, size_t words) {
  __shared__ unsigned int s_item;
  __shared__ int s_count;
  unsigned int* bits = bits_all + blockIdx.x*words;
  const unsigned int nitems = cells->count[bin];
  unsigned int idx = ~0u;
  while (true) {
    idx = mxmNextItem<false>(idx, grab, &s_item);
    if (idx >= nitems) break;
    const Index row = rows[idx];
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    int mine = 0;
    mxmRowProducts<long long>(__ldg(A_ptr + row), __ldg(A_ptr + row + 1),
        threadIdx.x >> 5, CT/32, A_ind, B_ptr,
        [&](long long, Index b) {
          const Index col = __ldg(B_ind + b);
          const unsigned int m = 1u << (col & 31);
          if (!(atomicOr(bits + (col >> 5), m) & m)) ++mine;
        });
    mine = warpSum(mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_count, mine);
    __syncthreads();
    if (threadIdx.x == 0) row_val[row] = s_count;
    for (size_t w = threadIdx.x; w < words; w += CT) bits[w] = 0u;
  }
}

// Semiring add of v into a 32-bit cell: native for plus (keeping float subnormals,
// atomicAddIeee), CAS loop otherwise.
__device__ __forceinline__ void mxmAdd(float* cell, float v) { atomicAddIeee(cell, v); }
__device__ __forceinline__ void mxmAdd(int* cell, int v) { atomicAdd(cell, v); }

template <bool PLUS, typename T, typename AddOp>
__device__ __forceinline__ void mxmCombine(T* cell, T v, AddOp add_op) {
  if (PLUS) mxmAdd(cell, v);
  else atomicCombine(cell, v, add_op);
}

// In-place ascending bitonic sort of n (a power of two) keys with their values by
// one group of GT threads.
template <int GT, bool WARP, typename c>
__device__ __forceinline__ void mxmBitonicSort(int* keys, c* vals, int n, int gtid) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = gtid; t < (n >> 1); t += GT) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int l = i | j;
        const int ki = keys[i], kl = keys[l];
        if ((ki > kl) == ((i & k) == 0)) {
          keys[i] = kl; keys[l] = ki;
          const c vi = vals[i]; vals[i] = vals[l]; vals[l] = vi;
        }
      }
      mxmGroupSync<WARP>();
    }
  }
}

// Numeric: the row's entries, combined, sorted by column, at C_ptr[row].
template <int CT, bool WARP, int SLOTS, bool PLUS, typename c, typename a, typename b,
          typename MulOp, typename AddOp>
__global__ void __launch_bounds__(CT)
mxmNumericKernel(const Index* __restrict__ rows, const MxmCells* cells, int bin,
                 unsigned int* grab,
                 const Index* __restrict__ A_ptr, const Index* __restrict__ A_ind,
                 const a* __restrict__ A_val,
                 const Index* __restrict__ B_ptr, const Index* __restrict__ B_ind,
                 const b* __restrict__ B_val,
                 const Index* __restrict__ C_ptr, Index* __restrict__ C_ind,
                 c* __restrict__ C_val, MulOp mul_op, AddOp add_op, c identity) {
  constexpr int GT = WARP ? 32 : CT;
  extern __shared__ __align__(16) int mxm_smem[];
  __shared__ unsigned int s_item;
  const int gtid = WARP ? (threadIdx.x & 31) : threadIdx.x;
  int* keys = mxm_smem + (WARP ? (threadIdx.x >> 5)*2*SLOTS : 0);
  c* vals = reinterpret_cast<c*>(keys + SLOTS);
  const unsigned int nitems = cells->count[bin];
  unsigned int idx = ~0u;
  while (true) {
    idx = mxmNextItem<WARP>(idx, grab, &s_item);
    if (idx >= nitems) break;
    const Index row = rows[idx];
    const Index c_beg = __ldg(C_ptr + row);
    const Index cnt = __ldg(C_ptr + row + 1) - c_beg;
    const int lg = mxmTableLog(cnt, SLOTS);
    const int nslots = 1 << lg;
    for (int s = gtid; s < nslots; s += GT) { keys[s] = GB_MXM_EMPTY; vals[s] = identity; }
    mxmGroupSync<WARP>();
    mxmRowProducts<int>(__ldg(A_ptr + row), __ldg(A_ptr + row + 1),
        WARP ? 0 : threadIdx.x >> 5, WARP ? 1 : CT/32, A_ind, B_ptr,
        [&](long long pa, Index pb) {
          bool fresh;
          const unsigned int s = mxmTableSlot(keys, __ldg(B_ind + pb), 32 - lg,
                                              nslots - 1, &fresh);
          mxmCombine<PLUS>(vals + s, static_cast<c>(mul_op(A_val[pa], B_val[pb])), add_op);
        });
    mxmGroupSync<WARP>();
    mxmBitonicSort<GT, WARP>(keys, vals, nslots, gtid);
    for (Index t = gtid; t < cnt; t += GT) {
      C_ind[c_beg + t] = keys[t];
      C_val[c_beg + t] = vals[t];
    }
    if (WARP) __syncwarp();
  }
}

// Numeric, rows beyond the largest table: per CTA a dense accumulator over ncols
// (identity on entry and left so) and a bitmap of the columns hit (zero on entry and
// left so); the bitmap is read out in column order.
template <int CT, bool PLUS, typename c, typename a, typename b, typename MulOp,
          typename AddOp>
__global__ void __launch_bounds__(CT)
mxmNumericDenseKernel(const Index* __restrict__ rows, const MxmCells* cells, int bin,
                      unsigned int* grab,
                      const Index* __restrict__ A_ptr, const Index* __restrict__ A_ind,
                      const a* __restrict__ A_val,
                      const Index* __restrict__ B_ptr, const Index* __restrict__ B_ind,
                      const b* __restrict__ B_val,
                      const Index* __restrict__ C_ptr, Index* __restrict__ C_ind,
                      c* __restrict__ C_val, MulOp mul_op, AddOp add_op, c identity,
                      c* acc_all, unsigned int* bits_all, Index ncols, size_t words) {
  __shared__ unsigned int s_item;
  __shared__ int s_scan[CT/32 + 1];
  __shared__ Index s_out;
  c* acc = acc_all + blockIdx.x*static_cast<size_t>(ncols);
  unsigned int* bits = bits_all + blockIdx.x*words;
  unsigned int idx = ~0u;
  while (true) {
    idx = mxmNextItem<false>(idx, grab, &s_item);
    // the bin size is read per row: held across the row it is spilled
    if (idx >= cells->count[bin]) break;
    const Index row = rows[idx];
    // the row's output offset waits in shared memory (in a register it is spilled
    // across the product loop)
    if (threadIdx.x == 0) s_out = __ldg(C_ptr + row);
    mxmRowProducts<long long>(__ldg(A_ptr + row), __ldg(A_ptr + row + 1),
        threadIdx.x >> 5, CT/32, A_ind, B_ptr,
        [&](long long pa, Index pb) {
          const Index col = __ldg(B_ind + pb);
          atomicOr(bits + (col >> 5), 1u << (col & 31));
          mxmCombine<PLUS>(acc + col, static_cast<c>(mul_op(A_val[pa], B_val[pb])), add_op);
        });
    __syncthreads();
    // L1 may hold lines of these arrays from the previous row: read through L2
    Index out = s_out;
    for (size_t w0 = 0; w0 < words; w0 += CT) {
      const size_t w = w0 + threadIdx.x;
      unsigned int word = w < words ? __ldcg(bits + w) : 0u;
      int total;
      Index at = out + blockExclusiveScan<CT>(__popc(word), s_scan, &total);
      if (word) bits[w] = 0u;
      while (word) {
        const Index col = static_cast<Index>(32*w) + __ffs(word) - 1;
        word &= word - 1;
        C_ind[at] = col;
        C_val[at] = __ldcg(acc + col);
        acc[col] = identity;
        ++at;
      }
      out += total;
    }
  }
}

template <typename T>
__global__ void mxmFillKernel(T* __restrict__ out, size_t n, T v) {
  for (size_t i = blockIdx.x*static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x)*blockDim.x)
    out[i] = v;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_SPGEMM_UNMASKED_CUH_
