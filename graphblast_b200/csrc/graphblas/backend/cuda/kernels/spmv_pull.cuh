// graphblast_b200 backend — PULL direction kernels (dense frontier).
//
//  * spmvMergeKernel      : generic-semiring CSR SpMV, merge-path load balanced
//                           (rows + nonzeros split evenly across CTAs and threads),
//                           streaming loads of colind/val, gathers of the
//                           dense vector served from L2 (evict-last), shuffle-based
//                           segmented scan for rows that straddle threads, per-CTA
//                           carry-out fixed up by spmvCarryFixupKernel.
//                           Replaces mgpu::SpmvCsrBinary (reference spmv.hpp:188-190,
//                           ext/moderngpu/include/kernels/spmvcsr.cuh:334-413,489-587:
//                           5+ launches and 2 device syncs per SpMV).
//  * spmvMaskedOrPullKernel / spmvMaskedOrPullBitsKernel: fused mask + OR-AND +
//                           early-exit + operand-reuse Boolean pull (reference
//                           kernels/spmv.hpp:7-59).  The Bits form (identity 0) reads
//                           mask and frontier as bitmaps, decides most rows from a
//                           per-matrix first-neighbour summary, publishes the result
//                           as a bitmap + count (values are materialised lazily) and
//                           posts the count to the host mailbox.
//
// Algorithmic bytes per launch (SURVEY.md §8d):
//   merge SpMV : 4(n+1) rowptr + 8 nnz colind/val + 4n gather (once) + 4n write
//   Boolean    : 4(n+1) + 4 E_inspected + 4n mask + 4n write
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_SPMV_PULL_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_SPMV_PULL_CUH_

#include "graphblas/backend/cuda/kernels/common.cuh"
#include "graphblas/backend/cuda/kernels/util.cuh"

namespace graphblas {
namespace backend {

#define GB_SPMV_NT   128
#define GB_SPMV_IPT  9                               // merge items per thread
// Share of the SM's 256 KB given to shared memory.  The kernel needs ~4.7 KB per
// CTA; everything else should be L1, which is what holds the loads in flight and
// the hot part of the gathered vector (tools/spmv_lab.cu sweep, RMAT-22:
// 25 % -> 0.49 ms, 50 % -> 0.60 ms, 100 % -> 1.33 ms).
#define GB_SPMV_CARVEOUT 25
#define GB_SPMV_TILE (GB_SPMV_NT*GB_SPMV_IPT)        // merge items per CTA
// Resident CTAs per SM the register allocation must allow: full occupancy (2048
// threads).  Without the cap ptxas takes 40+ registers and the kernel loses 20 %.
#define GB_SPMV_MINB(NT) ((2048/(NT)) > 32 ? 32 : (2048/(NT)))

// Merge-path split: on diagonal d (d = rows consumed + nonzeros consumed) return
// the number of row-end items consumed.  List A is row_end[r] = rowptr[r+1],
// list B the nonzero indices 0..nnz-1; a row-end is consumed before the nonzero
// with the same value (that nonzero belongs to the next row).
__device__ __forceinline__ Index mergePathRows(long long d,
                                               const Index* __restrict__ rowptr,
                                               Index nrows, Index nnz) {
  long long lo = d - nnz; if (lo < 0) lo = 0;
  long long hi = d < nrows ? d : nrows;
  while (lo < hi) {
    long long mid = (lo + hi) >> 1;
    if (static_cast<long long>(__ldg(rowptr + mid + 1)) <= d - mid - 1)
      lo = mid + 1;
    else
      hi = mid;
  }
  return static_cast<Index>(lo);
}

// tile_rows[c] = rows consumed at the start of tile c, for c in [0, ntiles].
// Every search is an independent chain of ~log2(n) dependent loads; doing them
// all in parallel here (and caching the result per matrix, the partition only
// depends on rowptr) takes that latency chain out of every SpMV tile.
__global__ void spmvMergePartitionKernel(Index* __restrict__ tile_rows,
                                         const Index* __restrict__ rowptr,
                                         Index nrows, Index nnz, int ntiles,
                                         int tile_items) {
  int c = blockIdx.x*blockDim.x + threadIdx.x;
  if (c > ntiles) return;
  const long long total = static_cast<long long>(nrows) + nnz;
  long long d = static_cast<long long>(c)*tile_items;
  if (d > total) d = total;
  tile_rows[c] = mergePathRows(d, rowptr, nrows, nnz);
}

// Shared-memory slot of product p.  Threads store 8 consecutive products as two
// 128-bit words at a 32-byte lane stride, which on its own is a 2-way bank
// conflict in every quarter warp; swapping the two halves of every other group of
// four chunks (bit 5 of p selects, bit 2 is toggled) makes the stores conflict
// free, and the sequential readers pay one XOR.
__device__ __forceinline__ int prodSlot(int p) { return p ^ ((p >> 3) & 4); }

// LaneMajor: lanes of a warp take consecutive nonzeros with 32-bit loads (any
// alignment).  Otherwise every thread takes 8 consecutive nonzeros, read as two
// 128-bit loads per array (colind and val must be 32-byte aligned).
template <int NT, int IPT, bool LaneMajor,
          typename W, typename a, typename U,
          typename MulOp, typename AddOp>
__global__ void __launch_bounds__(NT, GB_SPMV_MINB(NT))
spmvMergeKernelT(W* __restrict__           w,
                const Index* __restrict__ tile_rows,
                Index* __restrict__       carry_row,
                W* __restrict__           carry_val,
                const Index* __restrict__ rowptr,
                const Index* __restrict__ colind,
                const a* __restrict__     val,
                const U* __restrict__     u,
                Index                     nrows,
                Index                     nnz,
                W                         identity,
                MulOp                     mul_op,
                AddOp                     add_op) {
  // One buffer: products grow from the bottom, row ends from the top.  A tile has
  // nr row ends and nk nonzeros with nr + nk <= NT*IPT, the product window adds at
  // most 14 slots of alignment slack and the row ends one entry (the open row).
  // Keeping the footprint at ~3.7 KB per CTA matters more than anything else in
  // this kernel: L1 capacity (what the shared-memory carve-out leaves) is what
  // bounds the loads in flight.
  static_assert(sizeof(W) == 4 && sizeof(Index) == 4, "32-bit values and indices");
  __shared__ __align__(32) unsigned int s_buf[(NT*IPT) + 40];
  W* const s_prod = reinterpret_cast<W*>(s_buf);
#define GB_S_ROWEND(i) (reinterpret_cast<Index*>(s_buf)[(NT*IPT) + 39 - (i)])
  __shared__ Index s_wkey[NT/32];
  __shared__ W     s_wval[NT/32];

  const int t    = threadIdx.x;
  const int lane = t & 31;
  const int wid  = t >> 5;

  const long long total = static_cast<long long>(nrows) + nnz;
  const long long d0 = static_cast<long long>(blockIdx.x)*(NT*IPT);
  long long d1 = d0 + (NT*IPT); if (d1 > total) d1 = total;
  const int tile_items = static_cast<int>(d1 - d0);

  const Index r0 = __ldg(tile_rows + blockIdx.x);
  const Index r1 = __ldg(tile_rows + blockIdx.x + 1);
  const Index k0 = static_cast<Index>(d0 - r0);
  const Index k1 = static_cast<Index>(d1 - r1);
  const int   nr = r1 - r0;          // rows that END in this tile
  const int   nk = k1 - k0;          // nonzeros consumed in this tile
  const Index k0a = k0 & ~7;         // 32-byte aligned load window start

  // ---- phase 1a: issue the streaming loads + gathers of this thread's chunks --
  // Products mul(A(k), u[col(k)]) for k in [k0, k1) go to s_prod[k - k0a].
  const uint64_t pol = makeEvictLastPolicy();
  const int nchunks = (nk > 0) ? ((k1 - k0a + 7) >> 3) : 0;
  if (LaneMajor) {
    // Lanes of a warp take CONSECUTIVE nonzeros (32-bit loads, 128 bytes per
    // instruction, same bytes per wavefront as the 256-bit form): one gather
    // instruction then covers 32 neighbouring entries of (usually) one row, whose
    // sorted column indices fall into far fewer 128-byte lines than 32 entries
    // taken 8 apart, and the product stores are conflict free.  The L1 data pipe
    // (wavefronts), not HBM, is what this kernel saturates.
    const int span = (nk > 0) ? (k1 - k0a) : 0;
    for (int g = wid*256; g < span; g += (NT/32)*256) {
      Index col[8];
      a     av[8];
      U     uv[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const Index k = k0a + g + j*32 + lane;
        col[j] = (k >= k0 && k < k1) ? ldStream(colind + k)
                                     : static_cast<Index>(-1);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const Index k = k0a + g + j*32 + lane;
        if (col[j] >= 0) av[j] = ldStream(val + k);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (col[j] >= 0) uv[j] = ldGather(u + col[j], pol);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int p = g + j*32 + lane;
        if (p < span)
          s_prod[prodSlot(p)] = (col[j] >= 0) ? mul_op(av[j], uv[j]) : identity;
      }
    }
  } else
  for (int c = t; c < nchunks; c += NT) {
    const Index kb = k0a + (c << 3);
    W prods[8];
    if (kb + 8 <= nnz) {
      const Word8 cw = ldStream256(colind + kb);
      const Word8 vw = ldStream256(val + kb);
      U uv[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) uv[j] = ldGather(u + cw.w[j], pol);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        a av;
        memcpy(&av, &vw.w[j], 4);
        prods[j] = mul_op(av, uv[j]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const Index k = kb + j;
        if (k >= k0 && k < k1) {
          const Index col = ldStream(colind + k);
          const a av = ldStream(val + k);
          prods[j] = mul_op(av, ldGather(u + col, pol));
        } else {
          prods[j] = identity;
        }
      }
    }
    float4 lo4, hi4;
    memcpy(&lo4, &prods[0], 16);
    memcpy(&hi4, &prods[4], 16);
    const int swap = c & 4;            // == prodSlot(8c) - 8c
    *reinterpret_cast<float4*>(&s_prod[(c << 3) + swap])       = lo4;
    *reinterpret_cast<float4*>(&s_prod[(c << 3) + (4 - swap)]) = hi4;
  }

  // ---- phase 1b: row-end offsets for rows r0 .. r1 (last = still-open row) ----
  for (int i = t; i <= nr; i += NT) {
    const Index r = r0 + i;
    GB_S_ROWEND(i) = (r < nrows) ? __ldg(rowptr + r + 1) : nnz;
  }
  __syncthreads();

  // ---- phase 2: thread partition without searching -----------------------------
  // Row-end i is merge item p_i = i + (rowend_i - k0).  Thread t owns items
  // [t*IPT, (t+1)*IPT) and starts at local row #{i : p_i < t*IPT}; p is increasing.
  // Every thread finds its own count with a binary search over the (at most
  // NT*IPT + 1) row ends in shared memory: ~log2(rows in tile) loads, no second
  // barrier, and no serial loop when one long row spans the whole tile (the
  // scatter form of this step let one thread write up to NT entries and kept the
  // other warps at the barrier — 28 % of this kernel's stall samples).
  int start_i;
  {
    const int target = t*IPT;
    int lo = 0, hi = nr;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (mid + (GB_S_ROWEND(mid) - k0) < target) lo = mid + 1; else hi = mid;
    }
    start_i = lo;
  }

  // ---- phase 3: sequential merge of this thread's IPT items ----------------------
  int ld = t*IPT;
  if (ld > tile_items) ld = tile_items;
  int nit = tile_items - ld;
  if (nit > IPT) nit = IPT;
  int   i = start_i;                  // local row
  Index k = k0 + (ld - i);            // global nonzero index
  const int first_i = i;
  W acc = identity;
  W head_val = identity;              // first row that ends in this thread's range
  Index rowend = GB_S_ROWEND(i);
#pragma unroll
  for (int it = 0; it < IPT; ++it) {
    if (it < nit) {
      if (k < rowend) {
        acc = add_op(acc, s_prod[prodSlot(k - k0a)]);
        ++k;
      } else {
        // A finished row goes straight to global memory (neighbouring threads
        // finish neighbouring rows); only the first one waits for the carry-in.
        if (i == first_i) head_val = acc; else w[r0 + i] = acc;
        acc = identity;
        ++i;
        rowend = GB_S_ROWEND(i);
      }
    }
  }

  // ---- phase 4: segmented scan of (open row, partial) over the CTA ----------------
  Index key = i;
  W     v   = acc;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    Index pk = __shfl_up_sync(GB_FULL_MASK, key, off);
    W     pv = __shfl_up_sync(GB_FULL_MASK, v, off);
    if (lane >= off && pk == key) v = add_op(pv, v);
  }
  if (lane == 31) { s_wkey[wid] = key; s_wval[wid] = v; }
  const Index key0 = __shfl_sync(GB_FULL_MASK, key, 0);
  const Index ekey = __shfl_up_sync(GB_FULL_MASK, key, 1);
  const W     eval = __shfl_up_sync(GB_FULL_MASK, v, 1);
  __syncthreads();
  // Fold the tails of the preceding warps.
  Index ck = -1;
  W     cv = identity;
#pragma unroll
  for (int ww = 0; ww < NT/32 - 1; ++ww) {
    if (ww < wid) {
      const Index wk = s_wkey[ww];
      const W     wv = s_wval[ww];
      if (wk == ck) cv = add_op(cv, wv);
      else { ck = wk; cv = wv; }
    }
  }
  W carry_in;
  if (lane == 0) {
    carry_in = (ck == first_i) ? cv : identity;
  } else {
    carry_in = eval;                                 // ekey == first_i always
    if (ekey == key0 && ck == ekey) carry_in = add_op(cv, eval);
  }

  if (i > first_i) w[r0 + first_i] = add_op(carry_in, head_val);

  if (t == NT - 1) {
    W out = (i > first_i) ? acc : add_op(carry_in, acc);
    carry_row[blockIdx.x] = (r0 + i < nrows) ? (r0 + i) : -1;
    carry_val[blockIdx.x] = out;
  }
#undef GB_S_ROWEND
}

// One thread per CTA carry: the first carry of a run of equal rows folds the
// whole run and adds it (on the left) to the row's stored tail.
template <typename W, typename AddOp>
__global__ void spmvCarryFixupKernel(W* __restrict__ w,
                                     const Index* __restrict__ carry_row,
                                     const W* __restrict__ carry_val,
                                     int ncarry, AddOp add_op) {
  int c = blockIdx.x*blockDim.x + threadIdx.x;
  if (c >= ncarry) return;
  const Index row = carry_row[c];
  if (row < 0) return;
  if (c > 0 && carry_row[c-1] == row) return;
  W total = carry_val[c];
  for (int c2 = c + 1; c2 < ncarry && carry_row[c2] == row; ++c2)
    total = add_op(total, carry_val[c2]);
  w[row] = add_op(total, w[row]);
}

// ---------------------------------------------------------------------------
// Fused masked Boolean pull.  One thread per row (rows with a satisfied mask
// test are skipped without touching the matrix; unvisited rows stop at the
// first frontier neighbour when early exit is on).
// ---------------------------------------------------------------------------
#define GB_PULL_NT 256
#define GB_PULL_WPI 4     // mask words (x32 rows) a warp handles per iteration

template <bool UseScmp, bool UseEarlyExit, bool UseOpReuse,
          typename W, typename M, typename U>
__global__ void __launch_bounds__(GB_PULL_NT)
spmvMaskedOrPullKernel(W* __restrict__           w,
                       const M* __restrict__     mask,
                       U                         identity,
                       Index                     nrows,
                       const Index* __restrict__ rowptr,
                       const Index* __restrict__ colind,
                       const U* __restrict__     u,
                       unsigned long long*       discovered,
                       unsigned long long*       inspected_bytes) {
  __shared__ int s_red[GB_PULL_NT/32];
  Index row = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  int found_total = 0;
  int inspected = 0;
  for (; row < nrows; row += stride) {
    bool found = false;
    const M m = mask[row];
    const bool masked_out = UseScmp ? (m != static_cast<M>(0))
                                    : (m == static_cast<M>(0));
    if (!masked_out) {
      Index k   = rowptr[row];
      Index end = rowptr[row + 1];
      for (; k < end; ++k) {
        const Index col = __ldg(colind + k);
        ++inspected;
        bool hit;
        if (UseOpReuse) hit = (__ldg(mask + col) != static_cast<M>(0));
        else            hit = (__ldg(u + col) != identity);
        if (hit) {
          found = true;
          if (UseEarlyExit) break;
        }
      }
    }
    w[row] = found ? static_cast<W>(1) : static_cast<W>(0);
    found_total += found ? 1 : 0;
  }
  int total = blockSum<GB_PULL_NT>(found_total, s_red);
  if (threadIdx.x == 0 && total)
    atomicAdd(discovered, static_cast<unsigned long long>(total));
  // Algorithmic bytes of the inspected colind entries (SURVEY.md §8d: E_insp).
  int insp = blockSum<GB_PULL_NT>(inspected, s_red);
  if (threadIdx.x == 0 && insp && inspected_bytes != NULL)
    atomicAdd(inspected_bytes, 4ull*static_cast<unsigned long long>(insp));
}

// ---------------------------------------------------------------------------
// Bitmap form of the fused masked Boolean pull (the one the BFS loop runs).
// mask_bits / u_bits hold one bit per vertex (bit == value != 0), so the visited
// test of a row is a broadcast word load and the neighbour test is a gather into
// an n/8-byte array (2 MB at RMAT-24) that lives in L1/L2 instead of a 4n-byte
// float array.  A warp owns 32 consecutive rows = one output word: the new
// frontier is written, through one ballot, as the bitmap shadow only; the caller
// holds the 0/1 values lazily (DenseVector::materialize).
// ---------------------------------------------------------------------------
// first[i] = -1 (empty row) | colind[rowptr[i]] | that value with bit 31 set when
// it is the row's only entry.  Computed once per matrix structure.
__global__ void pullFirstNeighbourKernel(Index* __restrict__ first,
                                         const Index* __restrict__ rowptr,
                                         const Index* __restrict__ colind,
                                         Index nrows) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < nrows; i += stride) {
    const Index beg = __ldg(rowptr + i);
    const Index len = __ldg(rowptr + i + 1) - beg;
    Index f = -1;
    if (len > 0) {
      f = __ldg(colind + beg);
      if (len == 1) f |= static_cast<Index>(0x80000000u);
    }
    first[i] = f;
  }
}

// The same encoding with the neighbour most likely to be visited instead of the first:
// probe[i] = -1 (empty row) | the entry u of row i with the longest row u
// (rowptr[u+1] - rowptr[u]; the earliest entry on a tie) | that value with bit 31 set
// when it is the row's only entry.  For a symmetric structure the row length is u's
// degree; for the CSC of a directed one it is u's in-degree, how reachable u is.  A
// warp per row, lanes striding the entries (R-MAT rows run to 10^6 entries); 2 nnz
// gathers of rowptr, once per matrix structure.
__global__ void pullMaxDegreeNeighbourKernel(Index* __restrict__ probe,
                                             const Index* __restrict__ rowptr,
                                             const Index* __restrict__ colind,
                                             Index nrows) {
  const int lane = threadIdx.x & 31;
  Index i = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
  const Index stride = (gridDim.x*blockDim.x) >> 5;
  for (; i < nrows; i += stride) {
    const Index beg = __ldg(rowptr + i);
    const Index len = __ldg(rowptr + i + 1) - beg;
    // key: row length above, the entry's position complemented below (the largest
    // key is the longest row, earliest entry)
    unsigned long long best = 0ull;
    for (Index k = lane; k < len; k += 32) {
      const Index u = __ldg(colind + beg + k);
      const unsigned long long d =
          static_cast<unsigned long long>(__ldg(rowptr + u + 1) - __ldg(rowptr + u));
      const unsigned long long key = (d << 32) | (0xffffffffu - static_cast<unsigned int>(k));
      if (key > best) best = key;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const unsigned long long o = __shfl_xor_sync(GB_FULL_MASK, best, off);
      if (o > best) best = o;
    }
    if (lane == 0) {
      Index f = -1;
      if (len > 0) {
        const Index k = static_cast<Index>(0xffffffffu - static_cast<unsigned int>(best));
        f = __ldg(colind + beg + k);
        if (len == 1) f |= static_cast<Index>(0x80000000u);
      }
      probe[i] = f;
    }
  }
}

// bits[w] bit b = row 32w+b has no entry (first == -1); rows past the end read 0.
// A traversal marks these rows visited up front: nothing can discover them, and a
// third of an R-MAT's rows would otherwise be looked at on every pull level.
__global__ void pullEmptyRowBitsKernel(unsigned int* __restrict__ bits,
                                       const Index* __restrict__ first, Index nrows) {
  const int lane = threadIdx.x & 31;
  Index row = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  const Index padded = ((nrows + 31) >> 5) << 5;
  for (; row < padded; row += stride) {            // whole warps: padded is a multiple of 32
    const bool empty = row < nrows && __ldg(first + row) == static_cast<Index>(-1);
    const unsigned int word = __ballot_sync(GB_FULL_MASK, empty);
    if (lane == 0) bits[row >> 5] = word;
  }
}

template <bool UseScmp, bool UseEarlyExit, bool UseOpReuse>
__global__ void __launch_bounds__(GB_PULL_NT)
spmvMaskedOrPullBitsKernel(unsigned int* __restrict__       w_bits,
                           const unsigned int* __restrict__ mask_bits,
                           const unsigned int* __restrict__ u_bits,
                           Index                            nrows,
                           const Index* __restrict__        first,
                           const Index* __restrict__        rowptr,
                           const Index* __restrict__        colind,
                           unsigned long long*              discovered,
                           unsigned long long*              inspected_bytes,
                           unsigned long long*              done,
                           unsigned long long*              mail,
                           unsigned long long               ticket) {
  __shared__ int s_red[GB_PULL_NT/32];
  const int lane = threadIdx.x & 31;
  const Index warp0  = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
  const Index nwarps = (gridDim.x*blockDim.x) >> 5;
  const Index nwords = (nrows + 31) >> 5;
  const Index ngroups = (nwords + GB_PULL_WPI - 1)/GB_PULL_WPI;
  const unsigned int* probe = UseOpReuse ? mask_bits : u_bits;
  int found_total = 0;
  int inspected = 0;
  // A warp owns GB_PULL_WPI consecutive mask words (128 rows) per iteration and
  // keeps that many independent load chains (mask word -> first neighbour ->
  // probe word) in flight per lane: with one word per iteration the late levels
  // of a traversal, where few rows are still unvisited, were bound by the
  // latency of one such chain per iteration.
  for (Index g = warp0; g < ngroups; g += nwarps) {
    unsigned int mword[GB_PULL_WPI];
#pragma unroll
    for (int j = 0; j < GB_PULL_WPI; ++j) {
      const Index word = g*GB_PULL_WPI + j;
      mword[j] = (word < nwords) ? __ldg(mask_bits + word)
                                 : (UseScmp ? 0xffffffffu : 0u);
    }
    // One coalesced 4-byte load answers most rows: the first (lowest-index)
    // neighbour of an R-MAT/social-graph row is usually a hub that is already
    // visited, and empty rows never touch rowptr/colind at all.  Only a miss on
    // a row with more entries walks the list (one 32-byte sector per row is
    // what the walk costs, against 4 bytes here).
    Index f[GB_PULL_WPI];
#pragma unroll
    for (int j = 0; j < GB_PULL_WPI; ++j) {
      const Index row = (g*GB_PULL_WPI + j)*32 + lane;
      const bool mbit = (mword[j] >> lane) & 1u;
      const bool active = (row < nrows) && (UseScmp ? !mbit : mbit);
      f[j] = static_cast<Index>(-1);
      if (active) {
        f[j] = __ldg(first + row);
        ++inspected;                      // = colind[rowptr[row]], one entry
      }
    }
    unsigned int pword[GB_PULL_WPI];
#pragma unroll
    for (int j = 0; j < GB_PULL_WPI; ++j) {
      pword[j] = 0u;
      if (f[j] != static_cast<Index>(-1))
        pword[j] = __ldg(probe + ((f[j] & 0x7fffffff) >> 5));
    }
#pragma unroll
    for (int j = 0; j < GB_PULL_WPI; ++j) {
      const Index word = g*GB_PULL_WPI + j;
      const Index row  = word*32 + lane;
      bool found = (pword[j] >> (f[j] & 31)) & 1u;
      if (f[j] >= 0 && !(found && UseEarlyExit)) {
        Index k         = __ldg(rowptr + row) + 1;
        const Index end = __ldg(rowptr + row + 1);
        for (; k < end; ++k) {
          const Index col = __ldg(colind + k);
          ++inspected;
          if ((__ldg(probe + (col >> 5)) >> (col & 31)) & 1u) {
            found = true;
            if (UseEarlyExit) break;
          }
        }
      }
      const unsigned int out = __ballot_sync(GB_FULL_MASK, found);
      if (lane == 0 && word < nwords) w_bits[word] = out;
      found_total += found ? 1 : 0;
    }
  }
  int total = blockSum<GB_PULL_NT>(found_total, s_red);
  if (threadIdx.x == 0 && total)
    atomicAdd(discovered, static_cast<unsigned long long>(total));
  int insp = blockSum<GB_PULL_NT>(inspected, s_red);
  if (threadIdx.x == 0 && insp && inspected_bytes != NULL)
    atomicAdd(inspected_bytes, 4ull*static_cast<unsigned long long>(insp));
  // The CTA that finishes last posts the discovered count to the host mailbox
  // (util.hpp): the level loop reads it without a stream synchronisation.
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(done, 1ull) == gridDim.x - 1) {
      const unsigned long long count =
          *reinterpret_cast<volatile unsigned long long*>(discovered);
      *done = 0ull;
      mailPost(mail, ticket, count);
    }
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_SPMV_PULL_CUH_
