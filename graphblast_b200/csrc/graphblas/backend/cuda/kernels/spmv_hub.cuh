// graphblast_b200 backend — hub-cached, TMA-staged generic-semiring pull SpMV.
//
// Same contract as spmvMergeKernelT, bit for bit wherever the fold's order does
// not matter: every product is rounded before it is added, as there (the
// multiplies functor's __fmul_rn; no FFMA).  (kernels/spmv_pull.cuh; replaces
// mgpu::SpmvCsrBinary, reference spmv.hpp:188-190 and
// ext/moderngpu/include/kernels/spmvcsr.cuh:334-413,489-587), built for what
// bounds that kernel: every gathered u[col] of a power-law graph is its own L1
// wavefront and its own 32-byte L2 sector, 128 M of them on RMAT-22 against
// 1.07 GB of streamed CSR.  Here
//
//  * the K most referenced columns ("hubs", chosen once per matrix) live in
//    SHARED memory: a per-call compact copy hub_vals[K] = u[hub_ids[K]] is
//    brought in with one TMA bulk copy per CTA, and the matrix carries an encoded
//    column array (bit 31 set: low bits = hub slot; clear: the column id), so a
//    hub reference costs a bank access instead of a sector;
//  * the kernel works on the NON-EMPTY rows only (a compacted row list built once
//    per matrix; 38 % of an R-MAT's rows are empty and would otherwise have to be
//    searched over inside the reduction); empty rows get the identity from the
//    pre-pass that also collects the hub values;
//  * tiles come from a WEIGHTED merge path over that list (a row end weighs
//    GB_HUB_RW nonzeros), so a tile has at most 253 row ends; its row-offset and
//    row-id windows (1 KB each) are staged into a double-buffered shared-memory
//    slot with cp.async.bulk + mbarrier, its boundaries are one 16-byte record;
//  * colind/val are streamed 8 consecutive nonzeros per thread (two 128-bit
//    loads each), the NEXT tile's pair is requested before this tile's reduction
//    starts (register double buffer), so a group always has a DRAM request and
//    its gathers in flight;
//  * the row that holds the first nonzero of every 8-entry chunk is precomputed
//    once per matrix as one byte (relative to the tile's first row), so a thread
//    starts its segmented reduction without searching;
//  * one persistent CTA per SM; independent 128-thread groups per CTA, each with
//    its own rowptr slots and named barrier — one barrier per tile;
//  * threads reduce their 8 products in registers (no product round trip through
//    shared memory); the cross-thread part is a shuffle-based segmented scan +
//    per-tile carry (spmvCarryFixupKernel folds the carries).
//
// The cold gathers are plain __ldg loads: unlike the streamed CSR arrays they
// allocate in L1.
//
// Algorithmic bytes per launch (SURVEY.md §8d): 4(n+1) + 8 nnz + 4n + 4n.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_SPMV_HUB_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_SPMV_HUB_CUH_

#include "graphblas/backend/cuda/kernels/common.cuh"

namespace graphblas {
namespace backend {

#define GB_HUB_GT    128                 // threads per tile group
#define GB_HUB_RW    4                   // weight of a row end in merge items
#define GB_HUB_TILE  1008                // weighted merge items per tile
#define GB_HUB_RPWIN 264                 // staged row entries (<= 253 + 2 + 6)
#define GB_HUB_PAD   16                  // slack entries behind the compact row arrays
#define GB_HUB_FLAG  0x80000000u         // encoded column: hub slot in the low bits

// ---------------------------------------------------------------------------
// mbarrier / bulk-copy (TMA, non-tensor form) primitives.
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smemAddr(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbarInit(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;"
               :: "r"(smemAddr(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void mbarFenceInit() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbarExpectTx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
               :: "r"(smemAddr(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ bool mbarTryWait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n"
               ".reg .pred p;\n"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
               "selp.u32 %0, 1, 0, p;\n"
               "}\n"
               : "=r"(ok) : "r"(smemAddr(bar)), "r"(parity) : "memory");
  return ok != 0;
}

__device__ __forceinline__ void mbarWait(uint64_t* bar, uint32_t parity) {
  while (!mbarTryWait(bar, parity)) { }
}

__device__ __forceinline__ uint64_t makeEvictFirstPolicy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;"
               : "=l"(pol));
  return pol;
}

// global -> shared bulk copy; dst, src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulkLoad(void* dst, const void* src,
                                         uint32_t bytes, uint64_t* bar,
                                         uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes"
               ".L2::cache_hint [%0], [%1], %2, [%3], %4;"
               :: "r"(smemAddr(dst)), "l"(src), "r"(bytes), "r"(smemAddr(bar)),
                  "l"(pol) : "memory");
}

// L2 prefetch of a window that a later bulk copy will read.
__device__ __forceinline__ void bulkPrefetchL2(const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;"
               :: "l"(src), "r"(bytes) : "memory");
}

__device__ __forceinline__ void groupBarrier(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------------------
// Compact list of the non-empty rows (once per matrix structure):
//   ne_rows[r] = id of the r-th non-empty row, ne_ptr[r] = its first nonzero
//   (so ne_ptr[r+1] is its end), for r in [0, m); both arrays carry GB_HUB_PAD
//   sentinel entries (row -1, offset nnz) so that 16-byte windows never leave
//   them.  empty_rows[] lists the others.
// Ordered compaction in three small kernels: per-block counts, one-block scan of
// the counts, per-block emit.
// ---------------------------------------------------------------------------
#define GB_HUB_CNT 1024

__global__ void __launch_bounds__(GB_HUB_CNT)
hubRowCountKernel(Index* __restrict__ block_nonempty,
                  const Index* __restrict__ rowptr, Index nrows) {
  __shared__ int s_red[GB_HUB_CNT/32];
  const Index r = blockIdx.x*GB_HUB_CNT + threadIdx.x;
  const int flag = (r < nrows && __ldg(rowptr + r + 1) > __ldg(rowptr + r)) ? 1 : 0;
  const int total = blockSum<GB_HUB_CNT>(flag, s_red);
  if (threadIdx.x == 0) block_nonempty[blockIdx.x] = total;
}

// In place: counts -> exclusive offsets; total[0] = sum.  One CTA.
__global__ void __launch_bounds__(GB_HUB_CNT)
hubRowScanKernel(Index* __restrict__ block_nonempty, int nblocks,
                 Index* __restrict__ total) {
  __shared__ int s_scan[GB_HUB_CNT/32 + 1];
  int running = 0;
  for (int base = 0; base < nblocks; base += GB_HUB_CNT) {
    const int idx = base + threadIdx.x;
    const int v = idx < nblocks ? block_nonempty[idx] : 0;
    int sum;
    const int excl = blockExclusiveScan<GB_HUB_CNT>(v, s_scan, &sum);
    if (idx < nblocks) block_nonempty[idx] = running + excl;
    running += sum;
  }
  if (threadIdx.x == 0) total[0] = running;
}

__global__ void __launch_bounds__(GB_HUB_CNT)
hubRowEmitKernel(Index* __restrict__ ne_rows, Index* __restrict__ ne_ptr,
                 Index* __restrict__ empty_rows,
                 const Index* __restrict__ block_offset,
                 const Index* __restrict__ rowptr, Index nrows) {
  __shared__ int s_scan[GB_HUB_CNT/32 + 1];
  const Index r = blockIdx.x*GB_HUB_CNT + threadIdx.x;
  Index beg = 0;
  int flag = 0;
  if (r < nrows) {
    beg = __ldg(rowptr + r);
    flag = (__ldg(rowptr + r + 1) > beg) ? 1 : 0;
  }
  int sum;
  const int excl = blockExclusiveScan<GB_HUB_CNT>(flag, s_scan, &sum);
  if (r < nrows) {
    const Index ne_before = block_offset[blockIdx.x] + excl;
    if (flag) { ne_rows[ne_before] = r; ne_ptr[ne_before] = beg; }
    else      empty_rows[r - ne_before] = r;
  }
}

__global__ void hubRowPadKernel(Index* __restrict__ ne_rows, Index* __restrict__ ne_ptr,
                                Index m, Index nnz) {
  const int i = threadIdx.x;
  if (i < GB_HUB_PAD) { ne_rows[m + i] = -1; ne_ptr[m + i] = nnz; }
}

// ---------------------------------------------------------------------------
// Weighted merge-path partition over the compact rows.  With
// f(r) = RW*r + ne_ptr[r] (items consumed when exactly r rows are finished), tile
// boundary c sits on diagonal d = c*TILE: rows consumed = max{r : f(r) <= d},
// nonzeros consumed = min(d - RW*r, ne_ptr[r+1]) (a row end cut by the diagonal
// goes to the next tile).  bounds[2c] = rows, bounds[2c+1] = nonzeros.
// ---------------------------------------------------------------------------
__global__ void hubPartitionKernel(Index* __restrict__ bounds,
                                   const Index* __restrict__ ne_ptr,
                                   Index m, Index nnz, int ntiles) {
  const int c = blockIdx.x*blockDim.x + threadIdx.x;
  if (c > ntiles) return;
  const long long total = static_cast<long long>(GB_HUB_RW)*m + nnz;
  long long d = static_cast<long long>(c)*GB_HUB_TILE;
  if (d > total) d = total;
  long long lo = 0, hi = m;                  // largest r with f(r) <= d
  while (lo < hi) {
    const long long mid = (lo + hi + 1) >> 1;
    if (GB_HUB_RW*mid + static_cast<long long>(__ldg(ne_ptr + mid)) <= d) lo = mid;
    else hi = mid - 1;
  }
  const Index r = static_cast<Index>(lo);
  long long k = d - static_cast<long long>(GB_HUB_RW)*r;
  const long long kmax = static_cast<long long>(__ldg(ne_ptr + r + 1));   // padded
  if (k > kmax) k = kmax;
  bounds[2*c]     = r;
  bounds[2*c + 1] = static_cast<Index>(k);
}

// Compact row that holds nonzero k: smallest r with ne_ptr[r+1] > k (k < nnz).
__device__ __forceinline__ Index hubRowOf(const Index* __restrict__ ne_ptr,
                                          Index m, Index k) {
  Index lo = 0, hi = m - 1;
  while (lo < hi) {
    const Index mid = (lo + hi) >> 1;
    if (__ldg(ne_ptr + mid + 1) <= k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// One 16-byte record per tile: {r0, k0, (nr << 8) | i0, nk}; i0 = local index of
// the row that holds the tile's first nonzero (where the thread owning k0 starts).
__global__ void hubTileDescKernel(int4* __restrict__ desc,
                                  const Index* __restrict__ bounds,
                                  const Index* __restrict__ ne_ptr,
                                  Index m, int ntiles) {
  const int c = blockIdx.x*blockDim.x + threadIdx.x;
  if (c >= ntiles) return;
  const Index r0 = bounds[2*c], k0 = bounds[2*c + 1];
  const Index r1 = bounds[2*c + 2], k1 = bounds[2*c + 3];
  Index i0 = r1 - r0;                         // no nonzero in the tile: the open row
  if (k1 > k0) i0 = hubRowOf(ne_ptr, m, k0) - r0;
  desc[c] = make_int4(r0, k0, ((r1 - r0) << 8) | i0, k1 - k0);
}

// chunk_rel[c] = compact row of nonzero 8c, relative to the first row of the tile
// that contains that nonzero (<= 253 by construction of the partition).
__global__ void hubChunkRowKernel(unsigned char* __restrict__ chunk_rel,
                                  const Index* __restrict__ bounds,
                                  const Index* __restrict__ ne_ptr,
                                  Index m, Index nnz, int ntiles) {
  Index c = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  const Index nchunks = (nnz + 7) >> 3;
  for (; c < nchunks; c += stride) {
    const Index k = c << 3;
    const Index row = hubRowOf(ne_ptr, m, k);
    int lo = 0, hi = ntiles - 1;              // largest tile T with k0(T) <= k
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(bounds + 2*mid + 1) <= k) lo = mid; else hi = mid - 1;
    }
    chunk_rel[c] = static_cast<unsigned char>(row - __ldg(bounds + 2*lo));
  }
}

// ---------------------------------------------------------------------------
// Hub selection (once per matrix structure).
// ---------------------------------------------------------------------------
// cnt[col] += 1 for every stored entry.
__global__ void hubCountKernel(int* __restrict__ cnt,
                               const Index* __restrict__ colind, Index nnz) {
  Index k = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; k < nnz; k += stride) atomicAdd(cnt + __ldg(colind + k), 1);
}

// out[0] = #{c : cnt[c] >= t}, out[1] = sum of those counts.
__global__ void hubAboveKernel(unsigned long long* __restrict__ out,
                               const int* __restrict__ cnt, Index n, int t) {
  __shared__ int s_red[256/32];
  Index c = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  int num = 0;
  unsigned long long sum = 0ull;
  for (; c < n; c += stride) {
    const int v = cnt[c];
    if (v >= t) { ++num; sum += static_cast<unsigned long long>(v); }
  }
  const int total = blockSum<256>(num, s_red);
  if (threadIdx.x == 0 && total)
    atomicAdd(out, static_cast<unsigned long long>(total));
  // 64-bit sum: warp shuffle, then one atomic per warp
#pragma unroll
  for (int off = 16; off > 0; off >>= 1)
    sum += __shfl_xor_sync(GB_FULL_MASK, sum, off);
  if ((threadIdx.x & 31) == 0 && sum) atomicAdd(out + 1, sum);
}

// Columns with cnt > t take a slot unconditionally (the host chose t so that they
// fit), columns with cnt == t while slots remain.  slot[c] = hub slot or -1.
// taken[0] = slots handed out, taken[1] = references covered.
__global__ void hubAssignKernel(Index* __restrict__ slot,
                                Index* __restrict__ hub_ids,
                                unsigned long long* __restrict__ taken,
                                const int* __restrict__ cnt, Index n, int t,
                                int capacity, int pass) {
  Index c = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; c < n; c += stride) {
    const int v = cnt[c];
    if (pass == 0) {
      Index s = -1;
      if (v > t) {
        s = static_cast<Index>(atomicAdd(taken, 1ull));
        hub_ids[s] = c;
        atomicAdd(taken + 1, static_cast<unsigned long long>(v));
      }
      slot[c] = s;
    } else if (v == t && v > 0) {
      const unsigned long long s = atomicAdd(taken, 1ull);
      if (s < static_cast<unsigned long long>(capacity)) {
        hub_ids[s] = c;
        slot[c] = static_cast<Index>(s);
        atomicAdd(taken + 1, static_cast<unsigned long long>(v));
      } else {
        atomicAdd(taken, static_cast<unsigned long long>(-1ll));
      }
    }
  }
}

// enc[k] = hub slot | FLAG, or the column id itself.
__global__ void hubEncodeKernel(Index* __restrict__ enc,
                                const Index* __restrict__ colind,
                                const Index* __restrict__ slot, Index nnz) {
  Index k = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; k < nnz; k += stride) {
    const Index c = __ldg(colind + k);
    const Index s = __ldg(slot + c);
    enc[k] = (s >= 0) ? static_cast<Index>(GB_HUB_FLAG | static_cast<unsigned>(s))
                      : c;
  }
}

// Per call, one launch: hub_vals[j] = u[hub_ids[j]] (slots past the count get
// `pad`), and w[row] = identity for every empty row.
template <typename W, typename U>
__global__ void hubPrepassKernel(U* __restrict__ hub_vals,
                                 const U* __restrict__ u,
                                 const Index* __restrict__ hub_ids,
                                 int count, int capacity, U pad,
                                 W* __restrict__ w,
                                 const Index* __restrict__ empty_rows,
                                 Index nempty, W identity) {
  const Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (Index j = i; j < capacity; j += stride)
    hub_vals[j] = (j < count) ? __ldg(u + __ldg(hub_ids + j)) : pad;
  for (Index e = i; e < nempty; e += stride) w[__ldg(empty_rows + e)] = identity;
}

// ---------------------------------------------------------------------------
// Shared-memory plan of the SpMV kernel (bytes), shared by host and device.
// ---------------------------------------------------------------------------
struct HubSmemPlan {
  int hub_bytes;        // K*4
  int group_bytes;      // 3 x (row-offset window + row-id window) + scan scratch
  int bar_offset;
  int total;
};

__host__ __device__ inline HubSmemPlan hubSmemPlan(int groups, int hub_k) {
  HubSmemPlan p;
  p.hub_bytes   = hub_k*4;
  // ptr[3][RPWIN] rows[3][RPWIN] wkey[2][4] wval[2][4]
  p.group_bytes = 6*GB_HUB_RPWIN*4 + 2*32;
  p.bar_offset  = p.hub_bytes + groups*p.group_bytes;
  p.total       = p.bar_offset + 8*(3*groups + 1) + 8;
  return p;
}

// Per-matrix arrays the kernel reads besides colind/val.
struct HubTiles {
  const int4*          desc;        // [ntiles] {r0, k0, (nr << 8) | i0, nk}
  const unsigned char* chunk_rel;   // [ceil(nnz/8)]
  const Index*         ne_ptr;      // [m + PAD] first nonzero of every compact row
  const Index*         ne_rows;     // [m + PAD] row id of every compact row
  Index                m;           // non-empty rows
  int                  ntiles;
};

template <int GROUPS, int HUB_K, typename W, typename a, typename U,
          typename MulOp, typename AddOp>
__global__ void __launch_bounds__(GROUPS*GB_HUB_GT, 1)
spmvHubKernel(W* __restrict__           w,
              HubTiles                  tiles,
              Index* __restrict__       carry_row,
              W* __restrict__           carry_val,
              const Index* __restrict__ enc_colind,
              const a* __restrict__     val,
              const U* __restrict__     u,
              const U* __restrict__     hub_vals,
              Index                     nnz,
              W                         identity,
              MulOp                     mul_op,
              AddOp                     add_op) {
  static_assert(sizeof(W) == 4 && sizeof(U) == 4 && sizeof(a) == 4 &&
                sizeof(Index) == 4, "32-bit values and indices");
  extern __shared__ __align__(128) unsigned char s_raw[];
  const HubSmemPlan plan = hubSmemPlan(GROUPS, HUB_K);
  const int ntiles = tiles.ntiles;

  const int tid  = threadIdx.x;
  const int g    = tid / GB_HUB_GT;            // group in CTA
  const int t    = tid % GB_HUB_GT;            // thread in group
  const int lane = t & 31;
  const int wid  = t >> 5;                     // warp in group (0..3)

  unsigned char* const s_group = s_raw + plan.hub_bytes + g*plan.group_bytes;
  Index* const st_ptr  = reinterpret_cast<Index*>(s_group);
  Index* const st_rows = st_ptr + 3*GB_HUB_RPWIN;
  Index* const s_wkey  = st_rows + 3*GB_HUB_RPWIN;
  W*     const s_wval  = reinterpret_cast<W*>(s_wkey + 8);
  uint64_t* const s_bar = reinterpret_cast<uint64_t*>(s_raw + plan.bar_offset);
  uint64_t* const bar_hub = s_bar + 3*GROUPS;
  uint64_t* const bar_rp  = s_bar + 3*g;       // [3] for this group

  if (tid == 0) {
    for (int i = 0; i < 3*GROUPS + 1; ++i) mbarInit(s_bar + i, 1);
    mbarFenceInit();
  }
  __syncthreads();

  const uint64_t pol_stream = makeEvictFirstPolicy();
  if (tid == 0 && HUB_K > 0) {
    mbarExpectTx(bar_hub, HUB_K*4);
    bulkLoad(s_raw, hub_vals, HUB_K*4, bar_hub, makeEvictLastPolicy());
  }

  const int gg      = blockIdx.x*GROUPS + g;   // global group id
  const int gstride = gridDim.x*GROUPS;

  // Producer step (thread 0 of the group): stage ne_ptr[r0 .. r0+nr+1] and
  // ne_rows[r0 .. r0+nr] of a tile into slot b.  The windows start at r0 & ~3;
  // the arrays are padded, so whole 16-byte windows stay inside them.
  // THREE slots: the slot of tile q-1 is refilled (for tile q+2) after the group
  // barrier of tile q, when every thread has left tile q-1 for good.  With two
  // slots the refill would follow the barrier of the tile that used the slot,
  // and a row id loaded before that barrier but consumed after it can still sit
  // in the shared-memory queue behind the hub reads when the bulk copy lands
  // (showing as a handful of results written to the wrong row).
  auto issueRows = [&](int b, int4 d) {
    const Index ra = d.x & ~3;
    const uint32_t bytes =
        static_cast<uint32_t>(((d.x + (d.z >> 8) + 2 + 3) & ~3) - ra)*4u;
    mbarExpectTx(bar_rp + b, 2u*bytes);
    bulkLoad(st_ptr + b*GB_HUB_RPWIN, tiles.ne_ptr + ra, bytes, bar_rp + b, pol_stream);
    bulkLoad(st_rows + b*GB_HUB_RPWIN, tiles.ne_rows + ra, bytes, bar_rp + b, pol_stream);
  };
  auto loadDesc = [&](int tile) {
    int4 d = make_int4(0, 0, 0, 0);
    if (tile < ntiles) d = __ldg(tiles.desc + tile);
    return d;
  };
  // This thread's 8 consecutive nonzeros of a tile: 256-bit streaming loads.
  struct Chunk { Word8 ci; Word8 vb; int rel; };
  auto loadChunk = [&](int4 d) {
    Chunk c;
    const Index kbase = (d.y & ~7) + 8*t;
    c.rel = 0;
    if (kbase < d.y + d.w) {
      if (kbase + 8 <= nnz) {
        c.ci = ldStream256(enc_colind + kbase);
        c.vb = ldStream256(val + kbase);
      } else {                                 // last chunk of the arrays
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const Index k = kbase + j < nnz ? kbase + j : nnz - 1;
          c.ci.w[j] = ldStream32(enc_colind + k);
          c.vb.w[j] = ldStream32(val + k);
        }
      }
      c.rel = tiles.chunk_rel[kbase >> 3];
    }
    return c;
  };

  int tile = gg;
  int4 cur = loadDesc(tile);
  int4 nxt = loadDesc(tile + gstride);
  Chunk cc = loadChunk(cur);
  if (t == 0) {
    if (tile < ntiles) issueRows(0, cur);
    if (tile + gstride < ntiles) issueRows(1, nxt);
  }
  int slot = 0;                                // q % 3
  int phase = 0;                               // (q / 3) & 1
  if (HUB_K > 0) mbarWait(bar_hub, 0);
  const uint32_t hub_base = smemAddr(s_raw);

  for (int q = 0; tile < ntiles; ++q, tile += gstride) {
    const int b = q & 1;                       // scan scratch buffer
    const Index r0 = cur.x, k0 = cur.y;
    const int   nr = cur.z >> 8;               // rows that END in this tile
    const Index k1 = k0 + cur.w;
    const Index kbase = (k0 & ~7) + 8*t;
    const bool  busy  = kbase < k1;

    // ---- gathers: cold columns from global memory (issued first), hub slots from
    // shared memory.  Positions outside [k0, k1) belong to the neighbouring tiles:
    // they are valid codes, gathered and never used.
    U uv[8];
    if (busy) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (cc.ci.w[j] >= 0) uv[j] = __ldg(u + cc.ci.w[j]);
      if (HUB_K > 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (cc.ci.w[j] < 0) {
            int bits;
            asm volatile("ld.shared.b32 %0, [%1];"
                         : "=r"(bits)
                         : "r"(hub_base + (static_cast<uint32_t>(cc.ci.w[j]) << 2)));
            memcpy(&uv[j], &bits, 4);
          }
        }
      }
    }
    // ---- request the next tile's entries and the record of the one after ---------
    const int4 nn = loadDesc(tile + 2*gstride);
    int vb[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) vb[j] = cc.vb.w[j];
    const int rel = cc.rel;
    cc = loadChunk(nxt);

    mbarWait(bar_rp + slot, phase);
    // rowStart(i) = rp[i], rowEnd(i) = rp[i+1], row id = rows[i], local i in [0, nr]
    const Index* const rp   = st_ptr  + slot*GB_HUB_RPWIN + (r0 & 3);
    const Index* const rows = st_rows + slot*GB_HUB_RPWIN + (r0 & 3);

    // A row whose nonzeros all lie in earlier tiles can still END here (its end
    // marker was cut off by the tile boundary): it gets the identity, the carry
    // fix-up adds the rest.
    if (t == 0 && nr > 0 && rp[1] <= k0) w[rows[0]] = identity;

    // ---- this thread's range and its first row ---------------------------------
    int i = nr;                                       // idle thread: the open row
    if (busy) i = (kbase >= k0) ? rel : (cur.z & 0xff);
    const int first_i = i;
    W acc  = identity;
    W head = identity;
    // warps whose 32 chunks all lie inside [k0, k1) skip the per-entry range test
    const bool all_full = __all_sync(GB_FULL_MASK, (kbase >= k0) && (kbase + 8 <= k1));
    if (busy) {
      int d = rp[i + 1] - kbase;               // entries of this chunk before the row ends
      if (all_full) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          a av;
          memcpy(&av, &vb[j], 4);
          const W prod = mul_op(av, uv[j]);
          if (j >= d) {                        // row i ended before this entry
            if (i == first_i) head = acc; else w[rows[i]] = acc;
            acc = identity;
            ++i;
            d = rp[i + 1] - kbase;
          }
          acc = add_op(acc, prod);
        }
        if (d <= 8 && i < nr) {                // the row ends with this chunk
          if (i == first_i) head = acc; else w[rows[i]] = acc;
          acc = identity;
          ++i;
        }
      } else {
        const int jlo = (k0 > kbase) ? (k0 - kbase) : 0;
        const int jhi = (k1 - kbase < 8) ? (k1 - kbase) : 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          a av;
          memcpy(&av, &vb[j], 4);
          const W prod = mul_op(av, uv[j]);
          if (j >= jlo && j < jhi) {
            if (j >= d) {
              if (i == first_i) head = acc; else w[rows[i]] = acc;
              acc = identity;
              ++i;
              d = rp[i + 1] - kbase;
            }
            acc = add_op(acc, prod);
          }
        }
        if (d <= jhi && i < nr) {
          if (i == first_i) head = acc; else w[rows[i]] = acc;
          acc = identity;
          ++i;
        }
      }
    }

    // ---- segmented scan of (open row, partial) over the group ---------------------
    Index key = i;
    W     v   = acc;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const Index pk = __shfl_up_sync(GB_FULL_MASK, key, off);
      const W     pv = __shfl_up_sync(GB_FULL_MASK, v, off);
      if (lane >= off && pk == key) v = add_op(pv, v);
    }
    Index* const wkey = s_wkey + 4*b;
    W*     const wval = s_wval + 4*b;
    if (lane == 31) { wkey[wid] = key; wval[wid] = v; }
    const Index key0 = __shfl_sync(GB_FULL_MASK, key, 0);
    const Index ekey = __shfl_up_sync(GB_FULL_MASK, key, 1);
    const W     eval = __shfl_up_sync(GB_FULL_MASK, v, 1);
    const Index head_row = (i > first_i) ? rows[first_i] : -1;
    const Index open_row = (t == GB_HUB_GT - 1) ? rows[i] : -1;   // -1 past the last row
    groupBarrier(1 + g, GB_HUB_GT);
    // every thread of the group has left tile q-1: its slot takes tile q+2
    const int refill = (slot == 0) ? 2 : slot - 1;
    if (t == 0 && tile + 2*gstride < ntiles) issueRows(refill, nn);
    if (slot == 2) { slot = 0; phase ^= 1; } else ++slot;

    Index ck = -1;
    W     cv = identity;
#pragma unroll
    for (int ww = 0; ww < GB_HUB_GT/32 - 1; ++ww) {
      if (ww < wid) {
        const Index wk = wkey[ww];
        const W     wv = wval[ww];
        if (wk == ck) cv = add_op(cv, wv);
        else { ck = wk; cv = wv; }
      }
    }
    W carry_in;
    if (lane == 0) {
      carry_in = (ck == first_i) ? cv : identity;
    } else {
      carry_in = eval;                         // ekey == first_i always
      if (ekey == key0 && ck == ekey) carry_in = add_op(cv, eval);
    }
    if (i > first_i) w[head_row] = add_op(carry_in, head);
    if (t == GB_HUB_GT - 1) {
      const W out = (i > first_i) ? acc : add_op(carry_in, acc);
      carry_row[tile] = open_row;
      carry_val[tile] = out;
    }
    cur = nxt;
    nxt = nn;
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_SPMV_HUB_CUH_
