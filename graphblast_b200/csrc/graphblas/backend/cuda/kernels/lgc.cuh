// graphblast_b200 backend — local graph clustering (algorithm::lgc; host side lgc.hpp):
// the approximate personalised PageRank push of Andersen, Chung and Lang on the lazy
// walk, pushed synchronously, as ONE persistent cooperative kernel with grid barriers
// between its phases, and the kernels of the conductance sweep cut over its result.
//
// Semantics (the reference's CPU checker SimpleReferenceLgc<float>, test_lgc.hpp, as
// its C++ evaluates it: alpha and eps are double, vectors are float).  d[v] = float(the
// row length of v); p = 0, r = 0, r[s] = 1, F = {s}; while F is not empty and fewer than
// max_rounds rounds have run:
//   for v in F:  p[v]  = float(double(p[v]) + alpha*double(r[v]))      (no FMA)
//                nr[v] = float((1 - alpha)*double(r[v])/2)
//   r2 = r;  r2[v] = nr[v] for v in F
//   for every w, over the v in F with A(v,w) stored, in ascending v:
//                r2[w] = r2[w] + float(nr[v]/d[v])                      (fp32 add, divide)
//   r = r2;  F = {v : double(r[v]) >= double(d[v])*eps}, less the no-op vertices with
//   d[v] = 0 and r[v] = 0.
// The reference's loop runs its max_niter rounds whatever F holds; once F is empty they
// change nothing, so stopping there gives the same floats.
//
// Determinism: the sums are pulled, never pushed with atomics.  A round is
//   A  every v in F (a list) updates p[v], sets r[v] = nr[v] and c[v] = float(nr[v]/d[v])
//      and stamps in_f[v] = round;
//   -- grid barrier --
//   B  every w that can change walks its in-list (the CSR row when A is symmetric, else
//      the CSC column) in stored order, adding c[v] for each v with in_f[v] == round to
//      r[w], commits r[w] and, when w meets the frontier test, appends it to the next
//      frontier list with its degree added to that frontier's volume;
//   -- grid barrier --
// Phase B reads only c[] and in_f[] of other vertices, so w commits its own r[w] in
// place.  The order of the frontier and touched lists (atomic appends) changes nothing:
// each vertex's update reads only its own words and its in-list.  With sorted column
// lists the in-list order is ascending v, the reference's order; an adopted CSR or CSC
// with unsorted lists gives a deterministic result in stored order instead.
//   Every value is non-negative, so adding +0.0f leaves a sum's bits alone: a warp
//   walking a long in-list loads GB_LGC_UNROLL chunks of 32 entries at once, then adds
//   each lane's contribution (0 for a non-member) chunk by chunk in lane order.
//
// Routes (which vertices phase B visits; both give the same bits):
//   sparse  phase A also claims v and its out-neighbours, T = F + N(F), once per round
//           by a round stamp in claim[] (nothing to clear), into the touched list; B
//           walks T.  Cost: vol(F) + the in-degree of T.
//   dense   B walks every row.  Cost: nnz, no claims.
// mode 1 (PUSHONLY) forces sparse rounds, mode 2 (PULLONLY) dense ones, mode 0 takes a
// dense round when the frontier's volume exceeds switchpoint * nnz.
//
// Lists of GB_LGC_WARP_MIN entries or more (in phase A the out-list, in phase B the
// in-list) take the whole warp, shorter ones a lane.
//
// Counter cells (64-bit, counters[]): the frontier count and volume of round k in
// cells k % 3 (three sets, so that the set of round k + 2 can be cleared during round k
// with no reader left), the touched count of round k in cell k % 2, then the rounds
// run, the total volume pushed and the number of dense rounds.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_LGC_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_LGC_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/common.cuh"

namespace graphblas {
namespace backend {

#define GB_LGC_NT        256           // CTA shape of the push kernel
#define GB_LGC_MINB      4             // resident CTAs per SM the register budget allows
#define GB_LGC_WARP_MIN  32            // shortest list the whole warp takes
#define GB_LGC_UNROLL    8             // 32-entry chunks of a warp's in-list per step

enum LgcCell {
  LGC_FCOUNT = 0,                      // [3] frontier size of round k in cell k % 3
  LGC_FVOL   = 3,                      // [3] frontier volume of round k in cell k % 3
  LGC_TCOUNT = 6,                      // [2] touched list size of round k in cell k % 2
  LGC_ROUNDS = 8,                      // rounds run
  LGC_PUSHED = 9,                      // sum over the rounds of the frontier volume
  LGC_DENSE  = 10,                     // rounds that took the dense route
  LGC_NCELLS = 11
};

struct LgcArgs {
  const Index* row_ptr;  const Index* row_ind;   // CSR: out-lists and degrees
  const Index* in_ptr;   const Index* in_ind;    // in-lists: the CSR again when symmetric
  Index n;
  Index source;
  long long nnz;
  double alpha, eps;
  int max_rounds;
  int mode;                      // 0 choose per round, 1 sparse only, 2 dense only
  float switchpoint;
  float* p;                      // [n] result
  float* r;                      // [n] residual
  float* c;                      // [n] c[v] = nr[v]/d[v] of the round's frontier
  int* in_f;                     // [n] the last round v was in the frontier, or -1
  int* claim;                    // [n] the last round v was in the touched set, or -1
  Index* front[2];               // [n] frontier lists of even and odd rounds
  Index* touched;                // [n] the touched list of a sparse round
  unsigned long long* counters;  // [LGC_NCELLS] LgcCell
};

__device__ __forceinline__ unsigned long long lgcCell(const LgcArgs& a, int cell) {
  return *reinterpret_cast<volatile unsigned long long*>(a.counters + cell);
}

// The lanes with `want` append x to list at counter *count, one atomic per warp; every
// lane of the warp calls it.  Returns nothing; *count grows by the number of wanting lanes.
__device__ __forceinline__ void lgcAppend(bool want, Index x, Index* list,
                                          unsigned long long* count) {
  const int lane = threadIdx.x & 31;
  const unsigned int m = __ballot_sync(GB_FULL_MASK, want);
  if (m == 0u) return;
  const int leader = __ffs(m) - 1;
  unsigned long long base = 0ull;
  if (lane == leader) base = atomicAdd(count, static_cast<unsigned long long>(__popc(m)));
  base = __shfl_sync(GB_FULL_MASK, base, leader);
  if (want) list[base + __popc(m & ((1u << lane) - 1u))] = x;
}

// Claims w for round k (want lanes only); the first claim appends it to the touched list.
__device__ __forceinline__ void lgcClaim(const LgcArgs& a, bool want, Index w, int k) {
  bool mine = false;
  if (want && __ldcg(a.claim + w) != k) mine = atomicExch(a.claim + w, k) != k;
  lgcAppend(mine, w, a.touched, a.counters + LGC_TCOUNT + (k & 1));
}

// Phase A for the frontier vertex v (valid lanes): the p and r updates and c[v].
__device__ __forceinline__ void lgcSettle(const LgcArgs& a, Index v, int k, double oma) {
  const float rv = __ldcg(a.r + v);
  const double rd = static_cast<double>(rv);
  a.p[v] = __double2float_rn(__dadd_rn(static_cast<double>(__ldcg(a.p + v)),
                                       __dmul_rn(a.alpha, rd)));
  const float nr = __double2float_rn(__dmul_rn(__dmul_rn(oma, rd), 0.5));
  const Index d = __ldg(a.row_ptr + v + 1) - __ldg(a.row_ptr + v);
  a.r[v] = nr;
  a.c[v] = d > 0 ? __fdiv_rn(nr, __int2float_rn(d)) : 0.f;
  a.in_f[v] = k;
}

// The contribution of in-list entry v in round k: c[v] when v is in the frontier, else 0.
__device__ __forceinline__ float lgcTerm(const LgcArgs& a, Index v, int k) {
  return __ldcg(a.in_f + v) == k ? __ldcg(a.c + v) : 0.f;
}

template <bool Dense>
__device__ __forceinline__ void lgcPull(const LgcArgs& a, int k, Index items,
                                        Index gwarp, Index gwarps, int lane) {
  const Index* list = a.touched;
  Index* next = a.front[(k + 1) & 1];
  unsigned long long* ncount = a.counters + LGC_FCOUNT + (k + 1) % 3;
  unsigned long long* nvol = a.counters + LGC_FVOL + (k + 1) % 3;
  for (Index i0 = gwarp*32; i0 < items; i0 += gwarps*32) {
    const Index i = i0 + lane;
    const bool valid = i < items;
    Index w = 0, b = 0, e = 0;
    float acc = 0.f;
    if (valid) {
      w = Dense ? i : __ldcg(list + i);
      b = __ldg(a.in_ptr + w);
      e = __ldg(a.in_ptr + w + 1);
      acc = __ldcg(a.r + w);
    }
    const bool heavy_v = e - b >= GB_LGC_WARP_MIN;
    if (!heavy_v)
      for (Index j = b; j < e; ++j) acc = acc + lgcTerm(a, __ldg(a.in_ind + j), k);
    unsigned int heavy = __ballot_sync(GB_FULL_MASK, heavy_v);
    while (heavy != 0u) {
      const int src = __ffs(heavy) - 1;
      heavy &= heavy - 1u;
      const Index hb = __shfl_sync(GB_FULL_MASK, b, src);
      const Index he = __shfl_sync(GB_FULL_MASK, e, src);
      float sum = __shfl_sync(GB_FULL_MASK, acc, src);
      // GB_LGC_UNROLL 32-entry chunks per step: every load of a step is issued before
      // its first add, so the latency of one chunk's in_ind -> in_f -> c chain overlaps
      // the others'; the adds then run chunk by chunk, lane by lane, in list order.
      for (Index base = hb; base < he; base += 32*GB_LGC_UNROLL) {
        Index v[GB_LGC_UNROLL];
        int f[GB_LGC_UNROLL];
        float t[GB_LGC_UNROLL];
#pragma unroll
        for (int u = 0; u < GB_LGC_UNROLL; ++u) {
          const Index j = base + u*32 + lane;
          v[u] = j < he ? __ldg(a.in_ind + j) : -1;
        }
#pragma unroll
        for (int u = 0; u < GB_LGC_UNROLL; ++u) f[u] = v[u] >= 0 ? __ldcg(a.in_f + v[u]) : -1;
#pragma unroll
        for (int u = 0; u < GB_LGC_UNROLL; ++u) t[u] = f[u] == k ? __ldcg(a.c + v[u]) : 0.f;
#pragma unroll
        for (int u = 0; u < GB_LGC_UNROLL; ++u) {
          if (__ballot_sync(GB_FULL_MASK, t[u] != 0.f) == 0u) continue;
#pragma unroll
          for (int l = 0; l < 32; ++l) sum = sum + __shfl_sync(GB_FULL_MASK, t[u], l);
        }
      }
      if (lane == src) acc = sum;
    }
    bool in_next = false;
    Index d = 0;
    if (valid) {
      a.r[w] = acc;
      d = __ldg(a.row_ptr + w + 1) - __ldg(a.row_ptr + w);
      in_next = static_cast<double>(acc) >= __dmul_rn(static_cast<double>(__int2float_rn(d)),
                                                      a.eps) &&
                !(d == 0 && acc == 0.f);
    }
    lgcAppend(in_next, w, next, ncount);
    unsigned long long vol = in_next ? static_cast<unsigned long long>(d) : 0ull;
    vol = __reduce_add_sync(GB_FULL_MASK, static_cast<unsigned int>(vol));
    if (lane == 0 && vol != 0ull) atomicAdd(nvol, vol);
  }
}

__global__ void __launch_bounds__(GB_LGC_NT, GB_LGC_MINB)
lgcKernel(LgcArgs a) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31;
  const Index gtid = blockIdx.x*GB_LGC_NT + threadIdx.x;
  const Index gthreads = gridDim.x*GB_LGC_NT;
  const Index gwarp = gtid >> 5;
  const Index gwarps = gthreads >> 5;
  const double oma = __dadd_rn(1.0, -a.alpha);

  // ---- init: p = 0, r = the source's unit vector, F_0 = {s} ---------------------------
  for (Index v = gtid; v < a.n; v += gthreads) {
    a.p[v] = 0.f;
    a.r[v] = v == a.source ? 1.f : 0.f;
    a.in_f[v] = -1;
    a.claim[v] = -1;
  }
  if (gtid == 0) {
    a.front[0][0] = a.source;
    a.counters[LGC_FCOUNT] = 1ull;
    a.counters[LGC_FVOL] = static_cast<unsigned long long>(
        __ldg(a.row_ptr + a.source + 1) - __ldg(a.row_ptr + a.source));
  }
  grid.sync();

  int k = 0;
  for (; k < a.max_rounds; ++k) {
    const Index nf = static_cast<Index>(lgcCell(a, LGC_FCOUNT + k % 3));
    if (nf == 0) break;
    const unsigned long long vol = lgcCell(a, LGC_FVOL + k % 3);
    const bool dense = a.mode == 2 ||
        (a.mode == 0 && static_cast<double>(vol) >
                        static_cast<double>(a.switchpoint)*static_cast<double>(a.nnz));
    if (gtid == 0) {                   // cells whose last reader is behind a barrier
      a.counters[LGC_FCOUNT + (k + 2) % 3] = 0ull;
      a.counters[LGC_FVOL + (k + 2) % 3] = 0ull;
      a.counters[LGC_TCOUNT + ((k + 1) & 1)] = 0ull;
      a.counters[LGC_PUSHED] += vol;
      a.counters[LGC_DENSE] += dense ? 1ull : 0ull;
    }

    // ---- A: settle the frontier; a sparse round also claims F + N(F) ------------------
    const Index* F = a.front[k & 1];
    for (Index i0 = gwarp*32; i0 < nf; i0 += gwarps*32) {
      const Index i = i0 + lane;
      const bool valid = i < nf;
      const Index v = valid ? __ldcg(F + i) : 0;
      if (valid) lgcSettle(a, v, k, oma);
      if (dense) continue;
      lgcClaim(a, valid, v, k);
      Index b = 0, e = 0;
      if (valid) { b = __ldg(a.row_ptr + v); e = __ldg(a.row_ptr + v + 1); }
      const bool heavy_v = e - b >= GB_LGC_WARP_MIN;
      if (heavy_v) e = b;
      // the short lists, one entry per lane per step
      const Index most = static_cast<Index>(__reduce_max_sync(GB_FULL_MASK,
                                                              static_cast<unsigned int>(e - b)));
      for (Index j = 0; j < most; ++j)
        lgcClaim(a, b + j < e, b + j < e ? __ldg(a.row_ind + b + j) : 0, k);
      unsigned int heavy = __ballot_sync(GB_FULL_MASK, heavy_v);
      while (heavy != 0u) {
        const int src = __ffs(heavy) - 1;
        heavy &= heavy - 1u;
        const Index hv = __shfl_sync(GB_FULL_MASK, v, src);
        const Index hb = __ldg(a.row_ptr + hv);
        const Index he = __ldg(a.row_ptr + hv + 1);
        for (Index base = hb; base < he; base += 32) {
          const Index j = base + lane;
          lgcClaim(a, j < he, j < he ? __ldg(a.row_ind + j) : 0, k);
        }
      }
    }
    grid.sync();

    // ---- B: pull, commit, next frontier ----------------------------------------------
    if (dense)
      lgcPull<true>(a, k, a.n, gwarp, gwarps, lane);
    else
      lgcPull<false>(a, k, static_cast<Index>(lgcCell(a, LGC_TCOUNT + (k & 1))),
                     gwarp, gwarps, lane);
    grid.sync();
  }
  if (gtid == 0) a.counters[LGC_ROUNDS] = static_cast<unsigned long long>(k);
}

// ---- sweep cut --------------------------------------------------------------------------
// U = {v : p[v] > 0 and d[v] > 0}, ordered by p[v]/d[v] (fp32) descending, ties by
// ascending id: key (~bits(p[v]/d[v]) << 32) | v, sorted ascending.  The key is a
// positive float, whose bits order as unsigned integers.

#define GB_SWEEP_NT 256

__global__ void __launch_bounds__(GB_SWEEP_NT)
lgcSweepKeysKernel(const float* p, const Index* row_ptr, Index n, unsigned long long* keys,
                   unsigned long long* count, Index* rank) {
  const Index stride = gridDim.x*GB_SWEEP_NT;
  for (Index i0 = blockIdx.x*GB_SWEEP_NT + (threadIdx.x & ~31); i0 < n; i0 += stride) {
    const Index v = i0 + (threadIdx.x & 31);
    bool in = false;
    unsigned long long key = 0ull;
    if (v < n) {
      rank[v] = 0x7fffffff;
      const Index d = __ldg(row_ptr + v + 1) - __ldg(row_ptr + v);
      const float pv = p != NULL ? p[v] : 0.f;       // p NULL: p holds no entry
      in = pv > 0.f && d > 0;
      if (in) {
        const unsigned int bits = __float_as_uint(__fdiv_rn(pv, __int2float_rn(d)));
        key = (static_cast<unsigned long long>(~bits) << 32) | static_cast<unsigned int>(v);
      }
    }
    const int lane = threadIdx.x & 31;
    const unsigned int m = __ballot_sync(GB_FULL_MASK, in);
    if (m == 0u) continue;
    const int leader = __ffs(m) - 1;
    unsigned long long base = 0ull;
    if (lane == leader) base = atomicAdd(count, static_cast<unsigned long long>(__popc(m)));
    base = __shfl_sync(GB_FULL_MASK, base, leader);
    if (in) keys[base + __popc(m & ((1u << lane) - 1u))] = key;
  }
}

__global__ void __launch_bounds__(GB_SWEEP_NT)
lgcSweepRankKernel(const unsigned long long* keys, Index m, Index* rank) {
  for (Index k = blockIdx.x*GB_SWEEP_NT + threadIdx.x; k < m; k += gridDim.x*GB_SWEEP_NT)
    rank[static_cast<unsigned int>(keys[k])] = k;
}

// The number of entries of list [b, e) of `ind` ranked before k, and the self-loops.
__device__ __forceinline__ void lgcSweepCount(const Index* ind, Index b, Index e, Index v,
                                              Index k, const Index* rank, int* before,
                                              int* self) {
  for (Index j = b; j < e; ++j) {
    const Index u = __ldg(ind + j);
    *self += u == v;
    *before += u != v && __ldg(rank + u) < k;
  }
}

// Position k of the order, vertex v: dcut[k] = d(v) - self(v) - out_before - in_before,
// dvol[k] = d(v).  A warp per position; a symmetric A (in_ptr NULL) counts once, twice.
__global__ void __launch_bounds__(GB_SWEEP_NT)
lgcSweepDeltaKernel(const unsigned long long* keys, Index m, const Index* row_ptr,
                    const Index* row_ind, const Index* in_ptr, const Index* in_ind,
                    const Index* rank, long long* dcut, long long* dvol) {
  const int lane = threadIdx.x & 31;
  const Index warps = gridDim.x*(GB_SWEEP_NT/32);
  for (Index k = blockIdx.x*(GB_SWEEP_NT/32) + (threadIdx.x >> 5); k < m; k += warps) {
    const Index v = static_cast<Index>(static_cast<unsigned int>(keys[k]));
    const Index b = __ldg(row_ptr + v), e = __ldg(row_ptr + v + 1);
    int out_before = 0, self = 0, in_before = 0, in_self = 0;
    for (Index j = b + lane; j < e; j += 32) lgcSweepCount(row_ind, j, j + 1, v, k, rank,
                                                           &out_before, &self);
    if (in_ptr != NULL) {
      const Index ib = __ldg(in_ptr + v), ie = __ldg(in_ptr + v + 1);
      for (Index j = ib + lane; j < ie; j += 32) lgcSweepCount(in_ind, j, j + 1, v, k, rank,
                                                               &in_before, &in_self);
    }
    out_before = __reduce_add_sync(GB_FULL_MASK, out_before);
    self = __reduce_add_sync(GB_FULL_MASK, self);
    in_before = in_ptr != NULL ? __reduce_add_sync(GB_FULL_MASK, in_before) : out_before;
    if (lane == 0) {
      dcut[k] = static_cast<long long>(e - b) - self - out_before - in_before;
      dvol[k] = static_cast<long long>(e - b);
    }
  }
}

// best[0] = min over the qualifying prefixes of phi's bits (phi >= 0 orders as its bits);
// with Second, best[1] = the smallest k whose phi has those bits.
template <bool Second>
__global__ void __launch_bounds__(GB_SWEEP_NT)
lgcSweepBestKernel(const long long* cut, const long long* vol, Index m, long long nnz,
                   unsigned long long* best) {
  for (Index k = blockIdx.x*GB_SWEEP_NT + threadIdx.x; k < m; k += gridDim.x*GB_SWEEP_NT) {
    const long long vk = vol[k];
    const long long den = vk < nnz - vk ? vk : nnz - vk;
    if (den <= 0) continue;
    const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(
        __ddiv_rn(static_cast<double>(cut[k]), static_cast<double>(den))));
    if (!Second) atomicMin(best, bits);
    else if (bits == best[0]) atomicMin(best + 1, static_cast<unsigned long long>(k));
  }
}

__global__ void __launch_bounds__(GB_SWEEP_NT)
lgcSweepOutKernel(const Index* rank, Index n, Index size, float* cluster) {
  for (Index v = blockIdx.x*GB_SWEEP_NT + threadIdx.x; v < n; v += gridDim.x*GB_SWEEP_NT)
    cluster[v] = rank[v] < size ? 1.f : 0.f;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_LGC_CUH_
