// graphblast_b200 backend — betweenness centrality (algorithm::bc; host side bc.hpp): a
// batched Brandes traversal (Brandes 2001) in the multi-source BFS style of Then et al.
// (VLDB 2014), 32 sources to a batch, one lane per source, ONE persistent cooperative
// kernel per batch with grid barriers between its phases.
//
// Semantics.  Each stored A(i,j) with i != j is an edge i -> j; self-loops and values are
// ignored.  For the sources S (a list; a repeated id counts once per entry),
//   bc[v] = sum over s in S, over t not in {s, v} reachable from s, of sigma_st(v)/sigma_st,
// sigma_st the number of shortest s -> t paths and sigma_st(v) those through v.  No
// normalisation, no halving.  sigma and the dependencies delta are fp64; the sum over
// sources is accumulated in fp64 per vertex and rounded to float once, at the end.
//
// State of a vertex v in a batch (lane s = the batch's s-th source):
//   seen[v]      the lanes that have reached v at the current depth or before;
//   fresh[p][v]  the lanes that reach v first at the level being built (p = its parity);
//   stamp[p][v]  (level << 32) | the lanes at which v lies at that level, for the last
//                level of parity p that listed v: an 8-byte word that tells a reader
//                whether, and for which lanes, v lies at a given level without loading
//                v's sigma line.  The level is 32 bits wide, so no traversal exceeds it;
//   sigma[v][32], delta[v][32]  row-major, one 256-byte line per vertex, so the lanes of
//                a warp read a neighbour's values in one coalesced access.
// Level lists.  Level d lists each vertex that some lane reaches at depth d once, as
// entries (v, chunk c, lanes, partial base): a vertex whose longer list (out or in) has
// L > GB_BC_CHUNK entries gets ceil(L / GB_BC_CHUNK) entries, chunk c covering entries
// [c*GB_BC_CHUNK, (c+1)*GB_BC_CHUNK) of whichever list a phase walks, so that a hub's
// list is spread over several warps.  All levels of a batch lie one after another in
// `entries`; level_start[d] is where level d begins.
//
// Phases (each ends at a grid barrier; a warp takes one entry at a time):
//   init      seen = 0 and stamps reset for every vertex; the sources are appended to
//             level 0 (a repeated source once, with all its lanes).
//   level 0   sigma[s][lanes] = 1, seen, stamp[0].
//   forward, level d -> d + 1:
//     discover  from the out-lists of level d: fresh[v] |= lanes(u) & ~seen[v]
//               (atomicOr, integers only); the first lane to touch v appends it to level
//               d + 1.  fresh of level d is cleared here.
//     pull      for v in level d + 1: lanes = fresh[v]; over v's in-list (the CSC, or the
//               CSR when A is symmetric), in stored order, sigma[v][s] += sigma[u][s] for
//               each u whose stamp says it lies at level d for lane s.  Then seen[v] and
//               the stamp of level d + 1.
//   backward, level d = D .. 1 (D the last level):
//               for u in level d, over u's out-list in stored order,
//               delta[u][s] += sigma[u][s] / sigma[v][s] * (1 + delta[v][s]) for each v at
//               level d + 1 for lane s; then total[u] += the sum of delta[u][s] over u's
//               lanes (a fixed xor-tree warp reduction) and u's stamp of level d is
//               written back for the level below.  Level 0 holds the sources, whose own
//               dependency is not counted, so it is not walked.
// A split list: each chunk writes its per-lane partial sums to `partial`; the warp that
// finishes last (an integer ticket) adds them in chunk order and commits.  No floating-
// point value goes through an atomic and every sum has a fixed order, so two calls give
// identical bytes.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_BC_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_BC_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/cooperative.cuh"

namespace graphblas {
namespace backend {

#define GB_BC_NT     256               // CTA shape of the traversal kernel
#define GB_BC_MINB   4                 // resident CTAs per SM the register budget allows
#define GB_BC_LANES  32                // sources per batch
#define GB_BC_CHUNK  1024              // list entries one warp walks at most
#define GB_BC_NONE   0xffffffff00000000ull   // a stamp that matches no level

enum BcCell {
  BC_ENTRIES = 0,                      // entries appended so far in the batch
  BC_PSLOTS  = 1,                      // partial slots reserved for the level being built
  BC_NCELLS  = 2
};

struct BcArgs {
  const Index* row_ptr;  const Index* row_ind;   // CSR: out-lists
  const Index* in_ptr;   const Index* in_ind;    // in-lists: the CSR again when symmetric
  Index n;
  const Index* sources;          // the call's source list; NULL: vertex i is source i
  Index first;                   // this batch's lane s takes source first + s
  int count;                     // lanes in this batch, 1..32
  unsigned int* seen;            // [n]
  unsigned int* fresh[2];        // [n] each; zero between levels of its parity
  unsigned long long* stamp[2];  // [n] each
  double* sigma;                 // [n][32]
  double* delta;                 // [n][32]
  double* total;                 // [n] the sum over the sources so far
  int4* entries;                 // (v, chunk, lanes, partial base or -1)
  Index* level_start;            // [n + 1]
  double* partial;               // [partial slots][32]
  int* ticket;                   // [partial slots] chunks done; 0 between uses
  unsigned long long* counters;  // [BC_NCELLS] BcCell
};

// The number of entries a level list gives v: one per GB_BC_CHUNK of its longer list.
__device__ __forceinline__ int bcChunks(const BcArgs& a, Index v) {
  const Index out = __ldg(a.row_ptr + v + 1) - __ldg(a.row_ptr + v);
  const Index in = __ldg(a.in_ptr + v + 1) - __ldg(a.in_ptr + v);
  const Index l = out > in ? out : in;
  return l > GB_BC_CHUNK ? static_cast<int>((l + GB_BC_CHUNK - 1)/GB_BC_CHUNK) : 1;
}

// The lanes with `want` append v (with its chunks) to the level being built, one atomic
// per warp; every lane of the warp calls it.
__device__ __forceinline__ void bcAppend(const BcArgs& a, bool want, Index v) {
  const int lane = threadIdx.x & 31;
  if (__ballot_sync(GB_FULL_MASK, want) == 0u) return;
  const int nch = want ? bcChunks(a, v) : 0;
  const int pch = nch > 1 ? nch : 0;
  int incl = nch, pincl = pch;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int t = __shfl_up_sync(GB_FULL_MASK, incl, off);
    const int pt = __shfl_up_sync(GB_FULL_MASK, pincl, off);
    if (lane >= off) { incl += t; pincl += pt; }
  }
  const int all = __shfl_sync(GB_FULL_MASK, incl, 31);
  const int pall = __shfl_sync(GB_FULL_MASK, pincl, 31);
  unsigned long long base = 0ull, pbase = 0ull;
  if (lane == 0) {
    base = atomicAdd(a.counters + BC_ENTRIES, static_cast<unsigned long long>(all));
    if (pall > 0) pbase = atomicAdd(a.counters + BC_PSLOTS, static_cast<unsigned long long>(pall));
  }
  base = __shfl_sync(GB_FULL_MASK, base, 0);
  pbase = __shfl_sync(GB_FULL_MASK, pbase, 0);
  const Index e0 = static_cast<Index>(base) + incl - nch;
  const int p0 = pch > 0 ? static_cast<int>(pbase) + pincl - pch : -1;
  for (int c = 0; c < nch; ++c) a.entries[e0 + c] = make_int4(v, c, 0, p0);
}

// Commits a warp's per-lane sum `acc` for chunk c of vertex v's entries, partial base pb:
// directly when the list is not split (pb < 0), else through the partial slots, the last
// chunk to finish adding them in chunk order.  Returns true in the warp that holds the
// final sums, which are then in *acc.
__device__ __forceinline__ bool bcGather(const BcArgs& a, double* acc, int c, int pb,
                                         Index v, int lane) {
  if (pb < 0) return true;
  const int nch = bcChunks(a, v);
  a.partial[static_cast<size_t>(pb + c)*GB_BC_LANES + lane] = *acc;
  __threadfence();
  __syncwarp();
  int done = 0;
  if (lane == 0) done = atomicAdd(a.ticket + pb, 1);
  done = __shfl_sync(GB_FULL_MASK, done, 0);
  if (done != nch - 1) return false;
  __threadfence();
  double sum = 0.0;
  for (int k = 0; k < nch; ++k)
    sum += __ldcg(a.partial + static_cast<size_t>(pb + k)*GB_BC_LANES + lane);
  if (lane == 0) a.ticket[pb] = 0;
  *acc = sum;
  return true;
}

// [cb, ce): chunk c of the list [b, e).
__device__ __forceinline__ void bcChunk(Index b, Index e, int c, Index* cb, Index* ce) {
  *cb = b + c*GB_BC_CHUNK;
  *ce = *cb + GB_BC_CHUNK < e ? *cb + GB_BC_CHUNK : e;
}

// The lanes of v's stamp in `stamp` when it names `level`, else 0.
__device__ __forceinline__ unsigned int bcLanesAt(const unsigned long long* stamp, Index v,
                                                  unsigned int level) {
  const unsigned long long st = __ldcg(stamp + v);
  return static_cast<unsigned int>(st >> 32) == level ? static_cast<unsigned int>(st) : 0u;
}

__global__ void __launch_bounds__(GB_BC_NT, GB_BC_MINB)
bcKernel(BcArgs a) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31;
  const Index gtid = blockIdx.x*GB_BC_NT + threadIdx.x;
  const Index gthreads = gridDim.x*GB_BC_NT;
  const Index gwarp = gtid >> 5;
  const Index gwarps = gthreads >> 5;
  const unsigned int me = 1u << lane;

  // ---- init: reset, and the sources into level 0 ---------------------------------------
  for (Index v = gtid; v < a.n; v += gthreads) {
    a.seen[v] = 0u;
    a.stamp[0][v] = GB_BC_NONE;
    a.stamp[1][v] = GB_BC_NONE;
  }
  if (gwarp == 0) {
    bool want = false;
    Index s = 0;
    if (lane < a.count) {
      s = a.sources != NULL ? __ldg(a.sources + a.first + lane) : a.first + lane;
      want = atomicOr(a.fresh[0] + s, me) == 0u;
    }
    bcAppend(a, want, s);
  }
  grid.sync();

  Index lo = 0;
  Index hi = static_cast<Index>(loadCell(a.counters + BC_ENTRIES));
  if (gtid == 0) {
    a.level_start[0] = 0;
    a.counters[BC_PSLOTS] = 0ull;
  }
  for (Index k = gwarp; k < hi; k += gwarps) {
    const int4 e = __ldcg(a.entries + k);
    const unsigned int lanes = __ldcg(a.fresh[0] + e.x);
    if (lane == 0) a.entries[k].z = static_cast<int>(lanes);
    if (e.y != 0) continue;
    if (lanes & me) a.sigma[static_cast<size_t>(e.x)*GB_BC_LANES + lane] = 1.0;
    if (lane == 0) {
      a.seen[e.x] = lanes;
      a.stamp[0][e.x] = static_cast<unsigned long long>(lanes);
    }
  }
  grid.sync();

  // ---- forward ----------------------------------------------------------------------------
  unsigned int d = 0;
  for (;; ++d) {
    // discover level d + 1 from the out-lists of level d
    unsigned int* fresh_next = a.fresh[(d + 1) & 1];
    for (Index k = lo + gwarp; k < hi; k += gwarps) {
      const int4 e = __ldcg(a.entries + k);
      const unsigned int lanes = static_cast<unsigned int>(e.z);
      if (e.y == 0 && lane == 0) a.fresh[d & 1][e.x] = 0u;
      Index cb, ce;
      bcChunk(__ldg(a.row_ptr + e.x), __ldg(a.row_ptr + e.x + 1), e.y, &cb, &ce);
      for (Index base = cb; base < ce; base += 32) {
        const Index j = base + lane;
        Index v = 0;
        bool want = false;
        if (j < ce) {
          v = __ldg(a.row_ind + j);
          const unsigned int bits = lanes & ~__ldcg(a.seen + v);
          if (bits != 0u && (__ldcg(fresh_next + v) & bits) != bits)
            want = atomicOr(fresh_next + v, bits) == 0u;
        }
        bcAppend(a, want, v);
      }
    }
    grid.sync();
    const Index next = static_cast<Index>(loadCell(a.counters + BC_ENTRIES));
    if (next == hi) break;
    if (gtid == 0) {
      a.level_start[d + 1] = hi;
      a.counters[BC_PSLOTS] = 0ull;    // level d + 1's slots are assigned; d + 2's start at 0
    }

    // pull the path counts of level d + 1 from the in-lists
    const unsigned long long* stamp_d = a.stamp[d & 1];
    for (Index k = hi + gwarp; k < next; k += gwarps) {
      const int4 e = __ldcg(a.entries + k);
      const Index v = e.x;
      const unsigned int lanes = __ldcg(fresh_next + v);
      if (lane == 0) a.entries[k].z = static_cast<int>(lanes);
      const Index ib = __ldg(a.in_ptr + v), ie = __ldg(a.in_ptr + v + 1);
      Index cb, ce;
      bcChunk(ib, ie, e.y, &cb, &ce);
      double acc = 0.0;
      for (Index base = cb; base < ce; base += 32) {
        const Index j = base + lane;
        Index u = 0;
        unsigned int m = 0u;
        if (j < ce) {
          u = __ldg(a.in_ind + j);
          m = bcLanesAt(stamp_d, u, d) & lanes;
        }
        unsigned int any = __ballot_sync(GB_FULL_MASK, m != 0u);
        while (any != 0u) {
          const int src = __ffs(any) - 1;
          any &= any - 1u;
          const Index uu = __shfl_sync(GB_FULL_MASK, u, src);
          const unsigned int mm = __shfl_sync(GB_FULL_MASK, m, src);
          if (mm & me) acc += __ldcg(a.sigma + static_cast<size_t>(uu)*GB_BC_LANES + lane);
        }
      }
      if (e.y == 0 && lane == 0) {
        a.seen[v] = __ldcg(a.seen + v) | lanes;
        a.stamp[(d + 1) & 1][v] = (static_cast<unsigned long long>(d + 1) << 32) | lanes;
      }
      if (bcGather(a, &acc, e.y, e.w, v, lane) && (lanes & me))
        a.sigma[static_cast<size_t>(v)*GB_BC_LANES + lane] = acc;
    }
    grid.sync();
    lo = hi;
    hi = next;
  }
  if (gtid == 0) a.level_start[d + 1] = hi;
  grid.sync();

  // ---- backward: levels d .. 1 ------------------------------------------------------------
  for (; d >= 1; --d) {
    const Index b0 = __ldcg(a.level_start + d), b1 = __ldcg(a.level_start + d + 1);
    const unsigned long long* stamp_next = a.stamp[(d + 1) & 1];
    for (Index k = b0 + gwarp; k < b1; k += gwarps) {
      const int4 e = __ldcg(a.entries + k);
      const Index u = e.x;
      const unsigned int lanes = static_cast<unsigned int>(e.z);
      const bool mine = (lanes & me) != 0u;
      const double su = mine ? __ldcg(a.sigma + static_cast<size_t>(u)*GB_BC_LANES + lane) : 0.0;
      Index cb, ce;
      bcChunk(__ldg(a.row_ptr + u), __ldg(a.row_ptr + u + 1), e.y, &cb, &ce);
      double acc = 0.0;
      for (Index base = cb; base < ce; base += 32) {
        const Index j = base + lane;
        Index v = 0;
        unsigned int m = 0u;
        if (j < ce) {
          v = __ldg(a.row_ind + j);
          m = bcLanesAt(stamp_next, v, d + 1) & lanes;
        }
        unsigned int any = __ballot_sync(GB_FULL_MASK, m != 0u);
        while (any != 0u) {
          const int src = __ffs(any) - 1;
          any &= any - 1u;
          const Index vv = __shfl_sync(GB_FULL_MASK, v, src);
          const unsigned int mm = __shfl_sync(GB_FULL_MASK, m, src);
          if (mm & me) {
            const size_t at = static_cast<size_t>(vv)*GB_BC_LANES + lane;
            acc += __ddiv_rn(su, __ldcg(a.sigma + at))*(1.0 + __ldcg(a.delta + at));
          }
        }
      }
      if (e.y == 0 && lane == 0)          // u's level-d stamp, for level d - 1
        a.stamp[d & 1][u] = (static_cast<unsigned long long>(d) << 32) | lanes;
      if (bcGather(a, &acc, e.y, e.w, u, lane)) {
        if (mine) a.delta[static_cast<size_t>(u)*GB_BC_LANES + lane] = acc;
        const double sum = warpReduce(mine ? acc : 0.0,
                                      [](double x, double y) { return x + y; });
        if (lane == 0) a.total[u] = __ldcg(a.total + u) + sum;
      }
    }
    grid.sync();
  }
  if (gtid == 0) {
    a.counters[BC_ENTRIES] = 0ull;
    a.counters[BC_PSLOTS] = 0ull;
  }
}

// bc[v] = float(total[v]), rounded once.
__global__ void __launch_bounds__(256)
bcFinishKernel(const double* total, Index n, float* bc) {
  for (Index v = blockIdx.x*256 + threadIdx.x; v < n; v += gridDim.x*256)
    bc[v] = __double2float_rn(total[v]);
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_BC_CUH_
