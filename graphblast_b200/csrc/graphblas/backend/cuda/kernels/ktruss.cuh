// graphblast_b200 backend — k-truss and truss decomposition (algorithm::ktruss,
// algorithm::trussness; host side ktruss.hpp): per-edge triangle support, then an
// edge peel with incremental support updates in ONE persistent cooperative kernel,
// grid barriers between rounds and no host wait.
//
// Graph.  The undirected simple graph G of a sorted, duplicate-free, structurally
// symmetric pattern (ptr, ind): entry p of row u with v = ind[p] is the edge {u, v};
// entries with v == u are skipped.  Each edge owns one slot, the position of its
// (min, max) entry (the CANONICAL entry); eid[p] is the slot of entry p's edge (-1 for
// a self-loop), so a triangle found from either endpoint charges the right counters.
//
// Work items.  An item (e, c) is chunk c of the intersection of e = {u, v}: entries
// [c*GB_KT_CHUNK, (c+1)*GB_KT_CHUNK) of the shorter of the two lists, each looked up in
// the longer one, so that one hub-hub edge is spread over several warps.  A warp takes
// one item at a time.  An edge whose shorter list has L entries has ceil(L/CHUNK) items.
//
// Support.  s(e) = |N(u) ∩ N(v)|: every item of every edge, integer atomicAdd of its
// warp's count, so the result does not depend on scheduling.
//
// Peel (Wang & Cheng, VLDB 2012, run in synchronous rounds).  state[e] is 0 while e is
// alive, r once e joins the frontier of round r; an edge whose state is below the
// current round is dead.  A level k takes as its first frontier the alive edges with
// s < k - 2.  Round r: for each e in F (state == r), each triangle {e, f, g} whose
// other edges are not dead; for each of f, g that is not in F, s is decremented, but
// only when e has the smallest slot among the triangle's F edges, so a triangle with
// several dying edges is charged once.  The thread whose atomicSub sees the old value
// k - 2 appends that edge to the next frontier (state r + 1), so each edge is appended
// once.  An edge appended during round r is neither in F nor dead for round r.  The
// next frontier empty, ktruss stops; trussness writes tau = k - 1 into s of each F
// edge as it goes and then takes the least support m of the alive edges and goes on
// with k = m + 3 (skipping the levels that would peel nothing) until no edge is alive.
// Supports never go below the triangle count of the remaining graph and every
// destroyed triangle is charged once, so at the end of a level s(e) is exactly the
// number of triangles of the remaining graph that contain e.
//
// Every edge joins a frontier at most once, so the frontiers lie one after another in
// one list of items (the support items' array, reused once they are counted); round r's
// frontier is [lo, hi), and its appends go to [hi, ...).  The items appended for round
// r's frontier are counted in their own cell, KT_COUNT + r % 3: it is written only
// before the barrier that opens round r, read by every thread right after it, and
// reset during round r + 2.  So every thread reads the same hi, however early it
// leaves the barrier and whatever other warps append meanwhile, and every thread runs
// the same rounds.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_KTRUSS_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_KTRUSS_CUH_

#include <climits>

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/cooperative.cuh"

namespace graphblas {
namespace backend {

#define GB_KT_NT     256               // CTA shape of the peel kernel
#define GB_KT_MINB   4                 // resident CTAs per SM the register budget allows
#define GB_KT_CHUNK  1024              // shorter-list entries one warp intersects at most
#define GB_KT_SKIP   (-1)              // state of a non-canonical entry or self-loop

enum KtCell {
  KT_COUNT      = 0,                   // [3] items of the frontier of round r, at r % 3
  KT_MIN        = 3,                   // [2] least alive support, by level parity
  KT_ROUNDS     = 5,                   // rounds that removed edges
  KT_LEVELS     = 6,                   // levels that removed edges
  KT_KMAX       = 7,                   // trussness: the largest tau
  KT_SUPPORT_US = 8,                   // the support pass, microseconds of globaltimer
  KT_NCELLS     = 9
};

struct KtArgs {
  const Index* ptr;  const Index* ind;   // the undirected pattern
  const Index* erow;                     // [nnz] the row of each entry
  const Index* eid;                      // [nnz] the slot of each entry's edge, -1 loop
  Index nnz;
  int* sup;                              // [nnz] support (tau once peeled, trussness)
  int* state;                            // [nnz] 0 alive, r frontier of round r, SKIP
  int2* items;                           // support items, then the peel list
  Index nitems;                          // support items
  int k;                                 // ktruss: k >= 2; trussness: 0
  int* cells;                            // [KT_NCELLS] KtCell
};

// The intersection items of the edge {u, v}: one per GB_KT_CHUNK of its shorter list.
__device__ __forceinline__ int ktChunksOf(const Index* ptr, Index u, Index v) {
  const Index du = __ldg(ptr + u + 1) - __ldg(ptr + u);
  const Index dv = __ldg(ptr + v + 1) - __ldg(ptr + v);
  const Index l = du < dv ? du : dv;
  return l > GB_KT_CHUNK ? static_cast<int>((l + GB_KT_CHUNK - 1)/GB_KT_CHUNK) : 1;
}

// The intersection items of the edge in canonical slot e.
__device__ __forceinline__ int ktChunks(const Index* ptr, const Index* ind,
                                        const Index* erow, Index e) {
  return ktChunksOf(ptr, __ldg(erow + e), __ldg(ind + e));
}

// One item's lists: [sb, se) the chunk of the shorter list, [lb, le) the longer list,
// u and v the edge's ends.
struct KtItem {
  Index sb, se, lb, le, u, v;
};

__device__ __forceinline__ KtItem ktItem(const KtArgs& a, Index e, int c) {
  KtItem it;
  it.u = __ldg(a.erow + e);
  it.v = __ldg(a.ind + e);
  const Index ub = __ldg(a.ptr + it.u), ue = __ldg(a.ptr + it.u + 1);
  const Index vb = __ldg(a.ptr + it.v), ve = __ldg(a.ptr + it.v + 1);
  const bool u_short = ue - ub <= ve - vb;
  const Index sb = u_short ? ub : vb, se = u_short ? ue : ve;
  it.lb = u_short ? vb : ub;
  it.le = u_short ? ve : ue;
  it.sb = sb + c*GB_KT_CHUNK;
  it.se = it.sb + GB_KT_CHUNK < se ? it.sb + GB_KT_CHUNK : se;
  return it;
}

// Whether entry j of the shorter list names a common neighbour w of u and v; then *q
// is w's entry in the longer list.  *lo is the lane's search start: the entries a lane
// visits increase, so their positions in the longer list do too.
__device__ __forceinline__ bool ktCommon(const KtArgs& a, const KtItem& it, Index j,
                                         Index* lo, Index* q) {
  const Index w = __ldg(a.ind + j);
  if (w == it.u || w == it.v) return false;
  *lo = findSorted(a.ind, *lo, it.le, w);
  *q = *lo;
  return *lo < it.le && __ldg(a.ind + *lo) == w;
}

// The lanes with `want` append edge f (with its items) to the frontier of `round`,
// which starts at item `start` of the peel list, and set its state to `round`; one
// atomic per warp on the round's count cell.  Every lane of the warp calls it.
__device__ __forceinline__ void ktAppend(const KtArgs& a, bool want, Index f, int round,
                                         Index start) {
  const int lane = threadIdx.x & 31;
  if (__ballot_sync(GB_FULL_MASK, want) == 0u) return;
  const int nch = want ? ktChunks(a.ptr, a.ind, a.erow, f) : 0;
  int incl = nch;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int t = __shfl_up_sync(GB_FULL_MASK, incl, off);
    if (lane >= off) incl += t;
  }
  const int all = __shfl_sync(GB_FULL_MASK, incl, 31);
  int base = 0;
  if (lane == 0) base = atomicAdd(a.cells + KT_COUNT + round % 3, all);
  base = start + __shfl_sync(GB_FULL_MASK, base, 0) + incl - nch;
  if (want) a.state[f] = round;
  for (int c = 0; c < nch; ++c) a.items[base + c] = make_int2(f, c);
}

// Decrements the support of f; true when f crossed below k - 2 here.
__device__ __forceinline__ bool ktDrop(const KtArgs& a, Index f, int k) {
  return atomicSub(a.sup + f, 1) == k - 2;
}

__global__ void __launch_bounds__(GB_KT_NT, GB_KT_MINB)
ktrussKernel(KtArgs a) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31;
  const Index gtid = blockIdx.x*GB_KT_NT + threadIdx.x;
  const Index gthreads = gridDim.x*GB_KT_NT;
  const Index gwarp = gtid >> 5;
  const Index gwarps = gthreads >> 5;
  const unsigned long long t0 = gtid == 0 ? globalTimerNs() : 0ull;

  // ---- support: every item of every edge ---------------------------------------------
  for (Index t = gwarp; t < a.nitems; t += gwarps) {
    const int2 e = __ldg(a.items + t);
    const KtItem it = ktItem(a, e.x, e.y);
    int count = 0;
    Index lo = it.lb, q;
    for (Index j = it.sb + lane; j < it.se; j += 32)
      count += ktCommon(a, it, j, &lo, &q) ? 1 : 0;
    count = warpReduce(count, [](int x, int y) { return x + y; });
    if (lane == 0 && count > 0) atomicAdd(a.sup + e.x, count);
  }
  grid.sync();
  if (gtid == 0) a.cells[KT_SUPPORT_US] = static_cast<int>((globalTimerNs() - t0)/1000ull);

  // ---- peel ----------------------------------------------------------------------------
  const bool truss = a.k == 0;
  int k = a.k;
  int r = 1;                            // the round about to run
  int level = 0;
  Index lo = 0;
  for (;;) {
    if (truss) {                        // the least support of the alive edges
      int m = INT_MAX;
      for (Index p = gtid; p < a.nnz; p += gthreads)
        if (__ldcg(a.state + p) == 0) {
          const int sp = __ldcg(a.sup + p);
          m = sp < m ? sp : m;
        }
      m = warpReduce(m, [](int x, int y) { return x < y ? x : y; });
      if (lane == 0 && m != INT_MAX) atomicMin(a.cells + KT_MIN + (level & 1), m);
      if (gtid == 0) a.cells[KT_MIN + ((level + 1) & 1)] = INT_MAX;
      grid.sync();
      m = loadCell(a.cells + KT_MIN + (level & 1));
      if (m == INT_MAX) break;
      k = m + 3;
    }
    // the level's first frontier: the alive edges with s < k - 2
    for (Index base = gwarp*32; base < a.nnz; base += gwarps*32) {
      const Index p = base + lane;
      const bool want = p < a.nnz && __ldcg(a.state + p) == 0 && __ldcg(a.sup + p) < k - 2;
      ktAppend(a, want, p, r, lo);
    }
    grid.sync();
    Index hi = lo + loadCell(a.cells + KT_COUNT + r % 3);
    if (hi > lo && gtid == 0) {
      a.cells[KT_LEVELS] += 1;
      a.cells[KT_KMAX] = k - 1;
    }
    while (hi > lo) {
      if (gtid == 0) a.cells[KT_COUNT + (r + 2) % 3] = 0;   // round r - 1's, read before it
      for (Index t = lo + gwarp; t < hi; t += gwarps) {
        const int2 ec = __ldcg(a.items + t);
        const Index e = ec.x;
        const KtItem it = ktItem(a, e, ec.y);
        if (truss && ec.y == 0 && lane == 0) a.sup[e] = k - 1;   // tau, final
        Index lo_l = it.lb;
        for (Index base = it.sb; base < it.se; base += 32) {
          const Index j = base + lane;
          Index q = 0;
          bool drop_f = false, drop_g = false;
          Index f = 0, g = 0;
          if (j < it.se && ktCommon(a, it, j, &lo_l, &q)) {
            f = __ldg(a.eid + j);
            g = __ldg(a.eid + q);
            const int sf = __ldcg(a.state + f), sg = __ldcg(a.state + g);
            const bool dead = (sf != 0 && sf < r) || (sg != 0 && sg < r);
            if (!dead) {
              const bool in_f = sf == r, in_g = sg == r;
              if (!in_f && (!in_g || e < g)) drop_f = ktDrop(a, f, k);
              if (!in_g && (!in_f || e < f)) drop_g = ktDrop(a, g, k);
            }
          }
          ktAppend(a, drop_f, f, r + 1, hi);
          ktAppend(a, drop_g, g, r + 1, hi);
        }
      }
      grid.sync();
      ++r;
      lo = hi;
      hi = lo + loadCell(a.cells + KT_COUNT + r % 3);
    }
    ++level;
    if (!truss) break;
  }
  if (gtid == 0) a.cells[KT_ROUNDS] = r - 1;
}

// erow, eid, state and the item count of every entry (0 unless canonical).
__global__ void __launch_bounds__(256)
ktrussPrepKernel(const Index* ptr, const Index* ind, Index n, Index nnz, Index* erow,
                 Index* eid, int* state, int* nitems) {
  for (Index p = blockIdx.x*256 + threadIdx.x; p < nnz; p += gridDim.x*256) {
    Index lo = 0, hi = n - 1;           // the largest row u with ptr[u] <= p
    while (lo < hi) {
      const Index mid = lo + (hi - lo + 1)/2;
      if (__ldg(ptr + mid) <= p) lo = mid; else hi = mid - 1;
    }
    const Index u = lo, v = __ldg(ind + p);
    erow[p] = u;
    Index slot = -1;
    if (u < v) slot = p;
    else if (u > v) slot = findSorted(ind, __ldg(ptr + v), __ldg(ptr + v + 1), u);
    eid[p] = slot;
    state[p] = u < v ? 0 : GB_KT_SKIP;
    nitems[p] = u < v ? ktChunksOf(ptr, u, v) : 0;
  }
}

// The support items of every canonical entry, from its scanned item offset.
__global__ void __launch_bounds__(256)
ktrussItemsKernel(const Index* ptr, const Index* ind, const Index* erow, const int* state,
                  const int* offset, Index nnz, int2* items) {
  for (Index p = blockIdx.x*256 + threadIdx.x; p < nnz; p += gridDim.x*256) {
    if (state[p] != 0) continue;
    const int nch = ktChunks(ptr, ind, erow, p);
    for (int c = 0; c < nch; ++c) items[offset[p] + c] = make_int2(p, c);
  }
}

// The entries of the result, one warp per row: those of every edge (keep_all), or of
// the alive ones.
__device__ __forceinline__ bool ktKeep(const Index* eid, const int* state, Index p,
                                       bool keep_all) {
  const Index e = __ldg(eid + p);
  return e >= 0 && (keep_all || __ldg(state + e) == 0);
}

__global__ void __launch_bounds__(256)
ktrussCountKernel(const Index* ptr, const Index* eid, const int* state, Index n,
                  bool keep_all, Index* count) {
  const int lane = threadIdx.x & 31;
  const Index warps = (gridDim.x*256) >> 5;
  for (Index u = (blockIdx.x*256 + threadIdx.x) >> 5; u < n; u += warps) {
    const Index b = __ldg(ptr + u), e = __ldg(ptr + u + 1);
    int kept = 0;
    for (Index p = b + lane; p < e; p += 32) kept += ktKeep(eid, state, p, keep_all) ? 1 : 0;
    kept = warpReduce(kept, [](int x, int y) { return x + y; });
    if (lane == 0) count[u] = kept;
  }
}

template <typename c>
__global__ void __launch_bounds__(256)
ktrussFillKernel(const Index* ptr, const Index* ind, const Index* eid, const int* state,
                 const int* sup, Index n, bool keep_all, const Index* rowptr,
                 Index* colind, c* val) {
  const int lane = threadIdx.x & 31;
  const Index warps = (gridDim.x*256) >> 5;
  for (Index u = (blockIdx.x*256 + threadIdx.x) >> 5; u < n; u += warps) {
    const Index b = __ldg(ptr + u), e = __ldg(ptr + u + 1);
    Index at = __ldg(rowptr + u);
    for (Index base = b; base < e; base += 32) {
      const Index p = base + lane;
      const bool keep = p < e && ktKeep(eid, state, p, keep_all);
      const unsigned int m = __ballot_sync(GB_FULL_MASK, keep);
      if (keep) {
        const Index o = at + __popc(m & ((1u << lane) - 1u));
        colind[o] = __ldg(ind + p);
        val[o] = static_cast<c>(__ldg(sup + __ldg(eid + p)));
      }
      at += __popc(m);
    }
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_KTRUSS_CUH_
