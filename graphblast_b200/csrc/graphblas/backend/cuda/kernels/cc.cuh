// graphblast_b200 backend — connected components as ONE persistent cooperative kernel
// (algorithm::cc; host side cc.hpp): Afforest (Sutton, Ben-Nun and Barak, IPDPS 2018),
// union-find over the pattern of A with grid barriers between its phases.
//
// Semantics.  i and j are joined when A(i,j) or A(j,i) is stored (stored zeros count,
// self-loops are ignored, values are never read).  out[i] = the smallest vertex id in
// the weakly connected component of i; counters[CC_COMPONENTS] = the number of
// components, the number of i with out[i] == i.  Only the CSR is read: union-find
// joins both ends of each stored entry, so a non-symmetric A needs no CSC.
//
// Forest.  parent[x] <= x for every x, and x is a root iff parent[x] == x.  A word only
// ever changes to a smaller vertex of x's tree:
//   link(u, v) — finds the roots p, q of u and v and hooks the larger under the smaller,
//     ONLY by atomicCAS(&parent[hi], hi, lo) on a word that still holds its own index;
//     a failed CAS means hi was hooked meanwhile, and link goes on from the new roots.
//     Never atomicMin: lowering a word that is no longer a root cuts its subtree off
//     the tree it was in.
//   find(x) — walks to the root, halving the path by CAS (parent[x]: p -> grandparent g,
//     only if it still holds p); g is in x's tree, so no tree is cut.
//   compress — parent[v] = root(v), plain (relaxed) stores, between grid barriers with
//     no link in flight.
// parent[] is read with ldRelaxed: other SMs hook and halve it while the kernel runs
// (the memory model of cooperative.cuh).
//
// Phases (grid barriers between them):
//   init      parent[v] = v.
//   rounds    r = 0, 1: every v with more than r entries links (v, colind[rowptr[v]+r]);
//             each round is followed by a compress.
//   sample    symmetric A only: CTA 0 counts the roots of GB_CC_SAMPLES hashed vertices
//             in shared memory and publishes the most frequent one, L, in CC_LARGEST.
//   finish    every v links its entries from position 2 on, except, for a symmetric A,
//             a v whose parent reads L (already in L's tree; each of its edges to a
//             vertex outside L's tree is the other end's entry, linked from there).
//             Remaining lists of fewer than GB_CC_LANE_MAX entries take a lane each,
//             longer ones the whole warp, and lists of GB_CC_GRID_MIN entries or more
//             are queued for the grid pass.
//   grid pass after a grid barrier, the whole grid links the queued lists: they are
//             cut into 32-entry chunks, numbered across all queued lists, and warp w
//             takes the chunks c with c % warps == w.  R-MAT hubs sit at low ids, so
//             one warp would otherwise own many of them (measured, DESIGN §4.15).
//   out       out[i] = (W) root(i), a read-only walk to the root (the last compress,
//             fused with the write), and a warp-reduced count of roots.
// With no stored entries (row_ptr NULL) only init and out run: out[i] = i.
//
// Determinism.  Each successful CAS joins two trees of one component, and trees never
// split, so at the end each component is one tree.  Its root is the only vertex whose
// parent is itself, and since parent[x] <= x along every path, it is the component's
// minimum.  Launch shape, timing and L change only how the trees get there.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_CC_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_CC_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/cooperative.cuh"

namespace graphblas {
namespace backend {

#define GB_CC_NT        512            // CTA shape of the components kernel
#define GB_CC_MINB      2              // resident CTAs per SM the register budget allows
#define GB_CC_LANE_MAX  32             // shortest remaining list the whole warp takes
#define GB_CC_GRID_MIN  1024           // shortest remaining list the grid pass takes
#define GB_CC_SAMPLES   1024           // vertices whose roots the sample counts
#define GB_CC_SLOTS     2048           // shared hash slots for the sampled roots

enum CcCell {
  CC_LARGEST    = 0,                   // L, the most frequent sampled root
  CC_COMPONENTS = 1,                   // the number of components
  CC_QUEUED     = 2,                   // the number of rows queued for the grid pass
  CC_NCELLS     = 3
};

struct CcArgs {
  const Index* row_ptr;  const Index* row_ind;   // CSR; row_ptr NULL: no stored entries
  Index n;
  int skip;                      // A is symmetric: the finish skips L's tree
  Index* parent;                 // [n] the union-find forest
  Index* queued;                 // [nnz / GB_CC_GRID_MIN + 1] rows for the grid pass
  unsigned long long* counters;  // [CC_NCELLS] CcCell
};

// The root of x, halving the path on the way by CAS.
__device__ __forceinline__ Index ccFind(Index* parent, Index x) {
  while (true) {
    const Index p = ldRelaxed(parent + x);
    if (p == x) return x;
    const Index g = ldRelaxed(parent + p);
    if (g == p) return p;
    atomicCAS(parent + x, p, g);       // only if parent[x] still holds p
    x = g;
  }
}

// Join the trees of u and v: the larger root is hooked under the smaller, by CAS on a
// word that still holds its own index; a failed CAS retries from the new roots.
__device__ __forceinline__ void ccLink(Index* parent, Index u, Index v) {
  Index p = ccFind(parent, u);
  Index q = ccFind(parent, v);
  while (p != q) {
    const Index hi = p > q ? p : q;
    const Index lo = p > q ? q : p;
    const Index old = atomicCAS(parent + hi, hi, lo);
    if (old == hi) return;
    p = ccFind(parent, old);           // hi was hooked under old meanwhile
    q = ccFind(parent, lo);
  }
}

// parent[v] = root(v) for v = first, first + stride, ... below n; no link is in flight.
__device__ __forceinline__ void ccCompress(Index* parent, Index n, Index first, Index stride) {
  for (Index v = first; v < n; v += stride) {
    Index r = ldRelaxed(parent + v);
    for (Index p = ldRelaxed(parent + r); p != r; p = ldRelaxed(parent + r)) r = p;
    stRelaxed(parent + v, r);
  }
}

// CTA 0: the most frequent root among GB_CC_SAMPLES hashed vertices (parent[] is
// compressed, so a vertex's parent is its root).  Ties go to the larger root; the
// result does not depend on which root L is.
__device__ __forceinline__ Index ccSample(const CcArgs& a) {
  __shared__ Index keys[GB_CC_SLOTS];
  __shared__ unsigned int counts[GB_CC_SLOTS];
  __shared__ unsigned long long best;
  for (int s = threadIdx.x; s < GB_CC_SLOTS; s += GB_CC_NT) { keys[s] = -1; counts[s] = 0u; }
  if (threadIdx.x == 0) best = 0ull;
  __syncthreads();
  for (int i = threadIdx.x; i < GB_CC_SAMPLES; i += GB_CC_NT) {
    const Index v = static_cast<Index>(fmix32(static_cast<unsigned int>(i)) %
                                       static_cast<unsigned int>(a.n));
    const Index r = ldRelaxed(a.parent + v);
    unsigned int slot = fmix32(static_cast<unsigned int>(r)) & (GB_CC_SLOTS - 1);
    while (true) {
      const Index k = atomicCAS(keys + slot, -1, r);
      if (k == -1 || k == r) { atomicAdd(counts + slot, 1u); break; }
      slot = (slot + 1) & (GB_CC_SLOTS - 1);
    }
  }
  __syncthreads();
  for (int s = threadIdx.x; s < GB_CC_SLOTS; s += GB_CC_NT)
    if (counts[s] != 0u)
      atomicMax(&best, (static_cast<unsigned long long>(counts[s]) << 32) |
                       static_cast<unsigned int>(keys[s]));
  __syncthreads();
  return static_cast<Index>(static_cast<unsigned int>(best));
}

template <typename W>
__global__ void __launch_bounds__(GB_CC_NT, GB_CC_MINB)
ccKernel(CcArgs a, W* out) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31;
  const Index gtid = blockIdx.x*GB_CC_NT + threadIdx.x;
  const Index gthreads = gridDim.x*GB_CC_NT;
  const Index gwarp = gtid >> 5;
  const Index gwarps = gthreads >> 5;

  // ---- init --------------------------------------------------------------------------
  for (Index v = gtid; v < a.n; v += gthreads) stRelaxed(a.parent + v, v);
  grid.sync();

  if (a.row_ptr != NULL) {
    // ---- neighbour rounds ------------------------------------------------------------
    for (int r = 0; r < 2; ++r) {
      for (Index v = gtid; v < a.n; v += gthreads) {
        const Index b = __ldg(a.row_ptr + v);
        if (__ldg(a.row_ptr + v + 1) - b > r) ccLink(a.parent, v, __ldg(a.row_ind + b + r));
      }
      grid.sync();
      ccCompress(a.parent, a.n, gtid, gthreads);
      grid.sync();
    }

    // ---- sample ----------------------------------------------------------------------
    if (a.skip && blockIdx.x == 0) {
      const Index L = ccSample(a);
      if (threadIdx.x == 0) a.counters[CC_LARGEST] = static_cast<unsigned long long>(L);
    }
    if (a.skip) grid.sync();
    const Index L = a.skip ? static_cast<Index>(loadCell(a.counters + CC_LARGEST)) : -1;

    // ---- finish: entries from position 2 on, a lane or a warp per list ---------------
    for (Index i0 = gwarp*32; i0 < a.n; i0 += gwarps*32) {
      const Index v = i0 + lane;
      Index b = 0, e = 0;
      if (v < a.n && (L < 0 || ldRelaxed(a.parent + v) != L)) {
        b = __ldg(a.row_ptr + v) + 2;
        e = __ldg(a.row_ptr + v + 1);
        if (e < b) e = b;
      }
      const bool grid_v = e - b >= GB_CC_GRID_MIN;
      if (grid_v) a.queued[atomicAdd(a.counters + CC_QUEUED, 1ull)] = v;
      const bool heavy_v = !grid_v && e - b >= GB_CC_LANE_MAX;
      if (!heavy_v && !grid_v)
        for (Index k = b; k < e; ++k) ccLink(a.parent, v, __ldg(a.row_ind + k));
      unsigned int heavy = __ballot_sync(GB_FULL_MASK, heavy_v);
      while (heavy != 0u) {
        const int src = __ffs(heavy) - 1;
        heavy &= heavy - 1u;
        const Index hv = __shfl_sync(GB_FULL_MASK, v, src);
        const Index hb = __shfl_sync(GB_FULL_MASK, b, src);
        const Index he = __shfl_sync(GB_FULL_MASK, e, src);
        for (Index k = hb + lane; k < he; k += 32) ccLink(a.parent, hv, __ldg(a.row_ind + k));
      }
    }
    grid.sync();

    // ---- grid pass: the queued lists in 32-entry chunks, chunk c to warp c % warps ----
    const Index nq = static_cast<Index>(__ldcg(a.counters + CC_QUEUED));
    Index before = 0;                  // chunks of the lists before q, modulo warps
    for (Index q = 0; q < nq; ++q) {
      const Index h = __ldcg(a.queued + q);
      const Index hb = __ldg(a.row_ptr + h) + 2;
      const Index he = __ldg(a.row_ptr + h + 1);
      const Index chunks = (he - hb + 31) >> 5;
      Index c = gwarp - before;
      if (c < 0) c += gwarps;
      for (; c < chunks; c += gwarps) {
        const Index k = hb + c*32 + lane;
        if (k < he) ccLink(a.parent, h, __ldg(a.row_ind + k));
      }
      before = static_cast<Index>((before + chunks) % gwarps);
    }
    grid.sync();
  }

  // ---- out: the root of every vertex, and the number of roots ------------------------
  unsigned int roots = 0u;
  for (Index v = gtid; v < a.n; v += gthreads) {
    Index r = v;
    for (Index p = ldRelaxed(a.parent + r); p != r; p = ldRelaxed(a.parent + r)) r = p;
    out[v] = static_cast<W>(r);
    roots += r == v ? 1u : 0u;
  }
  roots = __reduce_add_sync(GB_FULL_MASK, roots);
  if (lane == 0 && roots != 0u)
    atomicAdd(a.counters + CC_COMPONENTS, static_cast<unsigned long long>(roots));
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_CC_CUH_
