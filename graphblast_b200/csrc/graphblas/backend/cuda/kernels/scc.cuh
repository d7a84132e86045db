// graphblast_b200 backend — strongly connected components as ONE persistent cooperative
// kernel (algorithm::scc; host side scc.hpp): trim, forward–backward from a pivot, then
// colouring (Slota, Rajamanickam and Madduri, IPDPS 2014), with grid barriers between
// levels and no host wait.
//
// Graph.  The arc i -> j when A(i,j) is stored and i != j (stored zeros count, values
// are never read).  Out-lists come from the CSR (row_ptr, row_ind), in-lists from the
// CSC (col_ptr, col_ind); both are sorted and duplicate-free, so a list holds at most
// one self-loop, found by binary search.  out[i] = the smallest vertex id in the strongly
// connected component of i; cells[SCC_COMPONENTS] = the number of i with out[i] == i.
//
// A vertex is live while label[v] == -1; every phase settles whole components, so the
// components of the graph induced by the live vertices are components of the graph.
//   init      label = -1; live out- and in-degrees = list lengths without the self-loop;
//             the vertices with a zero degree form the first trim frontier.
//   trim      each frontier vertex x is settled (label = x) and decrements the live
//             degree of its out-neighbours' in-degrees and in-neighbours' out-degrees;
//             the thread whose atomicSub takes a degree to 0 queues that neighbour,
//             once, by atomicOr of SCC_QUEUED on its mark word.  Runs to its fixpoint,
//             so the trimmed set depends only on the pattern.
//   pivot     the live vertex with the largest (out + 1)(in + 1) (saturated at 2^32 - 1),
//             ties to the smallest id, by a 64-bit packed atomicMax.
//   FW–BW     its forward reach (over out-lists) and backward reach (over in-lists),
//             both in the same levels, marked by atomicOr of SCC_FW / SCC_BW.  The
//             pivot's component is their intersection; its label is the intersection's
//             minimum id (atomicMin), written by the colouring's first init.
//   colouring while live vertices remain: colour[v] = v, then the minimum is pushed
//             along live out-arcs by atomicMin from a work list (a vertex whose colour
//             dropped is queued once per level by an atomicExch of the level on its
//             stamp) until no colour drops.  colour[x] is then the smallest live id that
//             reaches x, so a live r with colour[r] == r is the minimum of its
//             component, and the vertices of colour r that reach r are exactly that
//             component: a backward reach from all roots at once, through live vertices
//             of the same colour, settles them (label = colour, by CAS from -1).  The
//             smallest live id is always a root, so every iteration settles something.
//   out       out[i] = (W) label[i], and a warp-reduced count of the i with label i.
//
// Frontiers.  A level expands the vertices q[lo, hi) of a frontier.  Lanes take one
// vertex each; a list of 32 entries or more is walked by the whole warp, and one of
// GB_SCC_GRID_MIN or more is deferred to a grid pass after a barrier, cut into 32-entry
// chunks numbered across all deferred lists (chunk c to warp c % warps), so that a hub
// does not hold up one warp.  Appends are counted per level in their own cell,
// buffered three ways as in ktruss.cuh (see `advance` in the kernel): every thread
// reads the same bound after the barrier that ends a level, however early it leaves
// that barrier and whatever other warps append meanwhile, so all threads run the same
// levels.  The trim and the colouring's settle, which settle each vertex once,
// lay their frontiers one after another in qa; the pivot's reaches do the same in qb
// and qc; the colour work lists alternate between qb and qc.
//
// Memory model (cooperative.cuh).  label, colour, degrees, marks, stamps and queue
// entries are written by other SMs while the kernel runs and are read with ldRelaxed;
// only the CSR and CSC are read through the non-coherent path.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_SCC_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_SCC_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/cooperative.cuh"

namespace graphblas {
namespace backend {

#define GB_SCC_NT        256           // CTA shape of the components kernel
#define GB_SCC_MINB      4             // resident CTAs per SM the register budget allows
#define GB_SCC_GRID_MIN  2048          // shortest list the grid pass takes

enum SccCell {
  SCC_FRONT      = 0,                  // [3] appends to a level's frontier, at lv % 3
  SCC_BACK       = 3,                  // [3] appends to a level's backward reach
  SCC_HEAVY      = 6,                  // [3] lists deferred to a level's grid pass
  SCC_PIVOT      = 9,                  // packed key of the pivot, 0: no live vertex
  SCC_MIN        = 10,                 // the smallest id of the pivot's component
  SCC_SIZE       = 11,                 // the size of the pivot's component
  SCC_TRIMMED    = 12,                 // vertices settled by the trim
  SCC_COLOURS    = 13,                 // colouring iterations
  SCC_BARRIERS   = 14,                 // grid barriers executed
  SCC_COMPONENTS = 15,                 // the number of components
  SCC_NCELLS     = 16
};

enum SccMark {                         // bits of mark[v]
  SCC_QUEUED = 1,                      // queued by the trim
  SCC_FW     = 2,                      // in the pivot's forward reach
  SCC_BW     = 4                       // in the pivot's backward reach
};

enum SccDir { SCC_OUT = 1, SCC_IN = 2 };

struct SccArgs {
  const Index* row_ptr;  const Index* row_ind;   // CSR: out-lists
  const Index* col_ptr;  const Index* col_ind;   // CSC: in-lists
  Index n;
  Index* label;                  // [n] -1 live, else the component's smallest id
  Index* dout;  Index* din;      // [n] live out- and in-degrees
  Index* mark;                   // [n] SccMark bits
  Index* colour;                 // [n]
  Index* stamp;                  // [n] the last level that queued v for the colour work list
  Index* qa;  Index* qb;  Index* qc;   // [n] each, the frontiers
  Index* heavy;                  // [2 (nnz / GB_SCC_GRID_MIN + 1)] x (out) or ~x (in)
  unsigned long long* counters;  // [SCC_NCELLS] SccCell
};

// The vertices q[lo, hi), expanded over their out-lists, in-lists or both (dirs).
struct SccFront {
  const Index* q;
  Index lo, hi;
  int dirs;
};

// The length of v's list without its self-loop.
__device__ __forceinline__ Index sccDegree(const Index* ptr, const Index* ind, Index v) {
  const Index b = __ldg(ptr + v), e = __ldg(ptr + v + 1);
  if (e == b) return 0;
  const Index k = findSorted(ind, b, e, v);
  return e - b - (k < e && __ldg(ind + k) == v ? 1 : 0);
}

// The light part of a level: visit(dir, x, y) for every entry y of each list of f,
// except lists of GB_SCC_GRID_MIN entries or more, which go to the heavy list.
template <typename Visit>
__device__ __forceinline__ void sccLight(const SccArgs& a, const SccFront& f,
                                         unsigned long long* heavy_cell, Visit& visit) {
  const int lane = threadIdx.x & 31;
  const Index gwarp = (blockIdx.x*GB_SCC_NT + threadIdx.x) >> 5;
  const Index gwarps = (gridDim.x*GB_SCC_NT) >> 5;
  for (int dir = SCC_OUT; dir <= SCC_IN; dir <<= 1) {
    if ((f.dirs & dir) == 0) continue;
    const Index* ptr = dir == SCC_OUT ? a.row_ptr : a.col_ptr;
    const Index* ind = dir == SCC_OUT ? a.row_ind : a.col_ind;
    for (Index i0 = f.lo + gwarp*32; i0 < f.hi; i0 += gwarps*32) {
      const Index i = i0 + lane;
      Index x = 0, b = 0, e = 0;
      if (i < f.hi) {
        x = ldRelaxed(f.q + i);
        b = __ldg(ptr + x);
        e = __ldg(ptr + x + 1);
      }
      const bool grid_x = e - b >= GB_SCC_GRID_MIN;
      if (grid_x) a.heavy[atomicAdd(heavy_cell, 1ull)] = dir == SCC_OUT ? x : ~x;
      const bool warp_x = !grid_x && e - b >= 32;
      if (!grid_x && !warp_x)
        for (Index k = b; k < e; ++k) visit(dir, x, __ldg(ind + k));
      unsigned int warps = __ballot_sync(GB_FULL_MASK, warp_x);
      while (warps != 0u) {
        const int src = __ffs(warps) - 1;
        warps &= warps - 1u;
        const Index wx = __shfl_sync(GB_FULL_MASK, x, src);
        const Index wb = __shfl_sync(GB_FULL_MASK, b, src);
        const Index we = __shfl_sync(GB_FULL_MASK, e, src);
        for (Index k = wb + lane; k < we; k += 32) visit(dir, wx, __ldg(ind + k));
      }
    }
  }
}

// The grid pass of a level: the nh deferred lists in 32-entry chunks, chunk c to warp
// c % warps, numbered across the lists (R-MAT hubs sit at low ids, so one warp would
// otherwise own many of them).
template <typename Visit>
__device__ __forceinline__ void sccHeavy(const SccArgs& a, Index nh, Visit& visit) {
  const int lane = threadIdx.x & 31;
  const Index gwarp = (blockIdx.x*GB_SCC_NT + threadIdx.x) >> 5;
  const Index gwarps = (gridDim.x*GB_SCC_NT) >> 5;
  Index before = 0;                    // chunks of the lists before h, modulo warps
  for (Index h = 0; h < nh; ++h) {
    const Index entry = ldRelaxed(a.heavy + h);
    const int dir = entry >= 0 ? SCC_OUT : SCC_IN;
    const Index x = entry >= 0 ? entry : ~entry;
    const Index* ptr = dir == SCC_OUT ? a.row_ptr : a.col_ptr;
    const Index* ind = dir == SCC_OUT ? a.row_ind : a.col_ind;
    const Index hb = __ldg(ptr + x), he = __ldg(ptr + x + 1);
    const Index chunks = (he - hb + 31) >> 5;
    Index c = gwarp - before;
    if (c < 0) c += gwarps;
    for (; c < chunks; c += gwarps) {
      const Index k = hb + c*32 + lane;
      if (k < he) visit(dir, x, __ldg(ind + k));
    }
    before = static_cast<Index>((before + chunks) % gwarps);
  }
}

template <typename W>
__global__ void __launch_bounds__(GB_SCC_NT, GB_SCC_MINB)
sccKernel(SccArgs a, W* out) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31;
  const Index gtid = blockIdx.x*GB_SCC_NT + threadIdx.x;
  const Index gthreads = gridDim.x*GB_SCC_NT;
  unsigned long long* const cells = a.counters;
  int lv = 0;                          // the level running; every thread runs the same
  int barriers = 0;

  // Level lv's appends count in cell lv % 3.  They are read at the start of level
  // lv + 1, before its first barrier; the cells of (lv + 1) % 3 are reset at level lv,
  // after the barrier that ended level lv - 1, where they were last read.
  auto advance = [&]() {
    ++lv;
    if (gtid == 0) {
      const int r = (lv + 1) % 3;
      cells[SCC_FRONT + r] = 0ull;
      cells[SCC_BACK + r] = 0ull;
      cells[SCC_HEAVY + r] = 0ull;
    }
  };
  auto next = [&]() {                  // end the level with a barrier
    grid.sync();
    ++barriers;
    advance();
  };
  auto count = [&](int cell) {         // the appends of the level before this one
    return static_cast<Index>(loadCell(cells + cell + (lv + 2) % 3));
  };
  // One frontier level over f and g: the light part, a barrier, and the grid pass with
  // its own barrier when a list was deferred.
  auto level = [&](const SccFront& f, const SccFront& g, auto& visit) {
    sccLight(a, f, cells + SCC_HEAVY + lv % 3, visit);
    sccLight(a, g, cells + SCC_HEAVY + lv % 3, visit);
    grid.sync();
    ++barriers;
    const Index nh = static_cast<Index>(loadCell(cells + SCC_HEAVY + lv % 3));
    if (nh > 0) {
      sccHeavy(a, nh, visit);
      grid.sync();
      ++barriers;
    }
    advance();
  };
  const SccFront none = {NULL, 0, 0, 0};

  // ---- init: level 0 queues the first trim frontier ------------------------------------
  if (gtid == 0) cells[SCC_MIN] = static_cast<unsigned long long>(a.n);
  for (Index v = gtid; v < a.n; v += gthreads) {
    const Index dout = sccDegree(a.row_ptr, a.row_ind, v);
    const Index din = sccDegree(a.col_ptr, a.col_ind, v);
    const bool dead = dout == 0 || din == 0;
    stRelaxed(a.label + v, -1);
    stRelaxed(a.dout + v, dout);
    stRelaxed(a.din + v, din);
    stRelaxed(a.mark + v, dead ? SCC_QUEUED : 0);
    stRelaxed(a.stamp + v, -1);
    if (dead) warpAppend(a.qa, 0, cells + SCC_FRONT + lv % 3, v);
  }
  next();

  // ---- trim, to its fixpoint -----------------------------------------------------------
  Index lo = 0, hi = count(SCC_FRONT);
  auto trim = [&](int dir, Index x, Index y) {
    if (y == x || (ldRelaxed(a.mark + y) & SCC_QUEUED) != 0) return;
    Index* deg = dir == SCC_OUT ? a.din : a.dout;    // x -> y, or y -> x
    if (atomicSub(deg + y, 1) == 1 && (atomicOr(a.mark + y, SCC_QUEUED) & SCC_QUEUED) == 0)
      warpAppend(a.qa, hi, cells + SCC_FRONT + lv % 3, y);
  };
  while (lo < hi) {
    for (Index i = lo + gtid; i < hi; i += gthreads) {
      const Index x = ldRelaxed(a.qa + i);
      stRelaxed(a.label + x, x);
    }
    level({a.qa, lo, hi, SCC_OUT | SCC_IN}, none, trim);
    lo = hi;
    hi += count(SCC_FRONT);
  }
  const Index trimmed = hi;

  // ---- pivot: the largest (out + 1)(in + 1) among the live, ties to the smallest id -----
  unsigned long long best = 0ull;
  for (Index v = gtid; v < a.n; v += gthreads) {
    if (ldRelaxed(a.label + v) != -1) continue;
    const unsigned long long score =
        static_cast<unsigned long long>(ldRelaxed(a.dout + v) + 1) *
        static_cast<unsigned long long>(ldRelaxed(a.din + v) + 1);
    const unsigned long long key =
        ((score < 0xFFFFFFFFull ? score : 0xFFFFFFFFull) << 32) |
        (0xFFFFFFFFull - static_cast<unsigned int>(v));
    best = key > best ? key : best;
  }
  best = warpReduce(best, [](unsigned long long x, unsigned long long y) { return x > y ? x : y; });
  if (lane == 0 && best != 0ull) atomicMax(cells + SCC_PIVOT, best);
  next();
  const unsigned long long pivot_key = loadCell(cells + SCC_PIVOT);
  Index pivot_min = -1;

  if (pivot_key != 0ull) {
    // ---- forward and backward reach of the pivot, in the same levels -------------------
    const Index p = static_cast<Index>(0xFFFFFFFFu - static_cast<unsigned int>(pivot_key));
    if (gtid == 0) {
      a.qb[0] = p;
      a.qc[0] = p;
      atomicOr(a.mark + p, SCC_FW | SCC_BW);
    }
    next();
    Index flo = 0, fhi = 1, blo = 0, bhi = 1;
    auto reach = [&](int dir, Index x, Index y) {
      if (y == x || ldRelaxed(a.label + y) != -1) return;
      const int bit = dir == SCC_OUT ? SCC_FW : SCC_BW;
      if ((ldRelaxed(a.mark + y) & bit) != 0 || (atomicOr(a.mark + y, bit) & bit) != 0) return;
      if (dir == SCC_OUT) warpAppend(a.qb, fhi, cells + SCC_FRONT + lv % 3, y);
      else                warpAppend(a.qc, bhi, cells + SCC_BACK + lv % 3, y);
    };
    while (flo < fhi || blo < bhi) {
      level({a.qb, flo, fhi, SCC_OUT}, {a.qc, blo, bhi, SCC_IN}, reach);
      flo = fhi;
      fhi += count(SCC_FRONT);
      blo = bhi;
      bhi += count(SCC_BACK);
    }

    // ---- the pivot's component: both reaches; its size and smallest id -----------------
    unsigned int size = 0u;
    for (Index i = gtid; i < fhi; i += gthreads) {
      const Index x = ldRelaxed(a.qb + i);
      if ((ldRelaxed(a.mark + x) & (SCC_FW | SCC_BW)) == (SCC_FW | SCC_BW)) {
        atomicMin(cells + SCC_MIN, static_cast<unsigned long long>(x));
        ++size;
      }
    }
    size = __reduce_add_sync(GB_FULL_MASK, size);
    if (lane == 0 && size != 0u) atomicAdd(cells + SCC_SIZE, static_cast<unsigned long long>(size));
    next();
    pivot_min = static_cast<Index>(loadCell(cells + SCC_MIN));
  }

  // ---- colouring, while live vertices remain -------------------------------------------
  Index settled = trimmed;             // the entries of qa so far
  int colours = 0;
  if (pivot_key != 0ull) {
    for (;;) {
      // init: colour[v] = v for every live v, all of them the first work list; the first
      // init also settles the pivot's component
      for (Index v = gtid; v < a.n; v += gthreads) {
        if (ldRelaxed(a.label + v) != -1) continue;
        if ((ldRelaxed(a.mark + v) & (SCC_FW | SCC_BW)) == (SCC_FW | SCC_BW)) {
          stRelaxed(a.label + v, pivot_min);
          continue;
        }
        stRelaxed(a.colour + v, v);
        warpAppend(a.qb, 0, cells + SCC_FRONT + lv % 3, v);
      }
      next();
      Index len = count(SCC_FRONT);
      if (len == 0) break;
      ++colours;

      // propagate the minimum along live out-arcs until no colour drops; the fixpoint
      // does not depend on the order of the atomicMins
      Index* cur = a.qb;
      Index* nxt = a.qc;
      auto push = [&](int, Index x, Index y) {
        if (y == x || ldRelaxed(a.label + y) != -1) return;
        const Index c = ldRelaxed(a.colour + x);
        if (atomicMin(a.colour + y, c) > c && atomicExch(a.stamp + y, lv) != lv)
          warpAppend(nxt, 0, cells + SCC_FRONT + lv % 3, y);
      };
      while (len > 0) {
        level({cur, 0, len, SCC_OUT}, none, push);
        len = count(SCC_FRONT);
        Index* t = cur;
        cur = nxt;
        nxt = t;
      }

      // settle: the roots, then backward through live vertices of their colour
      for (Index v = gtid; v < a.n; v += gthreads) {
        if (ldRelaxed(a.label + v) == -1 && ldRelaxed(a.colour + v) == v) {
          stRelaxed(a.label + v, v);
          warpAppend(a.qa, settled, cells + SCC_FRONT + lv % 3, v);
        }
      }
      next();
      Index slo = settled, shi = settled + count(SCC_FRONT);
      auto settle = [&](int, Index x, Index y) {
        if (y == x || ldRelaxed(a.label + y) != -1) return;
        const Index c = ldRelaxed(a.colour + x);
        if (ldRelaxed(a.colour + y) != c) return;
        if (atomicCAS(a.label + y, -1, c) == -1) warpAppend(a.qa, shi, cells + SCC_FRONT + lv % 3, y);
      };
      while (slo < shi) {
        level({a.qa, slo, shi, SCC_IN}, none, settle);
        slo = shi;
        shi += count(SCC_FRONT);
      }
      settled = shi;
    }
  }

  // ---- out: the label of every vertex, and the number of components --------------------
  unsigned int roots = 0u;
  for (Index v = gtid; v < a.n; v += gthreads) {
    const Index r = ldRelaxed(a.label + v);
    out[v] = static_cast<W>(r);
    roots += r == v ? 1u : 0u;
  }
  roots = __reduce_add_sync(GB_FULL_MASK, roots);
  if (lane == 0 && roots != 0u)
    atomicAdd(cells + SCC_COMPONENTS, static_cast<unsigned long long>(roots));
  if (gtid == 0) {
    cells[SCC_TRIMMED] = static_cast<unsigned long long>(trimmed);
    cells[SCC_COLOURS] = static_cast<unsigned long long>(colours);
    cells[SCC_BARRIERS] = static_cast<unsigned long long>(barriers);
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_SCC_CUH_
