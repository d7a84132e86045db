// graphblast_b200 backend — community detection by label propagation (LDBC Graphalytics
// CDLP) as ONE persistent cooperative kernel (algorithm::cdlp; host side cdlp.hpp): every
// iteration runs inside it, with grid barriers between them and no host wait.
//
// Semantics.  The arc i -> j when A(i,j) is stored and i != j (values never read, stored
// zeros count, self-loops ignored).  L_0(v) = v.  Iteration k: M(v) = the labels
// L_{k-1}(u) of v's out-neighbours (row v of the CSR) and of its in-neighbours (column v
// of the CSC), an arc stored both ways counted twice; L_k(v) = the smallest label of
// highest multiplicity in M(v), or L_{k-1}(v) when M(v) is empty.  A sameStructure() A
// (col_ptr NULL) is read through its CSR alone: both lists hold the same multiset, so
// every multiplicity doubles and the answer is the same.  The kernel stops after the
// first iteration that changes no label (a fixpoint) or after max_iter iterations.
//
// Classes, by the stored list length d(v) = out-degree + in-degree (CSR alone: the
// out-degree), self-loops included; fixed at the start of the kernel:
//   short  d <= GB_CDLP_SHORT_MAX (32).  A warp takes 32 consecutive vertices and packs
//          the lists of as many as fit into one round of 32 lanes, one entry per lane,
//          never cutting a list.  __match_any_sync on (vertex lane << 25 | label) gives
//          each entry its multiplicity, and __reduce_max_sync over the vertex's lanes on
//          (count << 25 | (2^25 - 1 - label)) picks the answer: a label takes 25 bits
//          (n <= 2^24 + 1), a count 6.
//   warp   d <= GB_CDLP_WARP_MAX (128).  One warp counts the list in its own
//          GB_CDLP_WARP_SLOTS-slot shared hash table (at most half full: no overflow),
//          then two warp reductions pick the highest count and the smallest label with it.
//   long   longer lists.  The list's labels are cut into P = ceil(d / GB_CDLP_PART)
//          partitions by hash(label) mod P; each (vertex, partition) pair is one work
//          item, and the items are dealt over every CTA of the grid, so one R-MAT hub
//          does not serialise on one CTA (cc's grid pass exists for the same reason).  A
//          CTA counts its item's partition in a shared table of up to GB_CDLP_SLOTS slots
//          (twice the partition's expected size, a power of two), and each warp combines
//          its best (count << 32 | ~label) into the vertex's best word by a 64-bit
//          atomicMax, which is order-independent.  A label that finds the table full is
//          counted by a scan of the whole list and combined the same way, so the result
//          never depends on the hash.  After a grid barrier every long vertex takes its
//          best word's label and clears the word.
//
// Phases (grid barriers between them):
//   setup   labels0[v] = v; each vertex's class; long vertices appended to the long list
//           with the first of their items (one 64-bit atomicAdd of 1 << 40 | P, so the
//           item bases rise with the list index); the community bitmap cleared.
//   iteration k = 1 .. max_iter, reading labels[(k - 1) & 1], writing labels[k & 1]:
//           short and warp vertices, then the long items; barrier; the long vertices'
//           labels; barrier; stop when cell CDLP_CHANGED + k % 3 is 0.
//   out     out[v] = (W) labels[T & 1][v] and the label's bit set in the bitmap; barrier;
//           the set bits counted: the number of communities.
// Changed counts are per iteration in their own cell, buffered three ways as in msf.cuh:
// iteration k adds to cell k % 3 and clears cell (k + 1) % 3, which no thread reads
// again before iteration k + 1 adds to it.  So every thread runs the same iterations.
//
// Determinism.  Every label of iteration k is a function of the labels of iteration
// k - 1: counts are exact and the tie rule is fixed, and the long path's partial answers
// meet in an atomicMax.  Launch shape, timing and the order of the long list change only
// who computes what.
//
// Memory model (cooperative.cuh).  Labels, best words and the bitmap are written while
// the kernel runs and read with __ldcg (from L2); the CSR and CSC take the non-coherent
// path.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_CDLP_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_CDLP_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/cooperative.cuh"

namespace graphblas {
namespace backend {

#define GB_CDLP_NT          256        // CTA shape of the label-propagation kernel
#define GB_CDLP_MINB        4          // resident CTAs per SM the register budget allows
#define GB_CDLP_SHORT_MAX   32         // longest list of the short class
#define GB_CDLP_WARP_MAX    128        // longest list of the warp class
#define GB_CDLP_WARP_SLOTS  256        // hash slots of one warp's table
#define GB_CDLP_PART        2048       // most entries of a long list's partition, d / P
#define GB_CDLP_SLOTS       4096       // hash slots of the CTA's table (2 GB_CDLP_PART)
#define GB_CDLP_LABEL_MASK  0x1ffffffu // 25 bits: a label, and the inverted label
#define GB_CDLP_ITEM_BITS   40         // the long cell: list length << 40 | items

enum CdlpCell {
  CDLP_CHANGED     = 0,                // [3] labels changed by an iteration, at k % 3
  CDLP_LONG        = 3,                // long vertices << 40 | their items
  CDLP_SHORT       = 4,                // vertices of the short class
  CDLP_WARP        = 5,                // vertices of the warp class
  CDLP_ITERATIONS  = 6,                // iterations run
  CDLP_BARRIERS    = 7,                // grid barriers executed
  CDLP_COMMUNITIES = 8,                // distinct labels at the end
  CDLP_NCELLS      = 9
};

struct CdlpArgs {
  const Index* row_ptr;  const Index* row_ind;   // CSR; row_ind NULL: no stored entries
  const Index* col_ptr;  const Index* col_ind;   // CSC; NULL when it is the CSR
  Index n;
  int max_iter;
  Index* labels0;  Index* labels1;     // [n] each, the labels of even and odd iterations
  Index* long_v;                       // [n] the long vertices
  Index* long_base;                    // [n] the first item of each long vertex
  unsigned long long* best;            // [n] each long vertex's best (count << 32 | ~label)
  unsigned int* bitmap;                // [n / 32 + 1] the labels of the result
  unsigned long long* counters;        // [CDLP_NCELLS] CdlpCell
};

// The entry k of v's list (out-list, then in-list): the neighbour's id.
struct CdlpList {
  Index ob, od, ib;                    // out-list start and length, in-list start
  __device__ __forceinline__ Index at(const CdlpArgs& a, Index k) const {
    return k < od ? __ldg(a.row_ind + ob + k) : __ldg(a.col_ind + ib + (k - od));
  }
};

__device__ __forceinline__ Index cdlpDegree(const CdlpArgs& a, Index v, CdlpList* l) {
  l->ob = __ldg(a.row_ptr + v);
  l->od = __ldg(a.row_ptr + v + 1) - l->ob;
  l->ib = 0;
  Index d = l->od;
  if (a.col_ptr != NULL) {
    l->ib = __ldg(a.col_ptr + v);
    d += __ldg(a.col_ptr + v + 1) - l->ib;
  }
  return d;
}

// Adds one occurrence of label x to the open-addressing table (keys, counts) of `mask`+1
// slots, starting at slot h & mask.  False when every slot holds another label.
__device__ __forceinline__ bool cdlpInsert(Index* keys, unsigned int* counts,
                                           unsigned int mask, unsigned int h, Index x) {
  for (unsigned int probe = 0; probe <= mask; ++probe) {
    const unsigned int s = (h + probe) & mask;
    const Index k = atomicCAS(keys + s, -1, x);
    if (k == -1 || k == x) { atomicAdd(counts + s, 1u); return true; }
  }
  return false;
}

// The larger of two (count, label) candidates: the higher count, then the smaller label.
__device__ __forceinline__ void cdlpBetter(unsigned int c, Index x, unsigned int* bc,
                                           Index* bx) {
  if (c > *bc || (c == *bc && c != 0u && x < *bx)) { *bc = c; *bx = x; }
}

template <typename W>
__global__ void __launch_bounds__(GB_CDLP_NT, GB_CDLP_MINB)
cdlpKernel(CdlpArgs a, W* out) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  __shared__ Index keys[GB_CDLP_SLOTS];
  __shared__ unsigned int counts[GB_CDLP_SLOTS];
  __shared__ int owner[GB_CDLP_NT];    // per warp: the lane whose list starts at a lane
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;    // warp in the CTA
  const Index gtid = blockIdx.x*GB_CDLP_NT + threadIdx.x;
  const Index gthreads = gridDim.x*GB_CDLP_NT;
  const Index gwarp = gtid >> 5;
  const Index gwarps = gthreads >> 5;
  const bool leader = gtid == 0;
  const bool stored = a.row_ind != NULL;
  int barriers = 0;

  // ---- setup -------------------------------------------------------------------------
  for (int s = threadIdx.x; s < GB_CDLP_SLOTS; s += GB_CDLP_NT) { keys[s] = -1; counts[s] = 0u; }
  for (Index w = gtid; w <= a.n/32; w += gthreads) a.bitmap[w] = 0u;
  unsigned int nshort = 0u, nwarp = 0u;
  for (Index v = gtid; v < a.n; v += gthreads) {
    a.labels0[v] = v;
    CdlpList l;
    const Index d = stored ? cdlpDegree(a, v, &l) : 0;
    nshort += d <= GB_CDLP_SHORT_MAX ? 1u : 0u;
    nwarp += d > GB_CDLP_SHORT_MAX && d <= GB_CDLP_WARP_MAX ? 1u : 0u;
    if (d > GB_CDLP_WARP_MAX) {
      const unsigned long long p = static_cast<unsigned long long>((d + GB_CDLP_PART - 1)/GB_CDLP_PART);
      const unsigned long long at =
          atomicAdd(a.counters + CDLP_LONG, (1ull << GB_CDLP_ITEM_BITS) | p);
      const Index i = static_cast<Index>(at >> GB_CDLP_ITEM_BITS);
      a.long_v[i] = v;
      a.long_base[i] = static_cast<Index>(at & ((1ull << GB_CDLP_ITEM_BITS) - 1ull));
      a.best[i] = 0ull;
    }
  }
  nshort = __reduce_add_sync(GB_FULL_MASK, nshort);
  nwarp = __reduce_add_sync(GB_FULL_MASK, nwarp);
  if (lane == 0 && nshort != 0u) atomicAdd(a.counters + CDLP_SHORT, static_cast<unsigned long long>(nshort));
  if (lane == 0 && nwarp != 0u) atomicAdd(a.counters + CDLP_WARP, static_cast<unsigned long long>(nwarp));
  grid.sync();
  ++barriers;
  const unsigned long long long_cell = loadCell(a.counters + CDLP_LONG);
  const Index nlong = static_cast<Index>(long_cell >> GB_CDLP_ITEM_BITS);
  const Index items = static_cast<Index>(long_cell & ((1ull << GB_CDLP_ITEM_BITS) - 1ull));

  int k = 1;
  for (; k <= a.max_iter; ++k) {
    const Index* in = (k & 1) ? a.labels0 : a.labels1;
    Index* next = (k & 1) ? a.labels1 : a.labels0;
    unsigned long long* changed_cell = a.counters + CDLP_CHANGED + k % 3;
    if (leader) a.counters[CDLP_CHANGED + (k + 1) % 3] = 0ull;
    unsigned int changed = 0u;

    // ---- short and warp vertices, 32 consecutive vertices to a warp -----------------
    for (Index v0 = gwarp*32; v0 < a.n; v0 += gwarps*32) {
      const Index v = v0 + lane;
      CdlpList l = {0, 0, 0};
      const Index d = v < a.n && stored ? cdlpDegree(a, v, &l) : 0;
      const Index old = v < a.n ? __ldcg(in + v) : 0;
      if (v < a.n && d == 0) next[v] = old;
      // short lists: packed into rounds of 32 lanes, a list never cut
      const int sd = v < a.n && d <= GB_CDLP_SHORT_MAX ? static_cast<int>(d) : 0;
      int incl = sd;
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(GB_FULL_MASK, incl, o);
        if (lane >= o) incl += t;
      }
      const int excl = incl - sd;
      unsigned int pending = __ballot_sync(GB_FULL_MASK, sd > 0);
      while (pending != 0u) {
        const int base = __shfl_sync(GB_FULL_MASK, excl, __ffs(pending) - 1);
        const bool mine = ((pending >> lane) & 1u) && incl - base <= 32;
        pending &= ~__ballot_sync(GB_FULL_MASK, mine);
        if (mine) owner[wib*32 + excl - base] = lane;
        const unsigned int starts = __reduce_or_sync(GB_FULL_MASK, mine ? 1u << (excl - base) : 0u);
        const int total = static_cast<int>(__reduce_max_sync(GB_FULL_MASK, mine ? incl - base : 0));
        __syncwarp();
        const bool valid_lane = lane < total;
        const int start = valid_lane ? 31 - __clz(starts & (0xffffffffu >> (31 - lane))) : 0;
        const int j = valid_lane ? owner[wib*32 + start] : 0;
        const Index u = __shfl_sync(GB_FULL_MASK, v, j);
        const Index uob = __shfl_sync(GB_FULL_MASK, l.ob, j);
        const Index uod = __shfl_sync(GB_FULL_MASK, l.od, j);
        const Index uib = __shfl_sync(GB_FULL_MASK, l.ib, j);
        const Index uold = __shfl_sync(GB_FULL_MASK, old, j);
        const CdlpList ul = {uob, uod, uib};
        const Index nb = valid_lane ? ul.at(a, lane - start) : u;
        const bool valid = valid_lane && nb != u;
        const unsigned int x = valid ? static_cast<unsigned int>(__ldcg(in + nb)) : 0u;
        const unsigned int key = valid ? (static_cast<unsigned int>(j) << 25) | x : 0xffffffffu;
        const unsigned int cnt = __popc(__match_any_sync(GB_FULL_MASK, key));
        const unsigned int packed = valid ? (cnt << 25) | (GB_CDLP_LABEL_MASK - x) : 0u;
        const unsigned int group = __match_any_sync(GB_FULL_MASK, valid_lane ? j : 32);
        const unsigned int top = __reduce_max_sync(group, packed);
        if (valid_lane && lane == start) {
          const Index lab = top != 0u ? static_cast<Index>(GB_CDLP_LABEL_MASK - (top & GB_CDLP_LABEL_MASK))
                                      : uold;
          next[u] = lab;
          changed += lab != uold ? 1u : 0u;
        }
        __syncwarp();
      }
      // warp lists: one at a time, in this warp's slice of the table
      unsigned int heavy = __ballot_sync(GB_FULL_MASK, d > GB_CDLP_SHORT_MAX && d <= GB_CDLP_WARP_MAX);
      Index* wkeys = keys + wib*GB_CDLP_WARP_SLOTS;
      unsigned int* wcounts = counts + wib*GB_CDLP_WARP_SLOTS;
      while (heavy != 0u) {
        const int src = __ffs(heavy) - 1;
        heavy &= heavy - 1u;
        const Index hv = __shfl_sync(GB_FULL_MASK, v, src);
        const Index hd = __shfl_sync(GB_FULL_MASK, d, src);
        const CdlpList hl = {__shfl_sync(GB_FULL_MASK, l.ob, src),
                             __shfl_sync(GB_FULL_MASK, l.od, src),
                             __shfl_sync(GB_FULL_MASK, l.ib, src)};
        const Index hold = __shfl_sync(GB_FULL_MASK, old, src);
        for (Index e = lane; e < hd; e += 32) {
          const Index nb = hl.at(a, e);
          if (nb == hv) continue;
          const Index x = __ldcg(in + nb);
          cdlpInsert(wkeys, wcounts, GB_CDLP_WARP_SLOTS - 1, fmix32(static_cast<unsigned int>(x)), x);
        }
        __syncwarp();
        unsigned int bc = 0u;
        Index bx = 0;
        for (int s = lane; s < GB_CDLP_WARP_SLOTS; s += 32) {
          cdlpBetter(wcounts[s], wkeys[s], &bc, &bx);
          wkeys[s] = -1;
          wcounts[s] = 0u;
        }
        const unsigned int top = __reduce_max_sync(GB_FULL_MASK, bc);
        const unsigned int lab = __reduce_min_sync(GB_FULL_MASK, bc == top ? static_cast<unsigned int>(bx)
                                                                             : 0xffffffffu);
        const Index nl = top != 0u ? static_cast<Index>(lab) : hold;
        if (lane == 0) {
          next[hv] = nl;
          changed += nl != hold ? 1u : 0u;
        }
        __syncwarp();
      }
    }

    // ---- long items: (vertex, partition) pairs dealt over the CTAs -------------------
    __syncthreads();                   // the warp slices are free
    for (Index it = blockIdx.x; it < items; it += gridDim.x) {
      Index lo = 0, hi = nlong - 1;    // the last long vertex whose base <= it
      while (lo < hi) {
        const Index mid = (lo + hi + 1) >> 1;
        if (__ldcg(a.long_base + mid) <= it) lo = mid; else hi = mid - 1;
      }
      const Index v = __ldcg(a.long_v + lo);
      const Index b = __ldcg(a.long_base + lo);
      CdlpList l;
      const Index d = cdlpDegree(a, v, &l);
      const unsigned int parts = static_cast<unsigned int>((d + GB_CDLP_PART - 1)/GB_CDLP_PART);
      const unsigned int part = static_cast<unsigned int>(it - b);
      const unsigned int per = static_cast<unsigned int>(d < GB_CDLP_PART ? d : GB_CDLP_PART);
      unsigned int slots = 256u;
      while (slots < 2u*per) slots <<= 1;
      const unsigned int mask = slots - 1u;
      for (Index e = threadIdx.x; e < d; e += GB_CDLP_NT) {
        const Index nb = l.at(a, e);
        if (nb == v) continue;
        const Index x = __ldcg(in + nb);
        const unsigned int h = fmix32(static_cast<unsigned int>(x));
        if (h % parts != part) continue;
        if (!cdlpInsert(keys, counts, mask, h/parts, x)) {
          unsigned int c = 0u;         // the table is full: count x by a scan of the list
          for (Index f = 0; f < d; ++f) {
            const Index y = l.at(a, f);
            c += y != v && __ldcg(in + y) == x ? 1u : 0u;
          }
          atomicMax(a.best + lo, (static_cast<unsigned long long>(c) << 32) |
                                 static_cast<unsigned int>(~static_cast<unsigned int>(x)));
        }
      }
      __syncthreads();
      unsigned int bc = 0u;
      Index bx = 0;
      for (unsigned int s = threadIdx.x; s < slots; s += GB_CDLP_NT) {
        cdlpBetter(counts[s], keys[s], &bc, &bx);
        keys[s] = -1;
        counts[s] = 0u;
      }
      const unsigned int top = __reduce_max_sync(GB_FULL_MASK, bc);
      const unsigned int lab = __reduce_min_sync(GB_FULL_MASK, bc == top ? static_cast<unsigned int>(bx)
                                                                           : 0xffffffffu);
      if (lane == 0 && top != 0u) {
        const unsigned long long w = (static_cast<unsigned long long>(top) << 32) | ~lab;
        if (w > __ldcg(a.best + lo)) atomicMax(a.best + lo, w);
      }
      __syncthreads();
    }
    grid.sync();
    ++barriers;

    // ---- the long vertices' labels ---------------------------------------------------
    for (Index i = gtid; i < nlong; i += gthreads) {
      const Index v = a.long_v[i];
      const unsigned long long w = __ldcg(a.best + i);
      const Index prev = __ldcg(in + v);
      const Index lab = w != 0ull ? static_cast<Index>(~static_cast<unsigned int>(w)) : prev;
      next[v] = lab;
      a.best[i] = 0ull;
      changed += lab != prev ? 1u : 0u;
    }
    changed = __reduce_add_sync(GB_FULL_MASK, changed);
    if (lane == 0 && changed != 0u) atomicAdd(changed_cell, static_cast<unsigned long long>(changed));
    grid.sync();
    ++barriers;
    if (loadCell(changed_cell) == 0ull) break;
  }
  const int iterations = k <= a.max_iter ? k : a.max_iter;

  // ---- out: the float labels, and the number of distinct labels ----------------------
  const Index* fin = (iterations & 1) ? a.labels1 : a.labels0;
  for (Index v = gtid; v < a.n; v += gthreads) {
    const Index x = __ldcg(fin + v);
    out[v] = static_cast<W>(x);
    const unsigned int bit = 1u << (x & 31);
    if ((__ldcg(a.bitmap + (x >> 5)) & bit) == 0u) atomicOr(a.bitmap + (x >> 5), bit);
  }
  grid.sync();
  ++barriers;
  unsigned int labels = 0u;
  for (Index w = gtid; w <= a.n/32; w += gthreads) labels += __popc(__ldcg(a.bitmap + w));
  labels = __reduce_add_sync(GB_FULL_MASK, labels);
  if (lane == 0 && labels != 0u)
    atomicAdd(a.counters + CDLP_COMMUNITIES, static_cast<unsigned long long>(labels));
  if (leader) {
    a.counters[CDLP_ITERATIONS] = static_cast<unsigned long long>(iterations);
    a.counters[CDLP_BARRIERS] = static_cast<unsigned long long>(barriers);
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_CDLP_CUH_
