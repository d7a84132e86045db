// graphblast_b200 backend — minimum spanning forest as ONE persistent cooperative kernel
// (algorithm::msf; host side msf.hpp): Borůvka rounds over cc.cuh's union-find, with grid
// barriers between phases and no host wait, and the kernels that build its input and
// read its result.
//
// Graph.  The canonical edge list (msfEmitKernel, msfCanonKernel): one slot per edge
// {u, v}, u < v, with A(u,v) or A(v,u) stored, in (u, v) order; its weight is the smaller
// of the stored values, kept as order-preserving bits (msfWeightBits): unsigned order
// of the bits is the numeric order of the weights, -0.0 and +0.0 have the same bits.
// The key (bits << 32) | slot orders edges by (w, u, v), a strict total order, so the
// minimum spanning forest is unique: Kruskal's forest under that order.
//
// Rounds (grid barriers between the phases):
//   init      parent[v] = v, best[v] = MSF_NONE.
//   pick      every edge of the live list whose endpoints have different roots takes
//             the atomicMin of its key into both roots' best words and is appended to
//             the next live list; an edge inside one tree is dropped for good.  No
//             append: no root picked, the forest is complete.  Round 0's live list is
//             every slot, read without a list.
//   link      every root with a pick flags the picked slot in forest[] and links its
//             endpoints (ccLink), then clears its best word.  Each pick is the lightest
//             edge leaving its tree, so by the cut property it is a forest edge; a
//             mutual pick names one slot twice and the second link is a no-op.
//   compress  ccCompress: parent[v] = root(v), so the next pick reads roots directly.
// Every round at least halves the trees that still have an edge leaving them, so at
// most ceil(log2 n) rounds pick and one more finds nothing: rounds <= ceil(log2 n) + 1.
//
// Live-list counts are per round in their own cell, buffered three ways as in
// ktruss.cuh: round r reads cell r % 3 after the barrier that ends round r - 1, appends
// to cell (r + 1) % 3, and clears cell (r + 2) % 3, which no thread reads again before
// round r + 2's appends.  So every thread runs the same rounds.
//
// Memory model (cooperative.cuh).  parent[] is read with ldRelaxed and best[] with
// __ldcg, both from L2: other SMs write them while the kernel runs, and a stale best
// word would skip a smaller pick.  The canonical list, which nothing writes, is read
// through the non-coherent path.
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_MSF_CUH_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_MSF_CUH_

#include <cooperative_groups.h>

#include "graphblas/backend/cuda/kernels/cc.cuh"
#include "graphblas/backend/cuda/kernels/cooperative.cuh"

namespace graphblas {
namespace backend {

#define GB_MSF_NT        512           // CTA shape of the forest kernel
#define GB_MSF_MINB      2             // resident CTAs per SM the register budget allows
#define GB_MSF_SUM_CTAS  256           // fixed shape of the weight sum, for its order
#define GB_MSF_SUM_NT    256
#define MSF_NONE         0xffffffffffffffffull   // a best word without a pick

enum MsfCell {
  MSF_LIVE     = 0,                    // [3] live edges of a round, at r % 3
  MSF_ROUNDS   = 3,                    // rounds with a pick phase
  MSF_BARRIERS = 4,                    // grid barriers executed
  MSF_NAN      = 5,                    // an FP32 NaN on an off-diagonal entry
  MSF_NCELLS   = 6
};

struct MsfArgs {
  const Index* eu;  const Index* ev;   // [m] the endpoints of each slot, eu < ev
  const unsigned int* ew;              // [m] the order-preserving weight bits
  Index n, m;
  Index* parent;                       // [n] cc.cuh's union-find forest
  unsigned long long* best;            // [n] the lightest key leaving each root
  Index* live0;  Index* live1;         // [m] each, the live lists of even and odd rounds
  int* forest;                         // [m] 1 on the slots of forest edges
  unsigned long long* counters;        // [MSF_NCELLS] MsfCell
};

// Order-preserving bits of a weight: the unsigned order of the bits is the numeric
// order of the weights.  Floats: -0.0 is +0.0 first; negative values have every bit
// flipped, the others their sign bit set.  Integers: the sign bit flipped.
__device__ __forceinline__ unsigned int msfWeightBits(float w) {
  const unsigned int u = __float_as_uint(w == 0.f ? 0.f : w);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ unsigned int msfWeightBits(int w) {
  return static_cast<unsigned int>(w) ^ 0x80000000u;
}

template <typename T> __device__ __forceinline__ T msfWeight(unsigned int b);
template <> __device__ __forceinline__ float msfWeight<float>(unsigned int b) {
  return __uint_as_float((b & 0x80000000u) ? (b ^ 0x80000000u) : ~b);
}
template <> __device__ __forceinline__ int msfWeight<int>(unsigned int b) {
  return static_cast<int>(b ^ 0x80000000u);
}

// Stored entry k of the CSR: keys[k] = min << bits | max of its row and column, pay[k]
// = its weight bits; a self-loop gets `loop`, the largest key, so loops sort last.  An
// FP32 NaN off the diagonal sets counters[MSF_NAN].
template <typename T>
__global__ void msfEmitKernel(const Index* __restrict__ rowptr,
                              const Index* __restrict__ colind, const T* __restrict__ val,
                              Index n, Index nnz, int bits, unsigned long long loop,
                              unsigned long long* __restrict__ keys,
                              unsigned int* __restrict__ pay,
                              unsigned long long* counters) {
  Index k = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; k < nnz; k += stride) {
    Index lo = 0, hi = n - 1;          // the row: the smallest r with rowptr[r+1] > k
    while (lo < hi) {
      const Index mid = (lo + hi) >> 1;
      if (__ldg(rowptr + mid + 1) <= k) lo = mid + 1; else hi = mid;
    }
    const Index c = __ldg(colind + k);
    if (c == lo) {
      keys[k] = loop;
      pay[k] = 0xffffffffu;
      continue;
    }
    const T w = __ldg(val + k);
    if (w != w && counters[MSF_NAN] == 0ull) atomicOr(counters + MSF_NAN, 1ull);
    const Index u = c < lo ? c : lo, v = c < lo ? lo : c;
    keys[k] = (static_cast<unsigned long long>(u) << bits) | static_cast<unsigned long long>(v);
    pay[k] = msfWeightBits(w);
  }
}

// first[i] = 1 where sorted key i starts a run and is no self-loop; first[nnz] = 0.
__global__ void msfFirstKernel(const unsigned long long* __restrict__ keys, Index nnz,
                               unsigned long long loop, int* __restrict__ first) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i <= nnz; i += stride)
    first[i] = i < nnz && keys[i] != loop && (i == 0 || keys[i - 1] != keys[i]) ? 1 : 0;
}

// The canonical list: the run of equal keys that starts at i (at most two entries,
// A(u,v) and A(v,u)) becomes slot first[i] (scanned), with the smaller weight bits.
__global__ void msfCanonKernel(const unsigned long long* __restrict__ keys,
                               const unsigned int* __restrict__ pay,
                               const int* __restrict__ first, Index nnz, int bits,
                               Index* __restrict__ eu, Index* __restrict__ ev,
                               unsigned int* __restrict__ ew) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < nnz; i += stride) {
    const int slot = first[i];
    if (first[i + 1] == slot) continue;
    const unsigned long long key = keys[i];
    unsigned int w = pay[i];
    for (Index j = i + 1; j < nnz && keys[j] == key; ++j) w = pay[j] < w ? pay[j] : w;
    eu[slot] = static_cast<Index>(key >> bits);
    ev[slot] = static_cast<Index>(key & ((1ull << bits) - 1ull));
    ew[slot] = w;
  }
}

__global__ void __launch_bounds__(GB_MSF_NT, GB_MSF_MINB)
msfKernel(MsfArgs a) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const Index gtid = blockIdx.x*GB_MSF_NT + threadIdx.x;
  const Index gthreads = gridDim.x*GB_MSF_NT;
  const bool leader = gtid == 0;
  int barriers = 0, rounds = 0;

  // ---- init --------------------------------------------------------------------------
  for (Index v = gtid; v < a.n; v += gthreads) {
    stRelaxed(a.parent + v, v);
    a.best[v] = MSF_NONE;
  }
  grid.sync();
  ++barriers;

  for (int r = 0;; ++r) {
    const Index len = static_cast<Index>(loadCell(a.counters + MSF_LIVE + r % 3));
    if (len == 0) break;
    ++rounds;
    const Index* in = (r & 1) ? a.live1 : a.live0;
    Index* out = (r & 1) ? a.live0 : a.live1;
    unsigned long long* next = a.counters + MSF_LIVE + (r + 1) % 3;
    if (leader) a.counters[MSF_LIVE + (r + 2) % 3] = 0ull;

    // ---- pick --------------------------------------------------------------------------
    for (Index i = gtid; i < len; i += gthreads) {
      const Index s = r == 0 ? i : __ldcg(in + i);
      const Index ru = ldRelaxed(a.parent + __ldg(a.eu + s));
      const Index rv = ldRelaxed(a.parent + __ldg(a.ev + s));
      if (ru == rv) continue;
      warpAppend(out, 0, next, s);
      const unsigned long long key =
          (static_cast<unsigned long long>(__ldg(a.ew + s)) << 32) | static_cast<unsigned int>(s);
      if (key < __ldcg(a.best + ru)) atomicMin(a.best + ru, key);
      if (key < __ldcg(a.best + rv)) atomicMin(a.best + rv, key);
    }
    grid.sync();
    ++barriers;
    if (loadCell(a.counters + MSF_LIVE + (r + 1) % 3) == 0ull) break;   // no root picked

    // ---- link --------------------------------------------------------------------------
    for (Index v = gtid; v < a.n; v += gthreads) {
      const unsigned long long b = __ldcg(a.best + v);
      if (b == MSF_NONE) continue;
      const Index s = static_cast<Index>(static_cast<unsigned int>(b));
      a.forest[s] = 1;
      ccLink(a.parent, __ldg(a.eu + s), __ldg(a.ev + s));
      a.best[v] = MSF_NONE;
    }
    grid.sync();
    ++barriers;

    // ---- compress ----------------------------------------------------------------------
    ccCompress(a.parent, a.n, gtid, gthreads);
    grid.sync();
    ++barriers;
  }

  if (leader) {
    a.counters[MSF_ROUNDS] = static_cast<unsigned long long>(rounds);
    a.counters[MSF_BARRIERS] = static_cast<unsigned long long>(barriers);
  }
}

// The forest as COO: slot s with off[s + 1] != off[s] (forest[] scanned over m + 1
// entries) goes to position off[s], its weight decoded.
template <typename T>
__global__ void msfForestKernel(const int* __restrict__ off, const Index* __restrict__ eu,
                                const Index* __restrict__ ev,
                                const unsigned int* __restrict__ ew, Index m,
                                Index* __restrict__ src, Index* __restrict__ dst,
                                T* __restrict__ val) {
  Index s = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; s < m; s += stride) {
    const int p = off[s];
    if (off[s + 1] == p) continue;
    src[p] = eu[s];
    dst[p] = ev[s];
    val[p] = msfWeight<T>(ew[s]);
  }
}

// out[b] = the fp64 sum of CTA b's share of x[0, count): strided partial sums, then a
// fixed tree.  Launched with GB_MSF_SUM_CTAS CTAs over the weights and then with one CTA
// over their partials, so the order of the additions depends on count alone.
template <typename T>
__global__ void __launch_bounds__(GB_MSF_SUM_NT)
msfSumKernel(const T* __restrict__ x, Index count, double* __restrict__ out) {
  __shared__ double part[GB_MSF_SUM_NT];
  double s = 0.0;
  for (Index i = blockIdx.x*GB_MSF_SUM_NT + threadIdx.x; i < count;
       i += gridDim.x*GB_MSF_SUM_NT)
    s += static_cast<double>(x[i]);
  part[threadIdx.x] = s;
  __syncthreads();
  for (int h = GB_MSF_SUM_NT/2; h > 0; h >>= 1) {
    if (threadIdx.x < h) part[threadIdx.x] += part[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = part[0];
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_MSF_CUH_
