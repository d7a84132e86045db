// graphblast_b200 backend — host side of local graph clustering (kernels/lgc.cuh): the
// input (graph_input.hpp), the scratch, the one cooperative launch of the push and the
// launches of the sweep cut.  algorithm::lgc and algorithm::lgcSweep come here.
#ifndef GRAPHBLAS_BACKEND_CUDA_LGC_HPP_
#define GRAPHBLAS_BACKEND_CUDA_LGC_HPP_

#include <cmath>
#include <limits>

#include <cub/cub.cuh>

#include "graphblas/backend/cuda/graph_input.hpp"
#include "graphblas/backend/cuda/ingest.hpp"
#include "graphblas/backend/cuda/kernels/lgc.cuh"

namespace graphblas {
namespace backend {

// p = the approximate personalised PageRank of source s (kernels/lgc.cuh states the
// arithmetic); r (when not NULL) = the final residual; *rounds = the rounds run, at most
// max_rounds (max_rounds <= 0 runs none: p = 0, r = the unit vector of s); *ms (when not
// NULL) = the device time, from CUDA events.  p and r become dense with nrows(A)
// entries.  mode: 0 chooses each round's route by the frontier volume against
// switchpoint*nnz, 1 takes only sparse rounds, 2 only dense rounds.  s, alpha and eps
// are checked by the caller.  Refusals: those of graphCheck (with the CSC), then r the
// same vector as p (GrB_INVALID_VALUE).  stats (when not NULL) = {pushed volume, dense
// rounds}.
// Scratch: the counter cells, seven n-word arrays (c, in_f, claim, two frontier lists,
// the touched list, r when not asked for) and the pattern's zero row pointers.
template <typename a>
Info lgcRun(Vector<float>* p, Vector<float>* r, const Matrix<a>* A, Index s, double alpha,
            double eps, int max_rounds, int mode, float switchpoint, int* rounds,
            float* ms = NULL, unsigned long long* stats = NULL) {
  CHECK(graphCheck("lgc", A, true, p, r));
  if (r == p) return GrB_INVALID_VALUE;
  const SparseMatrix<a>& S = A->sparse_;
  const Index n = S.nrows_;
  GpuTimer clock;
  clock.Start();
  if (rounds != NULL) *rounds = 0;
  if (stats != NULL) stats[0] = stats[1] = 0ull;
  cudaStream_t stream = gbStream();

  const size_t array = static_cast<size_t>(n)*sizeof(Index);   // bytes of an n-word array
  ScratchLayout l;
  const size_t counters = l.place(LGC_NCELLS*sizeof(unsigned long long));
  const size_t c = l.place(array), in_f = l.place(array), claim = l.place(array);
  const size_t front0 = l.place(array), front1 = l.place(array), touched = l.place(array);
  const size_t r_scratch = l.place(array);
  const size_t zero_rows = l.place(GraphPattern::zeroRowBytes(S));
  const DeviceBlock block(gbMalloc(l.bytes));
  const GraphPattern g(S, block.at<Index>(zero_rows));
  LgcArgs args;
  args.n = n;
  args.source = s;
  args.nnz = S.nvals_;
  args.alpha = alpha;
  args.eps = eps;
  args.max_rounds = max_rounds;
  args.mode = mode;
  args.switchpoint = switchpoint;
  args.counters = block.at<unsigned long long>(counters);
  args.c        = block.at<float>(c);
  args.in_f     = block.at<int>(in_f);
  args.claim    = block.at<int>(claim);
  args.front[0] = block.at<Index>(front0);
  args.front[1] = block.at<Index>(front1);
  args.touched  = block.at<Index>(touched);
  args.row_ptr = g.row_ptr;  args.row_ind = g.row_ind;
  args.in_ptr = g.in_ptr();
  args.in_ind = g.in_ind();
  CUDA_CALL(cudaMemsetAsync(args.counters, 0, LGC_NCELLS*sizeof(unsigned long long), stream));

  CHECK(p->setStorage(GrB_DENSE));
  CHECK(p->dense_.allocateGpu());
  args.p = p->dense_.d_val_;
  if (r != NULL) {
    CHECK(r->setStorage(GrB_DENSE));
    CHECK(r->dense_.allocateGpu());
    args.r = r->dense_.d_val_;
  } else {
    args.r = block.at<float>(r_scratch);
  }
  CHECK((launchCooperative<lgcKernel, GB_LGC_NT>(stream, args)));
  clock.Stop();
  p->dense_.touched();
  if (r != NULL) r->dense_.touched();
  unsigned long long cells[LGC_NCELLS];
  CUDA_CALL(cudaMemcpyAsync(cells, args.counters, sizeof(cells), cudaMemcpyDeviceToHost,
                            stream));
  runtime().sync();
  if (rounds != NULL) *rounds = static_cast<int>(cells[LGC_ROUNDS]);
  if (stats != NULL) { stats[0] = cells[LGC_PUSHED]; stats[1] = cells[LGC_DENSE]; }
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

// The sweep cut of p over A: the support U = {v : p[v] > 0 and d[v] > 0} ordered by
// p[v]/d[v] (fp32) descending, ties by ascending id; S_k its first k vertices;
// phi_k = cut(S_k)/min(vol(S_k), nnz - vol(S_k)) in double over the k whose denominator
// is positive, with vol and cut exact 64-bit counts (d = row lengths; cut counts the
// stored A(i,j) with i in S_k, j not, self-loops never).  cluster = 1 on S_k* for the
// smallest k* of least phi, else 0, dense; *size = k*, *conductance = phi_k*; when no k
// qualifies, an empty cluster, *size = 0 and *conductance = NaN.  Refusals: those of
// graphCheck (with the CSC), then cluster the same vector as p (GrB_INVALID_VALUE).
// Device work: the keys of U by an atomic append, the stable radix sort of
// ingest.hpp on them, rank[v], a warp per position counting its neighbours ranked
// before it, two inclusive 64-bit scans and a two-pass (phi, k) minimum.
template <typename a>
Info lgcSweepRun(Vector<float>* cluster, Vector<float>* p, const Matrix<a>* A, int* size,
                 double* conductance, float* ms = NULL) {
  CHECK(graphCheck("lgcSweep", A, true, cluster, p));
  if (cluster == p) return GrB_INVALID_VALUE;
  const SparseMatrix<a>& S = A->sparse_;
  const Index n = S.nrows_;
  const long long nnz = S.nvals_;
  GpuTimer clock;
  clock.Start();
  if (size != NULL) *size = 0;
  if (conductance != NULL) *conductance = std::numeric_limits<double>::quiet_NaN();
  cudaStream_t stream = gbStream();
  Storage p_type = GrB_UNKNOWN;
  CHECK(p->getStorage(&p_type));
  if (p_type == GrB_SPARSE) CHECK(p->sparse2dense(0.f));   // absent entries are 0
  if (p_type != GrB_UNKNOWN) CHECK(p->materialize());       // else p holds no entry
  CHECK(cluster->setStorage(GrB_DENSE));
  CHECK(cluster->dense_.allocateGpu());
  float* out = cluster->dense_.d_val_;
  if (n == 0) {
    clock.Stop();
    if (ms != NULL) *ms = clock.ElapsedMillis();
    return GrB_SUCCESS;
  }
  const float* pv = p_type != GrB_UNKNOWN ? p->dense_.d_val_ : NULL;
  const size_t nn = static_cast<size_t>(n);
  ScratchLayout l;
  const size_t cells_at = l.place(3*sizeof(unsigned long long));   // m, then (phi, k)
  const size_t keys_at = l.place(nn*8), keys_tmp_at = l.place(nn*8);
  const size_t rank_at = l.place(nn*sizeof(Index));
  const size_t zero_rows = l.place(GraphPattern::zeroRowBytes(S));
  const DeviceBlock block(gbMalloc(l.bytes));
  const GraphPattern g(S, block.at<Index>(zero_rows));
  unsigned long long* cells = block.at<unsigned long long>(cells_at);
  unsigned long long* keys = block.at<unsigned long long>(keys_at);
  unsigned long long* keys_tmp = block.at<unsigned long long>(keys_tmp_at);
  Index* rank = block.at<Index>(rank_at);
  CUDA_CALL(cudaMemsetAsync(cells, 0, sizeof(unsigned long long), stream));
  CUDA_CALL(cudaMemsetAsync(cells + 1, 0xff, 2*sizeof(unsigned long long), stream));
  const int gn = gridFor(nn, GB_SWEEP_NT);
  lgcSweepKeysKernel<<<gn, GB_SWEEP_NT, 0, stream>>>(pv, g.row_ptr, n, keys, cells, rank);
  GB_KERNEL_CHECK();
  const Index m = static_cast<Index>(runtime().fetch(cells));
  Index best_k = -1;
  double best_phi = std::numeric_limits<double>::quiet_NaN();
  if (m > 0) {
    radixSortPairs(&keys, NULL, &keys_tmp, NULL, m, 64);   // may swap the two buffers
    const unsigned long long* sorted = keys;
    const int gm = gridFor(static_cast<size_t>(m), GB_SWEEP_NT);
    lgcSweepRankKernel<<<gm, GB_SWEEP_NT, 0, stream>>>(sorted, m, rank);
    GB_KERNEL_CHECK();
    // dcut and dvol in the other key buffer and a fresh one, the scans in place
    long long* dcut = reinterpret_cast<long long*>(keys_tmp);
    const DeviceBlock dvol_block(gbMalloc(static_cast<size_t>(m)*8));
    long long* dvol = dvol_block.at<long long>();
    lgcSweepDeltaKernel<<<gridFor(static_cast<size_t>(m)*32, GB_SWEEP_NT), GB_SWEEP_NT, 0,
                          stream>>>(sorted, m, g.row_ptr, g.row_ind, g.col_ptr, g.col_ind,
                                    rank, dcut, dvol);
    GB_KERNEL_CHECK();
    size_t cub_bytes = 0;
    CUDA_CALL(cub::DeviceScan::InclusiveSum(NULL, cub_bytes, dcut, dcut, m, stream));
    const DeviceBlock cub_tmp(gbMalloc(cub_bytes));
    CUDA_CALL(cub::DeviceScan::InclusiveSum(cub_tmp.at<void>(), cub_bytes, dcut, dcut, m,
                                            stream));
    CUDA_CALL(cub::DeviceScan::InclusiveSum(cub_tmp.at<void>(), cub_bytes, dvol, dvol, m,
                                            stream));
    lgcSweepBestKernel<false><<<gm, GB_SWEEP_NT, 0, stream>>>(dcut, dvol, m, nnz, cells + 1);
    GB_KERNEL_CHECK();
    lgcSweepBestKernel<true><<<gm, GB_SWEEP_NT, 0, stream>>>(dcut, dvol, m, nnz, cells + 1);
    GB_KERNEL_CHECK();
    unsigned long long best[2];
    CUDA_CALL(cudaMemcpyAsync(best, cells + 1, sizeof(best), cudaMemcpyDeviceToHost, stream));
    runtime().sync();
    if (best[0] != ~0ull) {
      best_k = static_cast<Index>(best[1]);
      std::memcpy(&best_phi, &best[0], sizeof(best_phi));
    }
  }
  const Index members = best_k + 1;    // 0 when no prefix qualifies
  lgcSweepOutKernel<<<gn, GB_SWEEP_NT, 0, stream>>>(rank, n, members, out);
  GB_KERNEL_CHECK();
  clock.Stop();
  cluster->dense_.touched();
  if (size != NULL) *size = static_cast<int>(members);
  if (conductance != NULL) *conductance = best_phi;
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_LGC_HPP_
