// graphblast_b200 backend — host side of local graph clustering (kernels/lgc.cuh): the
// refusals, the scratch, the one cooperative launch of the push and the launches of the
// sweep cut.  algorithm::lgc and algorithm::lgcSweep come here.
#ifndef GRAPHBLAS_BACKEND_CUDA_LGC_HPP_
#define GRAPHBLAS_BACKEND_CUDA_LGC_HPP_

#include <cmath>
#include <limits>

#include <cub/cub.cuh>

#include "graphblas/backend/cuda/ingest.hpp"
#include "graphblas/backend/cuda/kernels/lgc.cuh"

namespace graphblas {
namespace backend {

// The refusals lgc and lgcSweep share, in this order and before anything is touched: a
// dense A (GrB_NOT_IMPLEMENTED, naming `what`); A not square, or x or y (when not
// NULL) not of size nrows(A) (GrB_DIMENSION_MISMATCH); an A with stored entries but
// without a device CSR, or non-symmetric without a device CSC (GrB_UNINITIALIZED_OBJECT).
template <typename a>
Info lgcCheck(const char* what, Vector<float>* x, Vector<float>* y, const Matrix<a>* A) {
  if (!A->isSparse()) {
    std::cout << "Error: " << what << " of a dense matrix is not implemented in this backend\n";
    return GrB_NOT_IMPLEMENTED;
  }
  const SparseMatrix<a>* S = &A->sparse_;
  const Index n = S->nrows_;
  if (n != S->ncols_) return GrB_DIMENSION_MISMATCH;
  for (Vector<float>* v : {x, y}) {
    if (v == NULL) continue;
    Index size = 0;
    CHECK(v->size(&size));
    if (size != n) return GrB_DIMENSION_MISMATCH;
  }
  if (n > 0 && S->nvals_ > 0 &&
      (S->d_csrRowPtr_ == NULL || (!S->sameStructure() && S->d_cscColPtr_ == NULL)))
    return GrB_UNINITIALIZED_OBJECT;
  return GrB_SUCCESS;
}

// p = the approximate personalised PageRank of source s (kernels/lgc.cuh states the
// arithmetic); r (when not NULL) = the final residual; *rounds = the rounds run, at most
// max_rounds (max_rounds <= 0 runs none: p = 0, r = the unit vector of s); *ms (when not
// NULL) = the device time, from CUDA events.  p and r become dense with nrows(A)
// entries.  mode: 0 chooses each round's route by the frontier volume against
// switchpoint*nnz, 1 takes only sparse rounds, 2 only dense rounds.  s, alpha and eps
// are checked by the caller.  Refusals as lgcCheck, then r the same vector as p
// (GrB_INVALID_VALUE).  stats (when not NULL) = {pushed volume, dense rounds}.
// Scratch: 256 bytes of counters, six n-word arrays (r when not asked for, c, in_f,
// claim, two frontier lists) and the touched list, freed after the launch.
template <typename a>
Info lgcRun(Vector<float>* p, Vector<float>* r, const Matrix<a>* A, Index s, double alpha,
            double eps, int max_rounds, int mode, float switchpoint, int* rounds,
            float* ms = NULL, unsigned long long* stats = NULL) {
  CHECK(lgcCheck("lgc", p, r, A));
  if (r == p) return GrB_INVALID_VALUE;
  const SparseMatrix<a>* S = &A->sparse_;
  const Index n = S->nrows_;
  GpuTimer clock;
  clock.Start();
  if (rounds != NULL) *rounds = 0;
  if (stats != NULL) stats[0] = stats[1] = 0ull;
  const int grid = cooperativeGrid<lgcKernel, GB_LGC_NT>();
  if (grid < 1) return GrB_PANIC;
  cudaStream_t stream = gbStream();
  const bool stored = S->nvals_ > 0;

  const size_t words = (static_cast<size_t>(n) + 63)/64*64;      // 256-byte aligned arrays
  const size_t rp_words = stored ? 0 : (static_cast<size_t>(n) + 64)/64*64;
  unsigned char* block = static_cast<unsigned char*>(gbMalloc(
      256 + (7*words + rp_words)*sizeof(Index)));
  Index* arrays = reinterpret_cast<Index*>(block + 256);
  LgcArgs args;
  args.n = n;
  args.source = s;
  args.nnz = S->nvals_;
  args.alpha = alpha;
  args.eps = eps;
  args.max_rounds = max_rounds;
  args.mode = mode;
  args.switchpoint = switchpoint;
  args.counters = reinterpret_cast<unsigned long long*>(block);
  args.c        = reinterpret_cast<float*>(arrays);
  args.in_f     = arrays + words;
  args.claim    = arrays + 2*words;
  args.front[0] = arrays + 3*words;
  args.front[1] = arrays + 4*words;
  args.touched  = arrays + 5*words;
  float* r_scratch = reinterpret_cast<float*>(arrays + 6*words);
  if (stored) {
    const bool same = S->sameStructure();
    args.row_ptr = S->d_csrRowPtr_;                 args.row_ind = S->d_csrColInd_;
    args.in_ptr = same ? S->d_csrRowPtr_ : S->d_cscColPtr_;
    args.in_ind = same ? S->d_csrColInd_ : S->d_cscRowInd_;
  } else {                             // no entries: every list is empty
    Index* zero_ptr = arrays + 7*words;
    CUDA_CALL(cudaMemsetAsync(zero_ptr, 0, (static_cast<size_t>(n) + 1)*sizeof(Index),
                              stream));
    args.row_ptr = zero_ptr;  args.row_ind = NULL;
    args.in_ptr = zero_ptr;   args.in_ind = NULL;
  }
  CUDA_CALL(cudaMemsetAsync(block, 0, LGC_NCELLS*sizeof(unsigned long long), stream));

  CHECK(p->setStorage(GrB_DENSE));
  CHECK(p->dense_.allocateGpu());
  args.p = p->dense_.d_val_;
  if (r != NULL) {
    CHECK(r->setStorage(GrB_DENSE));
    CHECK(r->dense_.allocateGpu());
    args.r = r->dense_.d_val_;
  } else {
    args.r = r_scratch;
  }
  void* params[] = { &args };
  CUDA_CALL(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(lgcKernel),
      dim3(grid), dim3(GB_LGC_NT), params, 0, stream));
  GB_KERNEL_CHECK();
  clock.Stop();
  p->dense_.touched();
  if (r != NULL) r->dense_.touched();
  unsigned long long cells[LGC_NCELLS];
  CUDA_CALL(cudaMemcpyAsync(cells, args.counters, sizeof(cells), cudaMemcpyDeviceToHost,
                            stream));
  runtime().sync();
  if (rounds != NULL) *rounds = static_cast<int>(cells[LGC_ROUNDS]);
  if (stats != NULL) { stats[0] = cells[LGC_PUSHED]; stats[1] = cells[LGC_DENSE]; }
  gbFree(block);
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

// The sweep cut of p over A: the support U = {v : p[v] > 0 and d[v] > 0} ordered by
// p[v]/d[v] (fp32) descending, ties by ascending id; S_k its first k vertices;
// phi_k = cut(S_k)/min(vol(S_k), nnz - vol(S_k)) in double over the k whose denominator
// is positive, with vol and cut exact 64-bit counts (d = row lengths; cut counts the
// stored A(i,j) with i in S_k, j not, self-loops never).  cluster = 1 on S_k* for the
// smallest k* of least phi, else 0, dense; *size = k*, *conductance = phi_k*; when no k
// qualifies, an empty cluster, *size = 0 and *conductance = NaN.  Refusals as lgcCheck,
// then cluster the same vector as p (GrB_INVALID_VALUE).
// Device work: the keys of U by an atomic append, the stable radix sort of
// ingest.hpp on them, rank[v], a warp per position counting its neighbours ranked
// before it, two inclusive 64-bit scans and a two-pass (phi, k) minimum.
template <typename a>
Info lgcSweepRun(Vector<float>* cluster, Vector<float>* p, const Matrix<a>* A, int* size,
                 double* conductance, float* ms = NULL) {
  CHECK(lgcCheck("lgcSweep", cluster, p, A));
  if (cluster == p) return GrB_INVALID_VALUE;
  const SparseMatrix<a>* S = &A->sparse_;
  const Index n = S->nrows_;
  const long long nnz = S->nvals_;
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
  const bool stored = nnz > 0;
  const bool same = S->sameStructure();
  const size_t nn = static_cast<size_t>(n);
  Index* zero_ptr = NULL;
  if (!stored) {
    zero_ptr = static_cast<Index*>(gbMalloc((nn + 1)*sizeof(Index)));
    CUDA_CALL(cudaMemsetAsync(zero_ptr, 0, (nn + 1)*sizeof(Index), stream));
  }
  const Index* row_ptr = stored ? S->d_csrRowPtr_ : zero_ptr;
  unsigned long long* cells = static_cast<unsigned long long*>(gbMalloc(
      4*sizeof(unsigned long long)));
  unsigned long long* const key_buf[2] = {
      static_cast<unsigned long long*>(gbMalloc(nn*8)),
      static_cast<unsigned long long*>(gbMalloc(nn*8))};
  unsigned long long* keys = key_buf[0];
  unsigned long long* keys_tmp = key_buf[1];
  Index* rank = static_cast<Index*>(gbMalloc(nn*sizeof(Index)));
  CUDA_CALL(cudaMemsetAsync(cells, 0, sizeof(unsigned long long), stream));
  CUDA_CALL(cudaMemsetAsync(cells + 1, 0xff, 2*sizeof(unsigned long long), stream));
  const int g = gridFor(nn, GB_SWEEP_NT);
  lgcSweepKeysKernel<<<g, GB_SWEEP_NT, 0, stream>>>(pv, row_ptr, n, keys, cells, rank);
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
    long long* dvol = static_cast<long long*>(gbMalloc(static_cast<size_t>(m)*8));
    lgcSweepDeltaKernel<<<gridFor(static_cast<size_t>(m)*32, GB_SWEEP_NT), GB_SWEEP_NT, 0,
                          stream>>>(sorted, m, row_ptr, S->d_csrColInd_,
        same ? NULL : S->d_cscColPtr_, same ? NULL : S->d_cscRowInd_, rank, dcut, dvol);
    GB_KERNEL_CHECK();
    size_t cub_bytes = 0;
    CUDA_CALL(cub::DeviceScan::InclusiveSum(NULL, cub_bytes, dcut, dcut, m, stream));
    void* cub_tmp = gbMalloc(cub_bytes);
    CUDA_CALL(cub::DeviceScan::InclusiveSum(cub_tmp, cub_bytes, dcut, dcut, m, stream));
    CUDA_CALL(cub::DeviceScan::InclusiveSum(cub_tmp, cub_bytes, dvol, dvol, m, stream));
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
    gbFree(cub_tmp);
    gbFree(dvol);
  }
  const Index members = best_k + 1;    // 0 when no prefix qualifies
  lgcSweepOutKernel<<<g, GB_SWEEP_NT, 0, stream>>>(rank, n, members, out);
  GB_KERNEL_CHECK();
  clock.Stop();
  cluster->dense_.touched();
  gbFree(key_buf[0]); gbFree(key_buf[1]); gbFree(rank); gbFree(cells); gbFree(zero_ptr);
  if (size != NULL) *size = static_cast<int>(members);
  if (conductance != NULL) *conductance = best_phi;
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_LGC_HPP_
