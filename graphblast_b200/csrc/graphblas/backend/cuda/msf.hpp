// graphblast_b200 backend — host side of the minimum spanning forest (kernels/msf.cuh):
// the input checks, the canonical weighted edge list, one cooperative launch, and the
// forest installed as a symmetric CSR.  algorithm::msf comes here.
#ifndef GRAPHBLAS_BACKEND_CUDA_MSF_HPP_
#define GRAPHBLAS_BACKEND_CUDA_MSF_HPP_

#include <type_traits>

#include "graphblas/backend/cuda/ewise_matrix.hpp"
#include "graphblas/backend/cuda/graph_input.hpp"
#include "graphblas/backend/cuda/ingest.hpp"
#include "graphblas/backend/cuda/kernels/msf.cuh"

namespace graphblas {
namespace backend {

// Of the last msfRun that ran: the rounds with a pick phase, the grid barriers of the
// kernel, and the device time of building the canonical edge list (CUDA events, ms).
struct MsfStats {
  int rounds = 0;
  int barriers = 0;
  float canon_ms = 0.f;
};

// F = the minimum spanning forest of the undirected graph G of A: the edge {i, j}, i !=
// j, when A(i,j) or A(j,i) is stored, weighted by the smaller stored value; edges ranked
// by (w, min(i,j), max(i,j)).  F(i,j) = F(j,i) = w({i,j}) on every forest edge, -0.0
// written as +0.0; F is n x n, a sorted CSR installed as symmetric, and may be A.
// *nedges = the forest's edges, *weight = their fp64 sum in an order fixed by the forest,
// *ms = the device time (CUDA events); each may be NULL.
// Refusals, F untouched: a dense A (GrB_NOT_IMPLEMENTED); A not square or F not n x n
// (GrB_DIMENSION_MISMATCH); a missing CSR (GrB_UNINITIALIZED_OBJECT); an FP32 A with a
// NaN on a stored off-diagonal entry (GrB_INVALID_VALUE).
// Memory, computed from the sizes and not measured.  The sort of the stored entries
// takes 24 bytes per entry (keys 2 x 8, weight payloads 2 x 4), 48 per canonical edge of
// a symmetric A.  The kernel holds 24 bytes per canonical edge (endpoints 2 x 4, weight
// bits 4, two live lists 2 x 4, forest flag 4) and 12 per vertex (parent 4, best word 8).
// At R-MAT-22 (128 312 156 stored entries, 64 156 078 edges) that is 3.1 GB for the sort
// and 1.6 GB for the kernel.  F costs what ingestCooToCsr needs for 2(n - 1) entries at
// most.
template <typename T>
Info msfRun(Matrix<T>* F, const Matrix<T>* A, long long* nedges, double* weight,
            float* ms = NULL) {
  static_assert(std::is_same<T, int>::value || std::is_same<T, float>::value,
                "msf reads int or float matrices");
  CHECK(graphCheck("msf", A, false, F));
  const SparseMatrix<T>& S = A->sparse_;
  const Index n = S.nrows_;
  const Index nnz = hasEntries(S) ? S.nvals_ : 0;
  const size_t nz = static_cast<size_t>(nnz);

  GpuTimer clock, canon;
  clock.Start();
  canon.Start();
  cudaStream_t s = gbStream();
  unsigned long long* cells = reinterpret_cast<unsigned long long*>(
      gbMalloc(MSF_NCELLS*sizeof(unsigned long long)));
  const DeviceBlock cells_block(cells);
  CUDA_CALL(cudaMemsetAsync(cells, 0, MSF_NCELLS*sizeof(unsigned long long), s));

  // ---- the canonical edge list ---------------------------------------------------------
  const int bits = ingestBitsFor(n);
  const unsigned long long loop = (1ull << (2*bits)) - 1ull;
  Index m = 0;
  ScratchLayout edges;
  size_t eu_at = 0, ev_at = 0, ew_at = 0;
  DeviceBlock list(NULL);
  if (nnz > 0) {
    DeviceBlock keys(gbMalloc(nz*8));
    DeviceBlock pay(gbMalloc(nz*4));
    msfEmitKernel<T><<<gridFor(nz, 256), 256, 0, s>>>(S.d_csrRowPtr_, S.d_csrColInd_,
        S.d_csrVal_, n, nnz, bits, loop, keys.at<unsigned long long>(), pay.at<unsigned int>(),
        cells);
    GB_KERNEL_CHECK();
    if (std::is_same<T, float>::value && runtime().fetch(cells + MSF_NAN) != 0ull)
      return GrB_INVALID_VALUE;
    {  // freed before `first` is allocated: the sort's peak stays 24 bytes per entry
      DeviceBlock keys_tmp(gbMalloc(nz*8));
      DeviceBlock pay_tmp(gbMalloc(nz*4));
      unsigned long long* k = keys.at<unsigned long long>();
      unsigned long long* k_tmp = keys_tmp.at<unsigned long long>();
      unsigned int* p = pay.at<unsigned int>();
      unsigned int* p_tmp = pay_tmp.at<unsigned int>();
      radixSortPairs(&k, &p, &k_tmp, &p_tmp, nnz, 2*bits);
      // the sort may have left its output in the other buffers: ownership follows it
      if (k != keys.at<unsigned long long>()) keys.swap(keys_tmp);
      if (p != pay.at<unsigned int>()) pay.swap(pay_tmp);
    }
    DeviceBlock first(gbMalloc((nz + 1)*sizeof(int)));
    msfFirstKernel<<<gridFor(nz + 1, 256), 256, 0, s>>>(keys.at<unsigned long long>(), nnz,
        loop, first.at<int>());
    GB_KERNEL_CHECK();
    m = static_cast<Index>(scanExclusiveInPlace(first.at<int>(), static_cast<long long>(nnz) + 1));
    const size_t slots = static_cast<size_t>(m);
    eu_at = edges.place(slots*sizeof(Index));
    ev_at = edges.place(slots*sizeof(Index));
    ew_at = edges.place(slots*sizeof(unsigned int));
    DeviceBlock canonical(m > 0 ? gbMalloc(edges.bytes) : NULL);
    list.swap(canonical);
    if (m > 0) {
      msfCanonKernel<<<gridFor(nz, 256), 256, 0, s>>>(keys.at<unsigned long long>(),
          pay.at<unsigned int>(), first.at<int>(), nnz, bits, list.at<Index>(eu_at),
          list.at<Index>(ev_at), list.at<unsigned int>(ew_at));
      GB_KERNEL_CHECK();
    }
  }  // first, pay and keys are freed here
  const size_t mm = static_cast<size_t>(m);
  const Index* eu = list.at<Index>(eu_at);
  const Index* ev = list.at<Index>(ev_at);
  const unsigned int* ew = list.at<unsigned int>(ew_at);
  canon.Stop();

  // ---- Borůvka rounds ------------------------------------------------------------------
  ScratchLayout l;
  const size_t parent_at = l.place(static_cast<size_t>(n)*sizeof(Index));
  const size_t best_at = l.place(static_cast<size_t>(n)*sizeof(unsigned long long));
  const size_t live0_at = l.place(mm*sizeof(Index));
  const size_t live1_at = l.place(mm*sizeof(Index));
  const size_t forest_at = l.place((mm + 1)*sizeof(int));
  const DeviceBlock block(m > 0 ? gbMalloc(l.bytes) : NULL);
  Index nf = 0;
  unsigned long long host_cells[MSF_NCELLS] = {};
  if (m > 0) {
    MsfArgs args;
    args.eu = eu;  args.ev = ev;  args.ew = ew;
    args.n = n;
    args.m = m;
    args.parent = block.at<Index>(parent_at);
    args.best = block.at<unsigned long long>(best_at);
    args.live0 = block.at<Index>(live0_at);
    args.live1 = block.at<Index>(live1_at);
    args.forest = block.at<int>(forest_at);
    args.counters = cells;
    const unsigned long long live = static_cast<unsigned long long>(m);
    CUDA_CALL(cudaMemcpyAsync(cells + MSF_LIVE, &live, sizeof(live), cudaMemcpyHostToDevice, s));
    CUDA_CALL(cudaMemsetAsync(args.forest, 0, (mm + 1)*sizeof(int), s));
    CHECK((launchCooperative<msfKernel, GB_MSF_NT>(s, args)));
    CUDA_CALL(cudaMemcpyAsync(host_cells, cells, sizeof(host_cells), cudaMemcpyDeviceToHost, s));
    nf = static_cast<Index>(scanExclusiveInPlace(args.forest, static_cast<long long>(m) + 1));
  }

  // ---- F: the forest both ways, and its weight -----------------------------------------
  const size_t nfz = static_cast<size_t>(nf);
  ScratchLayout coo;
  const size_t src_at = coo.place(nfz*sizeof(Index));
  const size_t dst_at = coo.place(nfz*sizeof(Index));
  const size_t val_at = coo.place(nfz*sizeof(T));
  const size_t sum_at = coo.place((GB_MSF_SUM_CTAS + 1)*sizeof(double));
  const DeviceBlock out(gbMalloc(coo.bytes));
  double* sums = out.at<double>(sum_at);
  if (nf > 0) {
    msfForestKernel<T><<<gridFor(mm, 256), 256, 0, s>>>(block.at<int>(forest_at), eu, ev, ew,
        m, out.at<Index>(src_at), out.at<Index>(dst_at), out.at<T>(val_at));
    GB_KERNEL_CHECK();
  }
  msfSumKernel<T><<<GB_MSF_SUM_CTAS, GB_MSF_SUM_NT, 0, s>>>(out.at<T>(val_at), nf, sums + 1);
  GB_KERNEL_CHECK();
  msfSumKernel<double><<<1, GB_MSF_SUM_NT, 0, s>>>(sums + 1, GB_MSF_SUM_CTAS, sums);
  GB_KERNEL_CHECK();
  double total = 0.0;
  CUDA_CALL(cudaMemcpyAsync(&total, sums, sizeof(double), cudaMemcpyDeviceToHost, s));
  Index* rowptr = NULL;
  Index* colind = NULL;
  T* val = NULL;
  const Index kept = ingestCooToCsr<T>(n, n, out.at<Index>(src_at), out.at<Index>(dst_at),
      out.at<T>(val_at), nf, GB_INGEST_SYMMETRIZE, &rowptr, &colind, &val);
  CHECK(installSymmetric(F, kept, rowptr, colind, val));
  clock.Stop();
  CUDA_CALL(cudaStreamSynchronize(s));
  MsfStats& stats = lastStats<MsfStats>();
  stats.rounds = static_cast<int>(host_cells[MSF_ROUNDS]);
  stats.barriers = static_cast<int>(host_cells[MSF_BARRIERS]);
  stats.canon_ms = canon.ElapsedMillis();
  if (nedges != NULL) *nedges = nf;
  if (weight != NULL) *weight = total;
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_MSF_HPP_
