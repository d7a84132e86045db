// graphblast_b200 backend — host side of k-truss and truss decomposition
// (kernels/ktruss.cuh): the input checks, the undirected view, the edge slots and
// support items, one cooperative launch, and the result installed as a symmetric CSR.
// algorithm::ktruss and algorithm::trussness come here.
#ifndef GRAPHBLAS_BACKEND_CUDA_KTRUSS_HPP_
#define GRAPHBLAS_BACKEND_CUDA_KTRUSS_HPP_

#include <climits>
#include <type_traits>

#include "graphblas/backend/cuda/ewise_matrix.hpp"
#include "graphblas/backend/cuda/graph_input.hpp"
#include "graphblas/backend/cuda/kernels/ktruss.cuh"

namespace graphblas {
namespace backend {

// Of the last ktrussRun: the rounds that removed edges, the levels that did, and the
// time of the support pass inside the kernel (globaltimer, milliseconds).
struct KtrussStats {
  int rounds = 0;
  int levels = 0;
  float support_ms = 0.f;
};

// k >= 2: C = the k-truss of the undirected simple graph G of A's pattern, C(i,j) =
// C(j,i) = the number of triangles of the k-truss that contain {i, j}; *count (when not
// NULL) = its undirected edges.  k == 0: C = the truss decomposition, C(i,j) = C(j,i) =
// tau({i, j}) on every edge of G; *count = the largest tau, 0 without an edge.  C is n x
// n, a sorted CSR installed as symmetric, and may be A.  *ms (when not NULL) = the
// device time, from CUDA events.
// Refusals, C untouched: a dense A (GrB_NOT_IMPLEMENTED); A not square or C not n x n
// (GrB_DIMENSION_MISMATCH); a missing CSR, or a missing CSC on an A that is not
// sameStructure() (GrB_UNINITIALIZED_OBJECT); an FP32 C with n > 2^24 (GrB_INVALID_VALUE);
// a symmetrised pattern or support item list past 2^31 - 1 entries (GrB_OUT_OF_MEMORY).
// The undirected view is A's CSR when A is sameStructure(), else pattern(A ∪ Aᵀ) built
// by the matrix eWiseAdd (ewise_matrix.hpp) into a temporary.
// Scratch, over the view's nnz entries (R-MAT-22: 128 312 156): per entry its row and
// its edge slot; per slot (indexed by the canonical entry) the support and the state;
// the item offsets (per entry, scanned in place); and the item list, one 8-byte item
// per edge plus one per extra chunk of a long shorter list, which holds the support
// items and then the peel list.  About 5 x 4 + 8/2 = 24 bytes per entry, 3.1 GB at
// R-MAT-22 (computed from the sizes, not measured), plus the counter cells and, for a
// non-symmetric A, the symmetrised pattern.
template <typename c, typename a>
Info ktrussRun(Matrix<c>* C, const Matrix<a>* A, int k, long long* count, float* ms = NULL) {
  static_assert(std::is_same<c, int>::value || std::is_same<c, float>::value,
                "ktruss writes int or float matrices");
  CHECK(graphCheck("k-truss", A, true, C));
  const SparseMatrix<a>& S = A->sparse_;
  const Index n = S.nrows_;
  if (std::is_same<c, float>::value && n > (1 << 24)) return GrB_INVALID_VALUE;

  GpuTimer clock;
  clock.Start();
  cudaStream_t s = gbStream();
  // the undirected view
  SparseMatrix<a> sym(n, n);
  sym.format_ = GrB_SPARSE_MATRIX_CSRONLY;
  const Index* ptr = S.d_csrRowPtr_;
  const Index* ind = S.d_csrColInd_;
  Index nnz = hasEntries(S) ? S.nvals_ : 0;
  if (nnz > 0 && !S.sameStructure()) {
    Descriptor tran;
    CHECK(tran.set(GrB_INP1, GrB_TRAN));
    CHECK((ewiseMatrix<true>(&sym, PlusMultipliesSemiring<a>(), &S, &S, &tran)));
    ptr = sym.d_csrRowPtr_;
    ind = sym.d_csrColInd_;
    nnz = sym.nvals_;
  }
  const size_t nz = static_cast<size_t>(nnz);

  ScratchLayout l;
  const size_t cells = l.place(KT_NCELLS*sizeof(int));
  const size_t erow = l.place(nz*sizeof(Index));
  const size_t eid = l.place(nz*sizeof(Index));
  const size_t sup = l.place(nz*sizeof(int));
  const size_t state = l.place(nz*sizeof(int));
  const size_t offset = l.place(nz*sizeof(int));
  const DeviceBlock block(gbMalloc(l.bytes));
  CUDA_CALL(cudaMemsetAsync(block.at<void>(cells), 0, KT_NCELLS*sizeof(int), s));
  DeviceBlock items(NULL);              // the support items, then the peel list
  if (nnz > 0) {
    CUDA_CALL(cudaMemsetAsync(block.at<void>(sup), 0, nz*sizeof(int), s));
    ktrussPrepKernel<<<gridFor(nz, 256), 256, 0, s>>>(ptr, ind, n, nnz, block.at<Index>(erow),
        block.at<Index>(eid), block.at<int>(state), block.at<int>(offset));
    GB_KERNEL_CHECK();
    const unsigned long long total = scanExclusiveInPlace(block.at<int>(offset), nnz);
    if (total > static_cast<unsigned long long>(INT_MAX)) return GrB_OUT_OF_MEMORY;
    const int nitems = static_cast<int>(total);
    DeviceBlock list(gbMalloc(static_cast<size_t>(nitems)*sizeof(int2)));
    items.swap(list);
    ktrussItemsKernel<<<gridFor(nz, 256), 256, 0, s>>>(ptr, ind, block.at<Index>(erow),
        block.at<int>(state), block.at<int>(offset), nnz, items.at<int2>());
    GB_KERNEL_CHECK();
    const int min_cell = INT_MAX;
    CUDA_CALL(cudaMemcpyAsync(block.at<int>(cells) + KT_MIN, &min_cell, sizeof(int),
                              cudaMemcpyHostToDevice, s));
    CUDA_CALL(cudaMemcpyAsync(block.at<int>(cells) + KT_MIN + 1, &min_cell, sizeof(int),
                              cudaMemcpyHostToDevice, s));
    KtArgs args;
    args.ptr = ptr;  args.ind = ind;
    args.erow = block.at<Index>(erow);
    args.eid = block.at<Index>(eid);
    args.nnz = nnz;
    args.sup = block.at<int>(sup);
    args.state = block.at<int>(state);
    args.items = items.at<int2>();
    args.nitems = nitems;
    args.k = k;
    args.cells = block.at<int>(cells);
    CHECK((launchCooperative<ktrussKernel, GB_KT_NT>(s, args)));
  }

  // the result: every kept entry of the view, in stored order
  const bool keep_all = k == 0;
  Index* rowptr = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(n) + 1)*sizeof(Index)));
  CUDA_CALL(cudaMemsetAsync(rowptr, 0, (static_cast<size_t>(n) + 1)*sizeof(Index), s));
  if (nnz > 0) {
    ktrussCountKernel<<<gridFor(static_cast<size_t>(n)*32, 256), 256, 0, s>>>(
        ptr, block.at<Index>(eid), block.at<int>(state), n, keep_all, rowptr);
    GB_KERNEL_CHECK();
  }
  const Index kept = static_cast<Index>(scanExclusiveInPlace(rowptr, static_cast<long long>(n) + 1));
  Index* colind = reinterpret_cast<Index*>(gbMalloc((kept > 0 ? kept : 1)*sizeof(Index)));
  c* val = reinterpret_cast<c*>(gbMalloc((kept > 0 ? kept : 1)*sizeof(c)));
  if (kept > 0) {
    ktrussFillKernel<c><<<gridFor(static_cast<size_t>(n)*32, 256), 256, 0, s>>>(
        ptr, ind, block.at<Index>(eid), block.at<int>(state), block.at<int>(sup), n, keep_all,
        rowptr, colind, val);
    GB_KERNEL_CHECK();
  }
  int host_cells[KT_NCELLS];
  CUDA_CALL(cudaMemcpyAsync(host_cells, block.at<int>(cells), sizeof(host_cells),
                            cudaMemcpyDeviceToHost, s));
  CUDA_CALL(cudaStreamSynchronize(s));
  DeviceBlock(NULL).swap(items);       // the items are freed before C takes the result
  CHECK(installSymmetric(C, kept, rowptr, colind, val));
  clock.Stop();
  KtrussStats& stats = lastStats<KtrussStats>();
  stats.rounds = host_cells[KT_ROUNDS];
  stats.levels = host_cells[KT_LEVELS];
  stats.support_ms = host_cells[KT_SUPPORT_US]*1e-3f;
  if (count != NULL) *count = keep_all ? host_cells[KT_KMAX] : kept/2;
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_KTRUSS_HPP_
