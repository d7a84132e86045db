// graphblast_b200 backend — assign into a sparse matrix: submatrices
// C(I, J) = accum(C(I, J), op(A)), columns C(I, j) = u, rows C(i, J) = u and
// constants C(I, J) = val.
//
// Every form is one merge of C with the embedded source E (kernels/assign.cuh):
//   1. the lists are checked on the host (range, ALL extent, repeats) and uploaded
//      once;
//   2. E is built: row offsets scattered through I and scanned, entries written in
//      place when J is increasing, through one radixSortPairs pass otherwise;
//   3. C' = C ∪ E on the tiles of ewise_matrix.cuh: count pass (its 64-bit total is
//      the one host read; past INT32_MAX: GrB_OUT_OF_MEMORY), scans, fill pass.
//      Without accum C's entries inside I x J are dropped and E's value wins; with
//      accum a matched pair writes accum(c, e);
//   4. C' is installed with replaceDevice.
// Nothing on the device that belongs to an operand changes before the result is
// complete, and a refusal leaves C as it was.  C may be A.
//
// A C marked symmetric stays so when I and J are the same list and, for the
// submatrix form, A is marked symmetric: then C' is symmetric too, and its CSC
// values (a CSRCSC C) come from a second fill pass over the same items with the
// other orientation's values of C and of E.  The row and column forms always
// clear the flag.
#ifndef GRAPHBLAS_BACKEND_CUDA_ASSIGN_MATRIX_HPP_
#define GRAPHBLAS_BACKEND_CUDA_ASSIGN_MATRIX_HPP_

#include <type_traits>
#include <vector>

#include "graphblas/backend/cuda/kernels/assign.cuh"
#include "graphblas/backend/cuda/kernels/kernels.hpp"
#include "graphblas/backend/cuda/extract.hpp"
#include "graphblas/backend/cuda/sparse_matrix.hpp"

namespace graphblas {
namespace backend {

// op(A) as the nrows x ncols CSR to embed: nrows + 1 pointers, nnz entries, and
// (may be NULL) the other orientation's values at the same slots.
template <typename T>
struct AssignSource {
  const Index* ptr;
  const Index* ind;
  const T*     val;
  const T*     oval;
  Index        nrows;
  Index        nnz;
};

// The embedded source E, an m x n CSR in fresh pool arrays (oval when asked for).
template <typename T>
struct AssignEmbedded {
  Index  nnz = 0;
  Index* ptr = NULL;
  Index* ind = NULL;
  T*     val = NULL;
  T*     oval = NULL;
  void release() { gbFree(ptr); gbFree(ind); gbFree(val); if (oval != NULL) gbFree(oval); }
};

// Both lists in range (GrB_INVALID_INDEX), then both free of repeats
// (GrB_INVALID_VALUE).
inline Info assignCheckLists(IndexList* I, const std::vector<Index>* rows, Index nI,
                             Index m, IndexList* J, const std::vector<Index>* cols,
                             Index nJ, Index n) {
  CHECK(I->check(rows, nI, m));
  CHECK(J->check(cols, nJ, n));
  if (!I->distinct(m) || !J->distinct(n)) return GrB_INVALID_VALUE;
  return GrB_SUCCESS;
}

// E's row offsets: the row lengths of S (ptr == NULL: len each) through I, scanned.
inline Index* assignRowOffsets(Index m, const IndexList& I, Index nI, const Index* ptr,
                               Index len) {
  cudaStream_t s = gbStream();
  Index* Eptr = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(m) + 1)*sizeof(Index)));
  CUDA_CALL(cudaMemsetAsync(Eptr, 0, (static_cast<size_t>(m) + 1)*sizeof(Index), s));
  if (nI > 0) {
    assignRowLengthsKernel<<<gridFor(nI, 256), 256, 0, s>>>(Eptr, I.device(), ptr, nI, len);
    GB_KERNEL_CHECK();
  }
  scanExclusiveAsync(Eptr, static_cast<long long>(m) + 1, NULL);
  return Eptr;
}

template <typename T>
void assignAllocEntries(AssignEmbedded<T>* E, Index nnz, bool with_oval) {
  const size_t nz = static_cast<size_t>(nnz > 0 ? nnz : 1);
  E->nnz = nnz;
  E->ind = reinterpret_cast<Index*>(gbMalloc(nz*sizeof(Index)));
  E->val = reinterpret_cast<T*>(gbMalloc(nz*sizeof(T)));
  E->oval = with_oval ? reinterpret_cast<T*>(gbMalloc(nz*sizeof(T))) : NULL;
}

// E = S placed at (I[p], J[q]) in an m x n matrix; n bounds J's entries.
template <typename T>
void assignEmbed(const AssignSource<T>& S, Index m, Index n, const IndexList& I,
                 const IndexList& J, bool with_oval, AssignEmbedded<T>* E) {
  cudaStream_t s = gbStream();
  E->ptr = assignRowOffsets(m, I, S.nrows, S.ptr, 0);
  assignAllocEntries(E, S.nnz, with_oval);
  if (S.nnz == 0) return;
  const size_t nz = static_cast<size_t>(S.nnz);
  const int grid = gridFor(nz, 256);
  if (J.nonDecreasing()) {
    assignEmbedKernel<T, false><<<grid, 256, 0, s>>>(E->ind, E->val, E->oval, E->ptr,
        I.device(), J.device(), S.ptr, S.ind, S.val, S.oval, S.nrows, S.nnz, 0, NULL, NULL);
    GB_KERNEL_CHECK();
    return;
  }
  // J unsorted (so given): sort each row's entries by their column in C
  const int cbits = ingestBitsFor(n);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(gbMalloc(nz*8));
  unsigned long long* keys_tmp = reinterpret_cast<unsigned long long*>(gbMalloc(nz*8));
  unsigned int* pay = reinterpret_cast<unsigned int*>(gbMalloc(nz*4));
  unsigned int* pay_tmp = reinterpret_cast<unsigned int*>(gbMalloc(nz*4));
  assignEmbedKernel<T, true><<<grid, 256, 0, s>>>(NULL, NULL, NULL, NULL, NULL, J.device(),
      S.ptr, S.ind, S.val, S.oval, S.nrows, S.nnz, cbits, keys, pay);
  GB_KERNEL_CHECK();
  radixSortPairs(&keys, &pay, &keys_tmp, &pay_tmp, S.nnz, ingestBitsFor(S.nrows) + cbits);
  assignSortedEmbedKernel<T><<<grid, 256, 0, s>>>(E->ind, E->val, E->oval, E->ptr,
      I.device(), S.ptr, S.val, S.oval, keys, pay, S.nnz, cbits);
  GB_KERNEL_CHECK();
  gbFree(pay_tmp); gbFree(pay); gbFree(keys_tmp); gbFree(keys);
}

// A bitmap of the list over extent, or NULL for ALL.
inline unsigned int* assignBitmap(const IndexList& L, Index n, Index extent) {
  if (L.all()) return NULL;
  cudaStream_t s = gbStream();
  const size_t words = (static_cast<size_t>(extent) + 31)/32;
  unsigned int* bits = reinterpret_cast<unsigned int*>(gbMalloc((words > 0 ? words : 1)*4));
  CUDA_CALL(cudaMemsetAsync(bits, 0, (words > 0 ? words : 1)*4, s));
  if (n > 0) {
    assignMarkKernel<<<gridFor(n, 256), 256, 0, s>>>(bits, L.device(), n);
    GB_KERNEL_CHECK();
  }
  return bits;
}

// The merge's count and fill passes, and C' installed.  Takes E (freed here).
template <typename c, typename Keep, typename Combine>
Info assignMergeWith(SparseMatrix<c>* C, AssignEmbedded<c>* E, Keep keep, Combine combine,
                     bool symmetric) {
  cudaStream_t s = gbStream();
  const Index m = C->nrows_;
  typename SparseMatrix<c>::View Cv = C->view(false);
  // a C never built is an empty m x n matrix
  Index* empty_ptr = NULL;
  const c* c_oval = symmetric ? C->view(true).val : NULL;
  if (!Cv.complete()) {
    empty_ptr = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(m) + 1)*sizeof(Index)));
    CUDA_CALL(cudaMemsetAsync(empty_ptr, 0, (static_cast<size_t>(m) + 1)*sizeof(Index), s));
    Cv.ptr = empty_ptr;
    Cv.ind = empty_ptr;
    Cv.val = E->val;
  }
  const Index c_nnz = empty_ptr != NULL ? 0 : C->nvals_;
  const long long total = static_cast<long long>(c_nnz) + E->nnz;
  const long long ntiles = (total + GB_EWM_TILE - 1)/GB_EWM_TILE;
  int* tiles = reinterpret_cast<int*>(gbMalloc(static_cast<size_t>(ntiles + 1)*sizeof(int)));
  unsigned long long* count = reinterpret_cast<unsigned long long*>(
      gbMalloc(sizeof(unsigned long long)));
  Index* rowptr = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(m) + 1)*sizeof(Index)));
  CUDA_CALL(cudaMemsetAsync(rowptr, 0, (static_cast<size_t>(m) + 1)*sizeof(Index), s));
  CUDA_CALL(cudaMemsetAsync(count, 0, sizeof(unsigned long long), s));
  if (ntiles > 0) {
    ewiseMatrixCountKernel<true, Keep><<<static_cast<unsigned int>(ntiles), GB_EWM_NT, 0, s>>>(
        Cv.ptr, Cv.ind, E->ptr, E->ind, m, total, tiles, rowptr, count, keep);
    GB_KERNEL_CHECK();
  }
  const unsigned long long nnz64 = runtime().fetch(count);
  gbFree(count);
  if (nnz64 > static_cast<unsigned long long>(INT32_MAX)) {
    gbFree(rowptr); gbFree(tiles);
    if (empty_ptr != NULL) gbFree(empty_ptr);
    E->release();
    return GrB_OUT_OF_MEMORY;
  }
  const Index nnz = static_cast<Index>(nnz64);
  scanExclusiveAsync(rowptr, static_cast<long long>(m) + 1, NULL);
  const size_t nz = static_cast<size_t>(nnz > 0 ? nnz : 1);
  Index* colind = reinterpret_cast<Index*>(gbMalloc(nz*sizeof(Index)));
  c* val = reinterpret_cast<c*>(gbMalloc(nz*sizeof(c)));
  c* oval = NULL;
  if (ntiles > 0) {
    scanExclusiveAsync(tiles, ntiles, NULL);
    const unsigned int grid = static_cast<unsigned int>(ntiles);
    ewiseMatrixFillKernel<true, c><<<grid, GB_EWM_NT, 0, s>>>(Cv.ptr, Cv.ind, Cv.val,
        E->ptr, E->ind, E->val, m, total, tiles, colind, val, combine, combine, keep);
    GB_KERNEL_CHECK();
    if (symmetric && E->oval != NULL) {
      // the same items again with the other orientation's values: C' is symmetric,
      // so these are its CSC values at its CSR slots
      oval = reinterpret_cast<c*>(gbMalloc(nz*sizeof(c)));
      Index* scratch = reinterpret_cast<Index*>(gbMalloc(nz*sizeof(Index)));
      ewiseMatrixFillKernel<true, c><<<grid, GB_EWM_NT, 0, s>>>(Cv.ptr, Cv.ind,
          c_nnz > 0 ? c_oval : Cv.val, E->ptr, E->ind, E->oval, m, total, tiles, scratch,
          oval, combine, combine, keep);
      GB_KERNEL_CHECK();
      gbFree(scratch);
    }
  } else if (symmetric && E->oval != NULL) {
    oval = reinterpret_cast<c*>(gbMalloc(nz*sizeof(c)));
  }
  gbFree(tiles);
  if (empty_ptr != NULL) gbFree(empty_ptr);
  E->release();
  C->replaceDevice(nnz, rowptr, colind, val, NULL, NULL, oval, symmetric);
  return GrB_SUCCESS;
}

// Without accum: C's entries in I x J go, E's values win.  With accum: a union
// combining matched pairs as accum(c, e).
template <typename c, typename AccumT>
Info assignMerge(SparseMatrix<c>* C, AssignEmbedded<c>* E, AccumT accum, const IndexList& I,
                 Index nI, const IndexList& J, Index nJ, bool symmetric) {
  if constexpr (AccumIsNull<AccumT>::value) {
    unsigned int* rbits = assignBitmap(I, nI, C->nrows_);
    unsigned int* cbits = assignBitmap(J, nJ, C->ncols_);
    const Info info = assignMergeWith(C, E, AssignKeep{rbits, cbits}, AssignTakeNew(),
                                      symmetric);
    if (rbits != NULL) gbFree(rbits);
    if (cbits != NULL) gbFree(cbits);
    return info;
  } else {
    return assignMergeWith(C, E, EwmKeepAll(), accum, symmetric);
  }
}

// Whether C' may stay symmetric, and whether its CSC values can be computed then
// (a CSRCSC C needs C's and E's other-orientation values).
template <typename c>
bool assignKeepsSymmetry(const SparseMatrix<c>* C, const IndexList& I, const IndexList& J,
                         bool source_symmetric, bool source_has_oval) {
  if (!C->symmetric_ || !source_symmetric || C->nrows_ != C->ncols_ || !I.sameAs(J))
    return false;
  if (C->format_ != GrB_SPARSE_MATRIX_CSRCSC) return true;
  return source_has_oval && (C->nvals_ == 0 || C->view(true).val != NULL);
}

// C(I, J) = accum(C(I, J), op(A)), op(A) = Aᵀ with transpose_a.  C may be A.
template <typename c, typename a, typename AccumT>
Info assignMatrix(SparseMatrix<c>* C, AccumT accum, const SparseMatrix<a>* A,
                  bool transpose_a, const std::vector<Index>* row_indices, Index nrows,
                  const std::vector<Index>* col_indices, Index ncols) {
  if constexpr (!std::is_same<c, a>::value) {
    return GrB_DOMAIN_MISMATCH;
  } else {
    const typename SparseMatrix<a>::View Av = A->view(transpose_a);
    const typename SparseMatrix<a>::View Ov = A->view(!transpose_a);
    // the frontend checks op(A)'s shape; checked again for callers that reach the
    // backend through the reference's frontend
    if (Av.dim != nrows || Av.other != ncols) return GrB_DIMENSION_MISMATCH;
    IndexList I, J;
    CHECK(assignCheckLists(&I, row_indices, nrows, C->nrows_, &J, col_indices, ncols,
                           C->ncols_));
    if (!Av.complete()) return GrB_UNINITIALIZED_OBJECT;
    const bool symmetric = assignKeepsSymmetry(C, I, J, A->symmetric_ && nrows == ncols,
                                               Ov.val != NULL);
    const bool with_oval = symmetric && C->format_ == GrB_SPARSE_MATRIX_CSRCSC;
    I.upload();
    J.upload();
    AssignSource<a> S = {Av.ptr, Av.ind, Av.val, with_oval ? Ov.val : NULL, nrows, A->nvals_};
    AssignEmbedded<c> E;
    assignEmbed(S, C->nrows_, C->ncols_, I, J, with_oval, &E);
    return assignMerge(C, &E, accum, I, nrows, J, ncols, symmetric);
  }
}

// C(I, J) = accum(C(I, J), val): every position of I x J ends up stored.
template <typename c, typename TS, typename AccumT>
Info assignConstant(SparseMatrix<c>* C, AccumT accum, TS val,
                    const std::vector<Index>* row_indices, Index nrows,
                    const std::vector<Index>* col_indices, Index ncols) {
  IndexList I, J;
  CHECK(assignCheckLists(&I, row_indices, nrows, C->nrows_, &J, col_indices, ncols,
                         C->ncols_));
  const long long block = static_cast<long long>(nrows)*ncols;
  if (block > static_cast<long long>(INT32_MAX)) return GrB_OUT_OF_MEMORY;
  const bool symmetric = assignKeepsSymmetry(C, I, J, true, true);
  const bool with_oval = symmetric && C->format_ == GrB_SPARSE_MATRIX_CSRCSC;
  I.upload();
  J.upload();
  cudaStream_t s = gbStream();
  AssignEmbedded<c> E;
  E.ptr = assignRowOffsets(C->nrows_, I, nrows, NULL, ncols);
  assignAllocEntries(&E, static_cast<Index>(block), with_oval);
  if (block > 0) {
    const int grid = gridFor(static_cast<size_t>(block), 256);
    if (J.nonDecreasing()) {
      assignConstKernel<c, Index><<<grid, 256, 0, s>>>(E.ind, E.val, E.oval, E.ptr,
          I.device(), J.device(), nrows, ncols, static_cast<c>(val));
    } else {
      // the sorted J: J's entries as keys, sorted
      const size_t nj = static_cast<size_t>(ncols);
      unsigned long long* keys = reinterpret_cast<unsigned long long*>(gbMalloc(nj*8));
      unsigned long long* keys_tmp = reinterpret_cast<unsigned long long*>(gbMalloc(nj*8));
      unsigned int* pay = reinterpret_cast<unsigned int*>(gbMalloc(nj*4));
      unsigned int* pay_tmp = reinterpret_cast<unsigned int*>(gbMalloc(nj*4));
      extractMapKeysKernel<<<gridFor(nj, 256), 256, 0, s>>>(keys, pay, J.device(), ncols);
      GB_KERNEL_CHECK();
      radixSortPairs(&keys, &pay, &keys_tmp, &pay_tmp, ncols, ingestBitsFor(C->ncols_));
      assignConstKernel<c, unsigned long long><<<grid, 256, 0, s>>>(E.ind, E.val, E.oval,
          E.ptr, I.device(), keys, nrows, ncols, static_cast<c>(val));
      gbFree(pay_tmp); gbFree(pay); gbFree(keys_tmp); gbFree(keys);
    }
    GB_KERNEL_CHECK();
  }
  return assignMerge(C, &E, accum, I, nrows, J, ncols, symmetric);
}

// C(I, j) = u (column, vertical) or C(i, J) = u (row): u as an nI x 1 or 1 x nJ
// matrix, its stored entries (every entry of a dense u).  i or j is `at`.
template <bool Column, typename c, typename U, typename AccumT>
Info assignVector(SparseMatrix<c>* C, AccumT accum, const Vector<U>* u,
                  const std::vector<Index>* indices, Index nindices, Index at) {
  if constexpr (!std::is_same<c, U>::value) {
    return GrB_DOMAIN_MISMATCH;
  } else {
    Index u_size;
    CHECK(const_cast<Vector<U>*>(u)->size(&u_size));
    const Index extent = Column ? C->nrows_ : C->ncols_;
    const Index other = Column ? C->ncols_ : C->nrows_;
    // the frontend checks these; checked again for the reference's frontend
    if (u_size != nindices || at >= other) return GrB_DIMENSION_MISMATCH;
    if (at < 0) return GrB_INVALID_INDEX;
    const std::vector<Index> one(1, at);
    IndexList L, P;
    CHECK(L.check(indices, nindices, extent));
    CHECK(P.check(&one, 1, other));
    if (!L.distinct(extent)) return GrB_INVALID_VALUE;
    if (u->vec_type_ != GrB_DENSE && u->vec_type_ != GrB_SPARSE)
      return GrB_UNINITIALIZED_OBJECT;
    CHECK(u->materialize());
    L.upload();
    P.upload();
    cudaStream_t s = gbStream();
    const bool dense = u->vec_type_ == GrB_DENSE;
    const Index nnz = dense ? u_size : u->sparse_.nvals_;
    const U* u_val = dense ? u->dense_.d_val_ : u->sparse_.d_val_;
    // the source's pointers and indices: a column is nI rows of at most one entry
    // (column 0), a row one row of u's indices
    const Index nptr = Column ? nindices + 1 : 2;
    Index* ptr = reinterpret_cast<Index*>(gbMalloc(static_cast<size_t>(nptr)*sizeof(Index)));
    Index* ind = reinterpret_cast<Index*>(gbMalloc(static_cast<size_t>(nnz > 0 ? nnz : 1)*sizeof(Index)));
    const Index* u_ind = dense ? NULL : u->sparse_.d_ind_;
    if (Column) {
      assignStoredBelowKernel<<<gridFor(static_cast<size_t>(nptr), 256), 256, 0, s>>>(ptr,
          u_ind, nnz, nindices, dense);
      CUDA_CALL(cudaMemsetAsync(ind, 0, static_cast<size_t>(nnz > 0 ? nnz : 1)*sizeof(Index), s));
    } else {
      const Index bounds[2] = {0, nnz};
      copyAsync(ptr, bounds, 2, cudaMemcpyHostToDevice);
      if (dense)
        assignStoredBelowKernel<<<gridFor(static_cast<size_t>(nnz) + 1, 256), 256, 0, s>>>(
            ind, NULL, 0, nnz > 0 ? nnz - 1 : 0, true);
      else if (nnz > 0)
        copyAsync(ind, u_ind, static_cast<size_t>(nnz), cudaMemcpyDeviceToDevice);
    }
    GB_KERNEL_CHECK();
    AssignSource<U> S = {ptr, ind, u_val, NULL, Column ? nindices : 1, nnz};
    AssignEmbedded<c> E;
    const IndexList& I = Column ? L : P;
    const IndexList& J = Column ? P : L;
    assignEmbed(S, C->nrows_, C->ncols_, I, J, false, &E);
    const Info info = assignMerge(C, &E, accum, I, Column ? nindices : 1, J,
                                  Column ? 1 : nindices, false);
    gbFree(ind);
    gbFree(ptr);
    return info;
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_ASSIGN_MATRIX_HPP_
