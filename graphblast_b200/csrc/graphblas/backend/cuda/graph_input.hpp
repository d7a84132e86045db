// graphblast_b200 backend — the input and output of the cooperative graph algorithms
// (cc.hpp, greedy_schedule.hpp, lgc.hpp, bc.hpp, ktruss.hpp, scc.hpp, msf.hpp, cdlp.hpp):
// one check of A and the results, one view of A's pattern as their kernels read it, one
// installer of a symmetric result matrix and the statistics of the last call.
#ifndef GRAPHBLAS_BACKEND_CUDA_GRAPH_INPUT_HPP_
#define GRAPHBLAS_BACKEND_CUDA_GRAPH_INPUT_HPP_

#include "graphblas/backend/cuda/ewise_matrix.hpp"

namespace graphblas {
namespace backend {

template <typename a>
bool hasEntries(const SparseMatrix<a>& S) { return S.nrows_ > 0 && S.nvals_ > 0; }

// The refusals the cooperative graph algorithms share, in this order and before
// anything is touched:
//   a dense A (GrB_NOT_IMPLEMENTED, naming `what`);
//   A not square, or one of the results (NULL ones skipped) not of size nrows(A): a
//   vector of another size, a matrix not nrows(A) x nrows(A) (GrB_DIMENSION_MISMATCH);
//   an A with stored entries but no device CSR, or, when needs_csc is set and A is not
//   sameStructure(), no device CSC (GrB_UNINITIALIZED_OBJECT).
// An algorithm's own refusals come after these.
template <typename W>
Info resultCheck(Vector<W>* v, Index n) {
  Index size = n;
  if (v != NULL) CHECK(v->size(&size));
  return size == n ? GrB_SUCCESS : GrB_DIMENSION_MISMATCH;
}
template <typename c>
Info resultCheck(Matrix<c>* C, Index n) {
  Index rows = n, cols = n;
  if (C != NULL) { CHECK(C->nrows(&rows)); CHECK(C->ncols(&cols)); }
  return rows == n && cols == n ? GrB_SUCCESS : GrB_DIMENSION_MISMATCH;
}

template <typename a, typename... R>
Info graphCheck(const char* what, const Matrix<a>* A, bool needs_csc, R*... results) {
  if (!A->isSparse()) {
    std::cout << "Error: " << what << " of a dense matrix is not implemented in this backend\n";
    return GrB_NOT_IMPLEMENTED;
  }
  const SparseMatrix<a>& S = A->sparse_;
  if (S.nrows_ != S.ncols_) return GrB_DIMENSION_MISMATCH;
  for (Info info : {resultCheck(results, S.nrows_)...})
    if (info != GrB_SUCCESS) return info;
  const bool no_csr = S.d_csrRowPtr_ == NULL || S.d_csrColInd_ == NULL;
  const bool no_csc = needs_csc && !S.sameStructure() &&
                      (S.d_cscColPtr_ == NULL || S.d_cscRowInd_ == NULL);
  if (hasEntries(S) && (no_csr || no_csc)) return GrB_UNINITIALIZED_OBJECT;
  return GrB_SUCCESS;
}

// A's pattern, for an A that passed graphCheck: its CSR out-lists, and its CSC in-lists
// or NULL when they are the CSR (sameStructure()).  When A stores no entry, every list
// is NULL except row_ptr, which is `zero_rows`: zeroRowBytes(S) bytes of the caller's
// scratch, set to zero here on the stream so that every row is empty (NULL when the
// caller wants no row pointers then).
struct GraphPattern {
  const Index* row_ptr;  const Index* row_ind;   // CSR
  const Index* col_ptr;  const Index* col_ind;   // CSC; NULL when it is the CSR

  template <typename a>
  static size_t zeroRowBytes(const SparseMatrix<a>& S) {
    return hasEntries(S) ? 0 : (static_cast<size_t>(S.nrows_) + 1)*sizeof(Index);
  }

  template <typename a>
  GraphPattern(const SparseMatrix<a>& S, Index* zero_rows)
      : row_ptr(zero_rows), row_ind(NULL), col_ptr(NULL), col_ind(NULL) {
    if (hasEntries(S)) {
      row_ptr = S.d_csrRowPtr_;  row_ind = S.d_csrColInd_;
      if (!S.sameStructure()) { col_ptr = S.d_cscColPtr_;  col_ind = S.d_cscRowInd_; }
    } else if (zero_rows != NULL) {
      CUDA_CALL(cudaMemsetAsync(zero_rows, 0, zeroRowBytes(S), gbStream()));
    }
  }

  bool stored() const { return row_ind != NULL; }   // A has stored entries
  // The in-lists: the CSC when it is held apart, else the CSR.
  const Index* in_ptr() const { return col_ptr != NULL ? col_ptr : row_ptr; }
  const Index* in_ind() const { return col_ptr != NULL ? col_ind : row_ind; }
};

// Installs the sorted CSR (rowptr, colind, val) of `count` entries as C, marked
// symmetric; C takes the arrays.  The values are symmetric too, so C's column-major
// values, when its format keeps them, are a copy of the CSR's.
template <typename c>
Info installSymmetric(Matrix<c>* C, Index count, Index* rowptr, Index* colind, c* val) {
  c* cscval = C->sparse_.format_ == GrB_SPARSE_MATRIX_CSRCSC ? copyOnDevice(val, count) : NULL;
  C->sparse_.replaceDevice(count, rowptr, colind, val, NULL, NULL, cscval, true);
  return C->setStorage(GrB_SPARSE);
}

// The statistics S of the last call of the algorithm that keeps them.
template <typename S>
S& lastStats() {
  static S stats;
  return stats;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_GRAPH_INPUT_HPP_
