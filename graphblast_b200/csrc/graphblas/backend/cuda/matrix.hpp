// graphblast_b200 backend — Matrix<T>: storage-tagged wrapper over SparseMatrix
// and DenseMatrix (the row-major array SpMM reads and writes).  Only the storage
// the tag names holds data: switching drops the other one, and with the sparse
// arrays every cache derived from them (SpMV tiles, hub index, pull summaries).
//
// Replaces reference graphblas/backend/cuda/matrix.hpp:21-352: same method set
// (the frontend graphblas::Matrix<T> forwards to every one of them) and the same
// members nrows_/ncols_/nvals_/sparse_/dense_/mat_type_ that the reference CPU
// verifiers and tests read (reference algorithm/bfs.hpp:101, test/gvxm.cu:44).
#ifndef GRAPHBLAS_BACKEND_CUDA_MATRIX_HPP_
#define GRAPHBLAS_BACKEND_CUDA_MATRIX_HPP_

#include <vector>
#include <iostream>

#include "graphblas/backend/cuda/sparse_matrix.hpp"
#include "graphblas/backend/cuda/dense_matrix.hpp"

namespace graphblas {
namespace backend {

template <typename T>
class Matrix {
 public:
  Matrix() : nrows_(0), ncols_(0), nvals_(0), sparse_(0, 0), dense_(0, 0),
             mat_type_(GrB_SPARSE) {}
  explicit Matrix(Index nrows, Index ncols)
      : nrows_(nrows), ncols_(ncols), nvals_(0), sparse_(nrows, ncols),
        dense_(nrows, ncols), mat_type_(GrB_SPARSE) {}
  ~Matrix() {}

  bool isSparse() const { return mat_type_ == GrB_SPARSE; }
  bool isDense()  const { return mat_type_ == GrB_DENSE; }

  Info nnew(Index nrows, Index ncols) {
    CHECK(sparse_.nnew(nrows, ncols));
    CHECK(dense_.nnew(nrows, ncols));
    nrows_ = nrows;
    ncols_ = ncols;
    return GrB_SUCCESS;
  }

  Info dup(const Matrix* rhs) {
    if (rhs->isDense()) {
      CHECK(dense_.dup(&rhs->dense_));
      return setStorage(GrB_DENSE);
    }
    CHECK(setStorage(rhs->mat_type_));
    if (isSparse()) return sparse_.dup(&rhs->sparse_);
    std::cout << "Error: Failed to call dup!\n";
    return GrB_UNINITIALIZED_OBJECT;
  }

  Info clear() {
    mat_type_ = GrB_UNKNOWN;
    nvals_    = 0;
    CHECK(sparse_.clear());
    CHECK(dense_.clear());
    return GrB_SUCCESS;
  }

  Info nrows(Index* out) {
    if (isSparse())     CHECK(sparse_.nrows(&nrows_));
    else if (isDense()) CHECK(dense_.nrows(&nrows_));
    *out = nrows_;
    return GrB_SUCCESS;
  }

  Info ncols(Index* out) {
    if (isSparse())     CHECK(sparse_.ncols(&ncols_));
    else if (isDense()) CHECK(dense_.ncols(&ncols_));
    *out = ncols_;
    return GrB_SUCCESS;
  }

  Info nvals(Index* out) {
    if (isSparse())     CHECK(sparse_.nvals(&nvals_));
    else if (isDense()) CHECK(dense_.nvals(&nvals_));
    *out = nvals_;
    return GrB_SUCCESS;
  }

  template <typename BinaryOpT>
  Info build(const std::vector<Index>* row_indices,
      const std::vector<Index>* col_indices, const std::vector<T>* values, Index nvals,
      BinaryOpT dup, char* dat_name) {
    CHECK(setStorage(GrB_SPARSE));
    if (sparse_.nvals_ > 0) sparse_.clear();
    return sparse_.build(row_indices, col_indices, values, nvals, dup,
        dat_name);
  }

  Info build(char* dat_name) {
    CHECK(setStorage(GrB_SPARSE));
    return sparse_.build(dat_name);
  }

  // Dense row-major values; on a refusal the matrix is left as it was.
  Info build(const std::vector<T>* values, Index nvals) {
    CHECK(dense_.build(values, nvals));
    return setStorage(GrB_DENSE);
  }
  Info buildDense(const T* h_values, long long nvals) {
    CHECK(dense_.build(h_values, nvals));
    return setStorage(GrB_DENSE);
  }
  // A caller-owned row-major device array, used in place.
  Info adoptDense(T* d_values) {
    CHECK(dense_.adopt(d_values));
    return setStorage(GrB_DENSE);
  }

  // Device CSR pointers, adopted without ownership.
  Info build(Index* row_ptr, Index* col_ind, T* values, Index nvals) {
    CHECK(setStorage(GrB_SPARSE));
    return sparse_.build(row_ptr, col_ind, values, nvals);
  }

  Info setElement(Index row_index, Index col_index) {
    if (isSparse()) return sparse_.setElement(row_index, col_index);
    return GrB_UNINITIALIZED_OBJECT;
  }

  Info extractElement(T* val, Index row_index, Index col_index) {
    if (isSparse()) return sparse_.extractElement(val, row_index, col_index);
    return GrB_UNINITIALIZED_OBJECT;
  }

  Info extractTuples(std::vector<Index>* row_indices, std::vector<Index>* col_indices,
      std::vector<T>* values, Index* n) {
    if (isSparse())
      return sparse_.extractTuples(row_indices, col_indices, values, n);
    return GrB_UNINITIALIZED_OBJECT;
  }

  Info extractTuples(std::vector<T>* values, Index* n) {
    if (isDense()) return dense_.extractTuples(values, n);
    return GrB_UNINITIALIZED_OBJECT;   // dense storage only (reference :204-209)
  }

  const T operator[](Index ind) {
    if (isSparse()) return sparse_[ind];
    std::cout << "Error: operator[] not defined for dense matrices!\n";
    return T();
  }

  Info print(bool force_update = false) {
    if (isSparse())     return sparse_.print(force_update);
    else if (isDense()) return dense_.print(force_update);
    return GrB_UNINITIALIZED_OBJECT;
  }

  Info check() {
    if (isSparse()) return sparse_.check();
    return GrB_UNINITIALIZED_OBJECT;
  }

  Info setNrows(Index nrows) {
    CHECK(sparse_.setNrows(nrows));
    CHECK(dense_.setNrows(nrows));
    return GrB_SUCCESS;
  }

  Info setNcols(Index ncols) {
    CHECK(sparse_.setNcols(ncols));
    CHECK(dense_.setNcols(ncols));
    return GrB_SUCCESS;
  }

  Info resize(Index nrows, Index ncols) {
    if (isSparse()) return sparse_.resize(nrows, ncols);
    return GrB_UNINITIALIZED_OBJECT;
  }

  // Storage for an output is sized by the operation that fills it (spgemmMasked
  // dups the mask pattern, spmm swaps in its result), so nothing is allocated
  // here; the storage left behind is released.
  Info setStorage(Storage mat_type) {
    if (mat_type == GrB_SPARSE && mat_type_ != GrB_SPARSE) CHECK(dense_.clear());
    if (mat_type == GrB_DENSE && mat_type_ != GrB_DENSE)   CHECK(sparse_.clear());
    mat_type_ = mat_type;
    return GrB_SUCCESS;
  }

  Info getStorage(Storage* mat_type) const {
    *mat_type = mat_type_;
    return GrB_SUCCESS;
  }

  Info getFormat(SparseMatrixFormat* format) const {
    if (isSparse()) return sparse_.getFormat(format);
    std::cout << "Error: Sparse matrix format is not defined for dense matrix!\n";
    return GrB_SUCCESS;
  }

  Info getSymmetry(bool* symmetry) const {
    if (isSparse()) return sparse_.getSymmetry(symmetry);
    std::cout << "Error: Matrix symmetry is not defined for dense matrix!\n";
    return GrB_SUCCESS;
  }

  template <typename U>
  Info fill(Index axis, Index nvals, U start) {
    if (isSparse()) return sparse_.fill(axis, nvals, start);
    return GrB_UNINITIALIZED_OBJECT;
  }

  template <typename U>
  Info fillAscending(Index axis, Index nvals, U start) {
    if (isSparse()) return sparse_.fillAscending(axis, nvals, start);
    return GrB_UNINITIALIZED_OBJECT;
  }

 public:  // (private in the reference; its drivers `#define private public`)
  Index nrows_;
  Index ncols_;
  Index nvals_;

  SparseMatrix<T> sparse_;
  DenseMatrix<T>  dense_;

  Storage mat_type_;
};

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_MATRIX_HPP_
