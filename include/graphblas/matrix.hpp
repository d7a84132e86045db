// graphblast_b200 frontend mirror — graphblas::Matrix<T>.
// The method set and argument checks of reference graphblas/matrix.hpp:14-252 over a
// backend::Matrix<T> held by value as `matrix_` (the CPU verifiers read
// matrix_.sparse_.h_csr*, reference algorithm/bfs.hpp:101-107).  As in vector.hpp a
// method names its pointer arguments and its backend call; `given` does the rest.
#ifndef GRAPHBLAS_MATRIX_HPP_
#define GRAPHBLAS_MATRIX_HPP_

#include <vector>

#include <graphblas/backend/cuda/matrix.hpp>

namespace graphblas {
template <typename T>
class Matrix {
  typedef backend::Matrix<T> Impl;

 public:
  Matrix() {}
  Matrix(Index nrows, Index ncols) : matrix_(nrows, ncols) {}

  // ---- shape, contents --------------------------------------------------------------------
  Info nnew(Index nrows, Index ncols) {
    return (nrows == 0 || ncols == 0) ? GrB_INVALID_VALUE : matrix_.nnew(nrows, ncols);
  }
  Info clear() { return matrix_.clear(); }
  Info dup(const Matrix* rhs) {
    return given([&](Impl& m) { return m.dup(&rhs->matrix_); }, rhs);
  }
  void operator=(const Matrix& rhs) { matrix_.dup(&rhs.matrix_); }
  Info nrows(Index* out) const { return given([&](Impl& m) { return m.nrows(out); }, out); }
  Info ncols(Index* out) const { return given([&](Impl& m) { return m.ncols(out); }, out); }
  Info nvals(Index* out) const { return given([&](Impl& m) { return m.nvals(out); }, out); }

  // ---- build ---------------------------------------------------------------------------------
  // Host COO triples.  The drivers' loader leaves the triples empty when a binary cache
  // exists: then dat_name alone says what to load (reference matrix.hpp:75-95).
  template <typename BinaryOpT>
  Info build(const std::vector<Index>* row_indices, const std::vector<Index>* col_indices,
             const std::vector<T>* values, Index nvals, BinaryOpT dup,
             char* dat_name = NULL) {
    return given([&](Impl& m) {
      const bool no_triples = row_indices->empty() && col_indices->empty() && values->empty();
      if (no_triples && dat_name == NULL) return GrB_NO_VALUE;
      if (dat_name != NULL && row_indices->empty()) return m.build(dat_name);
      return m.build(row_indices, col_indices, values, nvals, dup, dat_name);
    }, row_indices, col_indices, values);
  }
  Info build(const std::vector<T>* values, Index nvals) {
    return given([&](Impl& m) { return m.build(values, nvals); }, values);
  }
  // Dense row-major DEVICE values (nrows*ncols), adopted without ownership.
  Info adoptDense(T* d_values) {
    return given([&](Impl& m) { return m.adoptDense(d_values); }, d_values);
  }
  // DEVICE CSR arrays: row_ptr (nrows+1), col_ind (nvals), values (nvals).
  Info build(Index* d_row_ptr, Index* d_col_ind, T* d_values, Index nvals) {
    return given([&](Impl& m) {
      return nvals == 0 ? GrB_INVALID_VALUE : m.build(d_row_ptr, d_col_ind, d_values, nvals);
    }, d_row_ptr, d_col_ind, d_values);
  }

  // ---- element and tuple access ------------------------------------------------------------
  Info setElement(Index row, Index col) { return matrix_.setElement(row, col); }
  Info extractElement(T* out, Index row, Index col) {
    return given([&](Impl& m) { return m.extractElement(out, row, col); }, out);
  }
  Info extractTuples(std::vector<Index>* row_indices, std::vector<Index>* col_indices,
                     std::vector<T>* values, Index* n) {
    return given([&](Impl& m) { return m.extractTuples(row_indices, col_indices, values, n); },
                 row_indices, col_indices, values, n);
  }
  Info extractTuples(std::vector<T>* values, Index* n) {
    return given([&](Impl& m) { return m.extractTuples(values, n); }, values, n);
  }
  const T operator[](Index ind) { return matrix_[ind]; }

  // ---- handy methods -------------------------------------------------------------------------
  Info print(bool force_update = false)  { return matrix_.print(force_update); }
  Info check()                           { return matrix_.check(); }
  Info setNrows(Index nrows)             { return matrix_.setNrows(nrows); }
  Info setNcols(Index ncols)             { return matrix_.setNcols(ncols); }
  Info resize(Index nrows, Index ncols)  { return matrix_.resize(nrows, ncols); }
  Info setStorage(Storage kind)          { return matrix_.setStorage(kind); }
  Info getStorage(Storage* out) const {
    return given([&](Impl& m) { return m.getStorage(out); }, out);
  }
  template <typename U>
  Info fill(Index axis, Index nvals, U start) { return matrix_.fill(axis, nvals, start); }
  template <typename U>
  Info fillAscending(Index axis, Index nvals, U start) {
    return matrix_.fillAscending(axis, nvals, start);
  }

  Impl matrix_;

 private:
  // `work(backend object)` once none of `needed` is NULL (see vector.hpp).
  template <typename Work, typename... Pointers>
  Info given(Work&& work, const Pointers*... needed) const {
    const bool missing = ((needed == NULL) || ...);
    if (missing) return GrB_NULL_POINTER;
    return work(const_cast<Impl&>(matrix_));
  }
};
}  // namespace graphblas

#endif  // GRAPHBLAS_MATRIX_HPP_
