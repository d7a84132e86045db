// graphblast_b200 backend — DenseMatrix<T>: a row-major device array.
//
// Holds nrows x ncols values, every entry present (nvals = nrows * ncols), in one
// array from the stream-ordered pool (256-byte aligned), or in a caller-owned
// device array it adopts and never frees.  It is what SpMM (spmm.hpp) reads as B
// and writes as C.  Only float storage is built; other element types answer
// GrB_NOT_IMPLEMENTED.  A matrix of more than INT32_MAX elements is refused with
// GrB_OUT_OF_MEMORY, so that Index stays 32-bit, as for the nnz of a product.
#ifndef GRAPHBLAS_BACKEND_CUDA_DENSE_MATRIX_HPP_
#define GRAPHBLAS_BACKEND_CUDA_DENSE_MATRIX_HPP_

#include <algorithm>
#include <climits>
#include <cstdint>
#include <type_traits>
#include <vector>

#include "graphblas/backend/cuda/util.hpp"

namespace graphblas {
namespace backend {

template <typename T>
class DenseMatrix {
 public:
  DenseMatrix() : nrows_(0), ncols_(0), nvals_(0), d_val_(NULL), ownership_(false) {}
  DenseMatrix(Index nrows, Index ncols)
      : nrows_(nrows), ncols_(ncols), nvals_(0), d_val_(NULL), ownership_(false) {}
  ~DenseMatrix() { release(); }

  static constexpr bool kBuilt = std::is_same<T, float>::value;

  long long size() const { return static_cast<long long>(nrows_)*ncols_; }
  static bool fits(long long elements) { return elements <= INT32_MAX; }

  Info nnew(Index nrows, Index ncols) {
    nrows_ = nrows;
    ncols_ = ncols;
    return GrB_SUCCESS;
  }
  Info dup(const DenseMatrix* rhs) {
    if (nrows_ != rhs->nrows_ || ncols_ != rhs->ncols_) return GrB_DIMENSION_MISMATCH;
    if (rhs->d_val_ == NULL) return GrB_UNINITIALIZED_OBJECT;
    if (rhs == this) return GrB_SUCCESS;
    own();
    CUDA_CALL(cudaMemcpyAsync(d_val_, rhs->d_val_, size()*sizeof(T),
        cudaMemcpyDeviceToDevice, gbStream()));
    return GrB_SUCCESS;
  }
  Info clear() { release(); return GrB_SUCCESS; }
  Info nrows(Index* n) const { *n = nrows_; return GrB_SUCCESS; }
  Info ncols(Index* n) const { *n = ncols_; return GrB_SUCCESS; }
  Info nvals(Index* n) const { *n = nvals_; return GrB_SUCCESS; }

  // Row-major host values: more than nrows*ncols is GrB_DIMENSION_MISMATCH, fewer
  // leave the rest 0.
  Info build(const T* h_values, long long nvals) {
    if (!kBuilt) return GrB_NOT_IMPLEMENTED;
    if (nvals < 0) return GrB_INVALID_VALUE;
    if (nvals > size()) return GrB_DIMENSION_MISMATCH;
    if (!fits(size())) return GrB_OUT_OF_MEMORY;
    if (nvals > 0 && h_values == NULL) return GrB_NULL_POINTER;
    own();
    cudaStream_t s = gbStream();
    if (nvals < size())
      CUDA_CALL(cudaMemsetAsync(d_val_, 0, size()*sizeof(T), s));
    if (nvals > 0)
      CUDA_CALL(cudaMemcpyAsync(d_val_, h_values, nvals*sizeof(T),
          cudaMemcpyHostToDevice, s));
    runtime().sync();                      // the host values may go away after the call
    return GrB_SUCCESS;
  }
  Info build(const std::vector<T>* values, Index nvals) {
    if (static_cast<size_t>(nvals) > values->size()) return GrB_INVALID_VALUE;
    return build(values->data(), nvals);
  }

  // A caller-owned device array of nrows*ncols values, read and written in place.
  Info adopt(T* d_values) {
    if (!kBuilt) return GrB_NOT_IMPLEMENTED;
    if (!fits(size())) return GrB_OUT_OF_MEMORY;
    if (d_values == NULL) return GrB_NULL_POINTER;
    release();
    d_val_ = d_values;
    nvals_ = static_cast<Index>(size());
    return GrB_SUCCESS;
  }

  // A device array this object now owns (the result of an operation).
  void take(T* d_values) {
    release();
    d_val_ = d_values;
    ownership_ = true;
    nvals_ = static_cast<Index>(size());
  }

  // The first min(n, nvals) values in row-major order.  n > nvals copies nvals and
  // answers GrB_UNINITIALIZED_OBJECT, n < nvals GrB_INSUFFICIENT_SPACE.
  Info extract(T* h_out, long long n, long long* copied) const {
    if (d_val_ == NULL) return GrB_UNINITIALIZED_OBJECT;
    Info err = GrB_SUCCESS;
    if (n > nvals_) { err = GrB_UNINITIALIZED_OBJECT; n = nvals_; }
    else if (n < nvals_) err = GrB_INSUFFICIENT_SPACE;
    if (n > 0)
      CUDA_CALL(cudaMemcpyAsync(h_out, d_val_, n*sizeof(T), cudaMemcpyDeviceToHost,
          gbStream()));
    runtime().sync();
    if (copied != NULL) *copied = n;
    return err;
  }
  Info extractTuples(std::vector<T>* values, Index* n) {
    values->resize(static_cast<size_t>(std::max<Index>(0, std::min(*n, nvals_))));
    long long copied = 0;
    const Info err = extract(values->data(), *n, &copied);
    *n = static_cast<Index>(copied);
    return err;
  }

  Info print(bool force_update = false) { return GrB_SUCCESS; }
  Info setNrows(Index nrows) { nrows_ = nrows; return GrB_SUCCESS; }
  Info setNcols(Index ncols) { ncols_ = ncols; return GrB_SUCCESS; }
  Info resize(Index nrows, Index ncols) {
    nrows_ = nrows;
    ncols_ = ncols;
    return GrB_SUCCESS;
  }

  Index nrows_;
  Index ncols_;
  Index nvals_;          // nrows * ncols while values are held, else 0
  T*    d_val_;
  bool  ownership_;      // d_val_ came from the pool and is freed here

 private:
  // An owned array of the current size (kept when it already is one).
  void own() {
    if (!ownership_ || d_val_ == NULL) {
      release();
      d_val_ = reinterpret_cast<T*>(gbMalloc(std::max<long long>(size(), 1)*sizeof(T)));
      ownership_ = true;
    }
    nvals_ = static_cast<Index>(size());
  }
  void release() {
    if (ownership_) gbFree(d_val_);   // stream-ordered after the kernels reading it
    d_val_ = NULL;
    ownership_ = false;
    nvals_ = 0;
  }
};

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_DENSE_MATRIX_HPP_
