// graphblast_b200 backend — Vector<T>: dual-storage (sparse list / dense array)
// vector whose storage follows the traversal direction.
//
// Stands in for reference graphblas/backend/cuda/vector.hpp:27-454: same method
// set (the frontend forwards to it) and the members tests reach (sparse_, dense_,
// vec_type_).  Everything that merely hands a call to whichever storage is active
// goes through ONE helper (onActive) that visits the active storage with a generic
// callable; what is specific to this class is the storage state machine:
// the direction heuristic of convert() — the reference's (vector.hpp:292-323):
// with ratio = nnz/size, sparse->dense when ratio > switchpoint and growing,
// dense->sparse when ratio <= switchpoint and shrinking, otherwise remember ratio_ —
// and the conversions, which run as device kernels: sparse->dense = fill +
// scatter, dense->sparse = ordered compaction (kernels/compact.cuh).
#ifndef GRAPHBLAS_BACKEND_CUDA_VECTOR_HPP_
#define GRAPHBLAS_BACKEND_CUDA_VECTOR_HPP_

#include <vector>
#include <iostream>
#include <algorithm>

#include "graphblas/backend/cuda/util.hpp"
#include "graphblas/backend/cuda/descriptor.hpp"
#include "graphblas/backend/cuda/kernels/kernels.hpp"
#include "graphblas/backend/cuda/compact.hpp"
#include "graphblas/backend/cuda/sparse_vector.hpp"
#include "graphblas/backend/cuda/dense_vector.hpp"

namespace graphblas {
namespace backend {

template <typename T>
class Vector {
 public:
  Vector() : nsize_(0), nvals_(0), sparse_(0), dense_(0), vec_type_(GrB_UNKNOWN), ratio_(0) {}
  explicit Vector(Index nsize)
      : nsize_(nsize), nvals_(0), sparse_(nsize), dense_(nsize),
        vec_type_(GrB_UNKNOWN), ratio_(0) {}
  ~Vector() {}

  // ---- storage state ---------------------------------------------------------
  Info setStorage(Storage vec_type) {
    vec_type_ = vec_type;
    return onActive([](auto& active) { return active.allocateGpu(); }, GrB_SUCCESS);
  }
  Info getStorage(Storage* vec_type) const { *vec_type = vec_type_; return GrB_SUCCESS; }
  Info convert(T identity, float switchpoint, Descriptor* desc);
  Info sparse2dense(T identity, Descriptor* desc = NULL);
  Info dense2sparse(T identity, Descriptor* desc);
  Info swap(Vector* rhs);
  // Writes out lazily held values of a dense vector (dense_vector.hpp).
  Info materialize() { return vec_type_ == GrB_DENSE ? dense_.materialize() : GrB_SUCCESS; }
  Info materialize() const { return const_cast<Vector*>(this)->materialize(); }

  // ---- construction: the call decides the storage (fill / dense values -> dense,
  // index-value lists -> sparse; reference :150-156, 241-245) --------------------
  Info nnew(Index nsize) {
    nsize_ = nsize;
    CHECK(sparse_.nnew(nsize));
    return dense_.nnew(nsize);
  }
  template <typename BinaryOpT>
  Info build(const std::vector<Index>* indices, const std::vector<T>* values,
      Index nvals, BinaryOpT dup) {
    vec_type_ = GrB_SPARSE;
    return sparse_.build(indices, values, nvals, dup);
  }
  Info build(const std::vector<T>* values, Index nvals) {
    vec_type_ = GrB_DENSE;
    return dense_.build(values, nvals);
  }
  Info build(Index* indices, T* values, Index nvals) {
    vec_type_ = GrB_SPARSE;
    return sparse_.build(indices, values, nvals);
  }
  Info build(T* values, Index nvals) {
    vec_type_ = GrB_DENSE;
    return dense_.build(values, nvals);
  }
  Info fill(T val) {
    if (vec_type_ != GrB_DENSE) CHECK(setStorage(GrB_DENSE));
    return dense_.fill(val);
  }
  Info fillAscending(Index nvals) {
    if (vec_type_ != GrB_DENSE) CHECK(setStorage(GrB_DENSE));
    return dense_.fillAscending(nvals);
  }
  Info dup(const Vector* rhs) {
    vec_type_ = rhs->vec_type_;
    if (vec_type_ == GrB_SPARSE) return sparse_.dup(&rhs->sparse_);
    if (vec_type_ == GrB_DENSE)  return dense_.dup(&rhs->dense_);
    std::cout << "Error: dup of a vector without storage\n";
    return GrB_UNINITIALIZED_OBJECT;
  }
  // Storage becomes unknown; the dense side is not zero-filled here (the
  // reference does), the fill happens when a storage is chosen again.
  Info clear() {
    vec_type_ = GrB_UNKNOWN;
    nvals_ = 0;
    return sparse_.clear();
  }

  // ---- calls handed to the active storage ----------------------------------------
  Info size(Index* out) {
    return onActive([&](auto& active) { return active.size(&nsize_); }, GrB_SUCCESS,
                    [&] { *out = nsize_; });
  }
  Info nvals(Index* out) {
    return onActive([&](auto& active) { return active.nvals(&nvals_); }, GrB_SUCCESS,
                    [&] { *out = nvals_; });
  }
  Info setElement(T val, Index index) {
    return onActive([&](auto& active) { return active.setElement(val, index); });
  }
  Info extractElement(T* val, Index index) {
    return onActive([&](auto& active) { return active.extractElement(val, index); });
  }
  Info extractTuples(std::vector<Index>* indices, std::vector<T>* values, Index* n) {
    return onActive([&](auto& active) { return active.extractTuples(indices, values, n); });
  }
  // Values only: a sparse vector is densified with fill value 0 first
  // (reference :208-217).
  Info extractTuples(std::vector<T>* values, Index* n) {
    if (vec_type_ == GrB_SPARSE) CHECK(sparse2dense(static_cast<T>(0)));
    if (vec_type_ != GrB_DENSE) return GrB_UNINITIALIZED_OBJECT;
    return dense_.extractTuples(values, n);
  }
  Info resize(Index nvals) {
    return onActive([&](auto& active) { return active.resize(nvals); });
  }
  Info print(bool force_update = false) {
    return onActive([&](auto& active) { return active.print(force_update); }, GrB_SUCCESS);
  }
  Info countUnique(Index* count) { return GrB_SUCCESS; }
  const T& operator[](Index ind) {
    static T none = T();
    if (vec_type_ == GrB_SPARSE) return sparse_[ind];
    if (vec_type_ == GrB_DENSE)  return dense_[ind];
    return none;
  }

 public:  // (private in the reference; its drivers `#define private public`)
  Index           nsize_;
  Index           nvals_;
  SparseVector<T> sparse_;
  DenseVector<T>  dense_;
  Storage         vec_type_;
  float           ratio_;  // nnz/size seen at the previous convert()

 private:
  // Visits the active storage; `otherwise` is the answer when there is none.
  // `then` runs after a successful visit (or when there is no storage and
  // `otherwise` is success).
  template <typename Visit>
  Info onActive(Visit visit, Info otherwise = GrB_UNINITIALIZED_OBJECT) {
    return onActive(visit, otherwise, [] {});
  }
  template <typename Visit, typename Then>
  Info onActive(Visit visit, Info otherwise, Then then) {
    Info status = otherwise;
    if (vec_type_ == GrB_SPARSE)     status = visit(sparse_);
    else if (vec_type_ == GrB_DENSE) status = visit(dense_);
    if (status == GrB_SUCCESS) then();
    return status;
  }
};

// ---- storage state and conversions (the direction switch lives here) ----

// The direction switch.  fill = stored entries / length of the vector in its current
// storage.  A sparse vector turns dense once fill exceeds the switch point while
// still growing; a dense one turns sparse once fill is at or below it while
// shrinking; otherwise only the fill seen is remembered (hysteresis of reference
// vector.hpp:292-323).
template <typename T>
Info Vector<T>::convert(T identity, float switchpoint, Descriptor* desc) {
  if (vec_type_ != GrB_SPARSE && vec_type_ != GrB_DENSE) return GrB_UNINITIALIZED_OBJECT;
  const bool sparse_now = (vec_type_ == GrB_SPARSE);
  Index entries = 0, length = 0;
  if (sparse_now) {
    CHECK(sparse_.nvals(&entries));
    CHECK(sparse_.size(&length));
  } else {
    CHECK(dense_.computeNnz(&entries, identity, desc));
    CHECK(dense_.nvals(&length));
  }
  const float fill = static_cast<float>(entries)/length;
  if (desc->dirinfo())
    std::cout << "Nnz ratio: " << fill << " Switch point: " << switchpoint << std::endl;
  const bool to_dense  = sparse_now  && fill >  switchpoint && fill > ratio_;
  const bool to_sparse = !sparse_now && fill <= switchpoint && fill < ratio_;
  if (to_dense)  return sparse2dense(identity, desc);
  if (to_sparse) return dense2sparse(identity, desc);
  ratio_ = fill;
  return GrB_SUCCESS;
}

// With --opreuse the dense array is left untouched: the fused Boolean pull reads
// the mask instead of the frontier (reference vector.hpp:344-357).
template <typename T>
Info Vector<T>::sparse2dense(T identity, Descriptor* desc) {
  if (vec_type_ == GrB_DENSE) return GrB_SUCCESS;
  if (vec_type_ == GrB_UNKNOWN) {
    CHECK(setStorage(GrB_DENSE));
    return GrB_SUCCESS;
  }

  if (desc != NULL && desc->dirinfo())
    std::cout << "Converting from sparse to dense!\n";

  CHECK(setStorage(GrB_DENSE));
  const Index nvals = sparse_.nvals_;

  bool keep_bits = false;
  if (desc == NULL || !desc->opreuse()) {
    CHECK(dense_.fill(identity));
    if (nvals > 0) {
      const int nt = 256;
      if (desc != NULL && desc->struconly()) {
        scatterConstKernel<<<gridFor(nvals, nt), nt, 0, gbStream()>>>(
            dense_.d_val_, sparse_.d_ind_, (T)1, nvals);
        if (identity == static_cast<T>(0) && dense_.exactBits() != NULL) {
          GB_KERNEL_CHECK();
          scatterBitsKernel<<<gridFor(nvals, nt), nt, 0, gbStream()>>>(
              dense_.exactBits(), sparse_.d_ind_, nvals);
          keep_bits = true;
        }
      } else
        scatterValsKernel<<<gridFor(nvals, nt), nt, 0, gbStream()>>>(
            dense_.d_val_, sparse_.d_ind_, sparse_.d_val_, nvals);
      GB_KERNEL_CHECK();
    }
  }

  vec_type_ = GrB_DENSE;
  dense_.scattered(nvals, keep_bits);
  return GrB_SUCCESS;
}

template <typename T>
Info Vector<T>::dense2sparse(T identity, Descriptor* desc) {
  if (vec_type_ == GrB_SPARSE) return GrB_INVALID_OBJECT;

  if (desc->dirinfo())
    std::cout << "Converting from dense to sparse!\n";

  CHECK(dense_.allocateGpu());
  CHECK(sparse_.allocateGpu());
  const Index n = dense_.nvals_;
  const Index nitems = (n + 7)/8;

  LoadBalanceMode mxv_mode = getEnv("GRB_LOAD_BALANCE_MODE",
      GrB_LOAD_BALANCE_MERGE);

  // Lazy values are only tolerable on the structure-only bitmap path below.
  if (dense_.valuesStale() &&
      !(identity == static_cast<T>(0) && desc->struconly() &&
        mxv_mode == GrB_LOAD_BALANCE_MERGE))
    CHECK(dense_.materialize());

  Index count;
  const unsigned int* bits = dense_.exactBits();
  if (bits != NULL && identity == static_cast<T>(0)) {
    // Compact the bitmap shadow: n/32 words instead of n values.
    const Index nwords = (n + 31)/32;
    if (desc->struconly() && mxv_mode == GrB_LOAD_BALANCE_MERGE) {
      DenseBitsCompactSource<T, true> src;
      src.bits = bits; src.u = dense_.d_val_;
      src.out_ind = sparse_.d_ind_; src.out_val = sparse_.d_val_;
      count = compactOrdered(src, nwords, desc);
    } else {
      DenseBitsCompactSource<T, false> src;
      src.bits = bits; src.u = dense_.d_val_;
      src.out_ind = sparse_.d_ind_; src.out_val = sparse_.d_val_;
      count = compactOrdered(src, nwords, desc);
    }
  } else if (desc->struconly() && mxv_mode == GrB_LOAD_BALANCE_MERGE) {
    DenseCompactSource<T, true> src;
    src.u = dense_.d_val_; src.identity = identity; src.n = n;
    src.out_ind = sparse_.d_ind_; src.out_val = sparse_.d_val_;
    count = compactOrdered(src, nitems, desc);
  } else {
    DenseCompactSource<T, false> src;
    src.u = dense_.d_val_; src.identity = identity; src.n = n;
    src.out_ind = sparse_.d_ind_; src.out_val = sparse_.d_val_;
    count = compactOrdered(src, nitems, desc);
  }
  sparse_.computed(count);

  if (desc->debug()) {
    std::cout << "Dense frontier size: " << n << std::endl;
    std::cout << "Sparse frontier size: " << sparse_.nvals_ << std::endl;
  }

  vec_type_ = GrB_SPARSE;
  return GrB_SUCCESS;
}

template <typename T>
Info Vector<T>::swap(Vector* rhs) {  // NOLINT(build/include_what_you_use)
  // only vectors in the same, known storage can trade contents (reference :430-434)
  if (vec_type_ != rhs->vec_type_ || vec_type_ == GrB_UNKNOWN)
    return GrB_INVALID_OBJECT;
  if (vec_type_ == GrB_SPARSE) CHECK(sparse_.swap(&rhs->sparse_));
  else                         CHECK(dense_.swap(&rhs->dense_));
  std::swap(nsize_, rhs->nsize_);
  std::swap(nvals_, rhs->nvals_);
  std::swap(ratio_, rhs->ratio_);
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_VECTOR_HPP_
