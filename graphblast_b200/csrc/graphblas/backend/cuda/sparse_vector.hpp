// graphblast_b200 backend — SparseVector<T>: (index, value) lists with capacity
// nsize_ resident in HBM, host mirror materialised on demand.
//
// Stands in for reference graphblas/backend/cuda/sparse_vector.hpp:22-417: same
// method set and the member names its tests read (d_ind_, d_val_, nvals_, nsize_,
// need_update_; test/gvxm.cu:73).  Host and device sides are a pair of arrays each;
// everything that moves data goes through copyLists, everything that gives memory
// back through dropHost / dropDevice.  Storage appears on first use; device arrays
// adopted from the caller (build(Index*, T*, n)) are never freed here.
#ifndef GRAPHBLAS_BACKEND_CUDA_SPARSE_VECTOR_HPP_
#define GRAPHBLAS_BACKEND_CUDA_SPARSE_VECTOR_HPP_

#include <algorithm>
#include <iostream>
#include <unordered_set>
#include <vector>

#include "graphblas/backend/cuda/util.hpp"

namespace graphblas {
namespace backend {

template <typename T>
class DenseVector;

template <typename T>
class SparseVector {
 public:
  SparseVector() {}
  explicit SparseVector(Index nsize) : nsize_(nsize) {}
  ~SparseVector() { dropHost(); dropDevice(); }

  // ---- size and contents --------------------------------------------------------------
  // A new capacity discards the storage; the same capacity only empties the vector.
  Info nnew(Index nsize) {
    if (nsize != nsize_) { dropHost(); dropDevice(); }
    nsize_ = nsize;
    nvals_ = 0;
    return GrB_SUCCESS;
  }
  Info clear() { nvals_ = 0; return GrB_SUCCESS; }
  Info size(Index* out) const  { *out = nsize_; return GrB_SUCCESS; }
  Info nvals(Index* out) const { *out = nvals_; return GrB_SUCCESS; }

  Info dup(const SparseVector* rhs) {
    if (nsize_ != rhs->nsize_) CHECK(nnew(rhs->nsize_));
    nvals_ = rhs->nvals_;
    CHECK(allocateGpu());
    if (rhs->d_ind_ != NULL)
      copyLists(d_ind_, d_val_, rhs->d_ind_, rhs->d_val_, nvals_, cudaMemcpyDeviceToDevice);
    need_update_ = true;
    return GrB_SUCCESS;
  }

  // Host tuples -> vector (no duplicate handling: the callers build frontiers of
  // distinct vertices; `dup` is accepted for the signature).
  template <typename BinaryOpT>
  Info build(const std::vector<Index>* indices, const std::vector<T>* values, Index nvals,
             BinaryOpT dup) {
    if (nvals > nsize_) {
      std::cout << "Error: sparse vector build with more entries than its size\n";
      return GrB_PANIC;
    }
    if (nvals_ > 0) return GrB_OUTPUT_NOT_EMPTY;
    CHECK(allocate());
    std::copy(indices->begin(), indices->begin() + nvals, h_ind_);
    std::copy(values->begin(), values->begin() + nvals, h_val_);
    nvals_ = nvals;
    return cpuToGpu();
  }
  Info build(const std::vector<T>* values, Index nvals) {
    std::cout << "Error: a sparse vector cannot be built from a dense value list\n";
    return GrB_SUCCESS;                       // the reference reports and carries on
  }
  // Adopts device arrays; they stay the caller's.
  Info build(Index* indices, T* values, Index nvals) {
    dropDevice();
    d_ind_ = indices;
    d_val_ = values;
    owns_device_ = false;
    computed(nvals);
    return GrB_SUCCESS;
  }

  // Appends (index, val); the lists are not kept sorted by this call.
  Info setElement(T val, Index index) {
    if (nvals_ >= nsize_) return GrB_INSUFFICIENT_SPACE;
    CHECK(gpuToCpu());
    h_ind_[nvals_] = index;
    h_val_[nvals_] = val;
    ++nvals_;
    return cpuToGpu();
  }
  Info extractElement(T* val, Index index) { return GrB_SUCCESS; }   // no-op there too
  // *n must be the exact entry count.
  Info extractTuples(std::vector<Index>* indices, std::vector<T>* values, Index* n) {
    indices->clear();
    values->clear();
    if (*n != nvals_) {
      std::cout << "Error: extractTuples asked for " << *n << " entries, the vector has "
                << nvals_ << "\n";
      return (*n > nvals_) ? GrB_UNINITIALIZED_OBJECT : GrB_INSUFFICIENT_SPACE;
    }
    CHECK(gpuToCpu());
    indices->assign(h_ind_, h_ind_ + nvals_);
    values->assign(h_val_, h_val_ + nvals_);
    return GrB_SUCCESS;
  }
  // Value stored at `ind`, 0 when absent.
  const T& operator[](Index ind) {
    static T zero = T();
    gpuToCpu();
    const Index* hit = std::find(h_ind_, h_ind_ + nvals_, ind);
    return (hit == h_ind_ + nvals_) ? zero : h_val_[hit - h_ind_];
  }

  // New capacity, keeping the first min(nsize, nvals_) entries.
  Info resize(Index nsize) {
    CHECK(gpuToCpu());
    SparseVector old;                         // takes the current storage with it
    swap(&old);
    nsize_ = nsize;
    nvals_ = std::min(nsize, old.nvals_);
    CHECK(allocate());
    if (old.h_ind_ != NULL) {
      std::copy(old.h_ind_, old.h_ind_ + nvals_, h_ind_);
      std::copy(old.h_val_, old.h_val_ + nvals_, h_val_);
    }
    if (old.d_ind_ != NULL)
      copyLists(d_ind_, d_val_, old.d_ind_, old.d_val_, nvals_, cudaMemcpyDeviceToDevice);
    runtime().sync();                         // before `old` gives its arrays back
    return GrB_SUCCESS;
  }
  // Entries 0..nvals-1, all with value 0.
  Info fill(Index nvals) {
    if (nvals > nsize_) return GrB_INDEX_OUT_OF_BOUNDS;
    CHECK(allocate());
    for (Index i = 0; i < nvals; ++i) h_ind_[i] = i;
    std::fill(h_val_, h_val_ + nvals, T());
    nvals_ = nvals;
    return cpuToGpu();
  }
  Info print(bool force_update = false) {
    CHECK(gpuToCpu(force_update));
    if (nvals_ == 0) {
      std::cout << "Error: SpVec is empty!\n";
      return GrB_SUCCESS;
    }
    const Index shown = std::min(nvals_, 40);
    printArray("ind", h_ind_, shown);
    printArray("val", h_val_, shown);
    return GrB_SUCCESS;
  }
  // Number of distinct VALUES (what the colouring / components drivers ask for).
  Info countUnique(Index* count) {
    CHECK(gpuToCpu());
    *count = std::unordered_set<Index>(h_val_, h_val_ + nvals_).size();
    return GrB_SUCCESS;
  }
  Info swap(SparseVector* rhs) {
    std::swap(nsize_, rhs->nsize_);
    std::swap(nvals_, rhs->nvals_);
    std::swap(h_ind_, rhs->h_ind_);
    std::swap(h_val_, rhs->h_val_);
    std::swap(d_ind_, rhs->d_ind_);
    std::swap(d_val_, rhs->d_val_);
    std::swap(need_update_, rhs->need_update_);
    std::swap(owns_device_, rhs->owns_device_);
    return GrB_SUCCESS;
  }
  // The device lists hold nvals entries (from a kernel, or adopted) the host lacks.
  void computed(Index nvals) {
    nvals_ = nvals;
    need_update_ = true;
  }

  // ---- storage --------------------------------------------------------------------------
  Info allocateCpu() {
    if (nsize_ <= 0 || h_ind_ != NULL) return GrB_SUCCESS;
    const size_t cap = static_cast<size_t>(nsize_);
    h_ind_ = static_cast<Index*>(malloc(cap*sizeof(Index)));
    h_val_ = static_cast<T*>(malloc(cap*sizeof(T)));
    if (h_ind_ == NULL || h_val_ == NULL) {
      std::cout << "Error: CPU SpVec Out of memory!\n";
      return GrB_OUT_OF_MEMORY;
    }
    if (d_ind_ != NULL) need_update_ = true;  // the device side is the newer one
    return GrB_SUCCESS;
  }
  Info allocateGpu() {
    if (nsize_ <= 0 || d_ind_ != NULL) return GrB_SUCCESS;
    const size_t cap = static_cast<size_t>(nsize_);
    d_ind_ = static_cast<Index*>(gbMalloc(cap*sizeof(Index)));
    d_val_ = static_cast<T*>(gbMalloc(cap*sizeof(T)));
    owns_device_ = true;
    printMemory("SpVec");
    return GrB_SUCCESS;
  }
  Info allocate() { CHECK(allocateCpu()); return allocateGpu(); }

  Info cpuToGpu() {
    CHECK(allocate());
    if (nvals_ > 0) {
      copyLists(d_ind_, d_val_, h_ind_, h_val_, nvals_, cudaMemcpyHostToDevice);
      runtime().sync();
    }
    need_update_ = false;
    return GrB_SUCCESS;
  }
  Info gpuToCpu(bool force_update = false) {
    const bool host_was_missing = (h_ind_ == NULL);
    CHECK(allocate());
    if ((need_update_ || force_update || host_was_missing) && nvals_ > 0) {
      copyLists(h_ind_, h_val_, d_ind_, d_val_, nvals_, cudaMemcpyDeviceToHost);
      runtime().sync();
    }
    need_update_ = false;
    return GrB_SUCCESS;
  }

  // ---- data (private in the reference; its drivers `#define private public`) -----------
  Index  nsize_ = 0;       // capacity == logical length of the vector
  Index  nvals_ = 0;       // stored entries
  Index* h_ind_ = NULL;
  T*     h_val_ = NULL;
  Index* d_ind_ = NULL;
  T*     d_val_ = NULL;
  bool   need_update_ = false;   // device copy newer than host copy

 private:
  bool   owns_device_ = true;

  static void copyLists(Index* ind_to, T* val_to, const Index* ind_from, const T* val_from,
                        Index count, cudaMemcpyKind kind) {
    if (count <= 0) return;
    const size_t k = static_cast<size_t>(count);
    CUDA_CALL(cudaMemcpyAsync(ind_to, ind_from, k*sizeof(Index), kind, gbStream()));
    CUDA_CALL(cudaMemcpyAsync(val_to, val_from, k*sizeof(T), kind, gbStream()));
  }
  void dropHost() {
    free(h_ind_);
    free(h_val_);
    h_ind_ = NULL;
    h_val_ = NULL;
  }
  void dropDevice() {
    if (owns_device_) { gbFree(d_ind_); gbFree(d_val_); }
    d_ind_ = NULL;
    d_val_ = NULL;
    owns_device_ = true;
  }
};

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_SPARSE_VECTOR_HPP_
