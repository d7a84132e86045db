// graphblast_b200 backend — DenseVector<T>: n values resident in HBM with a
// lazily materialised host mirror.
//
// Stands in for reference graphblas/backend/cuda/dense_vector.hpp:22-438 (same public
// methods, and the member names its tests reach: nvals_, nnz_, h_val_, d_val_,
// need_update_).  What is different by design:
//  * device storage appears on first use, stream-ordered (util.hpp gbMalloc); device
//    arrays adopted from the caller (build(T*, n)) are never freed here;
//  * fill() / fillAscending() run on the device (the reference loops on the host and
//    copies 4n bytes, dense_vector.hpp:312-318), setElement() writes one element (the
//    reference round-trips the vector, :225-230);
//  * the vector carries facts ABOUT its contents that the traversal kernels leave
//    behind or consume: the count of non-identity entries (nnz_valid_, or still on
//    the device: count_pending_), "contents are exactly 0/1" (zero_one_), a bitmap
//    shadow (bits_valid_), and "only the bitmap is current" (vals_stale_).  They are
//    private: a write reports itself through touched(), wroteBooleanPull(),
//    wroteUnderMask() or scattered(); exactBits(), valuesStale(), holdsZeroOne() read.
#ifndef GRAPHBLAS_BACKEND_CUDA_DENSE_VECTOR_HPP_
#define GRAPHBLAS_BACKEND_CUDA_DENSE_VECTOR_HPP_

#include <algorithm>
#include <iostream>
#include <unordered_set>
#include <vector>

#include "graphblas/backend/cuda/util.hpp"
#include "graphblas/backend/cuda/descriptor.hpp"
#include "graphblas/backend/cuda/kernels/kernels.hpp"

namespace graphblas {
namespace backend {

template <typename T>
class SparseVector;

template <typename T>
class DenseVector {
 public:
  DenseVector() {}
  explicit DenseVector(Index nsize) : nvals_(nsize) {}
  ~DenseVector() {
    free(h_val_);
    if (owns_device_) gbFree(d_val_);
    gbFree(d_count_);
    gbFree(d_bits_);
  }

  // ---- size and contents --------------------------------------------------------------
  // A new length discards the storage; the facts about the contents go either way.
  Info nnew(Index nsize) {
    if (nsize != nvals_) {
      free(h_val_);
      h_val_ = NULL;
      if (owns_device_) gbFree(d_val_);
      d_val_ = NULL;
      owns_device_ = true;
      gbFree(d_bits_);
      d_bits_ = NULL;
    }
    nvals_ = nsize;
    const bool mirror_stale = need_update_;
    contentChanged();
    need_update_ = mirror_stale;
    return GrB_SUCCESS;
  }
  Info clear() { return fill(static_cast<T>(0)); }
  Info size(Index* out) const  { *out = nvals_; return GrB_SUCCESS; }
  Info nvals(Index* out) const { *out = nvals_; return GrB_SUCCESS; }
  Info nnz(Index* out) const   { *out = nnz_; return GrB_SUCCESS; }

  // Copies the values and what is known about them (not the bitmap).
  Info dup(const DenseVector* rhs) {
    if (nvals_ != rhs->nvals_) CHECK(nnew(rhs->nvals_));
    CHECK(allocateGpu());
    CHECK(const_cast<DenseVector*>(rhs)->materialize());
    if (rhs->d_val_ != NULL && rhs->d_val_ != d_val_)
      CUDA_CALL(cudaMemcpyAsync(d_val_, rhs->d_val_, bytes(nvals_), cudaMemcpyDeviceToDevice,
                                gbStream()));
    contentChanged();
    nnz_valid_    = rhs->nnz_valid_;
    nnz_          = rhs->nnz_;
    nnz_identity_ = rhs->nnz_identity_;
    zero_one_     = rhs->zero_one_;
    return GrB_SUCCESS;
  }

  // Entries != identity.  Free when the producing kernel left the count behind.
  Info computeNnz(Index* out, T identity, Descriptor* desc) {
    if (nvals_ == 0) return GrB_INVALID_OBJECT;
    const bool same_identity = (nnz_identity_ == identity);
    if (!(nnz_valid_ && same_identity)) {
      if (count_pending_ && same_identity && d_count_ != NULL) {
        // posted to the host mailbox by the producing kernel, or read from its cell
        unsigned long long posted;
        nnz_ = static_cast<Index>(
            (count_ticket_ != 0ull && runtime().mailWait(1, count_ticket_, &posted))
                ? posted : runtime().fetch(d_count_));
      } else {
        CHECK(allocateGpu());
        CHECK(materialize());
        unsigned long long* cell = desc->counters();
        CUDA_CALL(cudaMemsetAsync(cell, 0, sizeof(unsigned long long), gbStream()));
        countNonIdentityKernel<256><<<gridFor(nvals_, 256), 256, 0, gbStream()>>>(
            cell, d_val_, identity, nvals_);
        GB_KERNEL_CHECK();
        nnz_ = static_cast<Index>(runtime().fetch(cell));
        nnz_identity_ = identity;
      }
      nnz_valid_ = true;
      count_pending_ = false;
    }
    *out = nnz_;
    return GrB_SUCCESS;
  }

  template <typename BinaryOpT>
  Info build(const std::vector<Index>* indices, const std::vector<T>* values, Index nvals,
             BinaryOpT dup) {
    std::cout << "Error: a dense vector cannot be built from (index, value) tuples\n";
    return GrB_SUCCESS;                       // the reference reports and carries on
  }
  // The first nvals values from the host.
  Info build(const std::vector<T>* values, Index nvals) {
    if (nvals > nvals_) return GrB_INDEX_OUT_OF_BOUNDS;
    CHECK(allocate());
    CHECK(gpuToCpu());
    std::copy(values->begin(), values->begin() + nvals, h_val_);
    return cpuToGpu();
  }
  // Adopts a device array; it stays the caller's.
  Info build(T* values, Index nvals) {
    if (owns_device_) gbFree(d_val_);
    if (nvals != nvals_) { free(h_val_); h_val_ = NULL; }
    d_val_ = values;
    nvals_ = nvals;
    owns_device_ = false;
    contentChanged();
    return GrB_SUCCESS;
  }

  Info setElement(T val, Index index) {
    if (index < 0 || index >= nvals_) return GrB_INDEX_OUT_OF_BOUNDS;
    CHECK(allocateGpu());
    CHECK(materialize());
    T* stage = reinterpret_cast<T*>(runtime().h_pinned);
    runtime().sync();                         // the staging slot may be in flight
    *stage = val;
    CUDA_CALL(cudaMemcpyAsync(d_val_ + index, stage, sizeof(T), cudaMemcpyHostToDevice,
                              gbStream()));
    runtime().sync();
    const bool host_current = (h_val_ != NULL && !need_update_);
    contentChanged();
    if (host_current) {                       // keep the mirror in step instead of stale
      h_val_[index] = val;
      need_update_ = false;
    }
    return GrB_SUCCESS;
  }
  Info extractElement(T* val, Index index) {
    if (index < 0 || index >= nvals_) return GrB_INDEX_OUT_OF_BOUNDS;
    CHECK(allocateGpu());
    CHECK(materialize());
    *val = runtime().fetch(d_val_ + index);
    return GrB_SUCCESS;
  }
  Info extractTuples(std::vector<Index>* indices, std::vector<T>* values, Index* n) {
    std::cout << "Error: a dense vector has no (index, value) tuples to extract\n";
    return GrB_SUCCESS;
  }
  // *n must be the vector's length.
  Info extractTuples(std::vector<T>* values, Index* n) {
    values->clear();
    const Info fits = lengthMatches(*n);
    if (fits != GrB_SUCCESS) return fits;
    CHECK(gpuToCpu());
    values->assign(h_val_, h_val_ + nvals_);
    return GrB_SUCCESS;
  }
  // The same into caller memory (C ABI; no std::vector in between).
  Info extractRaw(T* values, Index n) {
    const Info fits = lengthMatches(n, false);
    if (fits != GrB_SUCCESS) return fits;
    CHECK(allocateGpu());
    CHECK(materialize());
    CUDA_CALL(cudaMemcpyAsync(values, d_val_, bytes(n), cudaMemcpyDeviceToHost, gbStream()));
    runtime().sync();
    return GrB_SUCCESS;
  }
  const T& operator[](Index ind) {
    static T zero = T();
    if (gpuToCpu() != GrB_SUCCESS) return zero;
    if (ind >= nvals_) {
      std::cout << "Error: Index out of bounds!\n";
      return zero;
    }
    return h_val_[ind];
  }

  // New length, keeping the first min(nsize, nvals_) values.
  Info resize(Index nsize) {
    CHECK(materialize());
    CHECK(gpuToCpu());
    T* const host_before = h_val_;
    T* const dev_before  = d_val_;
    const bool dev_was_ours = owns_device_;
    const Index kept = std::min(nsize, nvals_);
    h_val_ = NULL;
    d_val_ = NULL;
    owns_device_ = true;
    nvals_ = nsize;
    CHECK(allocate());
    if (host_before != NULL) std::copy(host_before, host_before + kept, h_val_);
    if (dev_before != NULL)
      CUDA_CALL(cudaMemcpyAsync(d_val_, dev_before, bytes(kept), cudaMemcpyDeviceToDevice,
                                gbStream()));
    free(host_before);
    if (dev_was_ours) gbFree(dev_before);     // stream-ordered: after the copy
    const bool mirror_stale = need_update_;
    contentChanged();
    need_update_ = mirror_stale;
    return GrB_SUCCESS;
  }

  // Constant vector; its bitmap shadow is all zero or all one (bits past the end stay
  // clear: consumers read whole words).
  Info fill(T val) {
    if (nvals_ == 0) return GrB_SUCCESS;
    CHECK(allocateGpu());
    fillKernel<<<gridFor(nvals_, 256), 256, 0, gbStream()>>>(d_val_, val, nvals_);
    GB_KERNEL_CHECK();
    contentChanged();
    fillBitmapKernel<<<gridFor(bitWords(), 256), 256, 0, gbStream()>>>(
        bitsStorage(), nvals_, val != static_cast<T>(0));
    GB_KERNEL_CHECK();
    bits_valid_ = true;
    return GrB_SUCCESS;
  }
  // 0, 1, 2, ...
  Info fillAscending(Index nvals) {
    if (nvals_ == 0) return GrB_SUCCESS;
    CHECK(allocateGpu());
    iotaKernel<<<gridFor(nvals_, 256), 256, 0, gbStream()>>>(d_val_, nvals_);
    GB_KERNEL_CHECK();
    contentChanged();
    return GrB_SUCCESS;
  }
  Info print(bool force_update = false) {
    CHECK(gpuToCpu(force_update));
    printArray("val", h_val_, std::min(nvals_, 40));
    return GrB_SUCCESS;
  }
  // Number of distinct values (colouring / components drivers).
  Info countUnique(Index* count) {
    CHECK(gpuToCpu());
    *count = std::unordered_set<Index>(h_val_, h_val_ + nvals_).size();
    return GrB_SUCCESS;
  }
  Info swap(DenseVector* rhs) {
    std::swap(nvals_, rhs->nvals_);
    std::swap(nnz_, rhs->nnz_);
    std::swap(h_val_, rhs->h_val_);
    std::swap(d_val_, rhs->d_val_);
    std::swap(need_update_, rhs->need_update_);
    std::swap(owns_device_, rhs->owns_device_);
    std::swap(nnz_valid_, rhs->nnz_valid_);
    std::swap(nnz_identity_, rhs->nnz_identity_);
    std::swap(d_count_, rhs->d_count_);
    std::swap(count_pending_, rhs->count_pending_);
    std::swap(count_ticket_, rhs->count_ticket_);
    std::swap(zero_one_, rhs->zero_one_);
    std::swap(d_bits_, rhs->d_bits_);
    std::swap(bits_valid_, rhs->bits_valid_);
    std::swap(bits_alloc_words_, rhs->bits_alloc_words_);
    std::swap(vals_stale_, rhs->vals_stale_);
    return GrB_SUCCESS;
  }

  // ---- storage --------------------------------------------------------------------------
  Info allocateCpu() {
    if (nvals_ <= 0 || h_val_ != NULL) return GrB_SUCCESS;
    h_val_ = static_cast<T*>(malloc(bytes(nvals_)));
    if (h_val_ == NULL) {
      std::cout << "Error: CPU DeVec Out of memory!\n";
      return GrB_OUT_OF_MEMORY;
    }
    if (d_val_ != NULL) need_update_ = true;  // the device side is the newer one
    return GrB_SUCCESS;
  }
  Info allocateGpu() {
    if (nvals_ <= 0 || d_val_ != NULL) return GrB_SUCCESS;
    d_val_ = static_cast<T*>(gbMalloc(bytes(nvals_)));
    owns_device_ = true;
    printMemory("DeVec");
    return GrB_SUCCESS;
  }
  Info allocate() { CHECK(allocateCpu()); return allocateGpu(); }

  Info cpuToGpu() {
    CHECK(allocate());
    CUDA_CALL(cudaMemcpyAsync(d_val_, h_val_, bytes(nvals_), cudaMemcpyHostToDevice,
                              gbStream()));
    runtime().sync();
    contentChanged();
    need_update_ = false;
    return GrB_SUCCESS;
  }
  Info gpuToCpu(bool force_update = false) {
    const bool host_was_missing = (h_val_ == NULL);
    CHECK(allocate());
    CHECK(materialize());
    if (need_update_ || force_update || host_was_missing) {
      CUDA_CALL(cudaMemcpyAsync(h_val_, d_val_, bytes(nvals_), cudaMemcpyDeviceToHost,
                                gbStream()));
      runtime().sync();
    }
    need_update_ = false;
    return GrB_SUCCESS;
  }

  // ---- facts about the contents -----------------------------------------------------------
  // A kernel wrote the values.
  void touched() { contentChanged(); }
  // The fused Boolean pull wrote 0/1 (with `bits_only`: the bitmap shadow alone) and
  // counted the ones into countCell() and, unless `ticket` is 0, the mailbox.
  void wroteBooleanPull(bool bits_only, unsigned long long ticket) {
    contentChanged();
    bits_valid_    = bits_only;
    vals_stale_    = bits_only;
    count_pending_ = true;
    count_ticket_  = ticket;
    zero_one_      = true;
    nnz_identity_  = T(0);
  }
  // A masked constant assign wrote the values; `bits_exact`: it kept the shadow in step.
  void wroteUnderMask(bool bits_exact) {
    contentChanged();
    bits_valid_ = bits_exact;
  }
  // A sparse vector of nnz entries was scattered into these values.  Under --opreuse
  // nothing was written, so the pending count, zero_one_ and vals_stale_ stay as they are.
  void scattered(Index nnz, bool bits_exact) {
    need_update_ = true;
    nnz_         = nnz;
    nnz_valid_   = false;
    bits_valid_  = bits_exact;
  }
  // The bitmap shadow when it is exact, else NULL.
  unsigned int* exactBits() const { return bits_valid_ ? d_bits_ : NULL; }
  bool valuesStale() const  { return vals_stale_; }
  bool holdsZeroOne() const { return zero_one_; }

  // Lazy values.  The fused Boolean pull publishes its 0/1 result through the
  // bitmap shadow only and sets vals_stale_; every consumer inside a traversal
  // (mask of assign, frontier of the next mxv, convert, count) reads the bitmap.
  // Anything that needs the value array calls materialize() first; anything that
  // overwrites the whole array clears the flag (contentChanged()).
  Info materialize() {
    if (vals_stale_) {
      CHECK(allocateGpu());
      bitmapToDenseKernel<<<gridFor(static_cast<size_t>(nvals_), 256), 256, 0,
          gbStream()>>>(d_val_, d_bits_, nvals_);
      GB_KERNEL_CHECK();
      vals_stale_ = false;
      need_update_ = true;
    }
    return GrB_SUCCESS;
  }

  size_t bitWords() const { return (static_cast<size_t>(nvals_) + 31)/32; }
  unsigned int* bitsStorage() {
    if (d_bits_ == NULL || bits_alloc_words_ < bitWords()) {
      gbFree(d_bits_);
      bits_alloc_words_ = bitWords() + 8;
      d_bits_ = static_cast<unsigned int*>(gbMalloc(bits_alloc_words_*sizeof(unsigned int)));
      bits_valid_ = false;
    }
    return d_bits_;
  }
  // A valid bitmap of the current contents, built if need be.
  unsigned int* ensureBits() {
    unsigned int* b = bitsStorage();
    if (!bits_valid_) {
      denseToBitmapKernel<<<gridFor(static_cast<size_t>(nvals_), 256), 256, 0,
          gbStream()>>>(b, d_val_, nvals_);
      GB_KERNEL_CHECK();
      bits_valid_ = true;
    }
    return b;
  }
  unsigned long long* countCell() {
    if (d_count_ == NULL)
      d_count_ = static_cast<unsigned long long*>(gbMalloc(sizeof(unsigned long long)));
    return d_count_;
  }

  // ---- data (private in the reference; its drivers `#define private public`) -----------
  Index nvals_ = 0;              // vector length
  Index nnz_ = 0;
  T*    h_val_ = NULL;
  T*    d_val_ = NULL;
  bool  need_update_ = false;    // device copy newer than host copy

 private:
  bool  owns_device_ = true;
  bool  nnz_valid_ = false;      // nnz_ counts entries != nnz_identity_ of the current data
  T     nnz_identity_ = T();
  // Count left on the device by the kernel that produced the current contents
  // (fused Boolean pull): *d_count_ = #entries != nnz_identity_.
  unsigned long long* d_count_ = NULL;
  bool  count_pending_ = false;
  unsigned long long count_ticket_ = 0ull;   // mailbox ticket of the pending count
  bool  zero_one_ = false;       // contents are exactly 0/1 (so a plus-reduce == count)

  // Bitmap shadow: bit i == (d_val_[i] != 0).  Kept by the operations of the
  // BFS loop (fill, fused Boolean pull, masked constant assign); any other write
  // invalidates it.  Lets masks and Boolean frontiers be read at 1 bit/vertex.
  unsigned int* d_bits_ = NULL;
  bool   bits_valid_ = false;
  size_t bits_alloc_words_ = 0;
  bool   vals_stale_ = false;    // only the bitmap is current

  static size_t bytes(Index count) { return static_cast<size_t>(count)*sizeof(T); }
  // The values were (or are about to be) overwritten: the host mirror is behind and
  // nothing derived from the old contents holds any more.
  void contentChanged() {
    need_update_ = true;
    nnz_valid_ = false;
    count_pending_ = false;
    zero_one_ = false;
    bits_valid_ = false;
    vals_stale_ = false;
  }
  // extractTuples / extractRaw take exactly the vector's length.
  Info lengthMatches(Index n, bool report = true) const {
    if (n == nvals_) return GrB_SUCCESS;
    if (report)
      std::cout << "Error: " << n << " values requested from a dense vector of " << nvals_
                << "\n";
    return (n > nvals_) ? GrB_UNINITIALIZED_OBJECT : GrB_INSUFFICIENT_SPACE;
  }
};

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_DENSE_VECTOR_HPP_
