// graphblast_b200 backend — SparseMatrix<T>: CSR + CSC with host mirrors.
//
// Takes the place of reference graphblas/backend/cuda/sparse_matrix.hpp:24-853.
// What is dictated by the drop-in boundary (SURVEY.md §8b) is kept: the method
// set the frontend forwards to, and the data members the unchanged drivers and
// CPU verifiers read through `#define private public`
// (matrix_.sparse_.h_csrRowPtr_ ..., reference algorithm/bfs.hpp:101-107).
// Everything else is this backend's own design:
//   * construction from tuples runs ON THE DEVICE (ingest.hpp: radix sort of
//     packed keys, CSR and CSC built there, then mirrored to the host) — the
//     reference sorts tuple vectors on the host and uploads;
//   * CSR and CSC are handled by the same code through a `Side` view (three
//     array references + the dimension) instead of parallel copies;
//   * the binary cache keeps values and says what it holds (header below); the
//     reference's headerless layout (nrows, nvals, rowptr, colind; values
//     implied 1, reference :328-407) is still read when found;
//   * device arrays come from the stream-ordered pool, 256-byte aligned (the
//     pull kernels' 256-bit loads rely on it); adopted arrays are never freed;
//   * derived per-matrix caches of the mxv kernels live here and are dropped
//     whenever the structure changes.
// Layout in HBM: int32 rowptr[nrows+1], int32 colind[nvals], T val[nvals], and the
// same triple for CSC; a structurally symmetric matrix (".ud." in the cache name,
// as in the reference) aliases the CSC index arrays to the CSR ones and keeps only
// cscVal separate.
#ifndef GRAPHBLAS_BACKEND_CUDA_SPARSE_MATRIX_HPP_
#define GRAPHBLAS_BACKEND_CUDA_SPARSE_MATRIX_HPP_

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <iostream>
#include <vector>

#include "graphblas/backend/cuda/util.hpp"
#include "graphblas/backend/cuda/hub_index.hpp"
#include "graphblas/backend/cuda/ingest.hpp"

namespace graphblas {
namespace backend {

template <typename T>
class DenseMatrix;

template <typename T>
class Vector;

// Header of this backend's binary cache files.
struct MatrixCacheHeader {
  char     magic[8];        // "GB2CSR01"
  int32_t  nrows;
  int32_t  ncols;
  int32_t  nvals;
  int32_t  value_bytes;     // sizeof(T) when values follow, 0 for a pattern
};

// Device words derived from one orientation's arrays, valid for the pointer array
// and entry count (the merge-path tiles: also the tile count) they were computed
// from.  Every structural change releases them; the key catches a path that forgot.
struct DerivedArray {
  Index*       d = NULL;
  const Index* key = NULL;
  Index        nvals = -1;
  int          count = 0;
  bool validFor(const Index* k, Index nv, int n = 0) const {
    return d != NULL && key == k && nvals == nv && count == n;
  }
  // Frees what is held, allocates `words` words and stamps the key; the caller fills d.
  Index* rebuild(size_t words, const Index* k, Index nv, int n = 0) {
    release();
    d = reinterpret_cast<Index*>(gbMalloc(words*sizeof(Index)));
    key = k; nvals = nv; count = n;
    return d;
  }
  void release() {
    if (d != NULL) gbFree(d);
    *this = DerivedArray();
  }
};

inline bool cacheFileExists(const char* path) {
  FILE* f = fopen(path, "rb");
  if (f == NULL) return false;
  fclose(f);
  return true;
}

template <typename T>
class SparseMatrix {
 public:
  // One orientation of the matrix: pointer array, index array, values, and how
  // many pointer entries there are (dim + 1).
  struct Side {
    Index*& ptr;
    Index*& ind;
    T*&     val;
    Index   dim;
  };
  // One stored orientation of the device side, read-only: the three arrays an
  // operation traverses as op(A), with the dimensions that go with them.
  struct View {
    const Index* ptr;
    const Index* ind;
    const T*     val;
    Index        dim;       // rows of this orientation (ptr has dim + 1 entries)
    Index        other;     // its columns
    int          which;     // 0 = CSR, 1 = CSC: the slot of the derived caches
    bool complete() const { return ptr != NULL && ind != NULL && val != NULL; }
  };

  SparseMatrix() { reset(0, 0); }
  explicit SparseMatrix(Index nrows, Index ncols) { reset(nrows, ncols); }
  ~SparseMatrix() { releaseHost(); releaseDevice(); }

  // ---- interface of the frontend ---------------------------------------------
  Info nnew(Index nrows, Index ncols) { nrows_ = nrows; ncols_ = ncols; return GrB_SUCCESS; }
  Info dup(const SparseMatrix* rhs);
  Info clear();
  Info nrows(Index* out) const { *out = nrows_; return GrB_SUCCESS; }
  Info ncols(Index* out) const { *out = ncols_; return GrB_SUCCESS; }
  Info nvals(Index* out) const { *out = nvals_; return GrB_SUCCESS; }
  template <typename BinaryOpT>
  Info build(const std::vector<Index>* row_indices,
      const std::vector<Index>* col_indices, const std::vector<T>* values, Index nvals,
      BinaryOpT dup, char* dat_name);
  Info build(char* dat_name);
  Info build(const std::vector<T>* values, Index nvals) { return GrB_NOT_IMPLEMENTED; }
  Info build(Index* row_ptr, Index* col_ind, T* values, Index nvals);
  // Tuples already in device memory (C ABI / generators): mode = IngestFlags.
  Info buildFromDeviceTuples(const Index* d_rows, const Index* d_cols,
      const T* d_vals, long long ntuples, int mode, bool symmetric);
  Info adoptCsc(Index* col_ptr, Index* row_ind, T* values, bool symmetric);
  Info setElement(Index row_index, Index col_index) { return GrB_NOT_IMPLEMENTED; }
  Info extractElement(T* val, Index row_index, Index col_index);
  Info extractTuples(std::vector<Index>* row_indices, std::vector<Index>* col_indices,
      std::vector<T>* values, Index* n);
  Info extractTuples(std::vector<T>* values, Index* n) { return GrB_NOT_IMPLEMENTED; }

  const T operator[](Index ind);
  Info print(bool force_update);
  Info check();
  Info setNrows(Index nrows) { nrows_ = nrows; return GrB_SUCCESS; }
  Info setNcols(Index ncols) { ncols_ = ncols; return GrB_SUCCESS; }
  Info setNvals(Index nvals) { nvals_ = nvals; return GrB_SUCCESS; }
  Info getFormat(SparseMatrixFormat* format) const { *format = format_; return GrB_SUCCESS; }
  // Reports false whatever symmetric_ says — a quirk of the reference (:578-582)
  // that the mxv dispatch depends on; symmetric_ still drives the aliasing.
  Info getSymmetry(bool* symmetry) const { *symmetry = false; return GrB_SUCCESS; }
  Info resize(Index nrows, Index ncols);
  template <typename U>
  Info fill(Index axis, Index nvals, U start);
  template <typename U>
  Info fillAscending(Index axis, Index nvals, U start);

  // ---- storage management (public: the drivers reach in) -------------------------
  Info allocateCpu();
  Info allocateGpu();
  Info allocate() { CHECK(allocateCpu()); return allocateGpu(); }
  Info cpuToGpu();
  Info gpuToCpu(bool force_update = false);
  Info syncCpu();            // host CSC rebuilt from the host CSR
  Info printCSR(const char* str) { return printSide(str, hostCsr(), ncols_); }
  Info printCSC(const char* str) { return printSide(str, hostCsc(), nrows_); }
  void dropDerived();
  // The contents replaced by a computed CSR of nnz entries in fresh arrays, which
  // this object takes (with cscptr != NULL, a ready CSC of the same entries too).
  // symmetric: the entry set is symmetric; the CSC index arrays are the CSR's and
  // cscval (needed when the format keeps a CSC) holds the column-major values.
  void replaceDevice(Index nnz, Index* rowptr, Index* colind, T* val,
      Index* cscptr = NULL, Index* cscind = NULL, T* cscval = NULL,
      bool symmetric = false);
  // The entry set stopped being symmetric (tril): from the next upload on the
  // column-major side owns its index arrays instead of borrowing the CSR's.
  void dropSymmetry() { if (symmetric_) { releaseDevice(); symmetric_ = false; } }
  // The CSC values become an array of this object's own when they are the CSR
  // value array (an adopted CSC may name it), so that an operation can scale the
  // two sides apart; a stream-ordered copy of the current values.
  void separateCscValues() {
    if (d_cscVal_ == NULL || d_cscVal_ != d_csrVal_) return;
    d_cscVal_ = devArray<T>(atLeastOne(nvals_));
    copyAsync(d_cscVal_, d_csrVal_, static_cast<size_t>(nvals_), cudaMemcpyDeviceToDevice);
    cscval_ownership_ = true;
  }

  Side hostCsr() { return Side{h_csrRowPtr_, h_csrColInd_, h_csrVal_, nrows_}; }
  Side hostCsc() { return Side{h_cscColPtr_, h_cscRowInd_, h_cscVal_, ncols_}; }
  Side devCsr()  { return Side{d_csrRowPtr_, d_csrColInd_, d_csrVal_, nrows_}; }
  Side devCsc()  { return Side{d_cscColPtr_, d_cscRowInd_, d_cscVal_, ncols_}; }
  View view(bool csc) const {
    return csc ? View{d_cscColPtr_, d_cscRowInd_, d_cscVal_, ncols_, nrows_, 1}
               : View{d_csrRowPtr_, d_csrColInd_, d_csrVal_, nrows_, ncols_, 0};
  }
  // Both orientations have the same structure: one pass over either serves for both.
  bool sameStructure() const { return symmetric_ || d_cscColPtr_ == d_csrRowPtr_; }

  Index nrows_;
  Index ncols_;
  Index nvals_;
  Index ncapacity_;         // entries the host / device arrays were sized for
  Index nempty_;

  Index* h_csrRowPtr_;
  Index* h_csrColInd_;
  T*     h_csrVal_;
  Index* h_cscColPtr_;
  Index* h_cscRowInd_;
  T*     h_cscVal_;

  Index* d_csrRowPtr_;
  Index* d_csrColInd_;
  T*     d_csrVal_;
  Index* d_cscColPtr_;
  Index* d_cscRowInd_;
  T*     d_cscVal_;

  bool need_update_;        // device copy newer than the host mirror
  bool csr_initialized_;
  bool csc_initialized_;
  bool csr_ownership_;      // device CSR arrays belong to this object
  bool csc_ownership_;      // device CSC index arrays belong to this object
  bool cscval_ownership_;   // device CSC values belong to this object
  bool symmetric_;
  SparseMatrixFormat format_;

  // Derived caches of the mxv kernels, one per traversed orientation (0 = CSR
  // rows, 1 = CSC columns), each valid for the arrays it was computed from:
  //   merge-path tile partition of the generic pull SpMV,
  //   first-neighbour summary of the Boolean pull,
  //   highest-degree-neighbour summary of the fused BFS pull,
  //   hub index of the hub-cached pull SpMV (hub_state_: 0 not built, 1 in use,
  //   2 rejected because too few entries reference the hub columns).
  DerivedArray tiles_[2];
  DerivedArray pull_first_[2];
  DerivedArray pull_maxdeg_[2];
  HubIndex     hub_[2];
  int          hub_state_[2] = {0, 0};

 private:
  void reset(Index nrows, Index ncols);
  void releaseHost();
  void releaseDevice();
  bool hostCscIsAlias() const { return h_cscColPtr_ == h_csrRowPtr_ && h_csrRowPtr_ != NULL; }
  static size_t atLeastOne(Index n) { return n > 0 ? static_cast<size_t>(n) : 1; }
  template <typename X>
  static X* hostArray(size_t count) { return reinterpret_cast<X*>(malloc(count*sizeof(X))); }
  template <typename X>
  static X* devArray(size_t count) { return reinterpret_cast<X*>(gbMalloc(count*sizeof(X))); }
  void transfer(Side dst, Side src, cudaMemcpyKind kind, bool with_indices) {
    if (with_indices) {
      copyAsync(dst.ptr, src.ptr, static_cast<size_t>(dst.dim) + 1, kind);
      copyAsync(dst.ind, src.ind, static_cast<size_t>(nvals_), kind);
    }
    copyAsync(dst.val, src.val, static_cast<size_t>(nvals_), kind);
  }
  Info finishDeviceBuild(bool build_csc);   // CSC side + host mirrors after a device CSR
  Info printSide(const char* str, Side side, Index other_dim);
  bool writeCache(const char* path);
  bool readCache(const char* path);
};

// ---------------------------------------------------------------------------

template <typename T>
void SparseMatrix<T>::reset(Index nrows, Index ncols) {
  nrows_ = nrows; ncols_ = ncols; nvals_ = 0; ncapacity_ = 0; nempty_ = 0;
  h_csrRowPtr_ = NULL; h_csrColInd_ = NULL; h_csrVal_ = NULL;
  h_cscColPtr_ = NULL; h_cscRowInd_ = NULL; h_cscVal_ = NULL;
  d_csrRowPtr_ = NULL; d_csrColInd_ = NULL; d_csrVal_ = NULL;
  d_cscColPtr_ = NULL; d_cscRowInd_ = NULL; d_cscVal_ = NULL;
  need_update_ = false;
  csr_initialized_ = false; csc_initialized_ = false;
  csr_ownership_ = false; csc_ownership_ = false; cscval_ownership_ = false;
  symmetric_ = false;
  format_ = getEnv("GRB_SPARSE_MATRIX_FORMAT", GrB_SPARSE_MATRIX_CSRCSC);
}

template <typename T>
void SparseMatrix<T>::dropDerived() {
  for (int k = 0; k < 2; ++k) {
    hub_[k].release();
    hub_state_[k] = 0;
    pull_first_[k].release();
    pull_maxdeg_[k].release();
    tiles_[k].release();
  }
}

template <typename T>
void SparseMatrix<T>::releaseHost() {
  const bool alias = hostCscIsAlias();
  free(h_csrRowPtr_); free(h_csrColInd_); free(h_csrVal_);
  if (!alias) { free(h_cscColPtr_); free(h_cscRowInd_); free(h_cscVal_); }
  h_csrRowPtr_ = NULL; h_csrColInd_ = NULL; h_csrVal_ = NULL;
  h_cscColPtr_ = NULL; h_cscRowInd_ = NULL; h_cscVal_ = NULL;
}

template <typename T>
void SparseMatrix<T>::releaseDevice() {
  dropDerived();
  if (csc_ownership_) {
    if (d_cscColPtr_ != d_csrRowPtr_) gbFree(d_cscColPtr_);
    if (d_cscRowInd_ != d_csrColInd_) gbFree(d_cscRowInd_);
  }
  if (cscval_ownership_ && d_cscVal_ != d_csrVal_) gbFree(d_cscVal_);
  if (csr_ownership_) { gbFree(d_csrRowPtr_); gbFree(d_csrColInd_); gbFree(d_csrVal_); }
  d_csrRowPtr_ = NULL; d_csrColInd_ = NULL; d_csrVal_ = NULL;
  d_cscColPtr_ = NULL; d_cscRowInd_ = NULL; d_cscVal_ = NULL;
  csr_ownership_ = false; csc_ownership_ = false; cscval_ownership_ = false;
}

template <typename T>
Info SparseMatrix<T>::clear() {
  releaseHost();
  releaseDevice();
  nvals_ = 0;
  ncapacity_ = 0;
  csr_initialized_ = false;
  csc_initialized_ = false;
  return GrB_SUCCESS;
}

// Deep copy of the device side (host mirrors follow lazily).  The derived caches
// describe the previous contents and are always dropped.
template <typename T>
Info SparseMatrix<T>::dup(const SparseMatrix* rhs) {
  if (nrows_ != rhs->nrows_ || ncols_ != rhs->ncols_) return GrB_DIMENSION_MISMATCH;
  SparseMatrix* src = const_cast<SparseMatrix*>(rhs);
  const bool reusable = csr_ownership_ && nvals_ == rhs->nvals_ &&
                        symmetric_ == rhs->symmetric_ && format_ == rhs->format_;
  if (!reusable) { releaseDevice(); releaseHost(); }
  dropDerived();
  nvals_     = rhs->nvals_;
  symmetric_ = rhs->symmetric_;
  format_    = rhs->format_;
  CHECK(allocateGpu());
  transfer(devCsr(), src->devCsr(), cudaMemcpyDeviceToDevice, true);
  if (format_ == GrB_SPARSE_MATRIX_CSRCSC && rhs->d_cscVal_ != NULL) {
    const bool own_indices = !symmetric_ && rhs->d_cscColPtr_ != NULL &&
                             rhs->d_cscRowInd_ != NULL;
    transfer(devCsc(), src->devCsc(), cudaMemcpyDeviceToDevice, own_indices);
    csc_initialized_ = true;
  }
  need_update_ = true;
  csr_initialized_ = true;
  return GrB_SUCCESS;
}

// The old arrays, and every cache built on them, go first: stream-ordered after the
// kernels queued so far, which may still read them through an operand that is this
// matrix.  Then the CSC, when the format keeps one, is the one given, the CSR's
// index arrays with the given values (symmetric), or is built here; what is given
// is freed when the format is CSR-only.  Unless the caller says so nothing is
// known about the result's symmetry.  The host mirrors follow lazily.
template <typename T>
void SparseMatrix<T>::replaceDevice(Index nnz, Index* rowptr, Index* colind, T* val,
    Index* cscptr, Index* cscind, T* cscval, bool symmetric) {
  clear();
  d_csrRowPtr_ = rowptr;
  d_csrColInd_ = colind;
  d_csrVal_ = val;
  csr_ownership_ = true;
  nvals_ = nnz;
  ncapacity_ = nnz;
  symmetric_ = symmetric;
  if (symmetric) {
    cscptr = rowptr;
    cscind = colind;
  }
  if (format_ == GrB_SPARSE_MATRIX_CSRCSC) {
    if (cscptr == NULL)
      ingestCsrToCsc<T>(nrows_, ncols_, nnz, rowptr, colind, val, &cscptr, &cscind, &cscval);
    d_cscColPtr_ = cscptr;
    d_cscRowInd_ = cscind;
    d_cscVal_ = cscval;
    csc_ownership_ = true;
    cscval_ownership_ = true;
    csc_initialized_ = true;
  } else {
    if (cscptr != NULL && !symmetric) { gbFree(cscptr); gbFree(cscind); }
    if (cscval != NULL) gbFree(cscval);
  }
  csr_initialized_ = true;
  need_update_ = true;
}

// After the device CSR is in place (owned): the CSC side, then the host mirrors
// the CPU verifiers read.
template <typename T>
Info SparseMatrix<T>::finishDeviceBuild(bool build_csc) {
  csr_initialized_ = true;
  ncapacity_ = nvals_;
  if (build_csc) {
    Index* colptr = NULL; Index* rowind = NULL; T* cval = NULL;
    if (symmetric_) {
      // same structure both ways: only the values need transposing
      ingestCsrToCsc<T>(nrows_, ncols_, nvals_, d_csrRowPtr_, d_csrColInd_, d_csrVal_,
          NULL, NULL, &cval);
      d_cscColPtr_ = d_csrRowPtr_;
      d_cscRowInd_ = d_csrColInd_;
    } else {
      ingestCsrToCsc<T>(nrows_, ncols_, nvals_, d_csrRowPtr_, d_csrColInd_, d_csrVal_,
          &colptr, &rowind, &cval);
      d_cscColPtr_ = colptr;
      d_cscRowInd_ = rowind;
    }
    d_cscVal_ = cval;
    csc_ownership_ = true;
    cscval_ownership_ = true;
    csc_initialized_ = true;
  }
  need_update_ = true;
  releaseHost();
  CHECK(gpuToCpu(true));
  return GrB_SUCCESS;
}

// Tuples in host vectors (the reference's Matrix::build after readMtx): upload,
// sort and convert on the device.  No symmetrising or dropping here — readMtx has
// done what the flags asked for; like the reference's coo2csr this only orders.
template <typename T>
template <typename BinaryOpT>
Info SparseMatrix<T>::build(const std::vector<Index>* row_indices,
    const std::vector<Index>* col_indices, const std::vector<T>* values, Index nvals,
    BinaryOpT dup, char* dat_name) {
  releaseHost();
  releaseDevice();
  if (dat_name != NULL) symmetric_ = (strstr(dat_name, ".ud.") != NULL);
  const size_t m = static_cast<size_t>(nvals);
  Index* d_r = devArray<Index>(atLeastOne(nvals));
  Index* d_c = devArray<Index>(atLeastOne(nvals));
  T*     d_v = devArray<T>(atLeastOne(nvals));
  copyAsync(d_r, row_indices->data(), m, cudaMemcpyHostToDevice);
  copyAsync(d_c, col_indices->data(), m, cudaMemcpyHostToDevice);
  copyAsync(d_v, values->data(), m, cudaMemcpyHostToDevice);
  runtime().sync();                      // the vectors may go away after the call
  nvals_ = ingestCooToCsr<T>(nrows_, ncols_, d_r, d_c, d_v, nvals, 0,
      &d_csrRowPtr_, &d_csrColInd_, &d_csrVal_);
  csr_ownership_ = true;
  gbFree(d_v); gbFree(d_c); gbFree(d_r);
  CHECK(finishDeviceBuild(format_ == GrB_SPARSE_MATRIX_CSRCSC));
  if (format_ == GrB_SPARSE_MATRIX_CSRONLY) {      // CSC names alias the CSR arrays
    h_cscColPtr_ = h_csrRowPtr_; h_cscRowInd_ = h_csrColInd_; h_cscVal_ = h_csrVal_;
  }
  if (dat_name != NULL) {
    if (!cacheFileExists(dat_name)) writeCache(dat_name);
    free(dat_name);
  }
  return GrB_SUCCESS;
}

template <typename T>
Info SparseMatrix<T>::buildFromDeviceTuples(const Index* d_rows, const Index* d_cols,
    const T* d_vals, long long ntuples, int mode, bool symmetric) {
  releaseHost();
  releaseDevice();
  symmetric_ = symmetric;
  nvals_ = ingestCooToCsr<T>(nrows_, ncols_, d_rows, d_cols, d_vals, ntuples, mode,
      &d_csrRowPtr_, &d_csrColInd_, &d_csrVal_);
  csr_ownership_ = true;
  return finishDeviceBuild(format_ == GrB_SPARSE_MATRIX_CSRCSC);
}

// Load from the binary cache named by readMtx (reference :354-407).
template <typename T>
Info SparseMatrix<T>::build(char* dat_name) {
  if (dat_name == NULL || !cacheFileExists(dat_name)) {
    std::cout << "Error: Unable to read file!\n";
    return GrB_SUCCESS;
  }
  releaseHost();
  releaseDevice();
  symmetric_ = (strstr(dat_name, ".ud.") != NULL);
  const bool ok = readCache(dat_name);
  free(dat_name);
  if (!ok) return GrB_SUCCESS;           // message printed; object left empty
  // host CSR is in place: device CSR from it, CSC on the device
  d_csrRowPtr_ = devArray<Index>(static_cast<size_t>(nrows_) + 1);
  d_csrColInd_ = devArray<Index>(atLeastOne(nvals_));
  d_csrVal_    = devArray<T>(atLeastOne(nvals_));
  csr_ownership_ = true;
  transfer(devCsr(), hostCsr(), cudaMemcpyHostToDevice, true);
  runtime().sync();
  CHECK(finishDeviceBuild(format_ == GrB_SPARSE_MATRIX_CSRCSC));
  if (format_ == GrB_SPARSE_MATRIX_CSRONLY) {
    h_cscColPtr_ = h_csrRowPtr_; h_cscRowInd_ = h_csrColInd_; h_cscVal_ = h_csrVal_;
  }
  return GrB_SUCCESS;
}

template <typename T>
bool SparseMatrix<T>::writeCache(const char* path) {
  FILE* f = fopen(path, "wb");
  if (f == NULL) {
    std::cout << "Error: Unable to open file for writing!\n";
    return false;
  }
  printf("Writing %s\n", path);
  MatrixCacheHeader h;
  memcpy(h.magic, "GB2CSR01", 8);
  h.nrows = nrows_; h.ncols = ncols_; h.nvals = nvals_;
  h.value_bytes = static_cast<int32_t>(sizeof(T));
  bool ok = fwrite(&h, sizeof(h), 1, f) == 1;
  ok = ok && fwrite(h_csrRowPtr_, sizeof(Index), static_cast<size_t>(nrows_) + 1, f) ==
                 static_cast<size_t>(nrows_) + 1;
  ok = ok && fwrite(h_csrColInd_, sizeof(Index), nvals_, f) == static_cast<size_t>(nvals_);
  ok = ok && fwrite(h_csrVal_, sizeof(T), nvals_, f) == static_cast<size_t>(nvals_);
  fclose(f);
  if (!ok) { std::cout << "Error: short write, cache removed\n"; remove(path); }
  return ok;
}

// Fills nrows_/ncols_/nvals_ and the host CSR.
template <typename T>
bool SparseMatrix<T>::readCache(const char* path) {
  FILE* f = fopen(path, "rb");
  if (f == NULL) {
    std::cout << "Error: Unable to open file for reading!\n";
    return false;
  }
  printf("Reading %s\n", path);
  MatrixCacheHeader h;
  bool ours = fread(&h, sizeof(h), 1, f) == 1 && memcmp(h.magic, "GB2CSR01", 8) == 0;
  bool values_follow = false;
  if (ours) {
    nrows_ = h.nrows; ncols_ = h.ncols; nvals_ = h.nvals;
    values_follow = (h.value_bytes == static_cast<int32_t>(sizeof(T)));
    if (h.value_bytes != 0 && !values_follow)
      std::cout << "Warning: cache holds values of another type; using 1\n";
  } else {
    // the reference's own layout: nrows, nvals, rowptr, colind (square, pattern)
    rewind(f);
    Index head[2];
    if (fread(head, sizeof(Index), 2, f) != 2) { fclose(f); return false; }
    if (ncols_ != head[0]) std::cout << "Error: nrows not equal to ncols!\n";
    nrows_ = head[0]; nvals_ = head[1];
  }
  h_csrRowPtr_ = hostArray<Index>(static_cast<size_t>(nrows_) + 1);
  h_csrColInd_ = hostArray<Index>(atLeastOne(nvals_));
  h_csrVal_    = hostArray<T>(atLeastOne(nvals_));
  bool ok = fread(h_csrRowPtr_, sizeof(Index), static_cast<size_t>(nrows_) + 1, f) ==
            static_cast<size_t>(nrows_) + 1;
  ok = ok && fread(h_csrColInd_, sizeof(Index), nvals_, f) == static_cast<size_t>(nvals_);
  if (ok && values_follow)
    ok = fread(h_csrVal_, sizeof(T), nvals_, f) == static_cast<size_t>(nvals_);
  else
    std::fill(h_csrVal_, h_csrVal_ + nvals_, static_cast<T>(1));
  fclose(f);
  if (!ok) std::cout << "Error: cache file is truncated\n";
  return ok;
}

// Device CSR arrays of the caller, used in place (reference :418-435).
template <typename T>
Info SparseMatrix<T>::build(Index* row_ptr, Index* col_ind, T* values, Index nvals) {
  releaseDevice();
  releaseHost();
  d_csrRowPtr_ = row_ptr;
  d_csrColInd_ = col_ind;
  d_csrVal_    = values;
  nvals_ = nvals;
  csr_ownership_ = false;
  csr_initialized_ = true;
  need_update_ = true;
  return GrB_SUCCESS;
}

// CSC of the caller.  symmetric: the index arrays alias the CSR (col_ptr/row_ind
// may be NULL).  values == NULL: an owned copy of the CSR values is made, which
// is only right when the values are symmetric too (pattern matrices) — a copy,
// not an alias, because per-row rescaling (PageRank) must be able to make the
// two sides differ.  values == the CSR value array is taken as given; the
// matrix x broadcast-vector eWiseMult (PageRank's normalisation) first gives the
// CSC its own copy (separateCscValues), and the matrix x scalar one scales the
// shared array once.
template <typename T>
Info SparseMatrix<T>::adoptCsc(Index* col_ptr, Index* row_ind, T* values,
    bool symmetric) {
  if (d_csrRowPtr_ == NULL) return GrB_UNINITIALIZED_OBJECT;
  dropDerived();
  symmetric_ = symmetric;
  const bool alias = symmetric && (col_ptr == NULL || row_ind == NULL);
  d_cscColPtr_ = alias ? d_csrRowPtr_ : col_ptr;
  d_cscRowInd_ = alias ? d_csrColInd_ : row_ind;
  csc_ownership_ = false;
  if (values != NULL) {
    d_cscVal_ = values;
    cscval_ownership_ = false;
  } else {
    d_cscVal_ = devArray<T>(atLeastOne(nvals_));
    copyAsync(d_cscVal_, d_csrVal_, static_cast<size_t>(nvals_), cudaMemcpyDeviceToDevice);
    cscval_ownership_ = true;
  }
  csc_initialized_ = true;
  need_update_ = true;
  return GrB_SUCCESS;
}

template <typename T>
Info SparseMatrix<T>::extractElement(T* val, Index row_index, Index col_index) {
  if (row_index < 0 || row_index >= nrows_ || col_index < 0 || col_index >= ncols_)
    return GrB_INDEX_OUT_OF_BOUNDS;
  CHECK(gpuToCpu());
  const Index* first = h_csrColInd_ + h_csrRowPtr_[row_index];
  const Index* last  = h_csrColInd_ + h_csrRowPtr_[row_index + 1];
  const Index* hit = std::lower_bound(first, last, col_index);
  if (hit == last || *hit != col_index) return GrB_NO_VALUE;
  *val = h_csrVal_[hit - h_csrColInd_];
  return GrB_SUCCESS;
}

template <typename T>
Info SparseMatrix<T>::extractTuples(std::vector<Index>* row_indices,
    std::vector<Index>* col_indices, std::vector<T>* values, Index* n) {
  if (*n > nvals_) {
    std::cout << "Error: Too many tuples requested!\n";
    return GrB_UNINITIALIZED_OBJECT;
  }
  if (*n < nvals_) {
    std::cout << "Error: Insufficient space!\n";
    return GrB_INSUFFICIENT_SPACE;
  }
  CHECK(gpuToCpu());
  row_indices->resize(nvals_);
  col_indices->assign(h_csrColInd_, h_csrColInd_ + nvals_);
  values->assign(h_csrVal_, h_csrVal_ + nvals_);
  for (Index r = 0; r < nrows_; ++r)
    std::fill(row_indices->begin() + h_csrRowPtr_[r],
              row_indices->begin() + h_csrRowPtr_[r + 1], r);
  return GrB_SUCCESS;
}

template <typename T>
const T SparseMatrix<T>::operator[](Index ind) {
  gpuToCpu(true);
  if (ind >= nvals_) std::cout << "Error: index out of bounds!\n";
  return h_csrColInd_[ind];
}

template <typename T>
Info SparseMatrix<T>::printSide(const char* str, Side side, Index other_dim) {
  const Index shown_major = std::min<Index>(20, side.dim);
  const Index shown_minor = std::min<Index>(20, other_dim);
  std::cout << str << ":\n";
  for (Index major = 0; major < shown_major; ++major) {
    Index k = side.ptr[major];
    const Index stop = side.ptr[major + 1];
    for (Index minor = 0; minor < shown_minor; ++minor) {
      const bool here = k < stop && side.ind[k] == minor;
      std::cout << ((here && side.val[k] > 0) ? "x " : "0 ");
      if (here) ++k;
    }
    std::cout << "\n";
  }
  return GrB_SUCCESS;
}

template <typename T>
Info SparseMatrix<T>::print(bool force_update) {
  CHECK(gpuToCpu(force_update));
  const int shown = std::min<Index>(nvals_, 40);
  printArray("csrColInd", h_csrColInd_, shown);
  printArray("csrRowPtr", h_csrRowPtr_, std::min<Index>(nrows_ + 1, 40));
  printArray("csrVal", h_csrVal_, shown);
  CHECK(printCSR("pretty print"));
  if (format_ == GrB_SPARSE_MATRIX_CSRCSC && h_cscColPtr_ != NULL) {
    printArray("cscRowInd", h_cscRowInd_, shown);
    printArray("cscColPtr", h_cscColPtr_, std::min<Index>(ncols_ + 1, 40));
    printArray("cscVal", h_cscVal_, shown);
    CHECK(printCSC("pretty print"));
  }
  return GrB_SUCCESS;
}

// Structural invariants of the CSR: offsets monotone, columns strictly
// increasing inside a row.  Returns GrB_INVALID_OBJECT on the first violation.
template <typename T>
Info SparseMatrix<T>::check() {
  CHECK(gpuToCpu());
  std::cout << "Begin check:\n";
  for (Index r = 0; r < nrows_; ++r) {
    if (h_csrRowPtr_[r + 1] < h_csrRowPtr_[r]) return GrB_INVALID_OBJECT;
    for (Index k = h_csrRowPtr_[r] + 1; k < h_csrRowPtr_[r + 1]; ++k)
      if (h_csrColInd_[k] <= h_csrColInd_[k - 1]) return GrB_INVALID_OBJECT;
  }
  return GrB_SUCCESS;
}

template <typename T>
Info SparseMatrix<T>::resize(Index nrows, Index ncols) {
  if (nrows > nrows_ || ncols > ncols_) return GrB_PANIC;   // shrink only
  nrows_ = nrows;
  ncols_ = ncols;
  return GrB_SUCCESS;
}

// axis: 0 row offsets, 1 column indices, 2 values (test helper of the reference).
template <typename T>
template <typename U>
Info SparseMatrix<T>::fill(Index axis, Index nvals, U start) {
  nvals_ = nvals;
  CHECK(allocate());
  if (axis == 0)      std::fill(h_csrRowPtr_, h_csrRowPtr_ + nvals, static_cast<Index>(start));
  else if (axis == 1) std::fill(h_csrColInd_, h_csrColInd_ + nvals, static_cast<Index>(start));
  else if (axis == 2) std::fill(h_csrVal_, h_csrVal_ + nvals, static_cast<T>(start));
  return cpuToGpu();
}

template <typename T>
template <typename U>
Info SparseMatrix<T>::fillAscending(Index axis, Index nvals, U start) {
  nvals_ = nvals;
  CHECK(allocate());
  for (Index i = 0; i < nvals; ++i) {
    if (axis == 0)      h_csrRowPtr_[i] = i + static_cast<Index>(start);
    else if (axis == 1) h_csrColInd_[i] = i + static_cast<Index>(start);
    else if (axis == 2) h_csrVal_[i] = static_cast<T>(i) + static_cast<T>(start);
  }
  return cpuToGpu();
}

template <typename T>
Info SparseMatrix<T>::allocateCpu() {
  ncapacity_ = nvals_;
  const size_t nv = atLeastOne(nvals_);
  if (h_csrRowPtr_ == NULL) h_csrRowPtr_ = hostArray<Index>(static_cast<size_t>(nrows_) + 1);
  if (h_csrColInd_ == NULL) h_csrColInd_ = hostArray<Index>(nv);
  if (h_csrVal_ == NULL)    h_csrVal_ = hostArray<T>(nv);
  if (format_ != GrB_SPARSE_MATRIX_CSRONLY) {
    if (h_cscColPtr_ == NULL) h_cscColPtr_ = hostArray<Index>(static_cast<size_t>(ncols_) + 1);
    if (h_cscRowInd_ == NULL) h_cscRowInd_ = hostArray<Index>(nv);
    if (h_cscVal_ == NULL)    h_cscVal_ = hostArray<T>(nv);
  }
  if (!h_csrRowPtr_ || !h_csrColInd_ || !h_csrVal_) return GrB_OUT_OF_MEMORY;
  return GrB_SUCCESS;
}

template <typename T>
Info SparseMatrix<T>::allocateGpu() {
  const size_t nv = atLeastOne(nvals_);
  if (d_csrRowPtr_ == NULL) {
    d_csrRowPtr_ = devArray<Index>(static_cast<size_t>(nrows_) + 1);
    d_csrColInd_ = devArray<Index>(nv);
    d_csrVal_    = devArray<T>(nv);
    csr_ownership_ = true;
    printMemory("csrVal");
  }
  if (format_ == GrB_SPARSE_MATRIX_CSRCSC && d_cscVal_ == NULL) {
    d_cscVal_ = devArray<T>(nv);
    d_cscColPtr_ = symmetric_ ? d_csrRowPtr_ : devArray<Index>(static_cast<size_t>(ncols_) + 1);
    d_cscRowInd_ = symmetric_ ? d_csrColInd_ : devArray<Index>(nv);
    csc_ownership_ = true;
    cscval_ownership_ = true;
    printMemory("cscVal");
  }
  return GrB_SUCCESS;
}

// Host -> device.  A changed entry count (tril) or foreign device arrays mean the
// device side is rebuilt; the derived caches never survive an upload.
template <typename T>
Info SparseMatrix<T>::cpuToGpu() {
  if (!csr_ownership_ || ncapacity_ != nvals_ || d_csrRowPtr_ == NULL) {
    releaseDevice();
    ncapacity_ = nvals_;
  }
  CHECK(allocateGpu());
  dropDerived();
  transfer(devCsr(), hostCsr(), cudaMemcpyHostToDevice, true);
  if (format_ == GrB_SPARSE_MATRIX_CSRCSC) {
    if (symmetric_) {
      d_cscColPtr_ = d_csrRowPtr_;
      d_cscRowInd_ = d_csrColInd_;
    }
    transfer(devCsc(), hostCsc(), cudaMemcpyHostToDevice, !symmetric_);
  }
  runtime().sync();
  need_update_ = false;
  return GrB_SUCCESS;
}

template <typename T>
Info SparseMatrix<T>::gpuToCpu(bool force_update) {
  const bool fresh_host = (h_csrRowPtr_ == NULL);
  if (fresh_host) CHECK(allocateCpu());
  if ((need_update_ || force_update || fresh_host) && d_csrRowPtr_ != NULL) {
    transfer(hostCsr(), devCsr(), cudaMemcpyDeviceToHost, true);
    const bool have_csc = format_ == GrB_SPARSE_MATRIX_CSRCSC && d_cscVal_ != NULL &&
        d_cscColPtr_ != NULL && d_cscRowInd_ != NULL && h_cscVal_ != NULL &&
        h_cscColPtr_ != NULL && h_cscRowInd_ != NULL && !hostCscIsAlias();
    if (have_csc)
      transfer(hostCsc(), devCsc(), cudaMemcpyDeviceToHost, true);
    runtime().sync();
  }
  need_update_ = false;
  return GrB_SUCCESS;
}

// Host CSC from the host CSR: counting sort by column (rows stay ordered inside a
// column because the CSR is walked row by row).  Takes the place of the
// reference's csr2csc call (:836-848).
template <typename T>
Info SparseMatrix<T>::syncCpu() {
  CHECK(allocateCpu());
  if (!h_csrRowPtr_ || !h_cscColPtr_ || hostCscIsAlias()) return GrB_INVALID_OBJECT;
  const Index nv = h_csrRowPtr_[nrows_];
  std::fill(h_cscColPtr_, h_cscColPtr_ + ncols_ + 1, 0);
  for (Index k = 0; k < nv; ++k) ++h_cscColPtr_[h_csrColInd_[k] + 1];
  for (Index c = 0; c < ncols_; ++c) h_cscColPtr_[c + 1] += h_cscColPtr_[c];
  std::vector<Index> next(h_cscColPtr_, h_cscColPtr_ + ncols_);
  for (Index r = 0; r < nrows_; ++r) {
    for (Index k = h_csrRowPtr_[r]; k < h_csrRowPtr_[r + 1]; ++k) {
      const Index at = next[h_csrColInd_[k]]++;
      h_cscRowInd_[at] = r;
      h_cscVal_[at] = h_csrVal_[k];
    }
  }
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_SPARSE_MATRIX_HPP_
