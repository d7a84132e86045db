// graphblast_b200 backend — extract: submatrices C = op(A)(I, J), columns
// w = op(A)(I, j) and subvectors w = u(I).
//
// All three cut one stored orientation S (kernels/extract.cuh): the submatrix cuts
// op(A) (A's CSR, or its CSC for Aᵀ); the column cuts row j of the other
// orientation with I as its column list; a sparse u is a one-row S over u's
// index list with I as its column list.  A dense u is a gather (indexed.hpp).
//
// extractCut, given device lists (NULL = ALL):
//   1. sel = the selected rows' lengths, scanned: a virtual CSR over the selected
//      entries (its 64-bit total is read; past INT32_MAX: GrB_OUT_OF_MEMORY);
//   2. J given: the column map, jpos = J's positions stably sorted by column
//      (radixSortPairs) and jptr = its bucket bounds over S's columns; count pass,
//      C's row offsets scanned from the per-row counts and the tile bases from the
//      per-tile counts (64-bit total read; past INT32_MAX: GrB_OUT_OF_MEMORY);
//      J = ALL: C's row offsets are sel, no count pass;
//   3. fill.  J non-decreasing (host check) gives every row in ascending column
//      order as it is written; otherwise the fill writes (row, column) keys with
//      their source slots, radixSortPairs sorts them and a store pass writes C.
// Nothing on the device that belongs to an operand changes before the result is
// complete, and a refusal leaves every operand as it was.
#ifndef GRAPHBLAS_BACKEND_CUDA_EXTRACT_HPP_
#define GRAPHBLAS_BACKEND_CUDA_EXTRACT_HPP_

#include <algorithm>
#include <vector>

#include "graphblas/backend/cuda/kernels/extract.cuh"
#include "graphblas/backend/cuda/kernels/kernels.hpp"
#include "graphblas/backend/cuda/sparse_matrix.hpp"
#include "graphblas/backend/cuda/indexed.hpp"

namespace graphblas {
namespace backend {

// One stored orientation to cut: nrows + 1 pointers, its index and value arrays,
// and (may be NULL) the values of the other orientation at the same slots, which
// a symmetric matrix keeps.
template <typename T>
struct ExtractSource {
  const Index* ptr;
  const Index* ind;
  const T*     val;
  const T*     oval;
  Index        nrows;
  Index        ncols;
};

// A computed CSR in fresh pool arrays; oval only when asked for.
template <typename T>
struct ExtractResult {
  Index  nnz = 0;
  Index* rowptr = NULL;
  Index* colind = NULL;
  T*     val = NULL;
  T*     oval = NULL;
};

// A host index list checked against its extent (NULL = ALL, which needs n ==
// extent) and uploaded once; device() stays NULL for ALL.
class IndexList {
 public:
  IndexList() : d_(NULL), h_(NULL), n_(0) {}
  ~IndexList() { if (d_ != NULL) gbFree(d_); }
  IndexList(const IndexList&) = delete;
  IndexList& operator=(const IndexList&) = delete;

  // GrB_INVALID_VALUE for a list shorter than n; GrB_INVALID_INDEX for an index
  // outside [0, extent) or ALL with n != extent.  Nothing is uploaded on a refusal.
  Info check(const std::vector<Index>* h, Index n, Index extent) {
    h_ = h; n_ = n;
    if (h == NULL) return n == extent ? GrB_SUCCESS : GrB_INVALID_INDEX;
    if (static_cast<Index>(h->size()) < n) return GrB_INVALID_VALUE;
    for (Index p = 0; p < n; ++p)
      if ((*h)[p] < 0 || (*h)[p] >= extent) return GrB_INVALID_INDEX;
    return GrB_SUCCESS;
  }
  void upload() {
    if (h_ == NULL || d_ != NULL) return;
    d_ = reinterpret_cast<Index*>(gbMalloc(static_cast<size_t>(n_ > 0 ? n_ : 1)*sizeof(Index)));
    copyAsync(d_, h_->data(), static_cast<size_t>(n_), cudaMemcpyHostToDevice);
  }
  const Index* device() const { return d_; }
  bool all() const { return h_ == NULL; }
  bool nonDecreasing() const {
    return h_ == NULL || std::is_sorted(h_->begin(), h_->begin() + n_);
  }
  // No index appears twice (ALL never repeats); extent bounds the checked list.
  bool distinct(Index extent) const {
    if (h_ == NULL) return true;
    std::vector<bool> seen(static_cast<size_t>(extent), false);
    for (Index p = 0; p < n_; ++p) {
      if (seen[(*h_)[p]]) return false;
      seen[(*h_)[p]] = true;
    }
    return true;
  }
  bool sameAs(const IndexList& o) const {
    if (all() || o.all()) return all() && o.all();
    return n_ == o.n_ && std::equal(h_->begin(), h_->begin() + n_, o.h_->begin());
  }

 private:
  Index* d_;
  const std::vector<Index>* h_;
  Index n_;
};

// C = S(rows, cols): nsel selected rows (rows == NULL: 0..nsel-1), ncut columns
// (cols == NULL: all of S's, ncut == S.ncols), sorted tells that cols is
// non-decreasing.  with_oval: C's entries of S.oval too.
template <typename T>
Info extractCut(const ExtractSource<T>& S, const Index* rows, Index nsel,
                const Index* cols, Index ncut, bool sorted, bool with_oval,
                ExtractResult<T>* out) {
  cudaStream_t s = gbStream();
  unsigned long long* count = reinterpret_cast<unsigned long long*>(
      gbMalloc(2*sizeof(unsigned long long)));
  CUDA_CALL(cudaMemsetAsync(count, 0, 2*sizeof(unsigned long long), s));

  // 1. the selected rows
  Index* sel = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(nsel) + 1)*sizeof(Index)));
  extractRowLengthsKernel<<<gridFor(static_cast<size_t>(nsel) + 1, 256), 256, 0, s>>>(
      sel, rows, S.ptr, nsel, count);
  GB_KERNEL_CHECK();
  const unsigned long long total64 = runtime().fetch(count);
  if (total64 > static_cast<unsigned long long>(INT32_MAX)) {
    gbFree(sel); gbFree(count);
    return GrB_OUT_OF_MEMORY;
  }
  scanExclusiveAsync(sel, static_cast<long long>(nsel) + 1, NULL);
  const long long total = static_cast<long long>(total64);
  const long long ntiles = (total + GB_EXT_TILE - 1)/GB_EXT_TILE;

  // 2. the column map, the count and C's row offsets
  Index* rowptr = sel;
  Index* jptr = NULL;
  unsigned int* jpos = NULL;
  int* tiles = NULL;
  Index nnz = static_cast<Index>(total);
  if (cols != NULL) {
    const size_t nc = static_cast<size_t>(ncut > 0 ? ncut : 1);
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(gbMalloc(nc*8));
    unsigned long long* keys_tmp = reinterpret_cast<unsigned long long*>(gbMalloc(nc*8));
    jpos = reinterpret_cast<unsigned int*>(gbMalloc(nc*4));
    unsigned int* pay_tmp = reinterpret_cast<unsigned int*>(gbMalloc(nc*4));
    if (ncut > 0) {
      extractMapKeysKernel<<<gridFor(ncut, 256), 256, 0, s>>>(keys, jpos, cols, ncut);
      GB_KERNEL_CHECK();
    }
    radixSortPairs(&keys, &jpos, &keys_tmp, &pay_tmp, ncut, ingestBitsFor(S.ncols));
    jptr = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(S.ncols) + 1)*sizeof(Index)));
    extractMapBoundsKernel<<<gridFor(static_cast<size_t>(S.ncols) + 1, 256), 256, 0, s>>>(
        jptr, keys, ncut, S.ncols);
    GB_KERNEL_CHECK();
    gbFree(pay_tmp); gbFree(keys_tmp); gbFree(keys);

    rowptr = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(nsel) + 1)*sizeof(Index)));
    CUDA_CALL(cudaMemsetAsync(rowptr, 0, (static_cast<size_t>(nsel) + 1)*sizeof(Index), s));
    tiles = reinterpret_cast<int*>(gbMalloc(static_cast<size_t>(ntiles > 0 ? ntiles : 1)*sizeof(int)));
    if (ntiles > 0) {
      extractCountKernel<<<static_cast<unsigned int>(ntiles), GB_EXT_NT, 0, s>>>(
          sel, rows, S.ptr, S.ind, jptr, nsel, total, tiles, rowptr, count + 1);
      GB_KERNEL_CHECK();
    }
    const unsigned long long nnz64 = runtime().fetch(count + 1);
    if (nnz64 > static_cast<unsigned long long>(INT32_MAX)) {
      gbFree(tiles); gbFree(rowptr); gbFree(jptr); gbFree(jpos); gbFree(sel); gbFree(count);
      return GrB_OUT_OF_MEMORY;
    }
    nnz = static_cast<Index>(nnz64);
    scanExclusiveAsync(rowptr, static_cast<long long>(nsel) + 1, NULL);
    if (ntiles > 0) scanExclusiveAsync(tiles, ntiles, NULL);
  }
  gbFree(count);

  // 3. fill
  const size_t nz = static_cast<size_t>(nnz > 0 ? nnz : 1);
  Index* colind = reinterpret_cast<Index*>(gbMalloc(nz*sizeof(Index)));
  T* val = reinterpret_cast<T*>(gbMalloc(nz*sizeof(T)));
  T* oval = with_oval ? reinterpret_cast<T*>(gbMalloc(nz*sizeof(T))) : NULL;
  const Index* jp = reinterpret_cast<const Index*>(jpos);
  if (ntiles > 0 && sorted) {
    const unsigned int grid = static_cast<unsigned int>(ntiles);
    if (cols != NULL)
      extractFillKernel<true, false, T><<<grid, GB_EXT_NT, 0, s>>>(sel, rows, S.ptr, S.ind,
          S.val, S.oval, jptr, jp, nsel, total, tiles, 0, colind, val, oval, NULL, NULL);
    else
      extractFillKernel<false, false, T><<<grid, GB_EXT_NT, 0, s>>>(sel, rows, S.ptr, S.ind,
          S.val, S.oval, NULL, NULL, nsel, total, NULL, 0, colind, val, oval, NULL, NULL);
    GB_KERNEL_CHECK();
  } else if (ntiles > 0 && nnz > 0) {
    // J unsorted (so given): sort each row's entries by column
    const int pbits = ingestBitsFor(ncut);
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(gbMalloc(nz*8));
    unsigned long long* keys_tmp = reinterpret_cast<unsigned long long*>(gbMalloc(nz*8));
    unsigned int* pay = reinterpret_cast<unsigned int*>(gbMalloc(nz*4));
    unsigned int* pay_tmp = reinterpret_cast<unsigned int*>(gbMalloc(nz*4));
    extractFillKernel<true, true, T><<<static_cast<unsigned int>(ntiles), GB_EXT_NT, 0, s>>>(
        sel, rows, S.ptr, S.ind, S.val, S.oval, jptr, jp, nsel, total, tiles, pbits,
        NULL, NULL, NULL, keys, pay);
    GB_KERNEL_CHECK();
    radixSortPairs(&keys, &pay, &keys_tmp, &pay_tmp, nnz, ingestBitsFor(nsel) + pbits);
    extractSortedStoreKernel<T><<<gridFor(nz, 256), 256, 0, s>>>(colind, val, oval, keys,
        pay, S.val, S.oval, nnz, pbits);
    GB_KERNEL_CHECK();
    gbFree(pay_tmp); gbFree(pay); gbFree(keys_tmp); gbFree(keys);
  }
  if (cols != NULL) {
    gbFree(tiles); gbFree(jptr); gbFree(jpos); gbFree(sel);
  }
  out->nnz = nnz;
  out->rowptr = rowptr;
  out->colind = colind;
  out->val = val;
  out->oval = oval;
  return GrB_SUCCESS;
}

// C = op(A)(I, J), op(A) = Aᵀ with transpose_a.  C may be A.  A symmetric A (its
// CSC index arrays are its CSR's) cut by one list both ways gives a symmetric C,
// installed the same way: its CSC is its CSR with the other orientation's values.
template <typename c, typename a>
Info extractMatrix(SparseMatrix<c>* C, const SparseMatrix<a>* A, bool transpose_a,
                   const std::vector<Index>* row_indices, Index nrows,
                   const std::vector<Index>* col_indices, Index ncols) {
  if constexpr (!std::is_same<c, a>::value) {
    return GrB_DOMAIN_MISMATCH;
  } else {
    const typename SparseMatrix<a>::View Av = A->view(transpose_a);
    const typename SparseMatrix<a>::View Ov = A->view(!transpose_a);
    // the frontend checks C's shape; checked again for callers that reach the
    // backend through the reference's frontend
    if (C->nrows_ != nrows || C->ncols_ != ncols) return GrB_DIMENSION_MISMATCH;
    IndexList I, J;
    CHECK(I.check(row_indices, nrows, Av.dim));
    CHECK(J.check(col_indices, ncols, Av.other));
    if (!Av.complete()) return GrB_UNINITIALIZED_OBJECT;
    // the CSC values of a symmetric C are A's other orientation's, cut alike
    const bool with_oval = C->format_ == GrB_SPARSE_MATRIX_CSRCSC;
    const bool symmetric = A->symmetric_ && Av.dim == Av.other && I.sameAs(J) &&
                           (Ov.val != NULL || !with_oval);
    I.upload();
    J.upload();
    ExtractSource<a> S = {Av.ptr, Av.ind, Av.val, symmetric ? Ov.val : NULL, Av.dim, Av.other};
    ExtractResult<a> R;
    CHECK(extractCut(S, I.device(), nrows, J.device(), ncols, J.nonDecreasing(),
                     symmetric && with_oval, &R));
    C->replaceDevice(R.nnz, R.rowptr, R.colind, R.val, NULL, NULL, R.oval, symmetric);
    return GrB_SUCCESS;
  }
}

// The sparse vector w (size n) takes a one-row result.
template <typename T>
void installSparseVector(SparseVector<T>* w, const ExtractResult<T>& R) {
  w->allocateGpu();
  copyAsync(w->d_ind_, R.colind, static_cast<size_t>(R.nnz), cudaMemcpyDeviceToDevice);
  copyAsync(w->d_val_, R.val, static_cast<size_t>(R.nnz), cudaMemcpyDeviceToDevice);
  w->computed(R.nnz);
  gbFree(R.rowptr); gbFree(R.colind); gbFree(R.val);
}

// w = op(A)(I, j): row j of the other orientation, I its column list.
template <typename W, typename a>
Info extractColumn(Vector<W>* w, const SparseMatrix<a>* A, bool transpose_a,
                   const std::vector<Index>* row_indices, Index nrows, Index col_index) {
  if constexpr (!std::is_same<W, a>::value) {
    return GrB_DOMAIN_MISMATCH;
  } else {
    const typename SparseMatrix<a>::View Ov = A->view(!transpose_a);
    Index w_size;
    CHECK(w->size(&w_size));
    if (w_size != nrows) return GrB_DIMENSION_MISMATCH;
    if (col_index < 0 || col_index >= Ov.dim) return GrB_INVALID_INDEX;
    IndexList I;
    CHECK(I.check(row_indices, nrows, Ov.other));
    if (!Ov.complete()) return GrB_UNINITIALIZED_OBJECT;
    I.upload();
    ExtractSource<a> S = {Ov.ptr, Ov.ind, Ov.val, NULL, Ov.dim, Ov.other};
    IndexList J;
    const std::vector<Index> one(1, col_index);
    J.check(&one, 1, Ov.dim);
    J.upload();
    ExtractResult<a> R;
    CHECK(extractCut(S, J.device(), 1, I.device(), nrows, I.nonDecreasing(), false, &R));
    installSparseVector(&w->sparse_, R);
    return w->setStorage(GrB_SPARSE);
  }
}

// w = u(I): a gather for a dense u, a one-row cut of u's index list for a sparse u.
template <typename W, typename U>
Info extractVector(Vector<W>* w, const Vector<U>* u, const std::vector<Index>* indices,
                   Index nindices) {
  if constexpr (!std::is_same<W, U>::value) {
    return GrB_DOMAIN_MISMATCH;
  } else {
    Index u_size, w_size;
    CHECK(const_cast<Vector<U>*>(u)->size(&u_size));
    CHECK(w->size(&w_size));
    if (w_size != nindices) return GrB_DIMENSION_MISMATCH;
    if (u->vec_type_ != GrB_DENSE && u->vec_type_ != GrB_SPARSE)
      return GrB_UNINITIALIZED_OBJECT;
    IndexList I;
    CHECK(I.check(indices, nindices, u_size));
    CHECK(u->materialize());
    I.upload();
    cudaStream_t s = gbStream();
    if (u->vec_type_ == GrB_DENSE) {
      // gathered apart, then copied: w may be u
      W* out = reinterpret_cast<W*>(gbMalloc(static_cast<size_t>(nindices)*sizeof(W)));
      if (I.all())
        copyAsync(out, u->dense_.d_val_, static_cast<size_t>(nindices), cudaMemcpyDeviceToDevice);
      else
        gatherByIndexKernel<<<gridFor(nindices, 256), 256, 0, s>>>(out, u_size, I.device(),
            u->dense_.d_val_, nindices);
      GB_KERNEL_CHECK();
      CHECK(w->setStorage(GrB_DENSE));
      CHECK(w->materialize());
      copyAsync(w->dense_.d_val_, out, static_cast<size_t>(nindices), cudaMemcpyDeviceToDevice);
      w->dense_.touched();
      gbFree(out);
      return GrB_SUCCESS;
    }
    // u's stored entries as the one row of a 1 x size(u) matrix
    const SparseVector<U>& su = u->sparse_;
    Index* ptr = reinterpret_cast<Index*>(gbMalloc(2*sizeof(Index)));
    const Index bounds[2] = {0, su.nvals_};
    copyAsync(ptr, bounds, 2, cudaMemcpyHostToDevice);
    ExtractSource<U> S = {ptr, su.d_ind_, su.d_val_, NULL, 1, u_size};
    ExtractResult<U> R;
    const Info info = extractCut(S, static_cast<const Index*>(NULL), 1, I.device(), nindices,
                                 I.nonDecreasing(), false, &R);
    gbFree(ptr);
    CHECK(info);
    installSparseVector(&w->sparse_, R);
    return w->setStorage(GrB_SPARSE);
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_EXTRACT_HPP_
