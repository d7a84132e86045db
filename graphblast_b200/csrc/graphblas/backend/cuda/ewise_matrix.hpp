// graphblast_b200 backend — element-wise operations on two sparse matrices and
// the matrix transpose.
//
//   ewiseMatrix<true>  : C = op(A) ⊕ op(B), the union of the two patterns; where
//                        both hold an entry C(i,j) = add(a, b) (the semiring's ADD,
//                        A's value first), where one does C takes its value
//                        unchanged — no identity is involved (the vector eWiseAdd,
//                        by contrast, has a dense result).
//   ewiseMatrix<false> : C = op(A) ⊗ op(B), the intersection, C(i,j) = mul(a, b)
//                        (the semiring's MUL, A's value first).
//   transposeSparse    : C = Aᵀ (C = A when the descriptor transposes A).
// op(X) is X, or Xᵀ (X's CSC) when GrB_INP0 / GrB_INP1 is GrB_TRAN.
//
// C comes out as a sorted, duplicate-free CSR with new arrays (C may be A, B or
// both); stored zeros stay stored and nothing is pruned.  C is replaced: accum is
// not applied, as in the unmasked mxm.  With C's format CSRCSC its CSC is built
// too, C's symmetric flag is cleared and every cache on its old arrays dropped.
#ifndef GRAPHBLAS_BACKEND_CUDA_EWISE_MATRIX_HPP_
#define GRAPHBLAS_BACKEND_CUDA_EWISE_MATRIX_HPP_

#include <type_traits>

#include "graphblas/backend/cuda/kernels/kernels.hpp"
#include "graphblas/backend/cuda/sparse_matrix.hpp"

namespace graphblas {
namespace backend {

template <bool IsAdd, typename c, typename a, typename b, typename SemiringT>
Info ewiseMatrix(SparseMatrix<c>* C, SemiringT op, const SparseMatrix<a>* A,
                 const SparseMatrix<b>* B, Descriptor* desc) {
  Desc_value inp0_mode, inp1_mode;
  CHECK(desc->get(GrB_INP0, &inp0_mode));
  CHECK(desc->get(GrB_INP1, &inp1_mode));
  const bool use_tran_A = inp0_mode == GrB_TRAN;
  const bool use_tran_B = inp1_mode == GrB_TRAN;

  const typename SparseMatrix<a>::View Av = A->view(use_tran_A);
  const typename SparseMatrix<b>::View Bv = B->view(use_tran_B);
  // the frontend checks the shapes of op(A), op(B) and C; they are checked again
  // for callers that reach the backend through the reference's frontend
  const Index m = C->nrows_, n = C->ncols_;
  if (Av.dim != m || Av.other != n || Bv.dim != m || Bv.other != n)
    return GrB_DIMENSION_MISMATCH;
  if (!Av.complete() || !Bv.complete()) return GrB_UNINITIALIZED_OBJECT;

  cudaStream_t s = gbStream();
  const long long total = static_cast<long long>(A->nvals_) + B->nvals_;
  const long long ntiles = (total + GB_EWM_TILE - 1)/GB_EWM_TILE;
  // tile counts (scanned in place into tile bases), then the 64-bit total
  const size_t tile_bytes = ((static_cast<size_t>(ntiles) + 1)*sizeof(int) + 7)/8*8;
  char* cells = reinterpret_cast<char*>(desc->scratch(GB_SCRATCH_VEC_A,
      tile_bytes + sizeof(unsigned long long)));
  int* tiles = reinterpret_cast<int*>(cells);
  unsigned long long* count = reinterpret_cast<unsigned long long*>(cells + tile_bytes);
  // per-row counts, then (scanned in place) C's row offsets
  Index* rowptr = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(m) + 1)*sizeof(Index)));
  CUDA_CALL(cudaMemsetAsync(rowptr, 0, (static_cast<size_t>(m) + 1)*sizeof(Index), s));
  CUDA_CALL(cudaMemsetAsync(count, 0, sizeof(unsigned long long), s));

  // 1. count: entries of C per tile, per row and in all
  if (ntiles > 0) {
    ewiseMatrixCountKernel<IsAdd><<<static_cast<unsigned int>(ntiles), GB_EWM_NT, 0, s>>>(
        Av.ptr, Av.ind, Bv.ptr, Bv.ind, m, total, tiles, rowptr, count, EwmKeepAll());
    GB_KERNEL_CHECK();
  }
  const unsigned long long nnz64 = runtime().fetch(count);
  if (nnz64 > static_cast<unsigned long long>(INT32_MAX)) {
    gbFree(rowptr);
    return GrB_OUT_OF_MEMORY;
  }
  const Index nnz = static_cast<Index>(nnz64);

  // 2. C's row offsets and the tile bases
  scanExclusiveAsync(rowptr, static_cast<long long>(m) + 1, NULL);
  Index* colind = reinterpret_cast<Index*>(gbMalloc((nnz > 0 ? nnz : 1)*sizeof(Index)));
  c* val = reinterpret_cast<c*>(gbMalloc((nnz > 0 ? nnz : 1)*sizeof(c)));

  // 3. fill
  if (ntiles > 0) {
    scanExclusiveAsync(tiles, ntiles, NULL);
    ewiseMatrixFillKernel<IsAdd, c><<<static_cast<unsigned int>(ntiles), GB_EWM_NT, 0, s>>>(
        Av.ptr, Av.ind, Av.val, Bv.ptr, Bv.ind, Bv.val, m, total, tiles, colind, val,
        extractMul(op), extractAdd(op), EwmKeepAll());
    GB_KERNEL_CHECK();
  }
  C->replaceDevice(nnz, rowptr, colind, val);
  return GrB_SUCCESS;
}

template <typename X>
X* copyOnDevice(const X* src, size_t count) {
  X* dst = reinterpret_cast<X*>(gbMalloc((count > 0 ? count : 1)*sizeof(X)));
  if (count > 0)
    CUDA_CALL(cudaMemcpyAsync(dst, src, count*sizeof(X), cudaMemcpyDeviceToDevice,
        gbStream()));
  return dst;
}

// C = Aᵀ, or C = A with transpose_a (GrB_INP0 = GrB_TRAN).  C's CSR is a copy of
// A's CSC when A has one and is built from A's CSR otherwise; C's CSC, when its
// format keeps one, is a copy of A's CSR.  C may be A.
template <typename c, typename a>
Info transposeSparse(SparseMatrix<c>* C, const SparseMatrix<a>* A, bool transpose_a) {
  if constexpr (!std::is_same<c, a>::value) {
    return GrB_DOMAIN_MISMATCH;
  } else {
    const Index m = transpose_a ? A->nrows_ : A->ncols_;
    const Index n = transpose_a ? A->ncols_ : A->nrows_;
    if (C->nrows_ != m || C->ncols_ != n) return GrB_DIMENSION_MISMATCH;
    if (A->d_csrRowPtr_ == NULL || A->d_csrColInd_ == NULL || A->d_csrVal_ == NULL)
      return GrB_UNINITIALIZED_OBJECT;
    if (transpose_a && reinterpret_cast<const void*>(C) == reinterpret_cast<const void*>(A))
      return GrB_SUCCESS;
    const Index nnz = A->nvals_;
    const size_t nz = static_cast<size_t>(nnz);
    const bool has_csc = A->d_cscColPtr_ != NULL && A->d_cscRowInd_ != NULL &&
                         A->d_cscVal_ != NULL;
    const bool want_csc = C->format_ == GrB_SPARSE_MATRIX_CSRCSC;
    // (ptr, ind, val) of A's CSR and, when present, of A's CSC
    Index* csr[2] = {NULL, NULL};  c* csr_val = NULL;
    Index* csc[2] = {NULL, NULL};  c* csc_val = NULL;
    const bool need_csr = transpose_a || want_csc;
    const bool need_csc = !transpose_a || want_csc;
    if (need_csr) {
      csr[0] = copyOnDevice(A->d_csrRowPtr_, static_cast<size_t>(A->nrows_) + 1);
      csr[1] = copyOnDevice(A->d_csrColInd_, nz);
      csr_val = copyOnDevice(A->d_csrVal_, nz);
    }
    if (need_csc) {
      if (has_csc) {
        csc[0] = copyOnDevice(A->d_cscColPtr_, static_cast<size_t>(A->ncols_) + 1);
        csc[1] = copyOnDevice(A->d_cscRowInd_, nz);
        csc_val = copyOnDevice(A->d_cscVal_, nz);
      } else {
        ingestCsrToCsc<c>(A->nrows_, A->ncols_, nnz, A->d_csrRowPtr_, A->d_csrColInd_,
            A->d_csrVal_, &csc[0], &csc[1], &csc_val);
      }
    }
    if (transpose_a) C->replaceDevice(nnz, csr[0], csr[1], csr_val, csc[0], csc[1], csc_val);
    else             C->replaceDevice(nnz, csc[0], csc[1], csc_val, csr[0], csr[1], csr_val);
    return GrB_SUCCESS;
  }
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_EWISE_MATRIX_HPP_
