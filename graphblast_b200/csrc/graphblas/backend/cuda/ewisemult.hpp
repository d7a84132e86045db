// graphblast_b200 backend — eWiseMult hosts.
//
// Replaces reference graphblas/backend/cuda/ewisemult.hpp:32-622 for the variants
// the hot-path algorithms reach (SURVEY.md §8 a11): vector (x) vector in its
// storage combinations, matrix (x) scalar and matrix (x) broadcast vector (the
// PageRank pre-normalisation A = alpha*A ./ outdeg, reference example/gpr.cu:81-86).
// All apply the semiring's MUL.  Quirks kept: the dense-dense kernel returns
// identity when either input equals identity (kernels/ewisemult.hpp:22-25);
// sparse-dense writes 0 for identity inputs (:108-113).
#ifndef GRAPHBLAS_BACKEND_CUDA_EWISEMULT_HPP_
#define GRAPHBLAS_BACKEND_CUDA_EWISEMULT_HPP_

#include <iostream>
#include <string>

#include "graphblas/backend/cuda/kernels/kernels.hpp"

namespace graphblas {
namespace backend {

// In a sparse result, entries whose dense mask is 0 are set to identity
// (reference zeroDenseIdentityKernel, kernels/util.hpp:34-50).
template <typename W, typename M>
__global__ void zeroWhereMaskZeroKernel(const M* mask, W identity, const Index* w_ind,
    W* w_val, Index nvals) {
  Index k = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; k < nvals; k += stride)
    if (mask[w_ind[k]] == static_cast<M>(0)) w_val[k] = identity;
}

// dense (x) dense -> dense (no mask, or dense mask)
template <typename W, typename U, typename V, typename M,
          typename BinaryOpT,     typename SemiringT>
Info eWiseMultInner(DenseVector<W>* w, const Vector<M>* mask, BinaryOpT accum,
    SemiringT op, const DenseVector<U>* u, const DenseVector<V>* v, Descriptor* desc) {
  Index n;
  u->nvals(&n);
  CHECK(w->allocateGpu());
  if (n > 0) {
    if (mask != NULL)
      ewiseMultDenseMaskedKernel<<<gridFor(n, 256), 256, 0, gbStream()>>>(
          w->d_val_, mask->dense_.d_val_, op.identity(), extractMul(op),
          u->d_val_, v->d_val_, n);
    else
      ewiseMultDenseKernel<<<gridFor(n, 256), 256, 0, gbStream()>>>(
          w->d_val_, op.identity(), extractMul(op), u->d_val_, v->d_val_, n);
    GB_KERNEL_CHECK();
  }
  w->touched();
  return GrB_SUCCESS;
}

// dense (x) dense under a sparse mask -> sparse with the mask's pattern
template <typename W, typename U, typename V, typename M,
          typename BinaryOpT,     typename SemiringT>
Info eWiseMultInner(SparseVector<W>* w, const SparseVector<M>* mask, BinaryOpT accum,
    SemiringT op, const DenseVector<U>* u, const DenseVector<V>* v, Descriptor* desc) {
  Index mask_nvals;
  mask->nvals(&mask_nvals);
  CHECK(w->allocateGpu());
  if (mask_nvals > 0) {
    ewiseMultSparseMaskKernel<<<gridFor(mask_nvals, 256), 256, 0, gbStream()>>>(
        w->d_ind_, w->d_val_, mask->d_ind_, mask->d_val_, mask_nvals,
        extractMul(op), u->d_val_, v->d_val_);
    GB_KERNEL_CHECK();
  }
  w->computed(mask_nvals);
  return GrB_SUCCESS;
}

// sparse (x) dense -> sparse with u's pattern; reverse swaps the mul arguments
template <typename W, typename U, typename V, typename M,
          typename BinaryOpT,     typename SemiringT>
Info eWiseMultInner(SparseVector<W>* w, const Vector<M>* mask, BinaryOpT accum,
    SemiringT op, const SparseVector<U>* u, const DenseVector<V>* v, bool reverse,
    Descriptor* desc) {
  Storage mask_type = GrB_UNKNOWN;
  if (mask != NULL) mask->getStorage(&mask_type);
  if (mask != NULL && mask_type == GrB_SPARSE) {
    // the result takes the mask's pattern (reference ewisemult.hpp:220-237)
    const SparseVector<M>* ms = &mask->sparse_;
    Index mask_nvals, nu;
    ms->nvals(&mask_nvals);
    u->nvals(&nu);
    CHECK(w->allocateGpu());
    if (mask_nvals > 0) {
      ewiseMultSparseDenseSparseMaskKernel<<<gridFor(mask_nvals, 256), 256, 0,
          gbStream()>>>(w->d_ind_, w->d_val_, ms->d_ind_, ms->d_val_, mask_nvals,
          op.identity(), extractMul(op), u->d_ind_, u->d_val_, nu, v->d_val_, reverse);
      GB_KERNEL_CHECK();
    }
    w->computed(mask_nvals);
    return GrB_SUCCESS;
  }
  Index u_nvals;
  u->nvals(&u_nvals);
  CHECK(w->allocateGpu());
  cudaStream_t s = gbStream();
  if (u_nvals > 0) {
    ewiseMultSparseDenseKernel<<<gridFor(u_nvals, 256), 256, 0, s>>>(w->d_ind_,
        w->d_val_, op.identity(), extractMul(op), u->d_ind_, u->d_val_, u_nvals,
        v->d_val_, reverse);
    GB_KERNEL_CHECK();
    if (mask != NULL && mask_type == GrB_DENSE) {
      zeroWhereMaskZeroKernel<<<gridFor(u_nvals, 256), 256, 0, s>>>(
          mask->dense_.d_val_, static_cast<W>(op.identity()), w->d_ind_,
          w->d_val_, u_nvals);
      GB_KERNEL_CHECK();
    }
  }
  w->computed(u_nvals);
  return GrB_SUCCESS;
}

// sparse matrix (x) scalar: both value arrays are scaled (reference :275-341)
template <typename c, typename a, typename b, typename m,
          typename BinaryOpT,     typename SemiringT>
Info eWiseMultInner(SparseMatrix<c>* C, const Matrix<m>* mask, BinaryOpT accum,
    SemiringT op, const SparseMatrix<a>* A, b val, Descriptor* desc) {
  if (mask != NULL) {
    std::cout << "eWiseMult Sparse Matrix Broadcast Scalar with Mask\n";
    std::cout << "Error: Feature not implemented yet!\n";
    return GrB_SUCCESS;
  }
  Index A_nvals;
  A->nvals(&A_nvals);
  if (A != C) CHECK(C->dup(A));
  cudaStream_t s = gbStream();
  if (A_nvals > 0) {
    ewiseScalarKernel<<<gridFor(A_nvals, 256), 256, 0, s>>>(C->d_csrVal_,
        extractMul(op), A->d_csrVal_, A_nvals, val);
    GB_KERNEL_CHECK();
    C->csr_initialized_ = true;
    if (A->format_ == GrB_SPARSE_MATRIX_CSRCSC && A->d_cscVal_ != NULL &&
        A->d_cscVal_ != A->d_csrVal_) {
      ewiseScalarKernel<<<gridFor(A_nvals, 256), 256, 0, s>>>(C->d_cscVal_,
          extractMul(op), A->d_cscVal_, A_nvals, val);
      GB_KERNEL_CHECK();
      C->csc_initialized_ = true;
    }
  }
  C->need_update_ = true;
  return GrB_SUCCESS;
}

// sparse matrix (x) column vector: C(i,j) = mul(A(i,j), b[i])  (reference :470-545)
template <typename c, typename a, typename b, typename m,
          typename BinaryOpT,     typename SemiringT>
Info eWiseMultColInner(SparseMatrix<c>* C, const Matrix<m>* mask, BinaryOpT accum,
    SemiringT op, const SparseMatrix<a>* A, const DenseVector<b>* B, Descriptor* desc) {
  if (mask != NULL) {
    std::cout << "eWiseMult Sparse Matrix Broadcast Col Vector with Mask\n";
    std::cout << "Error: Feature not implemented yet!\n";
    return GrB_SUCCESS;
  }
  Index A_nrows, A_nvals;
  A->nrows(&A_nrows);
  A->nvals(&A_nvals);
  if (A != C) CHECK(C->dup(A));
  // a CSC sharing the CSR's value array would be scaled twice, once per side
  C->separateCscValues();
  cudaStream_t s = gbStream();
  if (A_nvals > 0) {
    ewiseMultRowBroadcastKernel<<<gridFor(static_cast<size_t>(A_nrows)*32, 256),
        256, 0, s>>>(C->d_csrVal_, extractMul(op), A->d_csrRowPtr_,
        A->d_csrVal_, A_nrows, B->d_val_);
    GB_KERNEL_CHECK();
    C->csr_initialized_ = true;
    if (A->format_ == GrB_SPARSE_MATRIX_CSRCSC && A->d_cscVal_ != NULL) {
      // CSC entry k sits in row cscRowInd[k].
      ewiseMultIndexBroadcastKernel<<<gridFor(A_nvals, 256), 256, 0, s>>>(
          C->d_cscVal_, extractMul(op), A->d_cscRowInd_, A->d_cscVal_, A_nvals,
          B->d_val_);
      GB_KERNEL_CHECK();
      C->csc_initialized_ = true;
    }
  }
  C->need_update_ = true;
  return GrB_SUCCESS;
}

// sparse matrix (x) row vector: C(i,j) = mul(A(i,j), b[j])  (reference :547-618)
template <typename c, typename a, typename b, typename m,
          typename BinaryOpT,     typename SemiringT>
Info eWiseMultRowInner(SparseMatrix<c>* C, const Matrix<m>* mask, BinaryOpT accum,
    SemiringT op, const SparseMatrix<a>* A, const DenseVector<b>* B, Descriptor* desc) {
  if (mask != NULL) {
    std::cout << "eWiseMult Sparse Matrix Broadcast Row Vector with Mask\n";
    std::cout << "Error: Feature not implemented yet!\n";
    return GrB_SUCCESS;
  }
  Index A_ncols, A_nvals;
  A->ncols(&A_ncols);
  A->nvals(&A_nvals);
  if (A != C) CHECK(C->dup(A));
  C->separateCscValues();
  cudaStream_t s = gbStream();
  if (A_nvals > 0) {
    ewiseMultIndexBroadcastKernel<<<gridFor(A_nvals, 256), 256, 0, s>>>(
        C->d_csrVal_, extractMul(op), A->d_csrColInd_, A->d_csrVal_, A_nvals,
        B->d_val_);
    GB_KERNEL_CHECK();
    C->csr_initialized_ = true;
    if (A->format_ == GrB_SPARSE_MATRIX_CSRCSC && A->d_cscVal_ != NULL) {
      ewiseMultRowBroadcastKernel<<<gridFor(static_cast<size_t>(A_ncols)*32,
          256), 256, 0, s>>>(C->d_cscVal_, extractMul(op), A->d_cscColPtr_,
          A->d_cscVal_, A_ncols, B->d_val_);
      GB_KERNEL_CHECK();
      C->csc_initialized_ = true;
    }
  }
  C->need_update_ = true;
  return GrB_SUCCESS;
}
}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_EWISEMULT_HPP_
