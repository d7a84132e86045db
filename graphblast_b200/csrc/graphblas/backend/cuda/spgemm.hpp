// graphblast_b200 backend — SpGEMM hosts.
//
// spgemmMasked replaces reference graphblas/backend/cuda/spgemm.hpp:22-110 (the
// triangle counting path): C takes the mask's pattern (C->dup(mask)) and one value
// per mask entry is computed as the dot product A(i,:) . B(:,j).
// spgemmUnmasked is the unmasked product, this project's own hash-row kernels
// (kernels/spgemm_unmasked.cuh) in place of the reference's cuSPARSE csrgemm2
// calls (:114-512), which no longer exist in CUDA 12.
#ifndef GRAPHBLAS_BACKEND_CUDA_SPGEMM_HPP_
#define GRAPHBLAS_BACKEND_CUDA_SPGEMM_HPP_

#include <iostream>

#include "graphblas/backend/cuda/kernels/kernels.hpp"

namespace graphblas {
namespace backend {

// One pass of the hash formulation: three launches, one per table size.  The
// largest tables go first (few items, long tails).
template <bool SWAP, typename c, typename TV, typename PV, typename m,
          typename MulOp, typename AddOp>
Info spgemmHashPass(c* C_val, const HashItem* lists, size_t stride,
    const unsigned int* counts, unsigned int* grabs,
    const Index* T_ptr, const Index* T_ind, const TV* T_val,
    const Index* P_ptr, const Index* P_ind, const PV* P_val,
    const Index* M_ptr, const Index* M_ind, const m* M_val,
    const Index* mask_rowptr, const Index* mask_colind,
    MulOp mul_op, AddOp add_op, c identity, unsigned long long* list_bytes,
    cudaStream_t s) {
  const int sms = runtime().sm_count;
  {
    typedef HashGroupSmem<GB_HASH_SLOTS_L, GB_HASH_CHUNK_L, TV> Smem;
    auto kernel = spgemmHashKernel<1024, false, GB_HASH_SLOTS_L, GB_HASH_SEG_L,
        GB_HASH_CHUNK_L, GB_HASH_UNROLL_L, SWAP, c, TV, PV, m, MulOp, AddOp>;
    static bool configured = false;          // per instantiation
    if (!configured) {
      CUDA_CALL(cudaFuncSetAttribute(kernel,
          cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(Smem))));
      configured = true;
    }
    kernel<<<sms*GB_HASH_CTAS_L, 1024, sizeof(Smem), s>>>(C_val, lists + 2*stride, counts + 2,
        grabs + 2, T_ptr, T_ind, T_val, P_ptr, P_ind, P_val, M_ptr, M_ind, M_val,
        mask_rowptr, mask_colind, mul_op, add_op, identity, list_bytes);
    GB_KERNEL_CHECK();
  }
  {
    typedef HashGroupSmem<GB_HASH_SLOTS_M, GB_HASH_CHUNK_M, TV> Smem;
    auto kernel = spgemmHashKernel<256, false, GB_HASH_SLOTS_M, GB_HASH_CAP_M,
        GB_HASH_CHUNK_M, GB_HASH_UNROLL_M, SWAP, c, TV, PV, m, MulOp, AddOp>;
    static bool configured = false;
    if (!configured) {
      CUDA_CALL(cudaFuncSetAttribute(kernel,
          cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(Smem))));
      configured = true;
    }
    kernel<<<sms*GB_HASH_CTAS_M, 256, sizeof(Smem), s>>>(C_val, lists + stride, counts + 1,
        grabs + 1, T_ptr, T_ind, T_val, P_ptr, P_ind, P_val, M_ptr, M_ind, M_val,
        mask_rowptr, mask_colind, mul_op, add_op, identity, list_bytes);
    GB_KERNEL_CHECK();
  }
  {
    typedef HashGroupSmem<GB_HASH_SLOTS_S, GB_HASH_CHUNK_S, TV> Smem;
    auto kernel = spgemmHashKernel<256, true, GB_HASH_SLOTS_S, GB_HASH_CAP_S,
        GB_HASH_CHUNK_S, 2, SWAP, c, TV, PV, m, MulOp, AddOp>;
    static bool configured = false;
    if (!configured) {
      CUDA_CALL(cudaFuncSetAttribute(kernel,
          cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(8*sizeof(Smem))));
      configured = true;
    }
    kernel<<<sms*4, 256, 8*sizeof(Smem), s>>>(C_val, lists, counts, grabs,
        T_ptr, T_ind, T_val, P_ptr, P_ind, P_val, M_ptr, M_ind, M_val,
        mask_rowptr, mask_colind, mul_op, add_op, identity, list_bytes);
    GB_KERNEL_CHECK();
  }
  return GrB_SUCCESS;
}

template <typename c, typename a, typename b, typename m,
          typename BinaryOpT,     typename SemiringT>
Info spgemmMasked(SparseMatrix<c>* C, const Matrix<m>* mask, BinaryOpT accum,
    SemiringT op, const SparseMatrix<a>* A, const SparseMatrix<b>* B,
    Descriptor* desc) {
  Desc_value scmp_mode, inp0_mode, inp1_mode;
  CHECK(desc->get(GrB_MASK, &scmp_mode));
  CHECK(desc->get(GrB_INP0, &inp0_mode));
  CHECK(desc->get(GrB_INP1, &inp1_mode));

  const bool use_mask   = (mask != NULL);
  const bool use_tran_A = inp0_mode == GrB_TRAN;
  const bool use_tran_B = inp1_mode == GrB_TRAN;

  // rows of op(A) against columns of op(B): B's CSC unless B is transposed
  const typename SparseMatrix<a>::View Av = A->view(use_tran_A);
  const typename SparseMatrix<b>::View Bv = B->view(!use_tran_B);
  const Index* A_csrRowPtr = Av.ptr;
  const Index* A_csrColInd = Av.ind;
  const a*     A_csrVal    = Av.val;
  const Index  A_nrows     = Av.dim;
  const Index* B_cscColPtr = Bv.ptr;
  const Index* B_cscRowInd = Bv.ind;
  const b*     B_cscVal    = Bv.val;

  if (A_csrRowPtr == NULL || B_cscColPtr == NULL)
    return GrB_UNINITIALIZED_OBJECT;

  if (use_mask) {
    Storage mask_mat_type;
    CHECK(mask->getStorage(&mask_mat_type));
    if (mask_mat_type == GrB_DENSE) {
      std::cout << "SpGEMM with dense mask\n";
      std::cout << "Error: Feature not implemented yet!\n";
    } else {
      if (reinterpret_cast<const void*>(C) != reinterpret_cast<const void*>(A) &&
          reinterpret_cast<const void*>(C) != reinterpret_cast<const void*>(B))
        CHECK(C->dup(&mask->sparse_));

      const SparseMatrix<m>* sparse_mask = &mask->sparse_;
      unsigned long long* work = desc->counters() + 3;
      cudaStream_t s = gbStream();
      CUDA_CALL(cudaMemsetAsync(work, 0, sizeof(unsigned long long), s));
      const int grid = runtime().sm_count*8;
      unsigned long long* prof_cell = NULL;
      if (profiler().enabled) {
        profiler().ensureCells(gbStream());
        prof_cell = profiler().d_cells + GB_PROF_SPGEMM;
      }
      profiler().begin(GB_PROF_SPGEMM, s);
      // Hash formulation (kernels/spgemm_hash.cuh) when the mask can also be walked
      // by columns; otherwise the search kernels.  A symmetric matrix borrows its
      // CSR arrays for the column side, which is right only for the whole
      // pattern — tril drops the flag.
      const bool mask_by_cols = sparse_mask->format_ == GrB_SPARSE_MATRIX_CSRCSC &&
          sparse_mask->d_cscColPtr_ != NULL && sparse_mask->d_cscRowInd_ != NULL &&
          sparse_mask->d_cscVal_ != NULL;
      const Index B_ncols = Bv.dim;
      const bool hashed = mask_by_cols &&
          sparse_mask->nrows_ == A_nrows && sparse_mask->ncols_ == B_ncols;
      if (hashed) {
        // work items per class: at most one partial chunk per owner plus the full ones
        const size_t stride = static_cast<size_t>(A_nrows > B_ncols ? A_nrows : B_ncols) +
            static_cast<size_t>(sparse_mask->nvals_)/GB_HASH_CHUNK_S + 1;
        const size_t list_ints = 2*2*GB_HASH_NCLASS*stride;
        Index* arena = reinterpret_cast<Index*>(desc->scratch(GB_SCRATCH_VEC_A,
            (list_ints + 32)*sizeof(Index)));
        HashItem* lists = reinterpret_cast<HashItem*>(arena);
        unsigned int* cells = reinterpret_cast<unsigned int*>(arena + list_ints);
        // cells: [0..2] item counts of pass 1, [4..6] of pass 2, [8..10] and
        // [12..14] the grab counters
        CUDA_CALL(cudaMemsetAsync(cells, 0, 32*sizeof(unsigned int), s));
        spgemmHashClassifyKernel<<<gridFor(A_nrows, 256), 256, 0, s>>>(A_csrRowPtr,
            sparse_mask->d_csrRowPtr_, A_nrows, false, lists, stride, cells);
        GB_KERNEL_CHECK();
        spgemmHashClassifyKernel<<<gridFor(B_ncols, 256), 256, 0, s>>>(B_cscColPtr,
            sparse_mask->d_cscColPtr_, B_ncols, true,
            lists + GB_HASH_NCLASS*stride, stride, cells + 4);
        GB_KERNEL_CHECK();
        CHECK((spgemmHashPass<false>(C->d_csrVal_, lists, stride, cells, cells + 8,
            A_csrRowPtr, A_csrColInd, A_csrVal, B_cscColPtr, B_cscRowInd, B_cscVal,
            sparse_mask->d_csrRowPtr_, sparse_mask->d_csrColInd_,
            sparse_mask->d_csrVal_, sparse_mask->d_csrRowPtr_,
            sparse_mask->d_csrColInd_, extractMul(op), extractAdd(op),
            static_cast<c>(op.identity()), prof_cell, s)));
        CHECK((spgemmHashPass<true>(C->d_csrVal_, lists + GB_HASH_NCLASS*stride,
            stride, cells + 4, cells + 12,
            B_cscColPtr, B_cscRowInd, B_cscVal, A_csrRowPtr, A_csrColInd, A_csrVal,
            sparse_mask->d_cscColPtr_, sparse_mask->d_cscRowInd_,
            sparse_mask->d_cscVal_, sparse_mask->d_csrRowPtr_,
            sparse_mask->d_csrColInd_, extractMul(op), extractAdd(op),
            static_cast<c>(op.identity()), prof_cell, s)));
      } else {
        // thread per mask entry; entries whose lists are both long are deferred
        // to a warp-per-entry kernel through a device-side list (`work` counts it)
        Index* heavy = reinterpret_cast<Index*>(desc->scratch(GB_SCRATCH_VEC_A,
            2*static_cast<size_t>(sparse_mask->nvals_ + 1)*sizeof(Index)));
        spgemmMaskedEdgeKernel<<<grid, GB_SPGEMM_NT, 0, s>>>(C->d_csrVal_,
            sparse_mask->d_csrRowPtr_, sparse_mask->d_csrColInd_,
            sparse_mask->d_csrVal_, extractMul(op), extractAdd(op),
            static_cast<c>(op.identity()), A_csrRowPtr, A_csrColInd, A_csrVal,
            B_cscColPtr, B_cscRowInd, B_cscVal, A_nrows, sparse_mask->nvals_,
            heavy, work, prof_cell);
        GB_KERNEL_CHECK();
        spgemmMaskedHeavyKernel<<<grid, GB_SPGEMM_NT, 0, s>>>(C->d_csrVal_,
            sparse_mask->d_csrColInd_, extractMul(op), extractAdd(op),
            static_cast<c>(op.identity()), A_csrRowPtr, A_csrColInd, A_csrVal,
            B_cscColPtr, B_cscRowInd, B_cscVal, heavy, work);
      }
      GB_KERNEL_CHECK();
      profiler().end(GB_PROF_SPGEMM, s, 8.0*(A_nrows + 1) +
          8.0*sparse_mask->nvals_);
    }
  }
  C->need_update_ = true;
  C->csr_initialized_ = true;
  C->csc_initialized_ = false;
  return GrB_SUCCESS;
}

// Semirings whose add is not associative (greater, less, not_equal_to): their fold
// depends on the order of the products, and a hash accumulator has none.
template <typename S> struct FoldNeedsOrder : std::false_type {};
template <typename X, typename Y, typename Z>
struct FoldNeedsOrder<GreaterPlusSemiring<X, Y, Z> > : std::true_type {};
template <typename X, typename Y, typename Z>
struct FoldNeedsOrder<CustomLessPlusSemiring<X, Y, Z> > : std::true_type {};
template <typename X, typename Y, typename Z>
struct FoldNeedsOrder<NotEqualToPlusSemiring<X, Y, Z> > : std::true_type {};
template <typename X, typename Y, typename Z>
struct FoldNeedsOrder<CustomLessLessSemiring<X, Y, Z> > : std::true_type {};

// Semirings whose add is plus: the numeric kernels combine with a native atomicAdd.
template <typename S> struct AddIsPlus : std::false_type {};
#define GB_MXM_PLUS_ADD(NAME)                                                 \
  template <typename X, typename Y, typename Z>                               \
  struct AddIsPlus<NAME<X, Y, Z> > : std::true_type {};
GB_MXM_PLUS_ADD(PlusMultipliesSemiring)
GB_MXM_PLUS_ADD(PlusDividesSemiring)
GB_MXM_PLUS_ADD(PlusGreaterSemiring)
GB_MXM_PLUS_ADD(PlusMinusSemiring)
GB_MXM_PLUS_ADD(PlusLessSemiring)
GB_MXM_PLUS_ADD(PlusNotEqualToSemiring)
#undef GB_MXM_PLUS_ADD

// Largest scratch the dense-accumulator kernels take for their per-CTA arrays; the
// CTA count shrinks to fit.
#define GB_MXM_DENSE_BYTES (size_t(1) << 29)

template <typename KernelT>
void mxmSetSmem(KernelT kernel, size_t bytes) {
  CUDA_CALL(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
      static_cast<int>(bytes)));
}

// Numeric launches of spgemmUnmasked, one per bin that holds rows.
template <bool PLUS, typename c, typename a, typename b, typename MulOp, typename AddOp>
void mxmNumericPass(const unsigned int* count, const Index* lists, size_t stride,
    MxmCells* cells, const Index* A_ptr, const Index* A_ind, const a* A_val,
    const Index* B_ptr, const Index* B_ind, const b* B_val, Index ncols,
    const Index* C_ptr, Index* C_ind, c* C_val, MulOp mul_op, AddOp add_op,
    c identity, Descriptor* desc, cudaStream_t s) {
  const int sms = runtime().sm_count;
  if (count[0]) {
    auto kernel = mxmNumericKernel<256, true, 2*GB_MXM_NUM_S, PLUS, c, a, b, MulOp, AddOp>;
    const size_t smem = GB_MXM_WARPS*2*(2*GB_MXM_NUM_S)*sizeof(int);
    static bool configured = false;
    if (!configured) { mxmSetSmem(kernel, smem); configured = true; }
    const unsigned int want = (count[0] + GB_MXM_WARPS - 1)/GB_MXM_WARPS;
    kernel<<<want < 6u*sms ? want : 6u*sms, 256, smem, s>>>(lists, cells, 0,
        cells->grab, A_ptr, A_ind, A_val, B_ptr, B_ind, B_val, C_ptr, C_ind, C_val,
        mul_op, add_op, identity);
    GB_KERNEL_CHECK();
  }
  if (count[1]) {
    auto kernel = mxmNumericKernel<256, false, 2*GB_MXM_NUM_M, PLUS, c, a, b, MulOp, AddOp>;
    const size_t smem = 2*(2*GB_MXM_NUM_M)*sizeof(int);
    static bool configured = false;
    if (!configured) { mxmSetSmem(kernel, smem); configured = true; }
    kernel<<<count[1] < 6u*sms ? count[1] : 6u*sms, 256, smem, s>>>(lists + stride,
        cells, 1, cells->grab + 1, A_ptr, A_ind, A_val, B_ptr, B_ind, B_val, C_ptr,
        C_ind, C_val, mul_op, add_op, identity);
    GB_KERNEL_CHECK();
  }
  if (count[2]) {
    auto kernel = mxmNumericKernel<1024, false, 2*GB_MXM_NUM_L, PLUS, c, a, b, MulOp, AddOp>;
    const size_t smem = 2*(2*GB_MXM_NUM_L)*sizeof(int);
    static bool configured = false;
    if (!configured) { mxmSetSmem(kernel, smem); configured = true; }
    kernel<<<count[2] < 1u*sms ? count[2] : 1u*sms, 1024, smem, s>>>(
        lists + 2*stride, cells, 2, cells->grab + 2, A_ptr, A_ind, A_val, B_ptr,
        B_ind, B_val, C_ptr, C_ind, C_val, mul_op, add_op, identity);
    GB_KERNEL_CHECK();
  }
  if (count[3]) {
    const size_t words = (static_cast<size_t>(ncols) + 31)/32;
    const size_t per_cta = static_cast<size_t>(ncols)*sizeof(c) + words*sizeof(unsigned int);
    size_t ctas = GB_MXM_DENSE_BYTES/per_cta;
    if (ctas > count[3]) ctas = count[3];
    if (ctas > static_cast<size_t>(sms)) ctas = sms;
    if (ctas < 1) ctas = 1;
    c* acc = reinterpret_cast<c*>(desc->scratch(GB_SCRATCH_VEC_B, ctas*per_cta));
    unsigned int* bits = reinterpret_cast<unsigned int*>(acc + ctas*ncols);
    mxmFillKernel<<<gridFor(ctas*ncols, 256), 256, 0, s>>>(acc, ctas*ncols, identity);
    GB_KERNEL_CHECK();
    CUDA_CALL(cudaMemsetAsync(bits, 0, ctas*words*sizeof(unsigned int), s));
    mxmNumericDenseKernel<1024, PLUS><<<static_cast<int>(ctas), 1024, 0, s>>>(
        lists + 3*stride, cells, 3, cells->grab + 3, A_ptr, A_ind, A_val, B_ptr,
        B_ind, B_val, C_ptr, C_ind, C_val, mul_op, add_op, identity, acc, bits, ncols,
        words);
    GB_KERNEL_CHECK();
  }
}

// C = A (+.x) B without a mask (kernels/spgemm_unmasked.cuh).  C gets new arrays:
// it may be A or B.  accum is ignored, as in the masked product: C is replaced.
// Returns GrB_OUT_OF_MEMORY, with C untouched, when nnz(C) would not fit an Index.
template <typename c, typename a, typename b, typename SemiringT>
Info spgemmUnmaskedProduct(SparseMatrix<c>* C, SemiringT op,
    const SparseMatrix<a>* A, const SparseMatrix<b>* B, Descriptor* desc);

template <typename c, typename a, typename b, typename BinaryOpT, typename SemiringT>
Info spgemmUnmasked(SparseMatrix<c>* C, BinaryOpT accum, SemiringT op,
    const SparseMatrix<a>* A, const SparseMatrix<b>* B, Descriptor* desc) {
  if constexpr (FoldNeedsOrder<SemiringT>::value) return GrB_NOT_IMPLEMENTED;
  else return spgemmUnmaskedProduct(C, op, A, B, desc);
}

template <typename c, typename a, typename b, typename SemiringT>
Info spgemmUnmaskedProduct(SparseMatrix<c>* C, SemiringT op,
    const SparseMatrix<a>* A, const SparseMatrix<b>* B, Descriptor* desc) {
  Desc_value inp0_mode, inp1_mode;
  CHECK(desc->get(GrB_INP0, &inp0_mode));
  CHECK(desc->get(GrB_INP1, &inp1_mode));
  const bool use_tran_A = inp0_mode == GrB_TRAN;
  const bool use_tran_B = inp1_mode == GrB_TRAN;

  const typename SparseMatrix<a>::View Av = A->view(use_tran_A);
  const typename SparseMatrix<b>::View Bv = B->view(use_tran_B);
  const Index* A_ptr = Av.ptr;
  const Index* A_ind = Av.ind;
  const a*     A_val = Av.val;
  const Index* B_ptr = Bv.ptr;
  const Index* B_ind = Bv.ind;
  const b*     B_val = Bv.val;
  // op(A) is m x k, op(B) k x n: the kernels index B's pointer array with A's
  // columns, and C's arrays with m and n
  const Index m = Av.dim, n = Bv.other;
  if (Av.other != Bv.dim || m != C->nrows_ || n != C->ncols_)
    return GrB_DIMENSION_MISMATCH;
  if (!Av.complete() || !Bv.complete()) return GrB_UNINITIALIZED_OBJECT;

  cudaStream_t s = gbStream();
  const int sms = runtime().sm_count;
  const size_t stride = m > 0 ? static_cast<size_t>(m) : 1;
  // row lists of the four bins, then the cells (8-byte aligned)
  Index* lists = reinterpret_cast<Index*>(desc->scratch(GB_SCRATCH_VEC_A,
      GB_MXM_NBIN*stride*sizeof(Index) + sizeof(MxmCells) + 8));
  MxmCells* cells = reinterpret_cast<MxmCells*>(lists + GB_MXM_NBIN*stride);
  // row bounds, then counts, then (scanned in place) C's row offsets
  Index* rowptr = reinterpret_cast<Index*>(gbMalloc((static_cast<size_t>(m) + 1)*sizeof(Index)));
  CUDA_CALL(cudaMemsetAsync(rowptr + m, 0, sizeof(Index), s));
  CUDA_CALL(cudaMemsetAsync(cells, 0, sizeof(MxmCells), s));

  // 1. bounds and symbolic bins
  if (m > 0) {
    mxmRowBoundKernel<<<gridFor(static_cast<size_t>(m), 256), 256, 0, s>>>(A_ptr, A_ind,
        B_ptr, m, n, rowptr);
    GB_KERNEL_CHECK();
    mxmClassifyKernel<<<gridFor(static_cast<size_t>(m), 256), 256, 0, s>>>(rowptr, m,
        A_ptr, GB_MXM_SYM_S, GB_MXM_SYM_M, GB_MXM_SYM_L, lists, stride, cells);
    GB_KERNEL_CHECK();
  }
  const MxmCells sym = runtime().fetch(cells);
  if (sym.exact > static_cast<unsigned long long>(INT32_MAX)) {
    gbFree(rowptr);
    return GrB_OUT_OF_MEMORY;
  }

  // 2. symbolic: distinct columns per row
  if (sym.count[0]) {
    auto kernel = mxmSymbolicKernel<256, true, 2*GB_MXM_SYM_S>;
    const size_t smem = GB_MXM_WARPS*(2*GB_MXM_SYM_S)*sizeof(int);
    static bool configured = false;
    if (!configured) { mxmSetSmem(kernel, smem); configured = true; }
    const unsigned int want = (sym.count[0] + GB_MXM_WARPS - 1)/GB_MXM_WARPS;
    kernel<<<want < 3u*sms ? want : 3u*sms, 256, smem, s>>>(lists, cells, 0,
        cells->grab, A_ptr, A_ind, B_ptr, B_ind, rowptr);
    GB_KERNEL_CHECK();
  }
  if (sym.count[1]) {
    auto kernel = mxmSymbolicKernel<256, false, 2*GB_MXM_SYM_M>;
    const size_t smem = (2*GB_MXM_SYM_M)*sizeof(int);
    static bool configured = false;
    if (!configured) { mxmSetSmem(kernel, smem); configured = true; }
    kernel<<<sym.count[1] < 6u*sms ? sym.count[1] : 6u*sms, 256, smem, s>>>(
        lists + stride, cells, 1, cells->grab + 1, A_ptr, A_ind, B_ptr, B_ind, rowptr);
    GB_KERNEL_CHECK();
  }
  if (sym.count[2]) {
    auto kernel = mxmSymbolicKernel<1024, false, 2*GB_MXM_SYM_L>;
    const size_t smem = (2*GB_MXM_SYM_L)*sizeof(int);
    static bool configured = false;
    if (!configured) { mxmSetSmem(kernel, smem); configured = true; }
    kernel<<<sym.count[2] < 1u*sms ? sym.count[2] : 1u*sms, 1024, smem, s>>>(
        lists + 2*stride, cells, 2, cells->grab + 2, A_ptr, A_ind, B_ptr, B_ind, rowptr);
    GB_KERNEL_CHECK();
  }
  if (sym.count[3]) {
    const size_t words = (static_cast<size_t>(n) + 31)/32;
    size_t ctas = GB_MXM_DENSE_BYTES/(words*sizeof(unsigned int));
    if (ctas > sym.count[3]) ctas = sym.count[3];
    if (ctas > static_cast<size_t>(sms)) ctas = sms;
    if (ctas < 1) ctas = 1;
    unsigned int* bits = reinterpret_cast<unsigned int*>(desc->scratch(GB_SCRATCH_VEC_B,
        ctas*words*sizeof(unsigned int)));
    CUDA_CALL(cudaMemsetAsync(bits, 0, ctas*words*sizeof(unsigned int), s));
    mxmSymbolicDenseKernel<1024><<<static_cast<int>(ctas), 1024, 0, s>>>(
        lists + 3*stride, cells, 3, cells->grab + 3, A_ptr, A_ind, B_ptr, B_ind,
        rowptr, bits, words);
    GB_KERNEL_CHECK();
  }

  // 3. numeric bins by the exact counts, their 64-bit total, C's row offsets
  CUDA_CALL(cudaMemsetAsync(cells, 0, sizeof(MxmCells), s));
  if (m > 0) {
    mxmClassifyKernel<<<gridFor(static_cast<size_t>(m), 256), 256, 0, s>>>(rowptr, m,
        NULL, GB_MXM_NUM_S, GB_MXM_NUM_M, GB_MXM_NUM_L, lists, stride, cells);
    GB_KERNEL_CHECK();
  }
  const MxmCells num = runtime().fetch(cells);
  if (num.total > static_cast<unsigned long long>(INT32_MAX)) {
    gbFree(rowptr);
    return GrB_OUT_OF_MEMORY;
  }
  const Index nnz = static_cast<Index>(num.total);
  scanExclusiveInPlace(rowptr, static_cast<long long>(m) + 1);
  Index* colind = reinterpret_cast<Index*>(gbMalloc((nnz > 0 ? nnz : 1)*sizeof(Index)));
  c* val = reinterpret_cast<c*>(gbMalloc((nnz > 0 ? nnz : 1)*sizeof(c)));

  // 4. numeric
  mxmNumericPass<AddIsPlus<SemiringT>::value>(num.count, lists, stride, cells, A_ptr,
      A_ind, A_val, B_ptr, B_ind, B_val, n, rowptr, colind, val, extractMul(op),
      extractAdd(op), static_cast<c>(op.identity()), desc, s);

  C->replaceDevice(nnz, rowptr, colind, val);
  return GrB_SUCCESS;
}
}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_SPGEMM_HPP_
