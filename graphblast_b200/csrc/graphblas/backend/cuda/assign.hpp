// graphblast_b200 backend — masked constant assign.
//
// Replaces reference graphblas/backend/cuda/assign.hpp:14-241.
//  * dense target : w[i] = val where the mask selects i (dense or sparse mask).
//  * sparse target: the reference overwrites selected entries with `val` and then
//    prunes every entry equal to `val` (3 kernels + scan + 2 D2D copies,
//    :172-221) — i.e. a masked delete.  Here: one ordered compaction that keeps
//    exactly the surviving entries, then one D2D copy back.
// Mask polarity: under GrB_SCMP entries with mask == 0 are selected.
#ifndef GRAPHBLAS_BACKEND_CUDA_ASSIGN_HPP_
#define GRAPHBLAS_BACKEND_CUDA_ASSIGN_HPP_

#include <iostream>

#include "graphblas/backend/cuda/kernels/kernels.hpp"
#include "graphblas/backend/cuda/compact.hpp"

namespace graphblas {
namespace backend {

template <typename W, typename T, typename M, typename I,
          typename BinaryOpT>
Info assignDense(DenseVector<W>* w, Vector<M>* mask, BinaryOpT accum, T val,
    const Vector<I>* indices, Index nindices, Descriptor* desc) {
  Desc_value scmp_mode, repl_mode;
  CHECK(desc->get(GrB_MASK, &scmp_mode));
  CHECK(desc->get(GrB_OUTP, &repl_mode));

  const bool use_mask = (mask != NULL);
  const bool use_all  = (indices == NULL);
  const bool use_scmp = (scmp_mode == GrB_SCMP);

  if (desc->debug()) {
    std::cout << "Executing assignDense\n";
    printState(use_mask, !AccumIsNull<BinaryOpT>::value, use_scmp,
        repl_mode == GrB_REPLACE, false);
  }
  if (!use_all) {
    std::cout << "Selective Indices DeVec Assign Constant\n";
    std::cout << "Error: Feature not implemented yet!\n";
    return GrB_SUCCESS;
  }
  if (!use_mask) {
    std::cout << "Unmasked DeVec Assign Constant\n";
    std::cout << "Error: Feature not implemented yet!\n";
    return GrB_SUCCESS;
  }

  CHECK(w->allocateGpu());
  cudaStream_t s = gbStream();
  Storage mask_vec_type;
  CHECK(mask->getStorage(&mask_vec_type));

  // The target's bitmap shadow survives a constant assign when the mask's
  // selection is available as bits (dense mask with a valid shadow, or a sparse
  // mask): exactly the assign(v<f> = level) of the BFS loop.
  bool bits_kept = false;
  if (mask_vec_type == GrB_DENSE) {
    const int grid = gridFor(w->nvals_, 256);
    const unsigned int* mask_bits = mask->dense_.exactBits();
    if (mask_bits != NULL) {
      unsigned int* w_bits = w->exactBits();
      if (use_scmp)
        assignDenseBitsMaskKernel<true><<<grid, 256, 0, s>>>(w->d_val_, w_bits,
            w->nvals_, mask_bits, static_cast<W>(val));
      else
        assignDenseBitsMaskKernel<false><<<grid, 256, 0, s>>>(w->d_val_, w_bits,
            w->nvals_, mask_bits, static_cast<W>(val));
      bits_kept = (w_bits != NULL);
    } else if (use_scmp) {
      assignDenseDenseMaskKernel<true><<<grid, 256, 0, s>>>(w->d_val_,
          w->nvals_, mask->dense_.d_val_, static_cast<W>(val));
    } else {
      assignDenseDenseMaskKernel<false><<<grid, 256, 0, s>>>(w->d_val_,
          w->nvals_, mask->dense_.d_val_, static_cast<W>(val));
    }
    GB_KERNEL_CHECK();
  } else if (mask_vec_type == GrB_SPARSE) {
    if (use_scmp) {
      std::cout << "All Indices DeVec Assign Constant Scmp Kernel\n";
      std::cout << "Error: Feature not implemented yet!\n";
    } else if (mask->sparse_.nvals_ > 0) {
      const int grid = gridFor(mask->sparse_.nvals_, 256);
      unsigned int* w_bits = w->exactBits();
      if (w_bits != NULL) {
        assignDenseSparseMaskBitsKernel<<<grid, 256, 0, s>>>(w->d_val_,
            w_bits, mask->sparse_.d_ind_, mask->sparse_.nvals_,
            static_cast<W>(val));
        bits_kept = true;
      } else {
        assignDenseSparseMaskKernel<<<grid, 256, 0, s>>>(w->d_val_,
            mask->sparse_.d_ind_, mask->sparse_.nvals_, static_cast<W>(val));
      }
      GB_KERNEL_CHECK();
    } else {
      bits_kept = (w->exactBits() != NULL);
    }
  } else {
    return GrB_UNINITIALIZED_OBJECT;
  }
  w->wroteUnderMask(bits_kept);
  return GrB_SUCCESS;
}

template <typename W, typename T, typename M,
          typename BinaryOpT>
Info assignSparse(SparseVector<W>* w, Vector<M>* mask, BinaryOpT accum, T val,
    const Vector<Index>* indices, Index nindices, Descriptor* desc) {
  Desc_value scmp_mode;
  CHECK(desc->get(GrB_MASK, &scmp_mode));
  const bool use_scmp = (scmp_mode == GrB_SCMP);

  if (mask == NULL) {
    std::cout << "Unmasked SpVec Assign Constant\n";
    std::cout << "Error: Feature not implemented yet!\n";
    return GrB_SUCCESS;
  }

  Index w_nvals;
  w->nvals(&w_nvals);
  if (w_nvals == 0) return GrB_SUCCESS;

  Storage mask_vec_type;
  CHECK(mask->getStorage(&mask_vec_type));
  if (mask_vec_type == GrB_SPARSE) {
    CHECK(mask->convert(static_cast<M>(0), 0.3, desc));
    CHECK(mask->getStorage(&mask_vec_type));
  }
  if (mask_vec_type != GrB_DENSE) {
    std::cout << "SpVec Assign Constant Sparse Mask\n";
    std::cout << "Error: Feature not implemented yet!\n";
    return GrB_SUCCESS;
  }

  Index* tmp_ind = reinterpret_cast<Index*>(desc->scratch(GB_SCRATCH_VEC_A,
      static_cast<size_t>(w_nvals)*sizeof(Index)));
  W* tmp_val = reinterpret_cast<W*>(desc->scratch(GB_SCRATCH_VEC_B,
      static_cast<size_t>(w_nvals)*sizeof(W)));

  Index kept;
  if (use_scmp) {
    SparseAssignFilterSource<W, M, true> src;
    src.in_ind = w->d_ind_; src.in_val = w->d_val_;
    src.mask = mask->dense_.d_val_; src.val = static_cast<W>(val);
    src.out_ind = tmp_ind; src.out_val = tmp_val;
    kept = compactOrdered(src, w_nvals, desc);
  } else {
    SparseAssignFilterSource<W, M, false> src;
    src.in_ind = w->d_ind_; src.in_val = w->d_val_;
    src.mask = mask->dense_.d_val_; src.val = static_cast<W>(val);
    src.out_ind = tmp_ind; src.out_val = tmp_val;
    kept = compactOrdered(src, w_nvals, desc);
  }

  if (kept > 0) {
    cudaStream_t s = gbStream();
    CUDA_CALL(cudaMemcpyAsync(w->d_ind_, tmp_ind, kept*sizeof(Index),
        cudaMemcpyDeviceToDevice, s));
    CUDA_CALL(cudaMemcpyAsync(w->d_val_, tmp_val, kept*sizeof(W),
        cudaMemcpyDeviceToDevice, s));
  }
  w->computed(kept);
  return GrB_SUCCESS;
}
}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_ASSIGN_HPP_
