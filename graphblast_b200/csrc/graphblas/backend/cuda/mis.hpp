// graphblast_b200 backend — host side of the maximal independent set (kernels/mis.cuh):
// an init pass over the candidates, then one cooperative launch.  algorithm::mis comes
// here.
#ifndef GRAPHBLAS_BACKEND_CUDA_MIS_HPP_
#define GRAPHBLAS_BACKEND_CUDA_MIS_HPP_

#include <type_traits>

#include "graphblas/backend/cuda/greedy_schedule.hpp"
#include "graphblas/backend/cuda/kernels/mis.cuh"

namespace graphblas {
namespace backend {

// v[i] = 1 when vertex i of A's pattern is in the greedy maximal independent set in
// decreasing priority order over the candidates, else 0; *nmembers (when not NULL) =
// the size of the set; *ms (when not NULL) = the device time, from CUDA events.
// candidates == NULL: every vertex is a candidate.  Otherwise vertex i is one when the
// vector holds a non-zero value for it (a dense value, or a stored sparse entry).  The
// candidate vector is read in the storage it has, never converted, and read completely
// before v is written, so it may be v itself.
// Refusals, before v is touched: those of graphCheck (with the CSC) for v and the
// candidates, then candidates without device arrays (GrB_UNINITIALIZED_OBJECT).
template <typename W, typename a>
Info misRun(Vector<W>* v, const Matrix<a>* A, unsigned int seed,
            const Vector<W>* candidates, int* nmembers, float* ms = NULL) {
  static_assert(std::is_same<W, int>::value || std::is_same<W, float>::value,
                "mis writes int or float vectors");
  Vector<W>* cand = const_cast<Vector<W>*>(candidates);    // read only
  CHECK(graphCheck("mis", A, true, v, cand));
  const Index n = A->sparse_.nrows_;

  // the candidates as device arrays, in the storage they have
  const Storage cand_type = cand != NULL ? cand->vec_type_ : GrB_UNKNOWN;
  const W* cand_val = NULL;
  const Index* cand_ind = NULL;
  Index cand_nvals = 0;
  if (cand_type == GrB_DENSE && n > 0) {
    CHECK(cand->dense_.materialize());       // values from the bitmap, when only it is current
    cand_val = cand->dense_.d_val_;
    if (cand_val == NULL) return GrB_UNINITIALIZED_OBJECT;
  } else if (cand_type == GrB_SPARSE) {
    cand_nvals = cand->sparse_.nvals_;
    cand_ind = cand->sparse_.d_ind_;
    cand_val = cand->sparse_.d_val_;
    if (cand_nvals > 0 && (cand_ind == NULL || cand_val == NULL))
      return GrB_UNINITIALIZED_OBJECT;
  }

  // init pass: everything it reads of the candidates is read before v is written
  return greedyRun<W, misKernel<W>>(v, &A->sparse_, seed, nmembers, ms,
      [&](unsigned int* state, cudaStream_t stream) {
        const int nt = 256;
        if (cand == NULL) {
          CUDA_CALL(cudaMemsetAsync(state, 0, static_cast<size_t>(n)*sizeof(unsigned int),
                                    stream));
        } else if (cand_type == GrB_DENSE) {
          misInitDenseKernel<W><<<gridFor(n, nt), nt, 0, stream>>>(state, cand_val, n);
          GB_KERNEL_CHECK();
        } else {                       // sparse, or no storage: only stored non-zeros count
          fillKernel<unsigned int><<<gridFor(n, nt), nt, 0, stream>>>(state, MIS_OUT, n);
          GB_KERNEL_CHECK();
          if (cand_nvals > 0) {
            misInitSparseKernel<W><<<gridFor(cand_nvals, nt), nt, 0, stream>>>(
                state, cand_ind, cand_val, cand_nvals, n);
            GB_KERNEL_CHECK();
          }
        }
      });
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_MIS_HPP_
