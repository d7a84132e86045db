// graphblast_b200 backend — host side of the graph colouring (kernels/color.cuh): one
// cooperative launch per colouring.  backend::graphColor (seed 0) and algorithm::gc
// (any seed, reports the colour count) both come here.
#ifndef GRAPHBLAS_BACKEND_CUDA_COLOR_HPP_
#define GRAPHBLAS_BACKEND_CUDA_COLOR_HPP_

#include <type_traits>

#include "graphblas/backend/cuda/greedy_schedule.hpp"
#include "graphblas/backend/cuda/kernels/color.cuh"

namespace graphblas {
namespace backend {

// v[i] = colour of vertex i of A's pattern (1-based), greedy first-fit in decreasing
// priority order; *ncolors (when not NULL) = the largest colour, 0 when A has no rows;
// *ms (when not NULL) = the device time of the colouring, from CUDA events.
// Every refusal comes before v is touched: A not square or v not of size nrows(A)
// (GrB_DIMENSION_MISMATCH), a dense A (GrB_NOT_IMPLEMENTED), an A without a device CSR,
// or a non-symmetric A without a device CSC (GrB_UNINITIALIZED_OBJECT).
template <typename W, typename a>
Info graphColorRun(Vector<W>* v, const Matrix<a>* A, unsigned int seed, int* ncolors,
                   float* ms = NULL) {
  static_assert(std::is_same<W, int>::value || std::is_same<W, float>::value,
                "graphColor writes int or float colours");
  const Info refused = greedyCheck("graphColor", v, A, static_cast<Vector<W>*>(NULL));
  if (refused != GrB_SUCCESS) return refused;
  const Index n = A->sparse_.nrows_;
  return greedyRun<W, graphColorKernel<W>>(v, &A->sparse_, seed, ncolors, ms,
      [n](unsigned int* colour, cudaStream_t stream) {          // 0 = uncoloured
        CUDA_CALL(cudaMemsetAsync(colour, 0, static_cast<size_t>(n)*sizeof(unsigned int),
                                  stream));
      });
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_COLOR_HPP_
