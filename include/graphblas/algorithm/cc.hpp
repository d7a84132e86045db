// graphblast_b200 — connected components on the device.
//
// v[i] = the smallest vertex id in the weakly connected component of i, over the graph
// of A's pattern: i and j are joined when A(i,j) or A(j,i) is stored (stored zeros
// count, self-loops are ignored, values are never read; FP32 and INT32 A).
// *ncomponents = the number of components, the number of i with v[i] == i.  The result
// depends only on A's pattern: not on launch shape, timing or any seed, so there is no
// seed parameter.  Only A's CSR is read, so a non-symmetric A needs no CSC.  v becomes
// dense with nrows(A) entries and is overwritten completely; an A with no stored
// entries gives v[i] = i and n components, and n = 0 gives 0 components.  The whole
// computation is one cooperative union-find kernel (Afforest,
// backend/cuda/kernels/cc.cuh).  A float v holds ids exactly only up to 2^24, so
// nrows(A) > 2^24 + 1 is refused with GrB_INVALID_VALUE.  Returns the device time in
// milliseconds ("tight"), or -1 with the failing status in algorithm::lastStatus().
// The reference's cc (algorithm/cc.hpp) runs FastSV as a loop of operations with a
// host round trip per iteration; it is not restated, and its fixed point (each
// component's minimum id) is this result.
#ifndef GRAPHBLAS_ALGORITHM_CC_HPP_
#define GRAPHBLAS_ALGORITHM_CC_HPP_

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

template <typename a>
float cc(Vector<float>* v, const Matrix<a>* A, Descriptor* desc, int* ncomponents) {
  if (v == NULL || A == NULL || desc == NULL) GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  int count = 0;
  float ms = 0.f;
  GB_ALGO_STEP(backend::ccRun(&v->vector_, &A->matrix_, &count, &ms));
  if (ncomponents != NULL) *ncomponents = count;
  if (desc->descriptor_.timing_ > 0)
    std::cout << "cc, " << count << " components, " << ms << "\n";
  return ms;
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_CC_HPP_
