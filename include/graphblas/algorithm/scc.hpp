// graphblast_b200 — strongly connected components on the device.
//
// v[i] = the smallest vertex id in the strongly connected component of i, over the
// arcs i -> j with A(i,j) stored and i != j (stored zeros count, self-loops are
// ignored, values are never read; FP32 and INT32 A).  *ncomponents = the number of
// components, the number of i with v[i] == i.  The result depends only on A's pattern:
// not on launch shape, timing or any seed, so there is no seed parameter.  Out-lists
// come from A's CSR and in-lists from its CSC, so a non-symmetric A needs its CSC.  An A
// marked symmetric, or whose CSC aliases its CSR, has the connected components of its
// pattern as its strong components, and backend::ccRun computes them.  Otherwise the
// whole computation is one cooperative kernel: trim, forward–backward from a pivot,
// then colouring (backend/cuda/kernels/scc.cuh).  v becomes dense with nrows(A)
// entries and is overwritten completely; an A with no stored entries gives v[i] = i
// and n components, and n = 0 gives 0 components.  A float v holds ids exactly only up
// to 2^24, so nrows(A) > 2^24 + 1 is refused with GrB_INVALID_VALUE.  The other
// refusals, v untouched: NULL v, A or desc (GrB_UNINITIALIZED_OBJECT); a dense A
// (GrB_NOT_IMPLEMENTED); A not square or v not of size nrows(A)
// (GrB_DIMENSION_MISMATCH); a missing CSR, or a missing CSC on a non-symmetric A
// (GrB_UNINITIALIZED_OBJECT).  Returns the device time in milliseconds ("tight"), or -1
// with the failing status in algorithm::lastStatus().  The reference has no strongly
// connected components.
#ifndef GRAPHBLAS_ALGORITHM_SCC_HPP_
#define GRAPHBLAS_ALGORITHM_SCC_HPP_

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

template <typename a>
float scc(Vector<float>* v, const Matrix<a>* A, Descriptor* desc, int* ncomponents) {
  if (v == NULL || A == NULL || desc == NULL) GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  int count = 0;
  float ms = 0.f;
  GB_ALGO_STEP(backend::sccRun(&v->vector_, &A->matrix_, &count, &ms));
  if (ncomponents != NULL) *ncomponents = count;
  if (desc->descriptor_.timing_ > 0) {
    const backend::SccStats& stats = backend::lastStats<backend::SccStats>();
    std::cout << "scc, " << count << " components, " << stats.trimmed << " trimmed, "
              << stats.colour_iterations << " colourings, " << ms << "\n";
  }
  return ms;
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_SCC_HPP_
