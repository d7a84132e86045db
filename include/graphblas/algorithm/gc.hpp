// graphblast_b200 — graph colouring: greedy Jones–Plassmann on the device.
//
// v[i] = colour of vertex i (1-based) in the undirected graph of A's pattern
// (i and j conflict when A(i,j) or A(j,i) is stored, i != j; self-loops are ignored).
// The colouring is sequential greedy first-fit in decreasing priority order, the
// priority of vertex i being (hash(seed, i), i) with the hash of
// backend/cuda/kernels/greedy_schedule.cuh, so it depends on seed and A only.  The whole
// colouring is one cooperative kernel (backend/cuda/color.hpp); *ncolors = the
// largest colour (0 for an empty graph).  A non-symmetric A is read through its CSR
// and its CSC and needs both on the device.
// Returns the device time of the colouring in milliseconds ("tight"), or -1 with the
// failing status in algorithm::lastStatus().  The reference builds its colourings
// from many small operations per round (algorithm/gc.hpp gcJP / gcIS / gcMIS); those
// are not restated.
#ifndef GRAPHBLAS_ALGORITHM_GC_HPP_
#define GRAPHBLAS_ALGORITHM_GC_HPP_

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

template <typename a>
float gc(Vector<float>* v, const Matrix<a>* A, int seed, Descriptor* desc, int* ncolors) {
  if (v == NULL || A == NULL || desc == NULL) GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  int count = 0;
  float ms = 0.f;
  GB_ALGO_STEP(backend::graphColorRun(&v->vector_, &A->matrix_,
                                      static_cast<unsigned int>(seed), &count, &ms));
  if (ncolors != NULL) *ncolors = count;
  if (desc->descriptor_.timing_ > 0)
    std::cout << "gc, " << count << " colours, " << ms << "\n";
  return ms;
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_GC_HPP_
