// graphblast_b200 — maximal independent set on the device.
//
// v[i] = 1 when vertex i is in the set, else 0, over the undirected graph of A's pattern
// (i and j conflict when A(i,j) or A(j,i) is stored, i != j; self-loops are ignored).
// The set is the sequential greedy MIS in decreasing priority order over the
// candidates: i joins iff no higher-priority candidate neighbour joined, the priority
// of i being (hash(seed, i), i) with the hash of backend/cuda/kernels/color.cuh, so it
// depends on A, seed and the candidates only.  With no candidate vector it equals
// colour class 1 of algorithm::gc with the same seed.  candidates (may be NULL: every
// vertex) makes vertex i a candidate when it holds a non-zero value for i, in the
// storage it has; it is never converted and may be v itself.  The whole set is one
// cooperative kernel after an init pass (backend/cuda/mis.hpp); *nmembers = its size.
// A non-symmetric A is read through its CSR and its CSC and needs both on the device.
// Returns the device time in milliseconds ("tight"), or -1 with the failing status in
// algorithm::lastStatus().  The reference's mis / misInner (algorithm/mis.hpp) run
// Luby rounds as many small operations with random weights; they are not restated.
#ifndef GRAPHBLAS_ALGORITHM_MIS_HPP_
#define GRAPHBLAS_ALGORITHM_MIS_HPP_

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

template <typename a>
float mis(Vector<float>* v, const Matrix<a>* A, int seed, Descriptor* desc, int* nmembers,
          const Vector<float>* candidates = NULL) {
  if (v == NULL || A == NULL || desc == NULL) GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  int count = 0;
  float ms = 0.f;
  GB_ALGO_STEP(backend::misRun(&v->vector_, &A->matrix_, static_cast<unsigned int>(seed),
                               candidates != NULL ? &candidates->vector_ : NULL,
                               &count, &ms));
  if (nmembers != NULL) *nmembers = count;
  if (desc->descriptor_.timing_ > 0)
    std::cout << "mis, " << count << " members, " << ms << "\n";
  return ms;
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_MIS_HPP_
