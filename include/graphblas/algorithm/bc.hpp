// graphblast_b200 — betweenness centrality on the device.
//
// Graph.  Each stored entry A(i,j) with i != j is a directed edge i -> j.  Self-loops are
// ignored, and values are ignored (unweighted BC).  FP32 and INT32 A give the same
// result.  A symmetric A is therefore the undirected graph, with each edge in both
// directions.  A non-symmetric A needs its CSC (the path counts are pulled over
// in-lists).
// Sources.  A host list S of vertex ids.  Each listed entry contributes once, so a
// repeated id counts twice.  A NULL list means every vertex 0..n-1, which is exact BC.
// Result.  bc[v] = sum over s in S, over t not in {s, v} reachable from s, of
// sigma_st(v) / sigma_st, sigma_st the number of shortest s -> t paths and sigma_st(v)
// the number that pass through v.  There is no normalisation and no halving.  For a
// symmetric A with all sources this is exactly 2x networkx's undirected unnormalised
// value, and it equals networkx.betweenness_centrality(DiGraph, normalized=False).
// Output vector.  v becomes dense with nrows(A) entries of float.  A vertex that lies on
// no counted path gets exactly 0.
// Precision.  sigma and the dependencies delta are fp64 on the device, and the sum over
// sources is accumulated in fp64.  The result is rounded to float once, at the end.
// Determinism.  No floating-point value goes through an atomic.  Every sum runs in a
// fixed order, which is list order within a list and a fixed tree across lanes and
// chunks.  Two calls therefore give identical bytes.
//
// The sources run in batches of 32, one cooperative kernel each (a Brandes traversal in
// the multi-source BFS style, backend/cuda/kernels/bc.cuh), and one finish kernel.
// Refusals, v untouched: NULL v, A or desc (GrB_UNINITIALIZED_OBJECT); nsources < 0
// (GrB_INVALID_VALUE); a NULL list whose count is not n, or an id outside [0, n)
// (GrB_INVALID_INDEX); then those of backend::graphCheck (a dense A, then sizes, then a
// missing CSR or CSC); a batch whose level lists could pass 2^31 - 1 entries
// (GrB_OUT_OF_MEMORY).  nsources == 0 with a non-NULL list gives all zeros.  Returns the
// device time in milliseconds ("tight"), or -1 with the failing status in
// algorithm::lastStatus().
#ifndef GRAPHBLAS_ALGORITHM_BC_HPP_
#define GRAPHBLAS_ALGORITHM_BC_HPP_

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

// A NULL list of n entries, or nsources ids in [0, n).
inline bool bcSourcesValid(const Index* sources, Index nsources, Index n) {
  if (sources == NULL) return nsources == n;
  for (Index i = 0; i < nsources; ++i)
    if (sources[i] < 0 || sources[i] >= n) return false;
  return true;
}

template <typename a>
float bc(Vector<float>* v, const Matrix<a>* A, const Index* sources, Index nsources,
         Descriptor* desc) {
  if (v == NULL || A == NULL || desc == NULL) GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  if (nsources < 0) GB_ALGO_STEP(GrB_INVALID_VALUE);
  Index n = 0;
  GB_ALGO_STEP(A->nrows(&n));
  if (!bcSourcesValid(sources, nsources, n)) GB_ALGO_STEP(GrB_INVALID_INDEX);
  float ms = 0.f;
  GB_ALGO_STEP(backend::bcRun(&v->vector_, &A->matrix_, sources, nsources, &ms));
  if (desc->descriptor_.timing_ > 0)
    std::cout << "bc, " << nsources << " sources, " << ms << "\n";
  return ms;
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_BC_HPP_
