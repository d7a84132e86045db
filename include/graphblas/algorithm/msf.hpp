// graphblast_b200 — minimum spanning forest on the device.
//
// Graph.  The undirected graph G with the edge {i, j}, i != j, when A(i,j) or A(j,i) is
// stored.  Its weight w({i,j}) is the smaller of the stored values among A(i,j) and
// A(j,i), so a non-symmetric A, or a symmetric pattern with unequal values, is well
// defined.  Self-loops are ignored; stored zeros are edges of weight 0 (scipy treats
// explicit zeros as missing).  Only A's CSR is read, so a non-symmetric A needs no CSC.
// Column lists must be sorted and free of duplicates, as the library's builds, loads and
// ingest leave them.
// Order.  Edges are ranked by the key (w, min(i,j), max(i,j)).  Weights compare as
// numbers, -0.0 equal to +0.0, ±inf allowed; INT32 weights compare as signed integers.
// This is a strict total order, so the minimum spanning forest is unique: F is Kruskal's
// forest under this order, whatever the scheduling.
// Output.  F is n x n, replaced, and holds both directions of every forest edge: F(i,j) =
// F(j,i) = w({i,j}), -0.0 written as +0.0.  F is a sorted CSR installed as structurally
// symmetric (replaceDevice(..., symmetric = true)), so cc, gc, mis and lgc take their
// symmetric paths on it.  F has A's element type and may be A.  Two calls give identical
// bytes.  *nedges = the undirected forest edges (n minus the number of trees); *weight =
// their sum in fp64, taken in an order that depends only on the forest, so two calls give
// identical bits; it is exact while every partial sum is an integer below 2^53.  An A
// with no stored off-diagonal entry gives an empty F, 0 edges and weight 0; n = 0 too.
//
// Borůvka rounds as one cooperative kernel over cc's union-find
// (backend/cuda/kernels/msf.cuh).  Refusals, F untouched: NULL F, A or desc
// (GrB_UNINITIALIZED_OBJECT); a dense A (GrB_NOT_IMPLEMENTED); A not square or F not n x n
// (GrB_DIMENSION_MISMATCH); an A with entries but no device CSR
// (GrB_UNINITIALIZED_OBJECT); an FP32 A with a NaN on a stored off-diagonal entry
// (GrB_INVALID_VALUE).  Returns the device time in milliseconds ("tight"), or -1 with the
// failing status in algorithm::lastStatus().  The reference has no spanning forest.
#ifndef GRAPHBLAS_ALGORITHM_MSF_HPP_
#define GRAPHBLAS_ALGORITHM_MSF_HPP_

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

template <typename T>
float msf(Matrix<T>* F, const Matrix<T>* A, Descriptor* desc, Index* nedges,
          double* weight) {
  if (F == NULL || A == NULL || desc == NULL) GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  long long count = 0;
  double total = 0.0;
  float ms = 0.f;
  GB_ALGO_STEP(backend::msfRun(&F->matrix_, &A->matrix_, &count, &total, &ms));
  if (nedges != NULL) *nedges = static_cast<Index>(count);
  if (weight != NULL) *weight = total;
  if (desc->descriptor_.timing_ > 0)
    std::cout << "msf, " << count << " edges, weight " << total << ", "
              << backend::lastStats<backend::MsfStats>().rounds << " rounds, " << ms << "\n";
  return ms;
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_MSF_HPP_
