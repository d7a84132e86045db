// graphblast_b200 — k-truss and truss decomposition on the device.
//
// Graph.  The undirected simple graph G of A's pattern: G has the edge {i, j}, i != j,
// when A(i,j) or A(j,i) is stored.  Values and self-loops are ignored, so FP32 and INT32
// A give the same result.  Column lists must be sorted and free of duplicates, as the
// library's builds, loads and ingest leave them.  A non-symmetric A needs its CSC.
// k-truss.  ktruss(C, A, k), k >= 2: starting from G, every edge that lies in fewer
// than k - 2 triangles of the remaining graph is deleted, again and again, until none
// is left to delete.  C(i,j) = C(j,i) = the number of triangles of that k-truss that
// contain {i, j}, at least k - 2 on every stored entry.  With k = 2 every edge stays and
// C(i,j) is its triangle count in G.  *nedges = the undirected edges kept.
// Truss decomposition.  trussness(T, A): T has G's pattern in both directions, and
// T(i,j) = T(j,i) = tau({i, j}), the largest k whose k-truss contains the edge (2 for an
// edge in no triangle).  *kmax = the largest tau, or 0 when G has no edge.
// Output.  C and T are n x n, sorted CSR, replaced, and installed as structurally
// symmetric (replaceDevice(..., symmetric = true)), so cc, gc, mis and lgc take their
// symmetric paths on them.  Each is FP32 or INT32, independently of A, and may be A.
// The values are integers computed with integer atomics only, so every call gives
// identical bytes.
//
// The whole peel is one cooperative kernel with grid barriers between its rounds
// (backend/cuda/kernels/ktruss.cuh).  Refusals, the output untouched: NULL C, T, A or
// desc (GrB_UNINITIALIZED_OBJECT); k < 2 (GrB_INVALID_VALUE); a dense A
// (GrB_NOT_IMPLEMENTED); A not square or the output not n x n (GrB_DIMENSION_MISMATCH);
// a missing CSR, or a missing CSC on a non-symmetric A (GrB_UNINITIALIZED_OBJECT); an
// FP32 output with n > 2^24, where supports and tau would no longer be exact
// (GrB_INVALID_VALUE); a symmetrised pattern past 2^31 - 1 entries (GrB_OUT_OF_MEMORY).
// Returns the device time in milliseconds ("tight"), or -1 with the failing status in
// algorithm::lastStatus().
#ifndef GRAPHBLAS_ALGORITHM_KTRUSS_HPP_
#define GRAPHBLAS_ALGORITHM_KTRUSS_HPP_

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

template <typename T, typename a>
float ktruss(Matrix<T>* C, const Matrix<a>* A, int k, Descriptor* desc, Index* nedges) {
  if (C == NULL || A == NULL || desc == NULL) GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  if (k < 2) GB_ALGO_STEP(GrB_INVALID_VALUE);
  long long count = 0;
  float ms = 0.f;
  GB_ALGO_STEP(backend::ktrussRun(&C->matrix_, &A->matrix_, k, &count, &ms));
  if (nedges != NULL) *nedges = static_cast<Index>(count);
  if (desc->descriptor_.timing_ > 0)
    std::cout << "ktruss, k " << k << ", " << count << " edges, "
              << backend::lastStats<backend::KtrussStats>().rounds << " rounds, " << ms << "\n";
  return ms;
}

template <typename T, typename a>
float trussness(Matrix<T>* C, const Matrix<a>* A, Descriptor* desc, int* kmax) {
  if (C == NULL || A == NULL || desc == NULL) GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  long long count = 0;
  float ms = 0.f;
  GB_ALGO_STEP(backend::ktrussRun(&C->matrix_, &A->matrix_, 0, &count, &ms));
  if (kmax != NULL) *kmax = static_cast<int>(count);
  if (desc->descriptor_.timing_ > 0) {
    const backend::KtrussStats& stats = backend::lastStats<backend::KtrussStats>();
    std::cout << "trussness, kmax " << count << ", " << stats.levels << " levels, "
              << stats.rounds << " rounds, " << ms << "\n";
  }
  return ms;
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_KTRUSS_HPP_
