// graphblast_b200 — community detection by label propagation on the device (LDBC
// Graphalytics CDLP, vertex ids 0..n-1 as the initial labels).
//
// Graph.  The arc i -> j when A(i,j) is stored and i != j.  Values are never read and
// stored zeros count, so FP32 and INT32 A give the same result; self-loops are ignored.
// Iterations.  L_0(v) = v.  Iteration k is synchronous: M(v) = the labels L_{k-1}(u) of
// v's out-neighbours (row v of the CSR) and of its in-neighbours (column v of the CSC),
// an arc stored both ways counted twice; L_k(v) = the smallest label of highest
// multiplicity in M(v), and a vertex whose M(v) is empty keeps its label.  An A marked
// symmetric, or whose CSC aliases its CSR, is read through its CSR alone: both lists
// hold the same multiset, so every multiplicity doubles and the answer is the same.
// max_iter >= 0 iterations are defined.  The kernel stops after the first iteration
// that changes no label, a fixpoint, so the result equals max_iter iterations exactly;
// *iterations = the iterations run, including the one that changed nothing, and
// max_iter = 0 gives v[i] = i.  Synchronous label propagation can oscillate (a star
// alternates with period 2): the iteration count is what makes the result well defined.
// Result.  v becomes dense with nrows(A) entries and is overwritten completely; v[i] =
// L_T(i).  *ncommunities = the number of distinct labels.  Two calls give identical
// bytes.
//
// One cooperative kernel runs every iteration (backend/cuda/kernels/cdlp.cuh): lists of
// at most 32 entries are packed several to a warp and counted with __match_any_sync,
// lists of at most 128 entries are counted in a warp's shared hash table, and longer
// lists are cut into label partitions of about 2048 entries, each (vertex, partition)
// pair a work item of the whole grid.  Scratch: 6 n + n / 32 + 1 words and the counter
// cells (n + 1 more when A stores no entry), none proportional to nnz.
// Refusals, in this order, v untouched: NULL v, A or desc (GrB_UNINITIALIZED_OBJECT); a
// dense A (GrB_NOT_IMPLEMENTED); A not square or v not of size nrows(A)
// (GrB_DIMENSION_MISMATCH); a missing CSR, or a non-symmetric A without its CSC
// (GrB_UNINITIALIZED_OBJECT); nrows(A) > 2^24 + 1, where a float v can no longer hold
// every id exactly (GrB_INVALID_VALUE); max_iter < 0 (GrB_INVALID_VALUE).  Returns the
// device time in milliseconds ("tight"), or -1 with the failing status in
// algorithm::lastStatus().  The reference has no label propagation.
#ifndef GRAPHBLAS_ALGORITHM_CDLP_HPP_
#define GRAPHBLAS_ALGORITHM_CDLP_HPP_

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

template <typename a>
float cdlp(Vector<float>* v, const Matrix<a>* A, int max_iter, Descriptor* desc,
           int* ncommunities, int* iterations) {
  if (v == NULL || A == NULL || desc == NULL) GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  int count = 0, iters = 0;
  float ms = 0.f;
  GB_ALGO_STEP(backend::cdlpRun(&v->vector_, &A->matrix_, max_iter, &count, &iters, &ms));
  if (ncommunities != NULL) *ncommunities = count;
  if (iterations != NULL) *iterations = iters;
  if (desc->descriptor_.timing_ > 0) {
    const backend::CdlpStats& stats = backend::lastStats<backend::CdlpStats>();
    std::cout << "cdlp, " << count << " communities, " << iters << " iterations, "
              << stats.long_items << " long items, " << ms << "\n";
  }
  return ms;
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_CDLP_HPP_
