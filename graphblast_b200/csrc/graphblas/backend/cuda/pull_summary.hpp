// graphblast_b200 backend — per-structure summaries the Boolean pull reads instead
// of the row offsets: first neighbour (or, for the fused BFS, highest-degree
// neighbour) of every row, and the bitmap of empty rows.
// Built once per traversed structure and kept with the matrix (dropped with the
// other derived caches whenever the structure changes).
#ifndef GRAPHBLAS_BACKEND_CUDA_PULL_SUMMARY_HPP_
#define GRAPHBLAS_BACKEND_CUDA_PULL_SUMMARY_HPP_

namespace graphblas {
namespace backend {

// first[i] as pullFirstNeighbourKernel defines it; the empty-row bitmap follows the
// array (pullEmptyRowBits).  side: 0 = the CSR arrays are pulled, 1 = the CSC arrays.
template <typename T>
const Index* pullFirstNeighbours(SparseMatrix<T>* S, int side, const Index* ptr,
                                 const Index* ind, Index nrows) {
  if (S->d_pull_first_[side] == NULL || S->pull_first_key_[side] != ptr ||
      S->pull_first_nvals_[side] != S->nvals_) {
    if (S->d_pull_first_[side] != NULL) gbFree(S->d_pull_first_[side]);
    const size_t nwords = (static_cast<size_t>(nrows) + 31)/32;
    S->d_pull_first_[side] = reinterpret_cast<Index*>(
        gbMalloc((static_cast<size_t>(nrows) + 1 + nwords)*sizeof(Index)));
    cudaStream_t s = gbStream();
    pullFirstNeighbourKernel<<<gridFor(nrows, 256, 8), 256, 0, s>>>(
        S->d_pull_first_[side], ptr, ind, nrows);
    GB_KERNEL_CHECK();
    pullEmptyRowBitsKernel<<<gridFor(nrows, 256, 8), 256, 0, s>>>(
        reinterpret_cast<unsigned int*>(S->d_pull_first_[side] + nrows + 1),
        S->d_pull_first_[side], nrows);
    GB_KERNEL_CHECK();
    S->pull_first_key_[side] = ptr;
    S->pull_first_nvals_[side] = S->nvals_;
  }
  return S->d_pull_first_[side];
}

// probe[i] as pullMaxDegreeNeighbourKernel defines it (the fused BFS probes it: the
// highest-degree neighbour is the one most likely to be visited), the empty-row
// bitmap following it as above.  Cached beside the first-neighbour summary, under
// the same key.
template <typename T>
const Index* pullMaxDegreeNeighbours(SparseMatrix<T>* S, int side, const Index* ptr,
                                     const Index* ind, Index nrows) {
  if (S->d_pull_maxdeg_[side] == NULL || S->pull_maxdeg_key_[side] != ptr ||
      S->pull_maxdeg_nvals_[side] != S->nvals_) {
    if (S->d_pull_maxdeg_[side] != NULL) gbFree(S->d_pull_maxdeg_[side]);
    const size_t nwords = (static_cast<size_t>(nrows) + 31)/32;
    S->d_pull_maxdeg_[side] = reinterpret_cast<Index*>(
        gbMalloc((static_cast<size_t>(nrows) + 1 + nwords)*sizeof(Index)));
    cudaStream_t s = gbStream();
    pullMaxDegreeNeighbourKernel<<<gridFor(static_cast<size_t>(nrows)*32, 256, 8), 256, 0,
                                   s>>>(S->d_pull_maxdeg_[side], ptr, ind, nrows);
    GB_KERNEL_CHECK();
    pullEmptyRowBitsKernel<<<gridFor(nrows, 256, 8), 256, 0, s>>>(
        reinterpret_cast<unsigned int*>(S->d_pull_maxdeg_[side] + nrows + 1),
        S->d_pull_maxdeg_[side], nrows);
    GB_KERNEL_CHECK();
    S->pull_maxdeg_key_[side] = ptr;
    S->pull_maxdeg_nvals_[side] = S->nvals_;
  }
  return S->d_pull_maxdeg_[side];
}

inline const unsigned int* pullEmptyRowBits(const Index* first, Index nrows) {
  return reinterpret_cast<const unsigned int*>(first + nrows + 1);
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_PULL_SUMMARY_HPP_
