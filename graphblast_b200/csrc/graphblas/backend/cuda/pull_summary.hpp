// graphblast_b200 backend — per-structure summaries the Boolean pull reads instead
// of the row offsets: first neighbour (or, for the fused BFS, highest-degree
// neighbour) of every row, and the bitmap of empty rows.
// Built once per traversed structure and kept with the matrix (dropped with the
// other derived caches whenever the structure changes).
#ifndef GRAPHBLAS_BACKEND_CUDA_PULL_SUMMARY_HPP_
#define GRAPHBLAS_BACKEND_CUDA_PULL_SUMMARY_HPP_

namespace graphblas {
namespace backend {

// One summary of nrows + 1 words with the bitmap of empty rows behind it
// (pullEmptyRowBits), cached in `slot` under the pointer array and entry count it is
// built from: fill(out) launches the kernel that writes the words.
template <typename Fill>
const Index* pullSummary(DerivedArray* slot, const Index* ptr, Index nvals, Index nrows,
                         Fill fill) {
  if (!slot->validFor(ptr, nvals)) {
    const size_t nwords = (static_cast<size_t>(nrows) + 31)/32;
    Index* out = slot->rebuild(static_cast<size_t>(nrows) + 1 + nwords, ptr, nvals);
    fill(out);
    GB_KERNEL_CHECK();
    pullEmptyRowBitsKernel<<<gridFor(nrows, 256, 8), 256, 0, gbStream()>>>(
        reinterpret_cast<unsigned int*>(out + nrows + 1), out, nrows);
    GB_KERNEL_CHECK();
  }
  return slot->d;
}

// first[i] as pullFirstNeighbourKernel defines it.  side: 0 = the CSR arrays are
// pulled, 1 = the CSC arrays.
template <typename T>
const Index* pullFirstNeighbours(SparseMatrix<T>* S, int side, const Index* ptr,
                                 const Index* ind, Index nrows) {
  return pullSummary(&S->pull_first_[side], ptr, S->nvals_, nrows, [&](Index* out) {
    pullFirstNeighbourKernel<<<gridFor(nrows, 256, 8), 256, 0, gbStream()>>>(
        out, ptr, ind, nrows);
  });
}

// probe[i] as pullMaxDegreeNeighbourKernel defines it (the fused BFS probes it: the
// highest-degree neighbour is the one most likely to be visited).  Cached beside the
// first-neighbour summary, under the same key.
template <typename T>
const Index* pullMaxDegreeNeighbours(SparseMatrix<T>* S, int side, const Index* ptr,
                                     const Index* ind, Index nrows) {
  return pullSummary(&S->pull_maxdeg_[side], ptr, S->nvals_, nrows, [&](Index* out) {
    pullMaxDegreeNeighbourKernel<<<gridFor(static_cast<size_t>(nrows)*32, 256, 8), 256, 0,
                                   gbStream()>>>(out, ptr, ind, nrows);
  });
}

inline const unsigned int* pullEmptyRowBits(const Index* first, Index nrows) {
  return reinterpret_cast<const unsigned int*>(first + nrows + 1);
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_PULL_SUMMARY_HPP_
