// graphblast_b200 backend — host side of connected components (kernels/cc.cuh): the
// input (graph_input.hpp), the scratch and one cooperative launch.  algorithm::cc comes
// here.
#ifndef GRAPHBLAS_BACKEND_CUDA_CC_HPP_
#define GRAPHBLAS_BACKEND_CUDA_CC_HPP_

#include <type_traits>

#include "graphblas/backend/cuda/graph_input.hpp"
#include "graphblas/backend/cuda/kernels/cc.cuh"

namespace graphblas {
namespace backend {

// v[i] = the smallest vertex id in the weakly connected component of i in A's pattern
// (i and j joined when A(i,j) or A(j,i) is stored; self-loops ignored); *ncomponents
// (when not NULL) = the number of components, 0 when A has no rows; *ms (when not NULL)
// = the device time, from CUDA events.  v becomes dense with nrows(A) entries and is
// overwritten completely, whatever it held.  Only A's CSR is read.  A symmetric A (one
// with symmetric_ set, or whose CSC aliases its CSR) lets the kernel skip the largest
// sampled component in its last phase; any other A is read without the skip.
// Refusals, before v is touched: those of graphCheck (no CSC needed), then a float v
// with nrows(A) > 2^24 + 1, where a float can no longer hold every vertex id exactly
// (GrB_INVALID_VALUE).
// Scratch: the counter cells, then the n-word parent array followed by nnz /
// GB_CC_GRID_MIN + 1 words for the rows of the grid pass (no more rows than that can
// hold GB_CC_GRID_MIN entries).
template <typename W, typename a>
Info ccRun(Vector<W>* v, const Matrix<a>* A, int* ncomponents, float* ms = NULL) {
  static_assert(std::is_same<W, int>::value || std::is_same<W, float>::value,
                "cc writes int or float vectors");
  CHECK(graphCheck("cc", A, false, v));
  const SparseMatrix<a>& S = A->sparse_;
  const Index n = S.nrows_;
  if (std::is_same<W, float>::value && n > (1 << 24) + 1) return GrB_INVALID_VALUE;

  GpuTimer clock;
  clock.Start();
  if (ncomponents != NULL) *ncomponents = 0;
  CHECK(v->setStorage(GrB_DENSE));
  if (n == 0) {
    clock.Stop();
    if (ms != NULL) *ms = clock.ElapsedMillis();
    return GrB_SUCCESS;
  }
  CHECK(v->dense_.allocateGpu());
  const GraphPattern g(S, NULL);       // row_ptr NULL: no stored entries
  const size_t queued_words = (g.stored() ? static_cast<size_t>(S.nvals_)/GB_CC_GRID_MIN : 0)
                              + 1;
  ScratchLayout l;
  const size_t counters = l.place(CC_NCELLS*sizeof(unsigned long long));
  const size_t parent = l.place((static_cast<size_t>(n) + queued_words)*sizeof(Index));
  const DeviceBlock block(gbMalloc(l.bytes));
  CcArgs args;
  args.n = n;
  args.row_ptr = g.row_ptr;
  args.row_ind = g.row_ind;
  args.skip = S.sameStructure() ? 1 : 0;
  args.counters = block.at<unsigned long long>(counters);
  args.parent = block.at<Index>(parent);
  args.queued = args.parent + n;
  cudaStream_t stream = gbStream();
  CUDA_CALL(cudaMemsetAsync(args.counters, 0, CC_NCELLS*sizeof(unsigned long long), stream));
  CHECK((launchCooperative<ccKernel<W>, GB_CC_NT>(stream, args, v->dense_.d_val_)));
  clock.Stop();
  v->dense_.touched();
  if (ncomponents != NULL)
    *ncomponents = static_cast<int>(runtime().fetch(args.counters + CC_COMPONENTS));
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_CC_HPP_
