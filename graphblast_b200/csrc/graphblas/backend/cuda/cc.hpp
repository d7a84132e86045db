// graphblast_b200 backend — host side of connected components (kernels/cc.cuh): the
// refusals, the scratch and one cooperative launch.  algorithm::cc comes here.
#ifndef GRAPHBLAS_BACKEND_CUDA_CC_HPP_
#define GRAPHBLAS_BACKEND_CUDA_CC_HPP_

#include <type_traits>

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
// Every refusal comes before v is touched: a dense A (GrB_NOT_IMPLEMENTED); A not
// square or v not of size nrows(A) (GrB_DIMENSION_MISMATCH); an A with stored entries
// but no device CSR (GrB_UNINITIALIZED_OBJECT); a float v with nrows(A) > 2^24 + 1,
// where a float can no longer hold every vertex id exactly (GrB_INVALID_VALUE).
// Scratch: 256 bytes of counters, the n-word parent array and nnz / GB_CC_GRID_MIN + 1
// words for the rows of the grid pass (no more rows than that can hold GB_CC_GRID_MIN
// entries), freed after the launch.
template <typename W, typename a>
Info ccRun(Vector<W>* v, const Matrix<a>* A, int* ncomponents, float* ms = NULL) {
  static_assert(std::is_same<W, int>::value || std::is_same<W, float>::value,
                "cc writes int or float vectors");
  if (!A->isSparse()) {
    std::cout << "Error: cc of a dense matrix is not implemented in this backend\n";
    return GrB_NOT_IMPLEMENTED;
  }
  const SparseMatrix<a>* S = &A->sparse_;
  const Index n = S->nrows_;
  if (n != S->ncols_) return GrB_DIMENSION_MISMATCH;
  Index vsize = 0;
  CHECK(v->size(&vsize));
  if (vsize != n) return GrB_DIMENSION_MISMATCH;
  const bool stored = n > 0 && S->nvals_ > 0;
  if (stored && (S->d_csrRowPtr_ == NULL || S->d_csrColInd_ == NULL))
    return GrB_UNINITIALIZED_OBJECT;
  if (std::is_same<W, float>::value && n > (1 << 24) + 1) return GrB_INVALID_VALUE;

  GpuTimer clock;
  clock.Start();
  if (ncomponents != NULL) *ncomponents = 0;
  if (n == 0) {
    CHECK(v->setStorage(GrB_DENSE));
    clock.Stop();
    if (ms != NULL) *ms = clock.ElapsedMillis();
    return GrB_SUCCESS;
  }
  const int grid = cooperativeGrid<ccKernel<W>, GB_CC_NT>();
  if (grid < 1) return GrB_PANIC;
  cudaStream_t stream = gbStream();

  CHECK(v->setStorage(GrB_DENSE));     // before the scratch, so a failure leaks nothing
  CHECK(v->dense_.allocateGpu());
  W* out = v->dense_.d_val_;
  const size_t queued_words = (stored ? static_cast<size_t>(S->nvals_)/GB_CC_GRID_MIN : 0) + 1;
  unsigned char* block = static_cast<unsigned char*>(gbMalloc(
      256 + (static_cast<size_t>(n) + queued_words)*sizeof(Index)));
  CcArgs args;
  args.n = n;
  args.row_ptr = stored ? S->d_csrRowPtr_ : NULL;
  args.row_ind = stored ? S->d_csrColInd_ : NULL;
  args.skip = S->sameStructure() ? 1 : 0;
  args.counters = reinterpret_cast<unsigned long long*>(block);
  args.parent = reinterpret_cast<Index*>(block + 256);
  args.queued = args.parent + n;
  CUDA_CALL(cudaMemsetAsync(block, 0, 3*sizeof(unsigned long long), stream));

  void* params[] = { &args, &out };
  CUDA_CALL(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(ccKernel<W>),
      dim3(grid), dim3(GB_CC_NT), params, 0, stream));
  GB_KERNEL_CHECK();
  clock.Stop();
  v->dense_.touched();
  if (ncomponents != NULL)
    *ncomponents = static_cast<int>(runtime().fetch(args.counters + 1));
  gbFree(block);
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_CC_HPP_
