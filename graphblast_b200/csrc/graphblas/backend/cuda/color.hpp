// graphblast_b200 backend — host side of the graph colouring (kernels/color.cuh): one
// cooperative launch per colouring.  backend::graphColor (seed 0) and algorithm::gc
// (any seed, reports the colour count) both come here.
#ifndef GRAPHBLAS_BACKEND_CUDA_COLOR_HPP_
#define GRAPHBLAS_BACKEND_CUDA_COLOR_HPP_

#include <type_traits>

#include "graphblas/backend/cuda/kernels/color.cuh"

namespace graphblas {
namespace backend {

// v[i] = colour of vertex i of A's pattern (1-based), greedy first-fit in decreasing
// priority order; *ncolors (when not NULL) = the largest colour, 0 when A has no rows;
// *ms (when not NULL) = the device time of the colouring, from CUDA events.
// Every refusal comes before v is touched: A not square or v not of size nrows(A)
// (GrB_DIMENSION_MISMATCH), a dense A (GrB_NOT_IMPLEMENTED), an A without a device CSR,
// or a non-symmetric A without a device CSC (GrB_UNINITIALIZED_OBJECT).
template <typename W, typename a>
Info graphColorRun(Vector<W>* v, const Matrix<a>* A, unsigned int seed, int* ncolors,
                   float* ms = NULL) {
  static_assert(std::is_same<W, int>::value || std::is_same<W, float>::value,
                "graphColor writes int or float colours");
  if (!A->isSparse()) {
    std::cout << "Error: graphColor of a dense matrix is not implemented in this backend\n";
    return GrB_NOT_IMPLEMENTED;
  }
  const SparseMatrix<a>* S = &A->sparse_;
  const Index n = S->nrows_;
  if (n != S->ncols_) return GrB_DIMENSION_MISMATCH;
  Index vsize = 0;
  CHECK(v->size(&vsize));
  if (vsize != n) return GrB_DIMENSION_MISMATCH;
  const bool same_structure = S->symmetric_ || S->d_cscColPtr_ == S->d_csrRowPtr_;
  const bool stored = n > 0 && S->nvals_ > 0;
  if (stored && (S->d_csrRowPtr_ == NULL || (!same_structure && S->d_cscColPtr_ == NULL)))
    return GrB_UNINITIALIZED_OBJECT;

  GpuTimer clock;
  clock.Start();
  CHECK(v->setStorage(GrB_DENSE));
  if (ncolors != NULL) *ncolors = 0;
  if (!stored) {                       // no edges: every vertex takes colour 1
    if (n > 0) CHECK(v->fill(static_cast<W>(1)));
    if (ncolors != NULL && n > 0) *ncolors = 1;
    clock.Stop();
    if (ms != NULL) *ms = clock.ElapsedMillis();
    return GrB_SUCCESS;
  }
  CHECK(v->dense_.allocateGpu());
  cudaStream_t stream = gbStream();

  const size_t words = (static_cast<size_t>(n) + 63)/64*64;     // 256-byte aligned arrays
  const size_t counters_bytes = 4*sizeof(unsigned long long);     // in the first 256 bytes
  unsigned char* block = static_cast<unsigned char*>(gbMalloc(
      256 + 5*words*sizeof(Index)));
  GcArgs args;
  args.row_ptr = S->d_csrRowPtr_;  args.row_ind = S->d_csrColInd_;
  args.col_ptr = same_structure ? NULL : S->d_cscColPtr_;
  args.col_ind = same_structure ? NULL : S->d_cscRowInd_;
  args.n = n;
  args.seed = seed;
  args.counters   = reinterpret_cast<unsigned long long*>(block);
  Index* arrays   = reinterpret_cast<Index*>(block + 256);
  args.colour     = reinterpret_cast<unsigned int*>(arrays);
  args.waiting_on = arrays + words;
  args.resume     = arrays + 2*words;
  args.list[0]    = arrays + 3*words;
  args.list[1]    = arrays + 4*words;
  CUDA_CALL(cudaMemsetAsync(block, 0, counters_bytes, stream));
  CUDA_CALL(cudaMemsetAsync(args.colour, 0, static_cast<size_t>(n)*sizeof(unsigned int),
                            stream));

  void (*kernel)(GcArgs, W*) = graphColorKernel<W>;
  static int resident = 0;             // CTAs that fit at once (cooperative launch)
  if (resident == 0) {
    int per_sm = 0;
    CUDA_CALL(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, GB_GC_NT, 0));
    resident = per_sm*runtime().sm_count;
    if (resident < 1) { gbFree(block); return GrB_PANIC; }
  }
  W* out = v->dense_.d_val_;
  void* params[] = { &args, &out };
  CUDA_CALL(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(kernel),
      dim3(resident), dim3(GB_GC_NT), params, 0, stream));
  GB_KERNEL_CHECK();
  clock.Stop();
  v->dense_.touched();
  if (ncolors != NULL)
    *ncolors = static_cast<int>(runtime().fetch(args.counters + 3));
  gbFree(block);
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_COLOR_HPP_
