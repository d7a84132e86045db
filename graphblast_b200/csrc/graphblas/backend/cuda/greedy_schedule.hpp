// graphblast_b200 backend — host side of the greedy schedule
// (kernels/greedy_schedule.cuh): the refusals, the scratch and the one cooperative
// launch that the graph colouring (color.hpp) and the maximal independent set
// (mis.hpp) share.
#ifndef GRAPHBLAS_BACKEND_CUDA_GREEDY_SCHEDULE_HPP_
#define GRAPHBLAS_BACKEND_CUDA_GREEDY_SCHEDULE_HPP_

#include "graphblas/backend/cuda/kernels/greedy_schedule.cuh"

namespace graphblas {
namespace backend {

// The refusals, in this order and all before anything is touched: a dense A
// (GrB_NOT_IMPLEMENTED, naming `what`); A not square, or v or cand (when not NULL) not
// of size nrows(A) (GrB_DIMENSION_MISMATCH); an A with stored entries but without a
// device CSR, or non-symmetric without a device CSC (GrB_UNINITIALIZED_OBJECT).
template <typename W, typename a>
Info greedyCheck(const char* what, Vector<W>* v, const Matrix<a>* A, Vector<W>* cand) {
  if (!A->isSparse()) {
    std::cout << "Error: " << what << " of a dense matrix is not implemented in this backend\n";
    return GrB_NOT_IMPLEMENTED;
  }
  const SparseMatrix<a>* S = &A->sparse_;
  const Index n = S->nrows_;
  if (n != S->ncols_) return GrB_DIMENSION_MISMATCH;
  Index vsize = 0;
  CHECK(v->size(&vsize));
  if (vsize != n) return GrB_DIMENSION_MISMATCH;
  if (cand != NULL) {
    Index csize = 0;
    CHECK(cand->size(&csize));
    if (csize != n) return GrB_DIMENSION_MISMATCH;
  }
  const bool same_structure = S->symmetric_ || S->d_cscColPtr_ == S->d_csrRowPtr_;
  if (n > 0 && S->nvals_ > 0 &&
      (S->d_csrRowPtr_ == NULL || (!same_structure && S->d_cscColPtr_ == NULL)))
    return GrB_UNINITIALIZED_OBJECT;
  return GrB_SUCCESS;
}

// One run of kernel K on an A that passed greedyCheck: init(state, stream) sets the
// n-word state on the stream before v is touched, then v becomes dense with
// nrows(A) entries and K writes it; *count (when not NULL) = K's counters[3], 0 when
// A has no rows; *ms (when not NULL) = the device time, from CUDA events.
// Scratch: 256 bytes of counters and five 256-byte aligned n-word arrays (state,
// waiting_on, resume, two lists), plus n + 1 zero row pointers when A has no stored
// entries, so that every list is empty.
template <typename W, void (*K)(GreedyArgs, W*), typename a, typename Init>
Info greedyRun(Vector<W>* v, const SparseMatrix<a>* S, unsigned int seed, int* count,
               float* ms, Init init) {
  const Index n = S->nrows_;
  GpuTimer clock;
  clock.Start();
  if (count != NULL) *count = 0;
  if (n == 0) {
    CHECK(v->setStorage(GrB_DENSE));
    clock.Stop();
    if (ms != NULL) *ms = clock.ElapsedMillis();
    return GrB_SUCCESS;
  }
  cudaStream_t stream = gbStream();
  const bool stored = S->nvals_ > 0;
  const bool same_structure = S->symmetric_ || S->d_cscColPtr_ == S->d_csrRowPtr_;

  const size_t words = (static_cast<size_t>(n) + 63)/64*64;      // 256-byte aligned arrays
  const size_t rp_words = stored ? 0 : (static_cast<size_t>(n) + 64)/64*64;
  const size_t counters_bytes = 4*sizeof(unsigned long long);      // in the first 256 bytes
  unsigned char* block = static_cast<unsigned char*>(gbMalloc(
      256 + (5*words + rp_words)*sizeof(Index)));
  GreedyArgs args;
  args.n = n;
  args.seed = seed;
  args.counters   = reinterpret_cast<unsigned long long*>(block);
  Index* arrays   = reinterpret_cast<Index*>(block + 256);
  args.state      = reinterpret_cast<unsigned int*>(arrays);
  args.waiting_on = arrays + words;
  args.resume     = arrays + 2*words;
  args.list[0]    = arrays + 3*words;
  args.list[1]    = arrays + 4*words;
  if (stored) {
    args.row_ptr = S->d_csrRowPtr_;  args.row_ind = S->d_csrColInd_;
    args.col_ptr = same_structure ? NULL : S->d_cscColPtr_;
    args.col_ind = same_structure ? NULL : S->d_cscRowInd_;
  } else {                             // no edges: every list is empty
    Index* zero_ptr = arrays + 5*words;
    CUDA_CALL(cudaMemsetAsync(zero_ptr, 0, (static_cast<size_t>(n) + 1)*sizeof(Index),
                              stream));
    args.row_ptr = zero_ptr;  args.row_ind = NULL;
    args.col_ptr = NULL;      args.col_ind = NULL;
  }
  CUDA_CALL(cudaMemsetAsync(block, 0, counters_bytes, stream));
  init(args.state, stream);

  CHECK(v->setStorage(GrB_DENSE));
  CHECK(v->dense_.allocateGpu());
  static int resident = 0;             // CTAs of K that fit at once (cooperative launch)
  if (resident == 0) {
    int per_sm = 0;
    CUDA_CALL(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, K, GB_GC_NT, 0));
    resident = per_sm*runtime().sm_count;
    if (resident < 1) { gbFree(block); return GrB_PANIC; }
  }
  W* out = v->dense_.d_val_;
  void* params[] = { &args, &out };
  CUDA_CALL(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(K),
      dim3(resident), dim3(GB_GC_NT), params, 0, stream));
  GB_KERNEL_CHECK();
  clock.Stop();
  v->dense_.touched();
  if (count != NULL)
    *count = static_cast<int>(runtime().fetch(args.counters + 3));
  gbFree(block);
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_GREEDY_SCHEDULE_HPP_
