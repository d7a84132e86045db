// graphblast_b200 backend — host side of the maximal independent set (kernels/mis.cuh):
// an init pass over the candidates, then one cooperative launch.  algorithm::mis comes
// here.
#ifndef GRAPHBLAS_BACKEND_CUDA_MIS_HPP_
#define GRAPHBLAS_BACKEND_CUDA_MIS_HPP_

#include <type_traits>

#include "graphblas/backend/cuda/kernels/mis.cuh"

namespace graphblas {
namespace backend {

// v[i] = 1 when vertex i of A's pattern is in the greedy maximal independent set in
// decreasing priority order over the candidates, else 0; *nmembers (when not NULL) =
// the size of the set; *ms (when not NULL) = the device time, from CUDA events.
// candidates == NULL: every vertex is a candidate.  Otherwise vertex i is one when the
// vector holds a non-zero value for it (a dense value, or a stored sparse entry).  The
// candidate vector is read in the storage it has, never converted, and read completely
// before v is written, so it may be v itself.
// Every refusal comes before v is touched: A not square, or v or the candidates not of
// size nrows(A) (GrB_DIMENSION_MISMATCH), a dense A (GrB_NOT_IMPLEMENTED), an A without
// a device CSR, or a non-symmetric A without a device CSC (GrB_UNINITIALIZED_OBJECT).
template <typename W, typename a>
Info misRun(Vector<W>* v, const Matrix<a>* A, unsigned int seed,
            const Vector<W>* candidates, int* nmembers, float* ms = NULL) {
  static_assert(std::is_same<W, int>::value || std::is_same<W, float>::value,
                "mis writes int or float vectors");
  if (!A->isSparse()) {
    std::cout << "Error: mis of a dense matrix is not implemented in this backend\n";
    return GrB_NOT_IMPLEMENTED;
  }
  const SparseMatrix<a>* S = &A->sparse_;
  const Index n = S->nrows_;
  if (n != S->ncols_) return GrB_DIMENSION_MISMATCH;
  Index vsize = 0;
  CHECK(v->size(&vsize));
  if (vsize != n) return GrB_DIMENSION_MISMATCH;
  Vector<W>* cand = const_cast<Vector<W>*>(candidates);    // read only
  if (cand != NULL) {
    Index csize = 0;
    CHECK(cand->size(&csize));
    if (csize != n) return GrB_DIMENSION_MISMATCH;
  }
  const bool same_structure = S->symmetric_ || S->d_cscColPtr_ == S->d_csrRowPtr_;
  const bool stored = n > 0 && S->nvals_ > 0;
  if (stored && (S->d_csrRowPtr_ == NULL || (!same_structure && S->d_cscColPtr_ == NULL)))
    return GrB_UNINITIALIZED_OBJECT;

  // the candidates as device arrays, in the storage they have
  const Storage cand_type = cand != NULL ? cand->vec_type_ : GrB_UNKNOWN;
  const W* cand_val = NULL;
  const Index* cand_ind = NULL;
  Index cand_nvals = 0;
  if (cand_type == GrB_DENSE && n > 0) {
    CHECK(cand->dense_.materialize());       // values from the bitmap, when only it is current
    cand_val = cand->dense_.d_val_;
    if (cand_val == NULL) return GrB_UNINITIALIZED_OBJECT;
  } else if (cand_type == GrB_SPARSE) {
    cand_nvals = cand->sparse_.nvals_;
    cand_ind = cand->sparse_.d_ind_;
    cand_val = cand->sparse_.d_val_;
    if (cand_nvals > 0 && (cand_ind == NULL || cand_val == NULL))
      return GrB_UNINITIALIZED_OBJECT;
  }

  GpuTimer clock;
  clock.Start();
  if (nmembers != NULL) *nmembers = 0;
  if (n == 0) {
    CHECK(v->setStorage(GrB_DENSE));
    clock.Stop();
    if (ms != NULL) *ms = clock.ElapsedMillis();
    return GrB_SUCCESS;
  }
  cudaStream_t stream = gbStream();

  const size_t words = (static_cast<size_t>(n) + 63)/64*64;      // 256-byte aligned arrays
  const size_t rp_words = stored ? 0 : (static_cast<size_t>(n) + 64)/64*64;
  const size_t counters_bytes = 4*sizeof(unsigned long long);      // in the first 256 bytes
  unsigned char* block = static_cast<unsigned char*>(gbMalloc(
      256 + (5*words + rp_words)*sizeof(Index)));
  MisArgs args;
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

  // init pass: everything it reads of the candidates is read before v is written
  const int nt = 256;
  if (cand == NULL) {
    CUDA_CALL(cudaMemsetAsync(args.state, 0, static_cast<size_t>(n)*sizeof(unsigned int),
                              stream));
  } else if (cand_type == GrB_DENSE) {
    misInitDenseKernel<W><<<gridFor(n, nt), nt, 0, stream>>>(args.state, cand_val, n);
    GB_KERNEL_CHECK();
  } else {                             // sparse, or no storage: only stored non-zeros count
    fillKernel<unsigned int><<<gridFor(n, nt), nt, 0, stream>>>(args.state, MIS_OUT, n);
    GB_KERNEL_CHECK();
    if (cand_nvals > 0) {
      misInitSparseKernel<W><<<gridFor(cand_nvals, nt), nt, 0, stream>>>(
          args.state, cand_ind, cand_val, cand_nvals, n);
      GB_KERNEL_CHECK();
    }
  }

  CHECK(v->setStorage(GrB_DENSE));
  CHECK(v->dense_.allocateGpu());
  void (*kernel)(MisArgs, W*) = misKernel<W>;
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
  if (nmembers != NULL)
    *nmembers = static_cast<int>(runtime().fetch(args.counters + 3));
  gbFree(block);
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_MIS_HPP_
