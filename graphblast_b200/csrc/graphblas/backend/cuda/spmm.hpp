// graphblast_b200 backend — SpMM host: C = op(A) (+.x) B with A sparse and B, C
// dense row-major fp32 (kernels/spmm.cuh).  The reference has no SpMM (its
// spmm.hpp prints "not implemented"); this is the backend's own.
//
// A warm call (same A and N, C already dense of the right shape and not B) makes
// no allocation and no host synchronisation, and launches two kernels: the SpMM
// and the carry fix-up.  The first call on a structure adds the partition launch
// (cached on A with the pull SpMV's tiles).
#ifndef GRAPHBLAS_BACKEND_CUDA_SPMM_HPP_
#define GRAPHBLAS_BACKEND_CUDA_SPMM_HPP_

#include <climits>
#include <type_traits>

#include "graphblas/backend/cuda/kernels/kernels.hpp"
#include "graphblas/backend/cuda/matrix.hpp"
#include "graphblas/backend/cuda/spmv.hpp"
#include "graphblas/backend/cuda/spgemm.hpp"

namespace graphblas {
namespace backend {

template <typename c, typename a, typename b, typename SemiringT>
Info spmmProduct(Matrix<c>* C, SemiringT op, const Matrix<a>* A, const Matrix<b>* B,
    Descriptor* desc);

// C is replaced; accum is not applied, as for the unmasked sparse product.  The
// order-dependent semirings and element types other than float are refused.
template <typename c, typename a, typename b, typename BinaryOpT, typename SemiringT>
Info spmm(Matrix<c>* C, BinaryOpT accum, SemiringT op, const Matrix<a>* A,
    const Matrix<b>* B, Descriptor* desc) {
  constexpr bool fp32 = std::is_same<c, float>::value && std::is_same<a, float>::value &&
                        std::is_same<b, float>::value;
  if constexpr (FoldNeedsOrder<SemiringT>::value || !fp32) return GrB_NOT_IMPLEMENTED;
  else return spmmProduct(C, op, A, B, desc);
}

template <bool ADJ, bool VEC, typename c, typename a, typename SemiringT>
void spmmLaunch(dim3 grid, c* out, const Index* tiles, Index* carry_row, c* carry_val,
    const Index* ptr, const Index* ind, const a* val, const c* B, Index m, Index nnz,
    int N, int lanes, int nslices, SemiringT op, cudaStream_t s) {
  spmmMergeKernel<ADJ, VEC><<<grid, GB_SPMM_NT, 0, s>>>(out, tiles, carry_row, carry_val,
      ptr, ind, val, B, m, nnz, N, lanes, nslices, static_cast<c>(op.identity()),
      extractMul(op), extractAdd(op));
  GB_KERNEL_CHECK();
}

template <typename c, typename a, typename b, typename SemiringT>
Info spmmProduct(Matrix<c>* C, SemiringT op, const Matrix<a>* A, const Matrix<b>* B,
    Descriptor* desc) {
  Desc_value inp0_mode;
  CHECK(desc->get(GrB_INP0, &inp0_mode));
  const bool tran = inp0_mode == GrB_TRAN;
  SparseMatrix<a>* S = const_cast<SparseMatrix<a>*>(&A->sparse_);
  const DenseMatrix<b>& D = B->dense_;
  const typename SparseMatrix<a>::View Av = S->view(tran);
  const Index* ptr = Av.ptr;
  const Index* ind = Av.ind;
  const a*     val = Av.val;
  const Index  m = Av.dim, k = Av.other;
  const long long N = D.ncols_;
  if (D.nrows_ != k || C->nrows_ != m || C->ncols_ != N) return GrB_DIMENSION_MISMATCH;
  // before anything is allocated: C keeps its contents (the kernel indexes columns
  // with int, a column slice past the last one included)
  if (!DenseMatrix<c>::fits(static_cast<long long>(m)*N) ||
      N > INT32_MAX - GB_SPMM_COL_TILE)
    return GrB_OUT_OF_MEMORY;
  if (!Av.complete() || D.d_val_ == NULL)
    return GrB_UNINITIALIZED_OBJECT;

  // The result goes into C's own array when it has one of this shape that B does
  // not share; otherwise into a fresh one, swapped in at the end (C may be A or B).
  DenseMatrix<c>& Cd = C->dense_;
  const bool in_place = C->isDense() && Cd.ownership_ && Cd.d_val_ != NULL &&
      Cd.nrows_ == m && Cd.ncols_ == N &&
      reinterpret_cast<const void*>(Cd.d_val_) != reinterpret_cast<const void*>(D.d_val_);
  const long long elements = static_cast<long long>(m)*N;
  c* out = in_place ? Cd.d_val_
                    : reinterpret_cast<c*>(gbMalloc((elements > 0 ? elements : 1)*sizeof(c)));

  if (elements > 0) {
    cudaStream_t s = gbStream();
    const int ntiles = mergeTiles(S, Av.which, ptr, m);
    const Index nnz = S->nvals_;
    Index* carry_row = reinterpret_cast<Index*>(desc->scratch(GB_SCRATCH_CARRY_ROW,
        static_cast<size_t>(ntiles)*sizeof(Index)));
    c* carry_val = reinterpret_cast<c*>(desc->scratch(GB_SCRATCH_CARRY_VAL,
        static_cast<size_t>(ntiles)*N*sizeof(c)));
    const int lanes = spmmLanes(N);
    const long long slices = (N + GB_SPMM_COL_TILE - 1)/GB_SPMM_COL_TILE;
    const dim3 grid(ntiles, static_cast<unsigned>(slices < 65535 ? slices : 65535));
    const int nslices = static_cast<int>(slices);
    const Index* tiles = S->tiles_[Av.which].d;
    const double alg_bytes = 4.0*(m + 1) + 8.0*nnz + 4.0*k*N + 4.0*m*N;
    profiler().begin(GB_PROF_SPMM, s);
    if (N % 4 != 0)
      spmmLaunch<false, false>(grid, out, tiles, carry_row, carry_val, ptr, ind, val,
          D.d_val_, m, nnz, static_cast<int>(N), lanes, nslices, op, s);
    else if (reinterpret_cast<uintptr_t>(D.d_val_) % 16 == 0 &&
             reinterpret_cast<uintptr_t>(out) % 16 == 0)
      spmmLaunch<true, true>(grid, out, tiles, carry_row, carry_val, ptr, ind, val,
          D.d_val_, m, nnz, static_cast<int>(N), lanes, nslices, op, s);
    else
      spmmLaunch<true, false>(grid, out, tiles, carry_row, carry_val, ptr, ind, val,
          D.d_val_, m, nnz, static_cast<int>(N), lanes, nslices, op, s);
    const long long fix = static_cast<long long>(ntiles)*N;
    spmmCarryFixupKernel<<<static_cast<unsigned>((fix + 255)/256), 256, 0, s>>>(out,
        carry_row, carry_val, ntiles, N, extractAdd(op));
    GB_KERNEL_CHECK();
    profiler().end(GB_PROF_SPMM, s, alg_bytes);
  }

  // swap in: the old storage (and every cache built on it) goes, stream-ordered
  // after the kernels above that may still read it through A or B
  if (!in_place) {
    CHECK(C->setStorage(GrB_DENSE));
    Cd.take(out);
  }
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_SPMM_HPP_
