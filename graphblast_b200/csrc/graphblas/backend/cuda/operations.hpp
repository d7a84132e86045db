// graphblast_b200 backend — operation dispatch: what every frontend template in
// graphblas/operations.hpp lands on.
//
// Stands in for reference graphblas/backend/cuda/operations.hpp:18-1435.  Template
// parameter orders are fixed by the explicit instantiations the frontend writes
// (backend::mxm<c,a,b,m>, vxm<W,U,a,M>, mxv<W,U,a,M>, applyVxm<W,U,a,M>;
// reference graphblas/operations.hpp:47,85,125,863).  Structure is this
// backend's own:
//   * vxm and mxv share one body (mxvDispatch) — vxm is mxv on the transposed
//     matrix, done by toggling GrB_INP1 for the duration of the call;
//   * binary vector operations classify their operands once (pairOf) and switch
//     on the pair instead of nesting storage tests per operation;
//   * operations no algorithm of the path reaches are declared (the frontend
//     must link) and answer GrB_NOT_IMPLEMENTED through one helper.
//
// Direction choice for vxm/mxv (reference :124-139, :252-266):
//   CSR-only non-symmetric matrix -> vxm forced to push, mxv forced to pull;
//   GrB_PUSHPULL  -> Vector::convert() heuristic on the input vector;
//   GrB_PUSHONLY / GrB_PULLONLY -> input converted if needed.
// desc->lastmxv_ records the direction taken.
#ifndef GRAPHBLAS_BACKEND_CUDA_OPERATIONS_HPP_
#define GRAPHBLAS_BACKEND_CUDA_OPERATIONS_HPP_

#include <vector>
#include <typeinfo>

#include "graphblas/backend/cuda/vector.hpp"
#include "graphblas/backend/cuda/matrix.hpp"
#include "graphblas/backend/cuda/spmv.hpp"
#include "graphblas/backend/cuda/spmspv.hpp"
#include "graphblas/backend/cuda/spgemm.hpp"
#include "graphblas/backend/cuda/spmm.hpp"
#include "graphblas/backend/cuda/ewiseadd.hpp"
#include "graphblas/backend/cuda/ewisemult.hpp"
#include "graphblas/backend/cuda/ewise_matrix.hpp"
#include "graphblas/backend/cuda/extract.hpp"
#include "graphblas/backend/cuda/assign.hpp"
#include "graphblas/backend/cuda/assign_matrix.hpp"
#include "graphblas/backend/cuda/reduce.hpp"
#include "graphblas/backend/cuda/apply.hpp"
#include "graphblas/backend/cuda/indexed.hpp"
#include "graphblas/backend/cuda/tri.hpp"
#include "graphblas/backend/cuda/color.hpp"
#include "graphblas/backend/cuda/mis.hpp"
#include "graphblas/backend/cuda/cc.hpp"
#include "graphblas/backend/cuda/lgc.hpp"
#include "graphblas/backend/cuda/bc.hpp"
#include "graphblas/backend/cuda/ktruss.hpp"
#include "graphblas/backend/cuda/scc.hpp"
#include "graphblas/backend/cuda/msf.hpp"
#include "graphblas/backend/cuda/cdlp.hpp"

namespace graphblas {
namespace backend {

// One place that says "declared, not built" (SURVEY.md §8b: must declare).
inline Info notBuilt(const char* what) {
  std::cout << "Error: " << what << " is not implemented in this backend\n";
  return GrB_NOT_IMPLEMENTED;
}

// Storage of a pair of vector operands, classified once.
enum OperandPair {
  GB_PAIR_DENSE_DENSE,
  GB_PAIR_SPARSE_DENSE,
  GB_PAIR_DENSE_SPARSE,
  GB_PAIR_SPARSE_SPARSE,
  GB_PAIR_INVALID
};

inline OperandPair pairOf(Storage first, Storage second) {
  const bool fd = first == GrB_DENSE, fs = first == GrB_SPARSE;
  const bool sd = second == GrB_DENSE, ss = second == GrB_SPARSE;
  if (fd && sd) return GB_PAIR_DENSE_DENSE;
  if (fs && sd) return GB_PAIR_SPARSE_DENSE;
  if (fd && ss) return GB_PAIR_DENSE_SPARSE;
  if (fs && ss) return GB_PAIR_SPARSE_SPARSE;
  return GB_PAIR_INVALID;
}

template <typename TU, typename TV>
OperandPair pairOf(const Vector<TU>* u, const Vector<TV>* v) {
  return pairOf(u->vec_type_, v->vec_type_);
}

// Lazily held values (dense_vector.hpp) written out for every operand given.
template <typename X>
Info settle(const Vector<X>* x) { return x == NULL ? GrB_SUCCESS : x->materialize(); }
template <typename X, typename... Rest>
Info settle(const Vector<X>* x, Rest... rest) {
  CHECK(settle(x));
  return settle(rest...);
}

// Operations that exist in the frontend but that no algorithm of the path reaches
// (SURVEY.md §8b "must declare"): whatever the call shape — the frontend names the
// template arguments of some of them explicitly — the answer is the same.
#define GB_DECLARED_ONLY(name, what)                                        \
  template <typename... Named, typename... Args>                            \
  Info name(Args... args) { return notBuilt(what); }

GB_DECLARED_ONLY(assignIndexed,     "assignIndexed")
GB_DECLARED_ONLY(traceMxmTranspose, "traceMxmTranspose")
GB_DECLARED_ONLY(applyVxm,          "applyVxm")
#undef GB_DECLARED_ONLY

// w = greedy Jones–Plassmann colouring of A's pattern with seed 0 (color.hpp); W is
// int or float.  algorithm::gc takes other seeds.
template <typename W, typename a>
Info graphColor(Vector<W>* w, const Matrix<a>* A, Descriptor* desc) {
  return graphColorRun(w, A, 0u, static_cast<int*>(NULL));
}

template <typename TC, typename TA, typename TB, typename TMask,
          typename AccumT,     typename SemiringT>
Info mxm(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, SemiringT op,
    const Matrix<TA>* A, const Matrix<TB>* B, Descriptor* desc) {
  if (A->isSparse() && B->isDense()) {
    if (mask != NULL) return notBuilt("masked mxm with a dense operand");
    Desc_value inp1_mode;
    CHECK(desc->get(GrB_INP1, &inp1_mode));
    if (inp1_mode == GrB_TRAN) return notBuilt("mxm with a transposed dense B");
    return spmm(C, accum, op, A, B, desc);
  }
  if (!A->isSparse() || !B->isSparse()) return notBuilt("mxm with a dense A (GEMM / dense x sparse)");
  // A dense C turns sparse only once the product has replaced it: a refused
  // product leaves it as it was.
  const bool was_dense = C->isDense();
  if (!was_dense) CHECK(C->setStorage(GrB_SPARSE));
  const Info info = (mask == NULL)
      ? spgemmUnmasked(&C->sparse_, accum, op, &A->sparse_, &B->sparse_, desc)
      : spgemmMasked(&C->sparse_, mask, accum, op, &A->sparse_, &B->sparse_, desc);
  if (info == GrB_SUCCESS && was_dense) CHECK(C->setStorage(GrB_SPARSE));
  return info;
}

// C = op(A) (+) op(B) (IsAdd: union) or op(A) (x) op(B) (intersection) of two
// sparse matrices (ewise_matrix.hpp).  The refusals come before anything changes;
// a dense C turns sparse only once the result has replaced it.
template <bool IsAdd, typename TC, typename TA, typename TB, typename TMask,
          typename SemiringT>
Info ewiseMatrixDispatch(Matrix<TC>* C, const Matrix<TMask>* mask, SemiringT op,
    const Matrix<TA>* A, const Matrix<TB>* B, Descriptor* desc) {
  if (mask != NULL)
    return notBuilt(IsAdd ? "masked eWiseAdd of two matrices" : "masked eWiseMult of two matrices");
  if (!A->isSparse() || !B->isSparse())
    return notBuilt(IsAdd ? "eWiseAdd with a dense matrix" : "eWiseMult with a dense matrix");
  const bool was_dense = C->isDense();
  if (!was_dense) CHECK(C->setStorage(GrB_SPARSE));
  const Info info = ewiseMatrix<IsAdd>(&C->sparse_, op, &A->sparse_, &B->sparse_, desc);
  if (info == GrB_SUCCESS && was_dense) CHECK(C->setStorage(GrB_SPARSE));
  return info;
}

// Shared body of vxm / mxv once the descriptor says which side is transposed.
// Step 1 puts the input vector into the storage the direction needs, step 2 runs
// the push (sparse input) or the pull (dense input).
template <bool IsVxm, typename TW, typename TU, typename TA, typename TMask,
          typename AccumT, typename SemiringT>
Info mxvDispatch(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
    const Matrix<TA>* A, const Vector<TU>* u, Descriptor* desc) {
  Vector<TU>* input = const_cast<Vector<TU>*>(u);
  if (!A->isSparse()) return notBuilt("mxv / vxm with a dense matrix (GEMV)");

  SparseMatrixFormat format;
  bool reported_symmetric;
  Desc_value mode;
  CHECK(A->getFormat(&format));
  CHECK(A->getSymmetry(&reported_symmetric));
  CHECK(desc->get(GrB_MXVMODE, &mode));
  const bool one_orientation = !reported_symmetric && format == GrB_SPARSE_MATRIX_CSRONLY;
  const bool both_orientations = reported_symmetric || format == GrB_SPARSE_MATRIX_CSRCSC;

  // ---- step 1: storage of the input ------------------------------------------------
  const TU identity = op.identity();
  const bool dense_in = (input->vec_type_ == GrB_DENSE);
  const bool sparse_in = (input->vec_type_ == GrB_SPARSE);
  if (one_orientation) {
    // only the CSR exists: vxm can only push over it, mxv can only pull over it
    if (IsVxm && dense_in)   CHECK(input->dense2sparse(identity, desc));
    if (!IsVxm && sparse_in) CHECK(input->sparse2dense(identity, desc));
  } else {
    switch (mode) {
      case GrB_PUSHPULL: CHECK(input->convert(identity, desc->switchpoint(), desc)); break;
      case GrB_PUSHONLY: if (dense_in)  CHECK(input->dense2sparse(identity, desc)); break;
      case GrB_PULLONLY: if (sparse_in) CHECK(input->sparse2dense(identity, desc)); break;
      default: break;
    }
  }

  // ---- step 2: push ------------------------------------------------------------------
  bool pull = (input->vec_type_ != GrB_SPARSE);
  if (!pull) {
    const LoadBalanceMode balance = getEnv("GRB_LOAD_BALANCE_MODE", GrB_LOAD_BALANCE_MERGE);
    if (balance != GrB_LOAD_BALANCE_MERGE)
      return notBuilt("push load balancing other than GrB_LOAD_BALANCE_MERGE");
    // w becomes a sparse vector only if the push really runs: on a hand-back its
    // previous storage (and with it a dense w that accum combines into) must
    // survive untouched, so the tag is restored below.
    const Storage w_before = w->vec_type_;
    CHECK(w->setStorage(GrB_SPARSE));
    // In the automatic mode the push may hand the call back when the frontier owns
    // too many of the edges (spmspv.hpp); both orientations must exist for that.
    bool hand_back = false;
    const bool may_hand_back = (mode == GrB_PUSHPULL) && both_orientations;
    CHECK(spmspvMerge(&w->sparse_, mask, accum, op, &A->sparse_, &u->sparse_, desc,
        may_hand_back ? &hand_back : NULL));
    if (hand_back) {
      w->vec_type_ = w_before;
      CHECK(input->sparse2dense(identity, desc));
      pull = true;
    } else {
      desc->lastmxv_ = GrB_PUSHONLY;
    }
  }
  // ---- step 2: pull ------------------------------------------------------------------
  if (pull) {
    if (IsVxm) CHECK(w->setStorage(GrB_DENSE));
    else       CHECK(w->sparse2dense(identity, desc));
    CHECK(spmv(&w->dense_, mask, accum, op, &A->sparse_, &u->dense_, desc));
    desc->lastmxv_ = GrB_PULLONLY;
  }
  return GrB_SUCCESS;
}

// Debug trace shared by the two entry points.
template <typename X>
void traceVector(Descriptor* desc, const char* banner, const Vector<X>* x) {
  if (!desc->debug()) return;
  std::cout << banner << "\n";
  const_cast<Vector<X>*>(x)->print();
}

// vxm = mxv on the transposed matrix: GrB_INP1 is toggled around the call.
template <typename TW, typename TU, typename TA, typename TMask,
          typename AccumT, typename SemiringT>
Info vxm(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
    const Vector<TU>* u, const Matrix<TA>* A, Descriptor* desc) {
  traceVector(desc, "===Begin vxm===", u);
  Desc_value inp0_mode;
  CHECK(desc->get(GrB_INP0, &inp0_mode));
  if (inp0_mode != GrB_DEFAULT) return GrB_INVALID_VALUE;
  CHECK(desc->toggle(GrB_INP1));
  const Info status = mxvDispatch<true>(w, mask, accum, op, A, u, desc);
  CHECK(desc->toggle(GrB_INP1));
  if (status == GrB_SUCCESS) traceVector(desc, "===End vxm===", w);
  return status;
}

template <typename TW, typename TA, typename TU, typename TMask,
          typename AccumT, typename SemiringT>
Info mxv(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
    const Matrix<TA>* A, const Vector<TU>* u, Descriptor* desc) {
  traceVector(desc, "===Begin mxv===", u);
  Desc_value inp1_mode;
  CHECK(desc->get(GrB_INP1, &inp1_mode));
  if (inp1_mode != GrB_DEFAULT) return GrB_INVALID_VALUE;
  const Info status = mxvDispatch<false>(w, mask, accum, op, A, u, desc);
  if (status == GrB_SUCCESS) traceVector(desc, "===End mxv===", w);
  return status;
}

// w = u .* v.  Results: dense x dense -> dense (sparse when the mask is sparse),
// anything with a sparse operand -> sparse; sparse x sparse reads v as dense, as
// the reference does by flipping its tag (operations.hpp:365-371).
template <typename TW, typename TU, typename TV, typename TMask,
          typename AccumT,     typename SemiringT>
Info eWiseMult(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
    const Vector<TU>* u, const Vector<TV>* v, Descriptor* desc) {
  CHECK(settle(u, v, w, mask));
  if (pairOf(u, v) == GB_PAIR_SPARSE_SPARSE)
    CHECK(const_cast<Vector<TV>*>(v)->setStorage(GrB_DENSE));
  switch (pairOf(u, v)) {
    case GB_PAIR_DENSE_DENSE:
      if (mask != NULL && mask->vec_type_ == GrB_SPARSE) {
        CHECK(w->setStorage(GrB_SPARSE));
        return eWiseMultInner(&w->sparse_, &mask->sparse_, accum, op, &u->dense_,
            &v->dense_, desc);
      }
      if (mask != NULL && mask->vec_type_ != GrB_DENSE) return GrB_INVALID_OBJECT;
      CHECK(w->setStorage(GrB_DENSE));
      return eWiseMultInner(&w->dense_, mask, accum, op, &u->dense_, &v->dense_, desc);
    case GB_PAIR_SPARSE_DENSE:
      CHECK(w->setStorage(GrB_SPARSE));
      return eWiseMultInner(&w->sparse_, mask, accum, op, &u->sparse_, &v->dense_,
          false, desc);
    case GB_PAIR_DENSE_SPARSE:          // operands swapped, the kernel is told
      CHECK(w->setStorage(GrB_SPARSE));
      return eWiseMultInner(&w->sparse_, mask, accum, op, &v->sparse_, &u->dense_,
          true, desc);
    default:
      return GrB_INVALID_OBJECT;
  }
}

template <typename TC, typename TA, typename TB, typename TMask,
          typename AccumT,     typename SemiringT>
Info eWiseMult(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, SemiringT op,
    const Matrix<TA>* A, const Matrix<TB>* B, Descriptor* desc) {
  return ewiseMatrixDispatch<false>(C, mask, op, A, B, desc);
}

// Extension: matrix (x) broadcast scalar
template <typename TC, typename TA, typename TB, typename TMask,
          typename AccumT,     typename SemiringT>
Info eWiseMult(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, SemiringT op,
    const Matrix<TA>* A, TB val, Descriptor* desc) {
  if (A->isDense()) return notBuilt("eWiseMult of a dense matrix and a scalar");
  if (!A->isSparse()) return GrB_INVALID_OBJECT;
  if (mask != NULL) return notBuilt("masked eWiseMult of a matrix and a scalar");
  CHECK(C->setStorage(GrB_SPARSE));
  return eWiseMultInner(&C->sparse_, mask, accum, op, &A->sparse_, val, desc);
}

// Extension: matrix (x) broadcast vector (column vector; row vector when
// GrB_INP1 is GrB_TRAN)
template <typename TC, typename TA, typename TB, typename TMask,
          typename AccumT,     typename SemiringT>
Info eWiseMult(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, SemiringT op,
    const Matrix<TA>* A, const Vector<TB>* B, Descriptor* desc) {
  Desc_value inp0_mode, inp1_mode;
  CHECK(desc->get(GrB_INP0, &inp0_mode));
  CHECK(desc->get(GrB_INP1, &inp1_mode));
  if (inp0_mode != GrB_DEFAULT) return GrB_INVALID_VALUE;
  CHECK(settle(B));
  if (A->isDense()) return notBuilt("eWiseMult of a dense matrix and a vector");
  if (!A->isSparse()) return GrB_INVALID_OBJECT;
  if (mask != NULL) return notBuilt("masked eWiseMult of a matrix and a vector");
  CHECK(C->setStorage(GrB_SPARSE));
  if (B->vec_type_ == GrB_SPARSE)
    return notBuilt("eWiseMult of a matrix and a sparse vector");
  if (inp1_mode == GrB_TRAN)
    return eWiseMultRowInner(&C->sparse_, mask, accum, op, &A->sparse_, &B->dense_, desc);
  return eWiseMultColInner(&C->sparse_, mask, accum, op, &A->sparse_, &B->dense_, desc);
}

// w = u + v, always dense.  A sparse operand that is also the output is
// densified first (reference :598-607).  The routes the reference does not
// build (any mask, sparse + sparse) are refused before anything changes, w's
// storage included; like the reference they report it and return success.
template <typename TW, typename TU, typename TV, typename TMask,
          typename AccumT,     typename SemiringT>
Info eWiseAdd(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
    const Vector<TU>* u, const Vector<TV>* v, Descriptor* desc) {
  CHECK(settle(u, v, w, mask));
  const void* out = reinterpret_cast<const void*>(w);
  // an operand that is w is dense by the time the kernels run
  const bool u_sparse = u->vec_type_ == GrB_SPARSE && reinterpret_cast<const void*>(u) != out;
  const bool v_sparse = v->vec_type_ == GrB_SPARSE && reinterpret_cast<const void*>(v) != out;
  if (mask != NULL) {
    std::cout << "Error: Masked eWiseAdd not implemented yet!\n";
    return GrB_SUCCESS;
  }
  if (u_sparse && v_sparse) {
    std::cout << "Error: eWiseAdd sparse-sparse not implemented yet!\n";
    return GrB_SUCCESS;
  }
  if (reinterpret_cast<const void*>(u) == out && u->vec_type_ == GrB_SPARSE)
    const_cast<Vector<TU>*>(u)->sparse2dense(op.identity(), desc);
  else if (reinterpret_cast<const void*>(v) == out && v->vec_type_ == GrB_SPARSE)
    const_cast<Vector<TV>*>(v)->sparse2dense(op.identity(), desc);
  const OperandPair pair = pairOf(u, v);
  CHECK(w->setStorage(GrB_DENSE));
  switch (pair) {
    case GB_PAIR_DENSE_DENSE:
      return eWiseAddInner(&w->dense_, mask, accum, op, &u->dense_, &v->dense_, desc);
    case GB_PAIR_SPARSE_SPARSE:
      return eWiseAddInner(&w->dense_, mask, accum, op, &u->sparse_, &v->sparse_, desc);
    case GB_PAIR_SPARSE_DENSE:
      return eWiseAddInner(&w->dense_, mask, accum, op, &u->sparse_, &v->dense_,
          false, desc);
    case GB_PAIR_DENSE_SPARSE:          // operands swapped, the kernel is told
      return eWiseAddInner(&w->dense_, mask, accum, op, &v->sparse_, &u->dense_,
          true, desc);
    default:
      std::cout << "Error: eWiseAdd backend invalid choice!\n";
      return GrB_INVALID_OBJECT;
  }
}

template <typename TC, typename TA, typename TB, typename TMask,
          typename AccumT,     typename SemiringT>
Info eWiseAdd(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, SemiringT op,
    const Matrix<TA>* A, const Matrix<TB>* B, Descriptor* desc) {
  return ewiseMatrixDispatch<true>(C, mask, op, A, B, desc);
}

// ---- extract (extract.hpp) --------------------------------------------------------
// Host index lists, NULL = GrB_ALL.  A mask and a dense matrix are refused before
// anything changes; a dense C turns sparse only once the result has replaced it.

// C = op(A)(I, J); C may be A.
template <typename TC, typename TMask, typename TA, typename AccumT>
Info extract(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, const Matrix<TA>* A,
    const std::vector<Index>* row_indices, Index nrows,
    const std::vector<Index>* col_indices, Index ncols, Descriptor* desc) {
  if (mask != NULL) return notBuilt("masked extract");
  if (!A->isSparse()) return notBuilt("extract from a dense matrix");
  Desc_value inp0_mode;
  CHECK(desc->get(GrB_INP0, &inp0_mode));
  const bool was_dense = C->isDense();
  if (!was_dense) CHECK(C->setStorage(GrB_SPARSE));
  const Info info = extractMatrix(&C->sparse_, &A->sparse_, inp0_mode == GrB_TRAN,
      row_indices, nrows, col_indices, ncols);
  if (info == GrB_SUCCESS && was_dense) CHECK(C->setStorage(GrB_SPARSE));
  return info;
}

// w = op(A)(I, j), sparse.
template <typename TW, typename TMask, typename TA, typename AccumT>
Info extract(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, const Matrix<TA>* A,
    const std::vector<Index>* row_indices, Index nrows, Index col_index, Descriptor* desc) {
  if (mask != NULL) return notBuilt("masked extract");
  if (!A->isSparse()) return notBuilt("extract from a dense matrix");
  Desc_value inp0_mode;
  CHECK(desc->get(GrB_INP0, &inp0_mode));
  CHECK(settle(w));
  return extractColumn(w, &A->sparse_, inp0_mode == GrB_TRAN, row_indices, nrows, col_index);
}

// w = u(I): dense for a dense u, sparse for a sparse u.
template <typename TW, typename TMask, typename TU, typename AccumT>
Info extract(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, const Vector<TU>* u,
    const std::vector<Index>* indices, Index nindices, Descriptor* desc) {
  if (mask != NULL) return notBuilt("masked extract");
  CHECK(settle(w));
  return extractVector(w, u, indices, nindices);
}

// ---- assign into a matrix (assign_matrix.hpp) ----------------------------------------
// Host index lists, NULL = GrB_ALL.  A mask, a dense C and a dense A are refused
// before anything changes; C turns sparse once the result has replaced it (a C
// never built counts as empty).

// Whether a matrix assign can run on C: no mask and a C that is not dense.
template <typename TC, typename TMask>
Info assignTarget(const Matrix<TC>* C, const TMask* mask) {
  if (mask != NULL) return notBuilt("masked assign");
  if (C->isDense()) return notBuilt("assign into a dense matrix");
  return GrB_SUCCESS;
}

// C(I, J) = accum(C(I, J), op(A)); C may be A.
template <typename TC, typename TMask, typename TA, typename AccumT>
Info assign(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, const Matrix<TA>* A,
    const std::vector<Index>* row_indices, Index nrows,
    const std::vector<Index>* col_indices, Index ncols, Descriptor* desc) {
  CHECK(assignTarget(C, mask));
  if (!A->isSparse()) return notBuilt("assign from a dense matrix");
  Desc_value inp0_mode;
  CHECK(desc->get(GrB_INP0, &inp0_mode));
  CHECK(assignMatrix(&C->sparse_, accum, &A->sparse_, inp0_mode == GrB_TRAN, row_indices,
                     nrows, col_indices, ncols));
  return C->setStorage(GrB_SPARSE);
}

// C(I, j) = accum(C(I, j), u).
template <typename TC, typename TMask, typename TU, typename AccumT>
Info assign(Matrix<TC>* C, const Vector<TMask>* mask, AccumT accum, const Vector<TU>* u,
    const std::vector<Index>* row_indices, Index nrows, Index col_index, Descriptor* desc) {
  CHECK(assignTarget(C, mask));
  CHECK(assignVector<true>(&C->sparse_, accum, u, row_indices, nrows, col_index));
  return C->setStorage(GrB_SPARSE);
}

// C(i, J) = accum(C(i, J), u).
template <typename TC, typename TMask, typename TU, typename AccumT>
Info assign(Matrix<TC>* C, const Vector<TMask>* mask, AccumT accum, const Vector<TU>* u,
    Index row_index, const std::vector<Index>* col_indices, Index ncols, Descriptor* desc) {
  CHECK(assignTarget(C, mask));
  CHECK(assignVector<false>(&C->sparse_, accum, u, col_indices, ncols, row_index));
  return C->setStorage(GrB_SPARSE);
}

// C(I, J) = accum(C(I, J), val).
template <typename TC, typename TMask, typename TS, typename AccumT>
Info assign(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, TS val,
    const std::vector<Index>* row_indices, Index nrows,
    const std::vector<Index>* col_indices, Index ncols, Descriptor* desc) {
  CHECK(assignTarget(C, mask));
  CHECK(assignConstant(&C->sparse_, accum, val, row_indices, nrows, col_indices, ncols));
  return C->setStorage(GrB_SPARSE);
}

// C = Aᵀ (C = A when GrB_INP0 is GrB_TRAN); C may be A.
template <typename TC, typename TMask, typename TA, typename AccumT>
Info transpose(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum,
    const Matrix<TA>* A, Descriptor* desc) {
  if (mask != NULL) return notBuilt("masked transpose");
  if (!A->isSparse()) return notBuilt("transpose of a dense matrix");
  Desc_value inp0_mode;
  CHECK(desc->get(GrB_INP0, &inp0_mode));
  const bool was_dense = C->isDense();
  if (!was_dense) CHECK(C->setStorage(GrB_SPARSE));
  const Info info = transposeSparse(&C->sparse_, &A->sparse_, inp0_mode == GrB_TRAN);
  if (info == GrB_SUCCESS && was_dense) CHECK(C->setStorage(GrB_SPARSE));
  return info;
}

// Extension: vector (+) broadcast scalar
template <typename TW, typename TU, typename TV, typename TMask,
          typename AccumT,     typename SemiringT>
Info eWiseAdd(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
    const Vector<TU>* u, TV val, Descriptor* desc) {
  CHECK(settle(u, w));
  const Storage u_type = u->vec_type_;
  if (u_type != GrB_DENSE && u_type != GrB_SPARSE) return GrB_INVALID_OBJECT;
  if (mask != NULL) return notBuilt("masked eWiseAdd of a vector and a scalar");
  CHECK(w->setStorage(GrB_DENSE));
  if (u_type == GrB_DENSE)
    return eWiseAddInner(&w->dense_, mask, accum, op, &u->dense_, val, desc);
  return eWiseAddInner(&w->dense_, mask, accum, op, &u->sparse_, val, desc);
}

// Masked constant assign.  The target is written in part, so its lazily held
// values are written out first; a dense mask is read through its bitmap shadow
// when that is current, except by the sparse-target filter, which reads values.
template <typename TW, typename TS, typename TMask,
          typename AccumT>
Info assign(Vector<TW>* w, Vector<TMask>* mask, AccumT accum, TS val,
    const Vector<Index>* indices, Index nindices, Descriptor* desc) {
  if (desc->debug()) std::cout << "===Begin assign===\nInput: " << val << std::endl;
  CHECK(settle(w));
  if (w->vec_type_ == GrB_SPARSE) {
    CHECK(settle(mask));
    CHECK(assignSparse(&w->sparse_, mask, accum, val, indices, nindices, desc));
  } else if (w->vec_type_ == GrB_DENSE) {
    CHECK(assignDense(&w->dense_, mask, accum, val, indices, nindices, desc));
  }
  if (desc->debug()) {
    std::cout << "===End assign===\n";
    CHECK(w->print());
  }
  return GrB_SUCCESS;
}

template <typename TW, typename TU, typename TMask,
          typename AccumT,     typename UnaryOpT>
Info apply(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, UnaryOpT op,
    const Vector<TU>* u, Descriptor* desc) {
  Vector<TU>* source = const_cast<Vector<TU>*>(u);
  CHECK(settle(u, w, mask));
  if (u->vec_type_ == GrB_SPARSE) {
    CHECK(w->setStorage(GrB_SPARSE));
    return applyStored(&w->sparse_, mask, op, &source->sparse_, desc, "a sparse vector");
  }
  if (u->vec_type_ == GrB_DENSE) {
    CHECK(w->setStorage(GrB_DENSE));
    return applyStored(&w->dense_, mask, op, &source->dense_, desc, "a dense vector");
  }
  return GrB_UNINITIALIZED_OBJECT;
}

template <typename TC, typename TA, typename TMask,
          typename AccumT,     typename UnaryOpT>
Info apply(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, UnaryOpT op,
    const Matrix<TA>* A, Descriptor* desc) {
  Matrix<TA>* source = const_cast<Matrix<TA>*>(A);
  if (A->isSparse()) {
    CHECK(C->setStorage(GrB_SPARSE));
    return applyStored(&C->sparse_, mask, op, &source->sparse_, desc, "a sparse matrix");
  }
  if (A->isDense()) return notBuilt("apply on a dense matrix");
  return GrB_UNINITIALIZED_OBJECT;
}

// matrix rows -> vector
template <typename TW, typename TA, typename TMask,
          typename AccumT,     typename MonoidT>
Info reduce(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, MonoidT op,
    const Matrix<TA>* A, Descriptor* desc) {
  CHECK(w->setStorage(GrB_DENSE));
  if (mask != NULL) return notBuilt("masked reduce");
  if (A->isSparse()) return reduceRows(&w->dense_, op, &A->sparse_, desc);
  if (A->isDense())  return notBuilt("row reduce of a dense matrix");
  return GrB_UNINITIALIZED_OBJECT;
}

// vector -> scalar
template <typename TS, typename TU,
          typename AccumT, typename MonoidT>
Info reduce(TS* val, AccumT accum, MonoidT op, const Vector<TU>* u, Descriptor* desc) {
  if (u->vec_type_ == GrB_SPARSE)
    CHECK(reduceStored(val, accum, op, &u->sparse_, desc));
  else if (u->vec_type_ == GrB_DENSE)
    CHECK(reduceDense(val, accum, op, const_cast<DenseVector<TU>*>(&u->dense_), desc));
  else
    return GrB_UNINITIALIZED_OBJECT;
  if (desc->debug()) std::cout << "reduce output: " << *val << std::endl;
  return GrB_SUCCESS;
}

// matrix -> scalar
template <typename TS, typename TA,
          typename AccumT,     typename MonoidT>
Info reduce(TS* val, AccumT accum, MonoidT op, const Matrix<TA>* A, Descriptor* desc) {
  if (A->isSparse()) return reduceStored(val, accum, op, &A->sparse_, desc);
  if (A->isDense())  return notBuilt("reduce of a dense matrix to a scalar");
  return GrB_UNINITIALIZED_OBJECT;
}

// ---- index-driven vector operations (indexed.hpp) ------------------------------

template <typename TW, typename TMask, typename TU, typename TS>
Info scatter(Vector<TW>* w, const Vector<TMask>* mask, const Vector<TU>* u, TS val,
    Descriptor* desc) {
  return scatterConstant(w, mask, u, val, desc);
}

template <typename TW, typename TU, typename TMask, typename TIndex,
          typename AccumT>
Info assignScatter(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum,
    const Vector<TU>* u, const Vector<TIndex>* indices, Descriptor* desc) {
  return indexedMove<false>(w, mask, u, indices, desc);
}

template <typename TW, typename TU, typename TMask, typename TIndex,
          typename AccumT>
Info extractGather(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum,
    const Vector<TU>* u, const Vector<TIndex>* indices, Descriptor* desc) {
  return indexedMove<true>(w, mask, u, indices, desc);
}

template <typename TC, typename TA>
Info tril(Matrix<TC>* C, Matrix<TA>* A, Descriptor* desc) {
  if (reinterpret_cast<void*>(C) != reinterpret_cast<void*>(A)) CHECK(C->dup(A));
  if (!A->isSparse()) return notBuilt("tril of a dense matrix");
  CHECK(C->setStorage(GrB_SPARSE));
  return trilSparse(&C->sparse_, &A->sparse_, desc);
}
}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_OPERATIONS_HPP_
