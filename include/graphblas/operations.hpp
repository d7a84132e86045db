// graphblast_b200 frontend mirror — the GraphBLAS operation templates.
//
// Same entry points, template-argument order and return codes as reference
// graphblas/operations.hpp:13-889 (callers name the value types explicitly:
// vxm<float, float, float, float>(...)).  An operation here is three statements:
//   1. its required operands are present   (else GrB_UNINITIALIZED_OBJECT; vxm / mxv
//      also refuse an input vector without stored values, reference :71-74, :111-114),
//   2. its shape contract holds            (else GrB_DIMENSION_MISMATCH; an absent
//      optional operand — the mask — satisfies every relation it appears in),
//   3. the backend objects are handed to backend::<op>.
// Variants the reference only declares answer GrB_NOT_IMPLEMENTED.
#ifndef GRAPHBLAS_OPERATIONS_HPP_
#define GRAPHBLAS_OPERATIONS_HPP_

#include <iostream>
#include <type_traits>
#include <vector>

#include <graphblas/backend/cuda/operations.hpp>

namespace graphblas {

namespace ops_detail {

// ---- 1. presence -------------------------------------------------------------------
inline bool anyAbsent() { return false; }
template <typename First, typename... Rest>
bool anyAbsent(const First* first, const Rest*... rest) {
  return first == NULL || anyAbsent(rest...);
}
template <typename T>
bool holdsNothing(const Vector<T>* u) {
  Index stored = 0;
  return u->nvals(&stored) != GrB_SUCCESS || stored == 0;
}

// ---- 2. shapes ---------------------------------------------------------------------
// One extent of an operand; `known` is false for an absent (optional) operand.
struct Extent {
  Index n;
  bool  known;
};
template <typename T> Extent rowsOf(const Matrix<T>* m) {
  Extent e = {0, m != NULL};
  if (e.known) m->nrows(&e.n);
  return e;
}
template <typename T> Extent colsOf(const Matrix<T>* m) {
  Extent e = {0, m != NULL};
  if (e.known) m->ncols(&e.n);
  return e;
}
template <typename T> Extent sizeOf(const Vector<T>* v) {
  Extent e = {0, v != NULL};
  if (e.known) v->size(&e.n);
  return e;
}
// stored entries of a vector: the count the index-driven operations run over
template <typename T> Extent nvalsOf(const Vector<T>* v) {
  Extent e = {0, v != NULL};
  if (e.known) v->nvals(&e.n);
  return e;
}
// A shape contract: relations are added one by one, the first one that fails is
// reported (with the reference's wording) and remembered.
class Contract {
 public:
  Contract() : verdict_(GrB_SUCCESS) {}
  Contract& equal(Extent lhs, Extent rhs, const char* broken) {
    if (verdict_ == GrB_SUCCESS && lhs.known && rhs.known && lhs.n != rhs.n) {
      std::cout << broken << std::endl;
      verdict_ = GrB_DIMENSION_MISMATCH;
    }
    return *this;
  }
  Contract& atMost(Extent lhs, Extent rhs, const char* broken) {
    if (verdict_ == GrB_SUCCESS && lhs.known && rhs.known && lhs.n > rhs.n) {
      std::cout << broken << std::endl;
      verdict_ = GrB_DIMENSION_MISMATCH;
    }
    return *this;
  }
  // two matrices of one shape
  template <typename X, typename Y>
  Contract& alike(const Matrix<X>* x, const Matrix<Y>* y, const char* rows_broken,
                  const char* cols_broken) {
    return equal(rowsOf(x), rowsOf(y), rows_broken).equal(colsOf(x), colsOf(y), cols_broken);
  }
  Info verdict() const { return verdict_; }
 private:
  Info verdict_;
};

// ---- 3. backend objects ------------------------------------------------------------
template <typename T> const backend::Vector<T>* raw(const Vector<T>* v) { return v ? &v->vector_ : NULL; }
template <typename T> backend::Vector<T>*       raw(Vector<T>* v)       { return v ? &v->vector_ : NULL; }
template <typename T> const backend::Matrix<T>* raw(const Matrix<T>* m) { return m ? &m->matrix_ : NULL; }
template <typename T> backend::Matrix<T>*       raw(Matrix<T>* m)       { return m ? &m->matrix_ : NULL; }
inline backend::Descriptor*                     raw(Descriptor* d)      { return d ? &d->descriptor_ : NULL; }

// Shapes of an element-wise operation on two matrices: op(A), op(B) and C alike,
// op(X) being Xᵀ when GrB_INP0 / GrB_INP1 is GrB_TRAN.
template <typename TC, typename TMask, typename TA, typename TB>
Contract ewiseShapes(const Matrix<TC>* C, const Matrix<TMask>* mask, const Matrix<TA>* A,
                     const Matrix<TB>* B, Descriptor* desc) {
  Desc_value inp0 = GrB_DEFAULT, inp1 = GrB_DEFAULT;
  desc->get(GrB_INP0, &inp0);
  desc->get(GrB_INP1, &inp1);
  const bool ta = inp0 == GrB_TRAN, tb = inp1 == GrB_TRAN;
  return Contract()
      .equal(ta ? colsOf(A) : rowsOf(A), rowsOf(C), "op(A).nrows != C.nrows")
      .equal(ta ? rowsOf(A) : colsOf(A), colsOf(C), "op(A).ncols != C.ncols")
      .equal(tb ? colsOf(B) : rowsOf(B), rowsOf(C), "op(B).nrows != C.nrows")
      .equal(tb ? rowsOf(B) : colsOf(B), colsOf(C), "op(B).ncols != C.ncols")
      .alike(C, mask, "C.nrows != mask.nrows", "C.ncols != mask.ncols");
}

inline Info declaredOnly(const char* what) {
  std::cout << "Error: " << what << " not implemented yet!\n";
  return GrB_NOT_IMPLEMENTED;
}
}  // namespace ops_detail

#define GB_REQUIRE(...) \
  if (ops_detail::anyAbsent(__VA_ARGS__)) return GrB_UNINITIALIZED_OBJECT
#define GB_SHAPES(contract) \
  do { const Info gb_shape__ = (contract).verdict(); \
       if (gb_shape__ != GrB_SUCCESS) return gb_shape__; } while (0)

// ---- products ------------------------------------------------------------------------

// C<mask> = accum(C, A (+.x) B)
template <typename TC, typename TMask, typename TA, typename TB, typename AccumT,
          typename SemiringT>
Info mxm(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, SemiringT op,
         const Matrix<TA>* A, const Matrix<TB>* B, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, A, B, desc);
  if (mask == NULL) {
    // the unmasked product multiplies op(A) by op(B), with op what GrB_INP0 /
    // GrB_INP1 name: its shapes are those of the transposes
    Desc_value inp0, inp1;
    CHECK(desc->get(GrB_INP0, &inp0));
    CHECK(desc->get(GrB_INP1, &inp1));
    const bool ta = inp0 == GrB_TRAN, tb = inp1 == GrB_TRAN;
    GB_SHAPES(Contract()
        .equal(tb ? colsOf(B) : rowsOf(B), ta ? rowsOf(A) : colsOf(A),
               "op(B).nrows != op(A).ncols")
        .equal(ta ? colsOf(A) : rowsOf(A), rowsOf(C), "op(A).nrows != C.nrows")
        .equal(tb ? rowsOf(B) : colsOf(B), colsOf(C), "op(B).ncols != C.ncols"));
  } else {
    GB_SHAPES(Contract()
        .equal(rowsOf(B), colsOf(A), "B.nrows != A.ncols")
        .equal(rowsOf(A), rowsOf(C), "A.nrows != C.nrows")
        .equal(colsOf(B), colsOf(C), "B.ncols != C.ncols")
        .alike(C, mask, "C.nrows != mask.nrows", "C.ncols != mask.ncols"));
  }
  return backend::mxm<TC, TA, TB, TMask>(raw(C), raw(mask), accum, op, raw(A), raw(B),
                                        raw(desc));
}

// w<mask> = accum(w, u (+.x) A)
template <typename TW, typename TMask, typename TU, typename TA, typename AccumT,
          typename SemiringT>
Info vxm(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
         const Vector<TU>* u, const Matrix<TA>* A, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, u, A, desc);
  if (holdsNothing(u)) return GrB_UNINITIALIZED_OBJECT;
  GB_SHAPES(Contract()
      .equal(rowsOf(A), sizeOf(u), "A.nrows != u.size")
      .equal(colsOf(A), sizeOf(w), "A.ncols != w.size")
      .equal(sizeOf(w), sizeOf(mask), "w.size  != mask.size"));
  return backend::vxm<TW, TU, TA, TMask>(raw(w), raw(mask), accum, op, raw(u), raw(A),
                                        raw(desc));
}

// w<mask> = accum(w, A (+.x) u)
template <typename TW, typename TMask, typename TA, typename TU, typename AccumT,
          typename SemiringT>
Info mxv(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
         const Matrix<TA>* A, const Vector<TU>* u, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, u, A, desc);
  if (holdsNothing(u)) return GrB_UNINITIALIZED_OBJECT;
  GB_SHAPES(Contract()
      .equal(colsOf(A), sizeOf(u), "A.ncols != u.size")
      .equal(rowsOf(A), sizeOf(w), "A.nrows != w.size")
      .equal(sizeOf(w), sizeOf(mask), "w.size  != mask.size"));
  return backend::mxv<TW, TU, TA, TMask>(raw(w), raw(mask), accum, op, raw(A), raw(u),
                                        raw(desc));
}

// Extension: vxm fused with an apply on the input (declared by the reference, not built)
template <typename TW, typename TMask, typename TU, typename TA, typename AccumT,
          typename SemiringT>
Info applyVxm(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
              const Vector<TU>* u, const Matrix<TA>* A, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, u, A, desc);
  if (holdsNothing(u)) return GrB_UNINITIALIZED_OBJECT;
  GB_SHAPES(Contract()
      .equal(rowsOf(A), sizeOf(u), "A.nrows != u.size")
      .equal(colsOf(A), sizeOf(w), "A.ncols != w.size")
      .equal(sizeOf(w), sizeOf(mask), "w.size  != mask.size"));
  return backend::applyVxm<TW, TU, TA, TMask>(raw(w), raw(mask), accum, op, raw(u), raw(A),
                                             raw(desc));
}

// Extension: val = trace(A * B^T)
template <typename T, typename TA, typename TB, typename SemiringT>
Info traceMxmTranspose(T* val, SemiringT op, const Matrix<TA>* A, const Matrix<TB>* B,
                       Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(val, A, B, desc);
  return backend::traceMxmTranspose(val, op, raw(A), raw(B), raw(desc));
}

// ---- element-wise ----------------------------------------------------------------------

// w<mask> = accum(w, u .* v)
template <typename TW, typename TMask, typename TU, typename TV, typename AccumT,
          typename SemiringT>
Info eWiseMult(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
               const Vector<TU>* u, const Vector<TV>* v, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, u, v, desc);
  GB_SHAPES(Contract()
      .equal(sizeOf(u), sizeOf(v), "u.size != v.size")
      .equal(sizeOf(u), sizeOf(w), "u.size != w.size")
      .equal(sizeOf(u), sizeOf(mask), "u.size != mask.size"));
  return backend::eWiseMult(raw(w), raw(mask), accum, op, raw(u), raw(v), raw(desc));
}

// C<mask> = accum(C, op(A) .* op(B)), op what GrB_INP0 / GrB_INP1 name: the
// shapes compared are those of the transposes
template <typename TC, typename TMask, typename TA, typename TB, typename AccumT,
          typename SemiringT>
Info eWiseMult(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, SemiringT op,
               const Matrix<TA>* A, const Matrix<TB>* B, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, A, B, desc);
  GB_SHAPES(ewiseShapes(C, mask, A, B, desc));
  return backend::eWiseMult(raw(C), raw(mask), accum, op, raw(A), raw(B), raw(desc));
}

// Extension: C = A .* val (scalar broadcast)
template <typename TC, typename TMask, typename TA, typename TScalar, typename AccumT,
          typename SemiringT>
Info eWiseMult(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, SemiringT op,
               const Matrix<TA>* A, TScalar val, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, A, desc);
  GB_SHAPES(Contract()
      .alike(A, C, "A.nrows != C.nrows", "A.ncols != C.ncols")
      .alike(A, mask, "A.nrows != mask.nrows", "A.ncols != mask.ncols"));
  return backend::eWiseMult(raw(C), raw(mask), accum, op, raw(A), val, raw(desc));
}

// Extension: C = A .* B with a vector B broadcast along rows (along columns when
// GrB_INP1 is GrB_TRAN)
template <typename TC, typename TMask, typename TA, typename TB, typename AccumT,
          typename SemiringT>
Info eWiseMult(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, SemiringT op,
               const Matrix<TA>* A, const Vector<TB>* B, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, A, B, desc);
  GB_SHAPES(Contract()
      .alike(A, C, "A.nrows != C.nrows", "A.ncols != C.ncols")
      .alike(A, mask, "A.nrows != mask.nrows", "A.ncols != mask.ncols"));
  return backend::eWiseMult(raw(C), raw(mask), accum, op, raw(A), raw(B), raw(desc));
}

// w<mask> = accum(w, u + v)
template <typename TW, typename TMask, typename TU, typename TV, typename AccumT,
          typename SemiringT>
Info eWiseAdd(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
              const Vector<TU>* u, const Vector<TV>* v, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, u, v, desc);
  GB_SHAPES(Contract()
      .equal(sizeOf(u), sizeOf(v), "u.size != v.size")
      .equal(sizeOf(u), sizeOf(w), "u.size != w.size")
      .equal(sizeOf(u), sizeOf(mask), "u.size != mask.size")
      .equal(sizeOf(v), sizeOf(mask), "v.size != mask.size")
      .equal(sizeOf(w), sizeOf(mask), "w.size != mask.size"));
  return backend::eWiseAdd(raw(w), raw(mask), accum, op, raw(u), raw(v), raw(desc));
}

// Extension: w = u + val (scalar broadcast)
template <typename TW, typename TMask, typename TU, typename TScalar, typename AccumT,
          typename SemiringT>
Info eWiseAdd(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, SemiringT op,
              const Vector<TU>* u, TScalar val, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, u, desc);
  GB_SHAPES(Contract()
      .equal(sizeOf(u), sizeOf(w), "u.size != w.size")
      .equal(sizeOf(u), sizeOf(mask), "u.size != mask.size"));
  return backend::eWiseAdd(raw(w), raw(mask), accum, op, raw(u), val, raw(desc));
}

// C<mask> = accum(C, op(A) + op(B)), shapes as in the matrix eWiseMult
template <typename TC, typename TMask, typename TA, typename TB, typename AccumT,
          typename SemiringT>
Info eWiseAdd(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, SemiringT op,
              const Matrix<TA>* A, const Matrix<TB>* B, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, A, B, desc);
  GB_SHAPES(ewiseShapes(C, mask, A, B, desc));
  return backend::eWiseAdd(raw(C), raw(mask), accum, op, raw(A), raw(B), raw(desc));
}

// C<mask> = accum(C, Aᵀ); C = A when GrB_INP0 is GrB_TRAN (the transpose of the
// transposed input)
template <typename TC, typename TMask, typename TA, typename AccumT>
Info transpose(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, const Matrix<TA>* A,
               Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, A, desc);
  Desc_value inp0;
  CHECK(desc->get(GrB_INP0, &inp0));
  const bool ta = inp0 == GrB_TRAN;
  GB_SHAPES(Contract()
      .equal(ta ? rowsOf(A) : colsOf(A), rowsOf(C), "C.nrows != A.ncols")
      .equal(ta ? colsOf(A) : rowsOf(A), colsOf(C), "C.ncols != A.nrows")
      .alike(C, mask, "C.nrows != mask.nrows", "C.ncols != mask.ncols"));
  return backend::transpose(raw(C), raw(mask), accum, raw(A), raw(desc));
}

// ---- apply, reduce, tril -----------------------------------------------------------------

// w<mask> = accum(w, op(u))
template <typename TW, typename TMask, typename TU, typename AccumT, typename UnaryOpT>
Info apply(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, UnaryOpT op,
           const Vector<TU>* u, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, u);
  GB_SHAPES(Contract()
      .equal(sizeOf(u), sizeOf(w), "u.size != w.size")
      .equal(sizeOf(u), sizeOf(mask), "u.size != mask.size"));
  return backend::apply(raw(w), raw(mask), accum, op, raw(u), raw(desc));
}

// C<mask> = accum(C, op(A))
template <typename TC, typename TMask, typename TA, typename AccumT, typename UnaryOpT>
Info apply(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, UnaryOpT op,
           const Matrix<TA>* A, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, A);
  GB_SHAPES(Contract()
      .alike(A, C, "A.nrows != C.nrows", "A.ncols != C.ncols")
      .alike(A, mask, "A.nrows != mask.nrows", "A.ncols != mask.ncols"));
  return backend::apply(raw(C), raw(mask), accum, op, raw(A), raw(desc));
}

// w<mask> = accum(w, reduce rows of A)
template <typename TW, typename TMask, typename TA, typename AccumT, typename MonoidT>
Info reduce(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, MonoidT op,
            const Matrix<TA>* A, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, A, desc);
  GB_SHAPES(Contract()
      .equal(rowsOf(A), sizeOf(w), "A.nrows != w.size")
      .equal(sizeOf(w), sizeOf(mask), "w.size  != mask.size"));
  return backend::reduce(raw(w), raw(mask), accum, op, raw(A), raw(desc));
}

// val = reduce(u)
template <typename T, typename TU, typename AccumT, typename MonoidT>
Info reduce(T* val, AccumT accum, MonoidT op, const Vector<TU>* u, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(val, u);
  return backend::reduce(val, accum, op, raw(u), raw(desc));
}

// val = reduce(A)
template <typename T, typename TA, typename AccumT, typename MonoidT>
Info reduce(T* val, AccumT accum, MonoidT op, const Matrix<TA>* A, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(val, A);
  return backend::reduce(val, accum, op, raw(A), raw(desc));
}

// Extension: C = lower triangle of A (row >= col)
template <typename TC, typename TA>
Info tril(Matrix<TC>* C, Matrix<TA>* A, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, A, desc);
  GB_SHAPES(Contract().alike(A, C, "A.nrows != C.nrows", "A.ncols != C.ncols"));
  return backend::tril(raw(C), raw(A), raw(desc));
}

template <typename TW, typename TA>
Info graphColor(Vector<TW>* w, const Matrix<TA>* A, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, A, desc);
  return backend::graphColor(raw(w), raw(A), raw(desc));
}

// ---- assign and the index-driven operations -------------------------------------------

// w<mask>[indices] = val (constant assign)
template <typename TW, typename TMask, typename TScalar, typename TIndex, typename AccumT>
Info assign(Vector<TW>* w, Vector<TMask>* mask, AccumT accum, TScalar val,
            const Vector<TIndex>* indices, Index nindices, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, desc);
  GB_SHAPES(Contract().equal(sizeOf(w), sizeOf(mask), "w.size  != mask.size"));
  return backend::assign(raw(w), raw(mask), accum, val, raw(indices), nindices, raw(desc));
}

template <typename TW, typename TMask, typename TU, typename AccumT>
Info assignIndexed(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum,
                   const Vector<TU>* u, int* indices, Index nindices, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, u, desc);
  GB_SHAPES(Contract().equal(sizeOf(w), sizeOf(mask), "w.size  != mask.size"));
  return backend::assignIndexed(raw(w), raw(mask), accum, raw(u), indices, nindices,
                                raw(desc));
}

// Extension: w[indices[i]] = mask .* val
template <typename TW, typename TMask, typename TIndex, typename TScalar>
Info scatter(Vector<TW>* w, const Vector<TMask>* mask, const Vector<TIndex>* indices,
             TScalar val, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(indices, w);
  return backend::scatter(raw(w), raw(mask), raw(indices), val, raw(desc));
}

// Extension: w[indices[i]] = u[i]
template <typename TW, typename TMask, typename TU, typename TIndex, typename AccumT>
Info assignScatter(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum,
                   const Vector<TU>* u, const Vector<TIndex>* indices, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, u, indices, desc);
  GB_SHAPES(Contract()
      .equal(sizeOf(w), sizeOf(mask), "w.size  != mask.size")
      .atMost(nvalsOf(indices), sizeOf(u), "indices.nvals > u.size"));
  return backend::assignScatter(raw(w), raw(mask), accum, raw(u), raw(indices), raw(desc));
}

// Extension: w[i] = u[indices[i]]
template <typename TW, typename TMask, typename TU, typename TIndex, typename AccumT>
Info extractGather(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum,
                   const Vector<TU>* u, const Vector<TIndex>* indices, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(u, w, indices, desc);
  GB_SHAPES(Contract()
      .equal(sizeOf(w), sizeOf(mask), "w.size  != mask.size")
      .atMost(nvalsOf(indices), sizeOf(w), "indices.nvals > w.size"));
  return backend::extractGather(raw(w), raw(mask), accum, raw(u), raw(indices), raw(desc));
}

// ---- extract ---------------------------------------------------------------------------
// Host index lists; GrB_ALL (NULL) means every index of that extent.  C (or w) is
// replaced: accum is not applied.  The backend refuses an index out of range
// (GrB_INVALID_INDEX) before anything changes.

// w<mask> = u(indices)
template <typename TW, typename TMask, typename TU, typename AccumT>
Info extract(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, const Vector<TU>* u,
             const std::vector<Index>* indices, Index nindices, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, u, desc);
  GB_SHAPES(Contract()
      .equal(sizeOf(w), Extent{nindices, true}, "w.size != nindices")
      .equal(sizeOf(w), sizeOf(mask), "w.size != mask.size"));
  return backend::extract(raw(w), raw(mask), accum, raw(u), indices, nindices, raw(desc));
}

// C<mask> = op(A)(row_indices, col_indices), op(A) = Aᵀ when GrB_INP0 is GrB_TRAN
template <typename TC, typename TMask, typename TA, typename AccumT>
Info extract(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, const Matrix<TA>* A,
             const std::vector<Index>* row_indices, Index nrows,
             const std::vector<Index>* col_indices, Index ncols, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, A, desc);
  GB_SHAPES(Contract()
      .equal(rowsOf(C), Extent{nrows, true}, "C.nrows != nrows")
      .equal(colsOf(C), Extent{ncols, true}, "C.ncols != ncols")
      .alike(C, mask, "C.nrows != mask.nrows", "C.ncols != mask.ncols"));
  return backend::extract(raw(C), raw(mask), accum, raw(A), row_indices, nrows, col_indices,
                          ncols, raw(desc));
}

// w<mask> = op(A)(row_indices, col_index), op(A) = Aᵀ when GrB_INP0 is GrB_TRAN
template <typename TW, typename TMask, typename TA, typename AccumT>
Info extract(Vector<TW>* w, const Vector<TMask>* mask, AccumT accum, const Matrix<TA>* A,
             const std::vector<Index>* row_indices, Index nrows, Index col_index,
             Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(w, A, desc);
  Desc_value inp0;
  CHECK(desc->get(GrB_INP0, &inp0));
  GB_SHAPES(Contract()
      .equal(sizeOf(w), Extent{nrows, true}, "w.size != nrows")
      .atMost(Extent{col_index + 1, true}, inp0 == GrB_TRAN ? rowsOf(A) : colsOf(A),
              "col_index >= op(A).ncols")
      .equal(sizeOf(w), sizeOf(mask), "w.size != mask.size"));
  return backend::extract(raw(w), raw(mask), accum, raw(A), row_indices, nrows, col_index,
                          raw(desc));
}

// ---- assign into a matrix -----------------------------------------------------------
// Host index lists; GrB_ALL (NULL) means every index of that extent, and a list may
// not repeat an index (GrB_INVALID_VALUE).  Without accum, C(I, J) takes op(A)'s
// pattern and values (entries of C inside the region that op(A) does not store are
// deleted); with accum, C(I, J) = accum(C(I, J), op(A)) over the union of the two,
// C's value first.  Outside the region C is unchanged.  The backend refuses an
// index out of range (GrB_INVALID_INDEX) before anything changes.

// C<mask>(row_indices, col_indices) = accum(C(..), op(A)), op(A) = Aᵀ when GrB_INP0
// is GrB_TRAN; op(A) is nrows x ncols
template <typename TC, typename TMask, typename TA, typename AccumT>
Info assign(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, const Matrix<TA>* A,
            const std::vector<Index>* row_indices, Index nrows,
            const std::vector<Index>* col_indices, Index ncols, Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, A, desc);
  Desc_value inp0;
  CHECK(desc->get(GrB_INP0, &inp0));
  const bool ta = inp0 == GrB_TRAN;
  GB_SHAPES(Contract()
      .equal(ta ? colsOf(A) : rowsOf(A), Extent{nrows, true}, "op(A).nrows != nrows")
      .equal(ta ? rowsOf(A) : colsOf(A), Extent{ncols, true}, "op(A).ncols != ncols")
      .alike(C, mask, "C.nrows != mask.nrows", "C.ncols != mask.ncols"));
  return backend::assign(raw(C), raw(mask), accum, raw(A), row_indices, nrows, col_indices,
                         ncols, raw(desc));
}

// C<mask>(row_indices, col_index) = accum(C(..), u), u of size nrows
template <typename TC, typename TMask, typename TU, typename AccumT>
Info assign(Matrix<TC>* C, const Vector<TMask>* mask, AccumT accum, const Vector<TU>* u,
            const std::vector<Index>* row_indices, Index nrows, Index col_index,
            Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, u, desc);
  GB_SHAPES(Contract()
      .equal(sizeOf(u), Extent{nrows, true}, "u.size != nrows")
      .atMost(Extent{col_index + 1, true}, colsOf(C), "col_index >= C.ncols")
      .equal(rowsOf(C), sizeOf(mask), "C.nrows != mask.size"));
  return backend::assign(raw(C), raw(mask), accum, raw(u), row_indices, nrows, col_index,
                         raw(desc));
}

// C<mask>(row_index, col_indices) = accum(C(..), u), u of size ncols
template <typename TC, typename TMask, typename TU, typename AccumT>
Info assign(Matrix<TC>* C, const Vector<TMask>* mask, AccumT accum, const Vector<TU>* u,
            Index row_index, const std::vector<Index>* col_indices, Index ncols,
            Descriptor* desc) {
  using namespace ops_detail;
  GB_REQUIRE(C, u, desc);
  GB_SHAPES(Contract()
      .equal(sizeOf(u), Extent{ncols, true}, "u.size != ncols")
      .atMost(Extent{row_index + 1, true}, rowsOf(C), "row_index >= C.nrows")
      .equal(colsOf(C), sizeOf(mask), "C.ncols != mask.size"));
  return backend::assign(raw(C), raw(mask), accum, raw(u), row_index, col_indices, ncols,
                         raw(desc));
}

// C<mask>(row_indices, col_indices) = accum(C(..), val): every position of the
// region ends up stored
template <typename TC, typename TMask, typename TScalar, typename AccumT>
Info assign(Matrix<TC>* C, const Matrix<TMask>* mask, AccumT accum, TScalar val,
            const std::vector<Index>* row_indices, Index nrows,
            const std::vector<Index>* col_indices, Index ncols, Descriptor* desc) {
  static_assert(std::is_arithmetic<TScalar>::value,
                "assign: val is a scalar; pass the source matrix as const Matrix<T>*");
  using namespace ops_detail;
  GB_REQUIRE(C, desc);
  GB_SHAPES(Contract().alike(C, mask, "C.nrows != mask.nrows", "C.ncols != mask.ncols"));
  return backend::assign(raw(C), raw(mask), accum, val, row_indices, nrows, col_indices,
                         ncols, raw(desc));
}

// ---- declared by the reference, implemented nowhere -------------------------------------

template <typename TB, typename TA, typename TScalar, typename MonoidT>
Info scale(Matrix<TB>* B, MonoidT op, const Matrix<TA>* A, TScalar val, Descriptor* desc) {
  return ops_detail::declaredOnly("scale matrix variant");
}
template <typename TW, typename TU, typename TScalar, typename MonoidT>
Info scale(Vector<TW>* w, MonoidT op, const Vector<TU>* u, TScalar val, Descriptor* desc) {
  return ops_detail::declaredOnly("scale vector variant");
}

#undef GB_REQUIRE
#undef GB_SHAPES

}  // namespace graphblas

#endif  // GRAPHBLAS_OPERATIONS_HPP_
