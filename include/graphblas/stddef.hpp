// graphblast_b200 frontend mirror — binary operators, monoids and semirings.
//
// Same names, template parameters, identities and host/device qualifiers as
// reference graphblas/stddef.hpp:14-277, because user code and the algorithm
// headers instantiate them by name (LogicalOrAndSemiring<float>() ...).  Notable
// identities kept as the reference defines them (:160-173): LogicalAndMonoid ->
// false, MaximumMonoid -> 0, GreaterMonoid -> numeric_limits::min().
// identity() is host-only in the reference; the backend passes it by value.
#ifndef GRAPHBLAS_STDDEF_HPP_
#define GRAPHBLAS_STDDEF_HPP_

#include <cstddef>
#include <cstdint>
#include <limits>
#include <algorithm>

// name, default (T_in2, T_out) types, expression in lhs/rhs
#define GB_DEFINE_BINARY_OP(NAME, DEF_IN1, DEF_IN2, DEF_OUT, EXPR)            \
template <typename T_in1 DEF_IN1, typename T_in2 DEF_IN2,                     \
          typename T_out DEF_OUT>                                             \
struct NAME {                                                                 \
  inline GRB_HOST_DEVICE T_out operator()(T_in1 lhs, T_in2 rhs) {             \
    return EXPR;                                                              \
  }                                                                           \
};

#define GB_SAME  = T_in1
#define GB_BOOL  = bool
#define GB_NONE

namespace graphblas {
// A float product is rounded before anything adds it: on the device __fmul_rn
// keeps the compiler from contracting mul_op and add_op into one FFMA, which
// would round a kernel's sums differently from another route's (and turn an
// overflowing product next to -FLT_MAX into a finite sum).
template <typename T_in1, typename T_in2>
inline GRB_HOST_DEVICE auto gbMul(T_in1 lhs, T_in2 rhs) -> decltype(lhs * rhs) {
  return lhs * rhs;
}
inline GRB_HOST_DEVICE float gbMul(float lhs, float rhs) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(lhs, rhs);
#else
  return lhs * rhs;
#endif
}

GB_DEFINE_BINARY_OP(logical_or,   GB_BOOL, GB_BOOL, GB_BOOL, lhs || rhs)
GB_DEFINE_BINARY_OP(logical_and,   GB_BOOL, GB_BOOL, GB_BOOL, lhs && rhs)
GB_DEFINE_BINARY_OP(logical_xor,   GB_BOOL, GB_BOOL, GB_BOOL,
                    (lhs && !rhs) || (!lhs && rhs))
GB_DEFINE_BINARY_OP(equal,         GB_NONE, GB_SAME, GB_SAME, lhs == rhs)
GB_DEFINE_BINARY_OP(not_equal_to,  GB_NONE, GB_SAME, GB_SAME, lhs != rhs)
GB_DEFINE_BINARY_OP(greater,       GB_NONE, GB_SAME, GB_BOOL, lhs > rhs)
GB_DEFINE_BINARY_OP(less,          GB_NONE, GB_SAME, GB_BOOL, lhs < rhs)
GB_DEFINE_BINARY_OP(greater_equal, GB_NONE, GB_SAME, GB_BOOL, lhs >= rhs)
GB_DEFINE_BINARY_OP(less_equal,    GB_NONE, GB_SAME, GB_BOOL, lhs <= rhs)
GB_DEFINE_BINARY_OP(first,         GB_NONE, GB_SAME, GB_SAME, lhs)
GB_DEFINE_BINARY_OP(second,        GB_NONE, GB_SAME, GB_SAME, rhs)
GB_DEFINE_BINARY_OP(minimum,       GB_NONE, GB_SAME, GB_SAME, min(lhs, rhs))
GB_DEFINE_BINARY_OP(maximum,       GB_NONE, GB_SAME, GB_SAME, max(lhs, rhs))
GB_DEFINE_BINARY_OP(plus,          GB_NONE, GB_SAME, GB_SAME, lhs + rhs)
GB_DEFINE_BINARY_OP(minus,         GB_NONE, GB_SAME, GB_SAME, lhs - rhs)
GB_DEFINE_BINARY_OP(multiplies,    GB_NONE, GB_SAME, GB_SAME, gbMul(lhs, rhs))
GB_DEFINE_BINARY_OP(divides,       GB_NONE, GB_SAME, GB_SAME, lhs / rhs)
GB_DEFINE_BINARY_OP(select_second, GB_NONE, GB_SAME, GB_SAME, rhs)
}  // namespace graphblas

#undef GB_SAME
#undef GB_BOOL
#undef GB_NONE

// The vocabulary as two lists — (name, binary operator, identity) and (name, additive
// monoid, multiplicative operator) — from which the structs are generated.  Names and
// identities are the reference's (:160-213).  "less" is not a monoid (its two-sided
// identities differ, it is not associative); it is listed anyway for the SSSP
// improvement test, as there.
#define GB_MONOID_LIST(X)                                                     \
  X(PlusMonoid,       plus,         0)                                        \
  X(MultipliesMonoid, multiplies,   1)                                        \
  X(MinimumMonoid,    minimum,      std::numeric_limits<T_out>::max())        \
  X(MaximumMonoid,    maximum,      0)                                        \
  X(LogicalOrMonoid,  logical_or,   false)                                    \
  X(LogicalAndMonoid, logical_and,  false)                                    \
  X(GreaterMonoid,    greater,      std::numeric_limits<T_out>::min())        \
  X(CustomLessMonoid, less,         std::numeric_limits<T_out>::max())        \
  X(NotEqualToMonoid, not_equal_to, std::numeric_limits<T_out>::max())

#define GB_SEMIRING_LIST(X)                                                   \
  X(LogicalOrAndSemiring,         LogicalOrMonoid,  logical_and)              \
  X(PlusMultipliesSemiring,       PlusMonoid,       multiplies)               \
  X(MinimumPlusSemiring,          MinimumMonoid,    plus)                     \
  X(MaximumMultipliesSemiring,    MaximumMonoid,    multiplies)               \
  X(PlusDividesSemiring,          PlusMonoid,       divides)                  \
  X(PlusGreaterSemiring,          PlusMonoid,       greater)                  \
  X(GreaterPlusSemiring,          GreaterMonoid,    plus)                     \
  X(PlusMinusSemiring,            PlusMonoid,       minus)                    \
  X(PlusLessSemiring,             PlusMonoid,       less)                     \
  X(CustomLessPlusSemiring,       CustomLessMonoid, plus)                     \
  X(MinimumMultipliesSemiring,    MinimumMonoid,    multiplies)               \
  X(MultipliesMultipliesSemiring, MultipliesMonoid, multiplies)               \
  X(NotEqualToPlusSemiring,       NotEqualToMonoid, plus)                     \
  X(MinimumSelectSecondSemiring,  MinimumMonoid,    select_second)            \
  X(PlusNotEqualToSemiring,       PlusMonoid,       not_equal_to)             \
  X(CustomLessLessSemiring,       CustomLessMonoid, less)                     \
  X(MinimumNotEqualToSemiring,    MinimumMonoid,    not_equal_to)

namespace graphblas {

#define GB_MAKE_MONOID(NAME, OP, IDENTITY)                                    \
template <typename T_out>                                                     \
struct NAME {                                                                 \
  inline T_out identity() const { return static_cast<T_out>(IDENTITY); }      \
  inline __host__ __device__ T_out operator()(T_out lhs, T_out rhs) const {   \
    return OP<T_out>()(lhs, rhs);                                             \
  }                                                                           \
};
GB_MONOID_LIST(GB_MAKE_MONOID)
#undef GB_MAKE_MONOID

#define GB_MAKE_SEMIRING(NAME, ADD, MUL)                                      \
template <typename T_in1, typename T_in2 = T_in1, typename T_out = T_in1>     \
struct NAME {                                                                 \
  typedef T_out result_type;                                                  \
  typedef T_out T_out_type;                                                   \
  inline T_out identity() const { return ADD<T_out>().identity(); }           \
  inline __host__ __device__ T_out add_op(T_out lhs, T_out rhs) {             \
    return ADD<T_out>()(lhs, rhs);                                            \
  }                                                                           \
  inline __host__ __device__ T_out mul_op(T_in1 lhs, T_in2 rhs) {             \
    return MUL<T_in1, T_in2, T_out>()(lhs, rhs);                              \
  }                                                                           \
};
GB_SEMIRING_LIST(GB_MAKE_SEMIRING)
#undef GB_MAKE_SEMIRING

// Functor views of a semiring's two operations (what kernels are templated on).
template <typename SemiringT, bool IsAdd>
struct SemiringOpView {
  typedef typename SemiringT::T_out_type T_out_type;
  typedef typename SemiringT::T_out_type result_type;
  typedef typename SemiringT::T_out_type first_argument_type;
  typedef typename SemiringT::T_out_type second_argument_type;

  SemiringOpView() : sr() {}
  explicit SemiringOpView(SemiringT const& s) : sr(s) {}

  inline GRB_HOST_DEVICE T_out_type identity() const { return sr.identity(); }

  template <typename T_in1, typename T_in2>
  inline GRB_HOST_DEVICE T_out_type operator()(T_in1 lhs, T_in2 rhs) {
    return IsAdd ? sr.add_op(lhs, rhs) : sr.mul_op(lhs, rhs);
  }

 private:
  SemiringT sr;
};

template <typename SemiringT>
using AdditiveMonoidFromSemiring = SemiringOpView<SemiringT, true>;
template <typename SemiringT>
using MultiplicativeMonoidFromSemiring = SemiringOpView<SemiringT, false>;

template <typename SemiringT>
AdditiveMonoidFromSemiring<SemiringT> extractAdd(SemiringT const& sr) {
  return AdditiveMonoidFromSemiring<SemiringT>(sr);
}

template <typename SemiringT>
MultiplicativeMonoidFromSemiring<SemiringT> extractMul(SemiringT const& sr) {
  return MultiplicativeMonoidFromSemiring<SemiringT>(sr);
}
}  // namespace graphblas

#endif  // GRAPHBLAS_STDDEF_HPP_
