// graphblast_b200 — PageRank power iteration as a loop of GraphBLAS operations.
//
// A is expected pre-scaled to alpha * A(i,j) / outdeg(i) (prNormalize below does
// what reference example/gpr.cu:76-86 does in the driver).  Per iteration, as
// reference graphblas/algorithm/pr.hpp:50-84:
//   p_prev = p ; p_swap = p_prev (+.x) A ; p = p_swap + (1-alpha)/n ;
//   r = p - p_prev ; r_temp = r .* r ; error = sqrt(reduce(+, r_temp)) ;
//   stop when error <= eps or after max_niter iterations.
#ifndef GRAPHBLAS_ALGORITHM_PR_HPP_
#define GRAPHBLAS_ALGORITHM_PR_HPP_

#include <cmath>
#include <limits>
#include <vector>
#include <string>

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

// A = alpha * A ./ outdeg  (row broadcast), both CSR and CSC value arrays.
inline Info prNormalize(Matrix<float>* A, float alpha, Descriptor* desc) {
  Index n;
  CHECK(A->nrows(&n));
  Vector<float> outdegrees(n);
  CHECK((reduce<float, float, float>(&outdegrees, GrB_NULL, GrB_NULL, PlusMonoid<float>(), A, desc)));
  CHECK((eWiseMult<float, float, float, float>(A, GrB_NULL, GrB_NULL, PlusMultipliesSemiring<float>(), A, alpha, desc)));
  CHECK((eWiseMult<float, float, float, float>(A, GrB_NULL, GrB_NULL, PlusDividesSemiring<float>(), A, &outdegrees, desc)));
  return GrB_SUCCESS;
}

inline float pr(Vector<float>* p, const Matrix<float>* A, float alpha, float eps,
    Descriptor* desc) {
  Index n;
  GB_ALGO_STEP(A->nrows(&n));

  GB_ALGO_STEP(p->clear());
  GB_ALGO_STEP(p->fill(1.f/n));

  Vector<float> p_prev(n);
  Vector<float> p_swap(n);
  Vector<float> r(n);
  Vector<float> r_temp(n);
  GB_ALGO_STEP(r.fill(1.f));
  GB_ALGO_STEP(p_prev.fill(0.f));      // dense from the start: it trades places with p

  backend::Descriptor& d = desc->descriptor_;
  const bool verbose = (d.timing_ == 1);
  LoopTimer clock(verbose);
  float error = 1.f;
  int iter;
  clock.begin();

  for (iter = 1; error > eps && iter <= d.max_niter_; ++iter) {
    // p_prev = p ; p = p_prev (+.*) A + (1-alpha)/n ; error = |p - p_prev|_2.
    // Dense vectors (always, here): the old ranks change hands by a swap and the
    // update + difference + square + sum are one pass (backend loop_steps.hpp);
    // otherwise the reference's operations (algorithm/pr.hpp:49-66).
    GB_ALGO_STEP(p->swap(&p_prev));
    vxm<float, float, float, float>(&p_swap, GrB_NULL, GrB_NULL,
        PlusMultipliesSemiring<float>(), &p_prev, A, desc);
    // A push (mxvmode 1) leaves p_prev and p_swap sparse; the update below and the
    // next iteration's swap take them dense (no work when they already are).
    GB_ALGO_STEP(p_prev.sparse2dense(0.f));
    GB_ALGO_STEP(p_swap.sparse2dense(0.f));
    if (backend::prUpdateStep(&p->vector_, &p_swap.vector_, &p_prev.vector_,
                              (1.f - alpha)/n, &error, &desc->descriptor_) != GrB_SUCCESS) {
      eWiseAdd<float, float, float, float>(p, GrB_NULL, GrB_NULL,
          PlusMultipliesSemiring<float>(), &p_swap, (1.f - alpha)/n, desc);
      eWiseMult<float, float, float, float>(&r, GrB_NULL, GrB_NULL,
          PlusMinusSemiring<float>(), p, &p_prev, desc);
      eWiseAdd<float, float, float, float>(&r_temp, GrB_NULL, GrB_NULL,
          MultipliesMultipliesSemiring<float>(), &r, &r, desc);
      reduce<float, float>(&error, GrB_NULL, PlusMonoid<float>(), &r_temp, desc);
    }
    error = sqrt(error);

    if (verbose) {
      float ms = clock.lap();
      std::cout << iter << ", " << error << "/" << n << ", "
                << (d.lastmxv_ == GrB_PUSHONLY ? "push" : "pull") << ", "
                << ms << "\n";
    }
  }
  return clock.finish();
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_PR_HPP_
