// graphblast_b200 — local graph clustering on the device.
//
// lgc: p = the approximate personalised PageRank of source s on the lazy walk (Andersen,
// Chung and Lang's push), pushed synchronously one round at a time, bit for bit the
// floats of the reference's CPU checker SimpleReferenceLgc<float> (algorithm/
// test_lgc.hpp) for the same CSR, s, alpha, eps and max_niter.  backend/cuda/kernels/
// lgc.cuh states the arithmetic.  d[v] is the row length of v in A's pattern (values
// are never read; FP32 and INT32 A give the same result).  The round order the
// reference follows, ascending source vertex per target, is the stored order of the
// in-lists, so equality holds for sorted column lists, which the library's build and
// ingest always produce; an adopted CSR or CSC with unsorted lists still gives a
// deterministic result, but not necessarily the reference's.  A non-symmetric A needs
// its CSC (the pull reads in-lists).
//   r (when not NULL) = the final residual, bit-exact the same way; *rounds = the
// rounds run, at most desc's max_niter: the reference's loop always runs max_niter
// rounds, but those after the frontier empties change nothing.  max_niter <= 0 runs no
// round (p = 0, r = the unit vector of s).  desc's mxvmode picks the route of each
// round (GrB_PUSHONLY sparse, GrB_PULLONLY dense, the default by the frontier's volume
// against switchpoint * nnz); the result does not depend on it.  All rounds are one
// cooperative kernel.
//   Refusals, p and r untouched: NULL p, A or desc (GrB_UNINITIALIZED_OBJECT); s out
// of range (GrB_INVALID_INDEX); alpha outside (0, 1] or eps not > 0, NaN included
// (GrB_INVALID_VALUE); then those of backend::lgcCheck (a dense A, then sizes, then a
// missing CSC); r the same vector as p (GrB_INVALID_VALUE).
//
// lgcSweep: the sweep cut of p, the cluster a user of local clustering wants.  The
// support {v : p[v] > 0 and d[v] > 0} ordered by p[v]/d[v] descending (fp32, ties by
// ascending id); of its prefixes S_k, the one of least conductance
// cut(S_k)/min(vol(S_k), nnz - vol(S_k)) (exact 64-bit cut and volume, the quotient in
// double; prefixes with a zero denominator do not qualify), the smallest on a tie.
// cluster = 1 on its members, 0 elsewhere (dense); *size = its size and *conductance
// its conductance; no qualifying prefix gives an empty cluster, size 0 and NaN.  A p
// held sparse is converted to dense storage, its values unchanged.
//
// Both return the device time in milliseconds ("tight"), or -1 with the failing status
// in algorithm::lastStatus().
#ifndef GRAPHBLAS_ALGORITHM_LGC_HPP_
#define GRAPHBLAS_ALGORITHM_LGC_HPP_

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

template <typename a>
float lgc(Vector<float>* p, Vector<float>* r, const Matrix<a>* A, Index s, double alpha,
          double eps, Descriptor* desc, int* rounds) {
  if (p == NULL || A == NULL || desc == NULL) GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  Index n = 0;
  GB_ALGO_STEP(A->nrows(&n));
  if (s < 0 || s >= n) GB_ALGO_STEP(GrB_INVALID_INDEX);
  if (!(alpha > 0.0 && alpha <= 1.0) || !(eps > 0.0)) GB_ALGO_STEP(GrB_INVALID_VALUE);
  backend::Descriptor& d = desc->descriptor_;
  Desc_value mode;
  GB_ALGO_STEP(desc->get(GrB_MXVMODE, &mode));
  int count = 0;
  float ms = 0.f;
  GB_ALGO_STEP(backend::lgcRun(&p->vector_, r != NULL ? &r->vector_ : NULL, &A->matrix_, s,
      alpha, eps, d.max_niter_,
      mode == GrB_PUSHONLY ? 1 : (mode == GrB_PULLONLY ? 2 : 0), d.switchpoint(),
      &count, &ms));
  if (rounds != NULL) *rounds = count;
  if (d.timing_ > 0) std::cout << "lgc, " << count << " rounds, " << ms << "\n";
  return ms;
}

template <typename a>
float lgcSweep(Vector<float>* cluster, Vector<float>* p, const Matrix<a>* A,
               Descriptor* desc, int* size, double* conductance) {
  if (cluster == NULL || p == NULL || A == NULL || desc == NULL)
    GB_ALGO_STEP(GrB_UNINITIALIZED_OBJECT);
  int members = 0;
  double phi = 0.0;
  float ms = 0.f;
  GB_ALGO_STEP(backend::lgcSweepRun(&cluster->vector_, &p->vector_, &A->matrix_, &members,
                                    &phi, &ms));
  if (size != NULL) *size = members;
  if (conductance != NULL) *conductance = phi;
  if (desc->descriptor_.timing_ > 0)
    std::cout << "lgcSweep, " << members << " members, " << phi << ", " << ms << "\n";
  return ms;
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_LGC_HPP_
