/* graphblast_b200 — local graph clustering through the C ABI: the approximate
 * personalised PageRank push and its conductance sweep cut.  A companion of
 * graphblast_b200.h (handles, descriptors and GrB_* status codes are that header's),
 * exported by the same library.  include/graphblas/algorithm/lgc.hpp */
#ifndef GRAPHBLAST_B200_LGC_H_
#define GRAPHBLAST_B200_LGC_H_

#include "graphblast_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#pragma GCC visibility push(default)

/* p = the approximate personalised PageRank of `source` on the lazy walk of A's
 * pattern (ACL's push, synchronous rounds), bit for bit the floats of the reference's
 * CPU checker SimpleReferenceLgc<float> for the same CSR, source, alpha, eps and desc's
 * max_niter when the column lists are sorted (the library's build, load and ingest
 * sort them; adopted unsorted lists give a deterministic result in stored order).
 * r (may be NULL) = the final residual.  Both become dense.  *rounds (may be NULL) =
 * the rounds run; max_niter <= 0 runs none (p = 0, r = the unit vector of source).
 * FP32 and INT32 A give the same result; a non-symmetric A needs its CSC.  desc's
 * mxvmode picks the route of each round (1 sparse only, 2 dense only, 0 by the
 * frontier's volume against switchpoint * nnz) and never changes the result.
 * Refusals, in this order, leave p and r untouched: NULL p, A or desc
 * (GrB_UNINITIALIZED_OBJECT); a matrix of neither element type (GrB_DOMAIN_MISMATCH);
 * source out of range (GrB_INVALID_INDEX); alpha not in (0, 1] or eps not > 0
 * (GrB_INVALID_VALUE); no device (GrB_PANIC); a dense A (GrB_NOT_IMPLEMENTED, as
 * gb200_cc, gb200_gc and gb200_mis); A not square or p, r not of size n
 * (GrB_DIMENSION_MISMATCH); a non-symmetric A without its CSC
 * (GrB_UNINITIALIZED_OBJECT); r the same vector as p (GrB_INVALID_VALUE). */
int gb200_lgc(gb200_vector_t p, gb200_vector_t r, gb200_matrix_t A, int source,
              double alpha, double eps, gb200_desc_t desc, int* rounds, float* tight_ms);

/* The sweep cut of p: the vertices with p[v] > 0 and a non-empty row, ordered by
 * p[v]/d[v] (fp32) descending, ties by ascending id; of the prefixes S_k of that order,
 * the smallest k of least conductance cut(S_k)/min(vol(S_k), nnz - vol(S_k)) (d, vol
 * and cut count stored entries, self-loops never cut; prefixes with a zero denominator
 * do not qualify).  cluster = 1 on S_k, 0 elsewhere (dense); *size = k;
 * *conductance = its conductance.  No qualifying prefix: an empty cluster, size 0 and
 * NaN.  A p held sparse is converted to dense storage (its values unchanged); p is not
 * otherwise written.  Refusals as gb200_lgc where they apply (cluster and p of size
 * n), and cluster the same vector as p (GrB_INVALID_VALUE); each leaves cluster and p
 * untouched. */
int gb200_lgc_sweep(gb200_vector_t cluster, gb200_vector_t p, gb200_matrix_t A,
                    gb200_desc_t desc, int* size, double* conductance, float* tight_ms);

#pragma GCC visibility pop

#ifdef __cplusplus
}
#endif

#endif  /* GRAPHBLAST_B200_LGC_H_ */
