/* graphblast_b200 — k-truss and truss decomposition through the C ABI.  A companion
 * of graphblast_b200.h (handles, descriptors and GrB_* status codes are that header's),
 * exported by the same library.  include/graphblas/algorithm/ktruss.hpp */
#ifndef GRAPHBLAST_B200_KTRUSS_H_
#define GRAPHBLAST_B200_KTRUSS_H_

#include "graphblast_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#pragma GCC visibility push(default)

/* Graph: the undirected simple graph G of A's pattern, with the edge {i, j}, i != j,
 * when A(i,j) or A(j,i) is stored.  Values and self-loops are ignored, so FP32 and INT32
 * A give the same result.  Column lists are sorted and duplicate-free, as every build,
 * load and ingest of the library leaves them.  A non-symmetric A needs its CSC.
 *
 * Output: C (or T) is n x n, a sorted CSR, replaced, and installed as structurally
 * symmetric, so cc, gc, mis and lgc take their symmetric paths on it.  It is FP32 or
 * INT32, independently of A, and may be A.  The values are integers, so every call gives
 * identical bytes.
 *
 * Refusals, in this order, each leaving the output untouched:
 *   1. a NULL output, A or desc: GrB_UNINITIALIZED_OBJECT;
 *   2. an output or A of neither element type: GrB_DOMAIN_MISMATCH;
 *   3. k < 2 (gb200_ktruss): GrB_INVALID_VALUE;
 *   4. no device: GrB_PANIC;
 *   5. a dense A: GrB_NOT_IMPLEMENTED;
 *   6. A not square, or the output not n x n: GrB_DIMENSION_MISMATCH;
 *   7. a missing CSR, or a non-symmetric A without its CSC: GrB_UNINITIALIZED_OBJECT;
 *   8. an FP32 output with n > 2^24, where supports and tau would no longer be exact:
 *      GrB_INVALID_VALUE;
 *   9. a symmetrised pattern past 2^31 - 1 entries: GrB_OUT_OF_MEMORY. */

/* C = the k-truss of G, k >= 2: starting from G, every edge in fewer than k - 2
 * triangles of the remaining graph is deleted until none is left to delete.  C(i,j) =
 * C(j,i) = the number of triangles of the k-truss that contain {i, j}, at least k - 2.
 * With k = 2 every edge stays, with its triangle count in G.  *nedges (when not NULL) =
 * the undirected edges kept. */
int gb200_ktruss(gb200_matrix_t C, gb200_matrix_t A, int k, gb200_desc_t desc,
                 long long* nedges, float* tight_ms);

/* T = the truss decomposition of G: G's pattern in both directions, T(i,j) = T(j,i) =
 * the largest k whose k-truss contains {i, j} (2 for an edge in no triangle).  *kmax
 * (when not NULL) = the largest value, 0 when G has no edge. */
int gb200_trussness(gb200_matrix_t T, gb200_matrix_t A, gb200_desc_t desc, int* kmax,
                    float* tight_ms);

/* Of the last gb200_ktruss or gb200_trussness call of this process: the peel rounds
 * that removed edges, the levels that did (a k-truss runs one level), and the device
 * time of the support pass alone, in milliseconds.  Each pointer may be NULL. */
int gb200_ktruss_stats(int* rounds, int* levels, float* support_ms);

#pragma GCC visibility pop

#ifdef __cplusplus
}
#endif

#endif  /* GRAPHBLAST_B200_KTRUSS_H_ */
