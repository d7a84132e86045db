/* graphblast_b200 — minimum spanning forest through the C ABI.  A companion of
 * graphblast_b200.h (handles, descriptors and GrB_* status codes are that header's),
 * exported by the same library.  include/graphblas/algorithm/msf.hpp */
#ifndef GRAPHBLAST_B200_MSF_H_
#define GRAPHBLAST_B200_MSF_H_

#include "graphblast_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#pragma GCC visibility push(default)

/* Graph: the undirected graph G with the edge {i, j}, i != j, when A(i,j) or A(j,i) is
 * stored, of weight w({i,j}) = the smaller of the stored values among A(i,j) and A(j,i).
 * Self-loops are ignored; stored zeros are edges of weight 0 (scipy treats explicit
 * zeros as missing).  Only A's CSR is read, so a non-symmetric A needs no CSC.  Column
 * lists are sorted and duplicate-free, as every build, load and ingest of the library
 * leaves them.
 *
 * Order: edges are ranked by the key (w, min(i,j), max(i,j)).  Weights compare as
 * numbers, -0.0 equal to +0.0, +-inf allowed; INT32 weights compare as signed integers.
 * The order is strict and total, so the minimum spanning forest is unique: F is
 * Kruskal's forest under it, whatever the scheduling.
 *
 * Output: F is n x n, replaced, and holds both directions of every forest edge: F(i,j) =
 * F(j,i) = w({i,j}), -0.0 written as +0.0.  F is a sorted CSR installed as structurally
 * symmetric, so cc, gc, mis and lgc take their symmetric paths on it.  F has A's element
 * type and may be A.  Two calls give identical bytes.  *nedges (when not NULL) = the
 * undirected forest edges, n minus the number of trees.  *weight (when not NULL) = their
 * sum in fp64, taken in an order that depends only on the forest, so two calls give
 * identical bits; exact while every partial sum is an integer below 2^53.  An A with no
 * stored off-diagonal entry gives an empty F, 0 edges and weight 0.
 *
 * Refusals, in this order, each leaving F untouched:
 *   1. a NULL F, A or desc: GrB_UNINITIALIZED_OBJECT;
 *   2. F or A of neither element type, or F's element type different from A's:
 *      GrB_DOMAIN_MISMATCH;
 *   3. no device: GrB_PANIC;
 *   4. a dense A: GrB_NOT_IMPLEMENTED;
 *   5. A not square, or F not n x n: GrB_DIMENSION_MISMATCH;
 *   6. A with entries but no device CSR: GrB_UNINITIALIZED_OBJECT;
 *   7. an FP32 A with a NaN on a stored off-diagonal entry: GrB_INVALID_VALUE. */
int gb200_msf(gb200_matrix_t F, gb200_matrix_t A, gb200_desc_t desc, long long* nedges,
              double* weight, float* tight_ms);

/* Of the last gb200_msf call of this process that ran: the Boruvka rounds (at most
 * ceil(log2 n) + 1), the grid barriers the kernel executed, and the device time of
 * building the canonical edge list, in milliseconds.  Each pointer may be NULL. */
int gb200_msf_stats(int* rounds, int* barriers, float* canon_ms);

#pragma GCC visibility pop

#ifdef __cplusplus
}
#endif

#endif  /* GRAPHBLAST_B200_MSF_H_ */
