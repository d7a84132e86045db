/* graphblast_b200 — betweenness centrality through the C ABI.  A companion of
 * graphblast_b200.h (handles, descriptors and GrB_* status codes are that header's),
 * exported by the same library.  include/graphblas/algorithm/bc.hpp */
#ifndef GRAPHBLAST_B200_BC_H_
#define GRAPHBLAST_B200_BC_H_

#include "graphblast_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#pragma GCC visibility push(default)

/* v = the betweenness centrality of every vertex over the sources h_sources[0..nsources).
 *
 * Graph: each stored A(i,j) with i != j is a directed edge i -> j; self-loops and values
 * are ignored, so FP32 and INT32 A give the same result, and a symmetric A is the
 * undirected graph.  A non-symmetric A needs its CSC.
 * Sources: a host list; a repeated id counts once per entry.  A NULL list means every
 * vertex 0..n-1 (exact BC), and nsources must then be n.  nsources == 0 with a non-NULL
 * list gives all zeros.
 * Result: v[x] = sum over sources s, over t not in {s, x} reachable from s, of
 * sigma_st(x) / sigma_st (shortest-path counts), with no normalisation and no halving:
 * for a symmetric A and all sources, twice networkx's undirected unnormalised value.  v
 * becomes dense with nrows(A) floats; a vertex on no counted path is exactly 0.  Path
 * counts and dependencies are fp64, summed in fp64 in a fixed order and rounded to float
 * once, so two calls give identical bytes.
 *
 * Refusals, in this order, each leaving v untouched:
 *   1. a NULL v, A or desc: GrB_UNINITIALIZED_OBJECT;
 *   2. an A of neither element type: GrB_DOMAIN_MISMATCH;
 *   3. nsources < 0: GrB_INVALID_VALUE;
 *   4. a NULL list whose count is not n, or an id outside [0, n): GrB_INVALID_INDEX;
 *   5. no device: GrB_PANIC;
 *   6. a dense A: GrB_NOT_IMPLEMENTED; A not square or v not of size n:
 *      GrB_DIMENSION_MISMATCH; a missing CSR, or a missing CSC on a non-symmetric A:
 *      GrB_UNINITIALIZED_OBJECT;
 *   7. a graph so large that one batch's level lists could pass 2^31 - 1 entries:
 *      GrB_OUT_OF_MEMORY. */
int gb200_bc(gb200_vector_t v, gb200_matrix_t A, const int* h_sources, int nsources,
             gb200_desc_t desc, float* tight_ms);

#pragma GCC visibility pop

#ifdef __cplusplus
}
#endif

#endif  /* GRAPHBLAST_B200_BC_H_ */
