/* graphblast_b200 — strongly connected components through the C ABI.  A companion of
 * graphblast_b200.h (handles, descriptors and GrB_* status codes are that header's),
 * exported by the same library.  include/graphblas/algorithm/scc.hpp */
#ifndef GRAPHBLAST_B200_SCC_H_
#define GRAPHBLAST_B200_SCC_H_

#include "graphblast_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#pragma GCC visibility push(default)

/* Graph: the arc i -> j when A(i,j) is stored and i != j.  Values are never read and
 * stored zeros count, so FP32 and INT32 A give the same result.  Self-loops are
 * ignored: a vertex whose only arcs are self-loops is its own component.  Out-lists
 * come from A's CSR and in-lists from its CSC; column lists are sorted and
 * duplicate-free, as every build, load and ingest of the library leaves them.  An A
 * marked symmetric, or whose CSC aliases its CSR, has the connected components of its
 * pattern as its strong components, and gb200_cc's kernel computes them.
 *
 * Result: v becomes dense with nrows(A) entries and is overwritten completely; v[i] =
 * the smallest vertex id in the strongly connected component of i.  *ncomponents (when
 * not NULL) = the number of i with v[i] == i.  An A with no stored entries gives v[i] = i
 * and n components.  The result depends only on A's pattern, so two calls give
 * identical bytes and there is no seed.
 *
 * Refusals, in this order, each leaving v untouched:
 *   1. a NULL v, A or desc: GrB_UNINITIALIZED_OBJECT;
 *   2. an A of neither element type: GrB_DOMAIN_MISMATCH;
 *   3. no device: GrB_PANIC;
 *   4. a dense A: GrB_NOT_IMPLEMENTED;
 *   5. A not square, or v not of size nrows(A): GrB_DIMENSION_MISMATCH;
 *   6. a missing CSR, or a non-symmetric A without its CSC: GrB_UNINITIALIZED_OBJECT;
 *   7. nrows(A) > 2^24 + 1, where a float v can no longer hold every id exactly:
 *      GrB_INVALID_VALUE. */
int gb200_scc(gb200_vector_t v, gb200_matrix_t A, gb200_desc_t desc, int* ncomponents,
              float* tight_ms);

/* Of the last gb200_scc call of this process that ran: the vertices settled by the
 * trim, the size of the pivot's component settled by the forward-backward reach, the
 * colouring iterations, and the grid barriers the kernel executed.  The trim runs to
 * its fixpoint, so trimmed, pivot_size and colour_iterations depend only on A's
 * pattern; barriers also depends on how fast colours spread between the SMs.  After
 * an A marked symmetric (the connected-components kernel) all four are 0 except
 * barriers, which is -1.  Each pointer may be NULL. */
int gb200_scc_stats(long long* trimmed, long long* pivot_size, int* colour_iterations,
                    int* barriers);

#pragma GCC visibility pop

#ifdef __cplusplus
}
#endif

#endif  /* GRAPHBLAST_B200_SCC_H_ */
