/* graphblast_b200 — community detection by label propagation through the C ABI.  A
 * companion of graphblast_b200.h (handles, descriptors and GrB_* status codes are that
 * header's), exported by the same library.  include/graphblas/algorithm/cdlp.hpp */
#ifndef GRAPHBLAST_B200_CDLP_H_
#define GRAPHBLAST_B200_CDLP_H_

#include "graphblast_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#pragma GCC visibility push(default)

/* LDBC Graphalytics CDLP, with vertex ids 0..n-1 as the initial labels.
 *
 * Graph: the arc i -> j when A(i,j) is stored and i != j.  Values are never read and
 * stored zeros count, so FP32 and INT32 A give the same result.  Self-loops are
 * ignored.  Out-lists come from A's CSR and in-lists from its CSC.  An A marked
 * symmetric, or whose CSC aliases its CSR, is read through its CSR alone: both lists
 * hold the same multiset, so every multiplicity doubles and the answer is the same.
 *
 * Iterations: L_0(v) = v.  Iteration k is synchronous: M(v) = the labels L_{k-1}(u) of
 * v's out-neighbours (row v of the CSR) plus those of its in-neighbours (column v of the
 * CSC), an arc stored both ways counted twice.  L_k(v) = the smallest label of highest
 * multiplicity in M(v); a vertex whose M(v) is empty keeps its label.  max_iter >= 0
 * iterations are defined.  The kernel stops after the first iteration that changes no
 * label, a fixpoint, so the result equals max_iter iterations exactly.  *iterations
 * (when not NULL) = the iterations run, including the one that changed nothing;
 * max_iter = 0 gives v[i] = i.  Synchronous label propagation can oscillate (a star
 * alternates with period 2): the iteration count is what makes the result well defined.
 *
 * Result: v becomes dense with nrows(A) entries and is overwritten completely; v[i] =
 * L_T(i).  *ncommunities (when not NULL) = the number of distinct labels.  Two calls
 * give identical bytes.  Scratch: 6 n + n / 32 + 1 words and a few counter cells, none
 * proportional to the stored entries.
 *
 * Refusals, in this order, each leaving v untouched:
 *   1. a NULL v, A or desc: GrB_UNINITIALIZED_OBJECT;
 *   2. an A of neither element type: GrB_DOMAIN_MISMATCH;
 *   3. no device: GrB_PANIC;
 *   4. a dense A: GrB_NOT_IMPLEMENTED;
 *   5. A not square, or v not of size nrows(A): GrB_DIMENSION_MISMATCH;
 *   6. a missing CSR, or a non-symmetric A without its CSC: GrB_UNINITIALIZED_OBJECT;
 *   7. nrows(A) > 2^24 + 1, where a float v can no longer hold every id exactly:
 *      GrB_INVALID_VALUE;
 *   8. max_iter < 0: GrB_INVALID_VALUE. */
int gb200_cdlp(gb200_vector_t v, gb200_matrix_t A, int max_iter, gb200_desc_t desc,
               int* ncommunities, int* iterations, float* tight_ms);

/* Of the last gb200_cdlp call of this process that ran: the vertices whose list (out-
 * plus in-list, self-loops included) has at most 32 entries (short: packed several to a
 * warp), at most 128 (warp: one warp's hash table), and more (long), the (vertex,
 * partition) work items of the long lists, one per 2048 entries or part of it, and the
 * grid barriers the kernel executed: 2 per iteration and 2 more.  All depend only on A's
 * pattern and the iterations run.  Each pointer may be NULL. */
int gb200_cdlp_stats(long long* short_vertices, long long* warp_vertices,
                     long long* long_vertices, long long* long_items, int* barriers);

#pragma GCC visibility pop

#ifdef __cplusplus
}
#endif

#endif  /* GRAPHBLAST_B200_CDLP_H_ */
