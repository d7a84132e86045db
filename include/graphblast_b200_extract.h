/* graphblast_b200 — extract through the C ABI: submatrices, columns and subvectors
 * cut by host index lists.  A companion of graphblast_b200.h (handles, descriptors
 * and GrB_* status codes are that header's), exported by the same library.
 * include/graphblas/operations.hpp, extract */
#ifndef GRAPHBLAST_B200_EXTRACT_H_
#define GRAPHBLAST_B200_EXTRACT_H_

#include "graphblast_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#pragma GCC visibility push(default)

/* Index lists are host arrays of int.  A NULL list is GrB_ALL: every index of its
 * extent, in order, and its count must equal that extent.  Lists may be unsorted and
 * may repeat an index.  op(A) is A, or its transpose when desc's GrB_INP0 is GrB_TRAN
 * (read from A's CSC, which a non-symmetric A must then have).  Results are sorted by
 * index, duplicate-free, and keep stored zeros; the output is replaced (no accum).
 *
 * Refusals, in this order, each leaving the output untouched:
 *   1. a NULL output, source or desc handle: GrB_UNINITIALIZED_OBJECT;
 *   2. an index count < 1 (objects here cannot be empty): GrB_INVALID_VALUE;
 *   3. C and A of different element types, or a column from an INT32 A:
 *      GrB_DOMAIN_MISMATCH;
 *   4. no device: GrB_PANIC;
 *   5. a mask, or a dense A: GrB_NOT_IMPLEMENTED;
 *   6. shapes: C not nrows x ncols, w not of size nrows (nind), or col not below
 *      op(A)'s column count: GrB_DIMENSION_MISMATCH;
 *   7. an index outside op(A)'s (u's) range, a negative col, or a NULL list whose
 *      count is not the full extent: GrB_INVALID_INDEX;
 *   8. the orientation the cut reads is not stored (the CSC of a non-symmetric A for
 *      GrB_TRAN, or for a column without GrB_TRAN): GrB_UNINITIALIZED_OBJECT.
 * A result of more than 2^31 - 1 entries is GrB_OUT_OF_MEMORY, also leaving the
 * output untouched. */

/* C = op(A)(rows, cols), FP32 or INT32.  C may be A.  A symmetric A (built
 * undirected, or ingested from a symmetric file) cut by the same list both ways (both
 * NULL, or equal contents) gives a symmetric C, whose CSC is its CSR. */
int gb200_extract_matrix(gb200_matrix_t C, gb200_matrix_t mask, gb200_matrix_t A,
                         const int* h_rows, int nrows, const int* h_cols, int ncols,
                         gb200_desc_t desc);

/* w = op(A)(rows, col): a sparse vector of size nrows.  FP32 A only. */
int gb200_extract_column(gb200_vector_t w, gb200_vector_t mask, gb200_matrix_t A,
                         const int* h_rows, int nrows, int col, gb200_desc_t desc);

/* w = u(ind), of size nind: dense for a dense u, sparse (the entries where u(ind[i])
 * is stored) for a sparse u, whose indices ascend.  w may be u. */
int gb200_extract_vector(gb200_vector_t w, gb200_vector_t mask, gb200_vector_t u,
                         const int* h_ind, int nind, gb200_desc_t desc);

#pragma GCC visibility pop

#ifdef __cplusplus
}
#endif

#endif  /* GRAPHBLAST_B200_EXTRACT_H_ */
