/* graphblast_b200 — assign into a matrix through the C ABI: submatrices, columns, rows
 * and constants placed by host index lists.  A companion of graphblast_b200.h
 * (handles, descriptors, GB200_*_MONOID ids and GrB_* status codes are that
 * header's), exported by the same library.
 * include/graphblas/operations.hpp, assign */
#ifndef GRAPHBLAST_B200_ASSIGN_H_
#define GRAPHBLAST_B200_ASSIGN_H_

#include "graphblast_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#pragma GCC visibility push(default)

/* accum: no accumulator.  Any other accum is a GB200_*_MONOID id. */
#define GB200_NO_ACCUM (-1)

/* Index lists are host arrays of int.  A NULL list is GrB_ALL: every index of its
 * extent (C's rows for the row list, C's columns for the column list), in order, and
 * its count must equal that extent.  Lists may be unsorted but may not repeat an
 * index.  The region is rows x cols.
 *
 * Without accum (GB200_NO_ACCUM), C's region takes exactly op(A)'s pattern and
 * values: C(rows[p], cols[q]) = op(A)(p, q) where op(A) stores that entry, and C's
 * entries in the region that op(A) does not store are deleted.  With accum, the
 * region is the union of the two: where both store an entry the result is
 * accum(c, a), C's value first; where one does, its value.  Outside the region C is
 * unchanged.  C comes out sorted and duplicate-free, keeps stored zeros, and has its
 * CSC rebuilt when its format keeps one.  A C that was created and never built counts
 * as an empty matrix.
 *
 * Refusals, in this order, each leaving C untouched:
 *   1. a NULL C, source or desc handle: GrB_UNINITIALIZED_OBJECT;
 *   2. an index count < 1, or an accum that is neither GB200_NO_ACCUM nor a monoid
 *      id: GrB_INVALID_VALUE;
 *   3. element types (C and A both FP32 or both INT32; C FP32 for a row or column):
 *      GrB_DOMAIN_MISMATCH;
 *   4. no device: GrB_PANIC;
 *   5. a mask, a dense C or A, or an INT32 C with an accum other than
 *      GB200_PLUS_MONOID: GrB_NOT_IMPLEMENTED;
 *   6. shapes: op(A) not nrows x ncols, u not of size nrows (ncols), or col (row)
 *      not below C's column (row) count: GrB_DIMENSION_MISMATCH;
 *   7. an index outside C's range, a negative row or col, or a NULL list whose count
 *      is not the full extent: GrB_INVALID_INDEX;
 *   8. a list that repeats an index: GrB_INVALID_VALUE;
 *   9. the orientation that GrB_TRAN reads is not stored (the CSC of a non-symmetric
 *      A): GrB_UNINITIALIZED_OBJECT;
 *  10. a result of more than 2^31 - 1 entries (for a constant, a region of more than
 *      2^31 - 1 positions): GrB_OUT_OF_MEMORY. */

/* C(rows, cols) = accum(C(rows, cols), op(A)), FP32 or INT32; op(A) is A, or its
 * transpose when desc's GrB_INP0 is GrB_TRAN (read from A's CSC, which a
 * non-symmetric A must have).  C may be A.  A C marked symmetric (built undirected)
 * stays symmetric when A is marked symmetric and rows and cols are the same list
 * (both NULL, or equal contents). */
int gb200_assign_matrix(gb200_matrix_t C, gb200_matrix_t mask, int accum, gb200_matrix_t A,
                        const int* h_rows, int nrows, const int* h_cols, int ncols,
                        gb200_desc_t desc);

/* C(rows, cols) = accum(C(rows, cols), val), val cast to C's element type: every
 * position of the region ends up stored.  A C marked symmetric stays symmetric when
 * rows and cols are the same list. */
int gb200_assign_matrix_scalar(gb200_matrix_t C, gb200_matrix_t mask, int accum, double val,
                               const int* h_rows, int nrows, const int* h_cols, int ncols,
                               gb200_desc_t desc);

/* C(rows, col) = accum(C(rows, col), u), u of size nrows: its stored entries (every
 * entry of a dense u; a sparse u's indices ascend).  FP32 C only; GrB_INP0 is
 * ignored.  C's symmetric flag is cleared. */
int gb200_assign_column(gb200_matrix_t C, gb200_vector_t mask, int accum, gb200_vector_t u,
                        const int* h_rows, int nrows, int col, gb200_desc_t desc);

/* C(row, cols) = accum(C(row, cols), u), u of size ncols, as for a column. */
int gb200_assign_row(gb200_matrix_t C, gb200_vector_t mask, int accum, gb200_vector_t u,
                     int row, const int* h_cols, int ncols, gb200_desc_t desc);

#pragma GCC visibility pop

#ifdef __cplusplus
}
#endif

#endif  /* GRAPHBLAST_B200_ASSIGN_H_ */
