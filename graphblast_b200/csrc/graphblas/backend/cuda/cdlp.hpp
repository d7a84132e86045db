// graphblast_b200 backend — host side of community detection by label propagation
// (kernels/cdlp.cuh): the input (graph_input.hpp), the scratch and one cooperative
// launch.  algorithm::cdlp comes here.
#ifndef GRAPHBLAS_BACKEND_CUDA_CDLP_HPP_
#define GRAPHBLAS_BACKEND_CUDA_CDLP_HPP_

#include <type_traits>

#include "graphblas/backend/cuda/graph_input.hpp"
#include "graphblas/backend/cuda/kernels/cdlp.cuh"

namespace graphblas {
namespace backend {

// Of the last cdlpRun that ran: the vertices of each class (short: list of at most
// GB_CDLP_SHORT_MAX entries, warp: at most GB_CDLP_WARP_MAX, long: longer), the long
// lists' (vertex, partition) items, and the grid barriers of the kernel.
struct CdlpStats {
  long long short_vertices = 0;
  long long warp_vertices = 0;
  long long long_vertices = 0;
  long long long_items = 0;
  int barriers = 0;
};

// v[i] = L_T(i), the label of i after T iterations of synchronous label propagation
// (LDBC Graphalytics CDLP, kernels/cdlp.cuh): L_0(v) = v; L_k(v) = the smallest label of
// highest multiplicity among the labels L_{k-1}(u) of v's out-neighbours (A's CSR) and
// in-neighbours (A's CSC), an arc stored both ways counted twice, self-loops ignored;
// L_{k-1}(v) when v has no neighbour.  An A that is sameStructure() is read through its
// CSR alone (every multiplicity doubles, the answer is the same).  T = max_iter, or the
// first iteration that changes no label.  *ncommunities = the number of distinct labels,
// *iterations = T, *ms = the device time (CUDA events); each may be NULL.  v becomes
// dense with nrows(A) entries and is overwritten completely.
// Refusals, before v is touched: those of graphCheck (CSC needed), then nrows(A) >
// 2^24 + 1 for a float v, then max_iter < 0 (both GrB_INVALID_VALUE).
// Scratch: the counter cells, n + 1 zero row pointers when A stores no entry, and
// 6 n + n / 32 + 1 words: two label arrays, the long list and its item bases (n words
// each) and each long vertex's 64-bit best word, and the bitmap of the result's labels.
template <typename W, typename a>
Info cdlpRun(Vector<W>* v, const Matrix<a>* A, int max_iter, int* ncommunities,
             int* iterations, float* ms = NULL) {
  static_assert(std::is_same<W, int>::value || std::is_same<W, float>::value,
                "cdlp writes int or float vectors");
  CHECK(graphCheck("cdlp", A, true, v));
  const SparseMatrix<a>& S = A->sparse_;
  const Index n = S.nrows_;
  if (std::is_same<W, float>::value && n > (1 << 24) + 1) return GrB_INVALID_VALUE;
  if (max_iter < 0) return GrB_INVALID_VALUE;

  GpuTimer clock;
  clock.Start();
  if (ncommunities != NULL) *ncommunities = 0;
  if (iterations != NULL) *iterations = 0;
  CHECK(v->setStorage(GrB_DENSE));
  if (n == 0) {                        // the first iteration changes nothing
    if (iterations != NULL) *iterations = max_iter > 0 ? 1 : 0;
    clock.Stop();
    lastStats<CdlpStats>() = CdlpStats();
    if (ms != NULL) *ms = clock.ElapsedMillis();
    return GrB_SUCCESS;
  }
  CHECK(v->dense_.allocateGpu());
  const size_t nn = static_cast<size_t>(n);
  ScratchLayout l;
  const size_t counters = l.place(CDLP_NCELLS*sizeof(unsigned long long));
  const size_t zero_rows = l.place(GraphPattern::zeroRowBytes(S));
  const size_t best = l.place(nn*sizeof(unsigned long long));
  const size_t words = l.place(4*nn*sizeof(Index));
  const size_t bitmap = l.place((nn/32 + 1)*sizeof(unsigned int));
  const DeviceBlock block(gbMalloc(l.bytes));
  const GraphPattern g(S, block.at<Index>(zero_rows));
  CdlpArgs args;
  args.row_ptr = g.row_ptr;
  args.row_ind = g.row_ind;
  args.col_ptr = g.col_ptr;
  args.col_ind = g.col_ind;
  args.n = n;
  args.max_iter = max_iter;
  Index* w = block.at<Index>(words);
  args.labels0 = w;
  args.labels1 = w + nn;
  args.long_v = w + 2*nn;
  args.long_base = w + 3*nn;
  args.best = block.at<unsigned long long>(best);
  args.bitmap = block.at<unsigned int>(bitmap);
  args.counters = block.at<unsigned long long>(counters);
  cudaStream_t stream = gbStream();
  CUDA_CALL(cudaMemsetAsync(args.counters, 0, CDLP_NCELLS*sizeof(unsigned long long), stream));
  CHECK((launchCooperative<cdlpKernel<W>, GB_CDLP_NT>(stream, args, v->dense_.d_val_)));
  unsigned long long cells[CDLP_NCELLS];
  CUDA_CALL(cudaMemcpyAsync(cells, args.counters, sizeof(cells), cudaMemcpyDeviceToHost,
                            stream));
  clock.Stop();
  CUDA_CALL(cudaStreamSynchronize(stream));
  v->dense_.touched();
  CdlpStats& stats = lastStats<CdlpStats>();
  stats.short_vertices = static_cast<long long>(cells[CDLP_SHORT]);
  stats.warp_vertices = static_cast<long long>(cells[CDLP_WARP]);
  stats.long_vertices = static_cast<long long>(cells[CDLP_LONG] >> GB_CDLP_ITEM_BITS);
  stats.long_items = static_cast<long long>(cells[CDLP_LONG] &
                                            ((1ull << GB_CDLP_ITEM_BITS) - 1ull));
  stats.barriers = static_cast<int>(cells[CDLP_BARRIERS]);
  if (ncommunities != NULL) *ncommunities = static_cast<int>(cells[CDLP_COMMUNITIES]);
  if (iterations != NULL) *iterations = static_cast<int>(cells[CDLP_ITERATIONS]);
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_CDLP_HPP_
