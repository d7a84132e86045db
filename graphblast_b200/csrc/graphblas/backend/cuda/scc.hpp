// graphblast_b200 backend — host side of strongly connected components (kernels/scc.cuh):
// the input (graph_input.hpp), the scratch and one cooperative launch, or connected
// components for an A whose pattern is its own transpose.  algorithm::scc comes here.
#ifndef GRAPHBLAS_BACKEND_CUDA_SCC_HPP_
#define GRAPHBLAS_BACKEND_CUDA_SCC_HPP_

#include <type_traits>

#include "graphblas/backend/cuda/cc.hpp"
#include "graphblas/backend/cuda/graph_input.hpp"
#include "graphblas/backend/cuda/kernels/scc.cuh"

namespace graphblas {
namespace backend {

// Of the last sccRun that ran: vertices settled by the trim, vertices of the pivot's
// component, colouring iterations and grid barriers.  After the delegation to ccRun all
// are 0 except barriers, which is -1.
struct SccStats {
  long long trimmed = 0;
  long long pivot_size = 0;
  int colour_iterations = 0;
  int barriers = 0;
};

// v[i] = the smallest vertex id in the strongly connected component of i, over the arcs
// i -> j with A(i,j) stored and i != j; *ncomponents (when not NULL) = the number of
// components, 0 when A has no rows; *ms (when not NULL) = the device time, from CUDA
// events.  v becomes dense with nrows(A) entries and is overwritten completely.  Out-lists
// come from A's CSR, in-lists from its CSC.  An A that is sameStructure() (marked
// symmetric, or whose CSC aliases its CSR) has the connected components of its pattern
// as its strong components: ccRun computes them.
// Refusals, before v is touched: those of graphCheck (CSC needed), then a float v with
// nrows(A) > 2^24 + 1 (GrB_INVALID_VALUE), as in ccRun.
// Scratch: the counter cells, n + 1 zero row pointers when A stores no entry, nine n-word
// arrays (label, degrees, marks, colour, stamp, three queues) and 2 (nnz /
// GB_SCC_GRID_MIN + 1) words for the lists of a level's grid pass.
template <typename W, typename a>
Info sccRun(Vector<W>* v, const Matrix<a>* A, int* ncomponents, float* ms = NULL) {
  static_assert(std::is_same<W, int>::value || std::is_same<W, float>::value,
                "scc writes int or float vectors");
  CHECK(graphCheck("scc", A, true, v));
  const SparseMatrix<a>& S = A->sparse_;
  const Index n = S.nrows_;
  if (std::is_same<W, float>::value && n > (1 << 24) + 1) return GrB_INVALID_VALUE;
  if (S.sameStructure()) {
    CHECK(ccRun(v, A, ncomponents, ms));
    lastStats<SccStats>() = SccStats();
    lastStats<SccStats>().barriers = -1;
    return GrB_SUCCESS;
  }

  GpuTimer clock;
  clock.Start();
  if (ncomponents != NULL) *ncomponents = 0;
  CHECK(v->setStorage(GrB_DENSE));
  if (n == 0) {
    clock.Stop();
    lastStats<SccStats>() = SccStats();
    if (ms != NULL) *ms = clock.ElapsedMillis();
    return GrB_SUCCESS;
  }
  CHECK(v->dense_.allocateGpu());
  const size_t nn = static_cast<size_t>(n);
  const size_t heavy_words = 2*((hasEntries(S) ? static_cast<size_t>(S.nvals_) : 0)/
                                GB_SCC_GRID_MIN + 1);
  ScratchLayout l;
  const size_t counters = l.place(SCC_NCELLS*sizeof(unsigned long long));
  const size_t zero_rows = l.place(GraphPattern::zeroRowBytes(S));
  const size_t words = l.place((9*nn + heavy_words)*sizeof(Index));
  const DeviceBlock block(gbMalloc(l.bytes));
  const GraphPattern g(S, block.at<Index>(zero_rows));
  SccArgs args;
  args.n = n;
  args.row_ptr = g.row_ptr;
  args.row_ind = g.row_ind;
  args.col_ptr = g.in_ptr();
  args.col_ind = g.in_ind();
  args.counters = block.at<unsigned long long>(counters);
  Index* w = block.at<Index>(words);
  args.label = w;
  args.dout = w + nn;
  args.din = w + 2*nn;
  args.mark = w + 3*nn;
  args.colour = w + 4*nn;
  args.stamp = w + 5*nn;
  args.qa = w + 6*nn;
  args.qb = w + 7*nn;
  args.qc = w + 8*nn;
  args.heavy = w + 9*nn;
  cudaStream_t stream = gbStream();
  CUDA_CALL(cudaMemsetAsync(args.counters, 0, SCC_NCELLS*sizeof(unsigned long long), stream));
  CHECK((launchCooperative<sccKernel<W>, GB_SCC_NT>(stream, args, v->dense_.d_val_)));
  unsigned long long cells[SCC_NCELLS];
  CUDA_CALL(cudaMemcpyAsync(cells, args.counters, sizeof(cells), cudaMemcpyDeviceToHost,
                            stream));
  clock.Stop();
  CUDA_CALL(cudaStreamSynchronize(stream));
  v->dense_.touched();
  SccStats& stats = lastStats<SccStats>();
  stats.trimmed = static_cast<long long>(cells[SCC_TRIMMED]);
  stats.pivot_size = static_cast<long long>(cells[SCC_SIZE]);
  stats.colour_iterations = static_cast<int>(cells[SCC_COLOURS]);
  stats.barriers = static_cast<int>(cells[SCC_BARRIERS]);
  if (ncomponents != NULL) *ncomponents = static_cast<int>(cells[SCC_COMPONENTS]);
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_SCC_HPP_
