// graphblast_b200 backend — host side of betweenness centrality (kernels/bc.cuh): the
// input (graph_input.hpp), the scratch, one cooperative launch per batch of 32 sources
// and the finish.  algorithm::bc comes here.
#ifndef GRAPHBLAS_BACKEND_CUDA_BC_HPP_
#define GRAPHBLAS_BACKEND_CUDA_BC_HPP_

#include <climits>

#include "graphblas/backend/cuda/graph_input.hpp"
#include "graphblas/backend/cuda/kernels/bc.cuh"

namespace graphblas {
namespace backend {

// v[i] = the betweenness centrality of i over the sources (kernels/bc.cuh states the
// sum): `sources` a host list of nsources ids, each checked by the caller, or NULL for
// every vertex 0..n-1 (nsources = n).  v becomes dense with nrows(A) entries.  *ms (when
// not NULL) = the device time, from CUDA events.  Refusals: those of graphCheck (with
// the CSC), then a batch whose level lists could pass 2^31 - 1 entries
// (GrB_OUT_OF_MEMORY).  Launches: one cooperative kernel per batch of 32 sources and the
// finish; the host does not wait between them.
// Scratch: the counter cells, the fp64 totals, the source list, and, when there is a
// source: seen, two fresh words and two stamps per vertex, sigma and delta
// (2 x 32 doubles per vertex), the level starts, the level lists (lanes x (n + 2 nnz /
// GB_BC_CHUNK) 16-byte entries, lanes = min(32, nsources)), 4 nnz / GB_BC_CHUNK + 32
// partial slots of 32 doubles and their tickets, and the pattern's zero row pointers.
template <typename a>
Info bcRun(Vector<float>* v, const Matrix<a>* A, const Index* sources, Index nsources,
           float* ms = NULL) {
  CHECK(graphCheck("betweenness centrality", A, true, v));
  const SparseMatrix<a>& S = A->sparse_;
  const Index n = S.nrows_;
  const size_t nn = static_cast<size_t>(n);
  const size_t nnz = hasEntries(S) ? static_cast<size_t>(S.nvals_) : 0;
  const Index batches = (nsources + GB_BC_LANES - 1)/GB_BC_LANES;
  const size_t lanes = nsources < GB_BC_LANES ? static_cast<size_t>(nsources) : GB_BC_LANES;
  const size_t entries = lanes*(nn + (2*nnz + GB_BC_CHUNK - 1)/GB_BC_CHUNK);
  if (entries > static_cast<size_t>(INT_MAX)) return GrB_OUT_OF_MEMORY;
  const size_t slots = batches > 0 ? 4*nnz/GB_BC_CHUNK + 32 : 0;
  const size_t per_vertex = batches > 0 ? nn : 0;   // the traversal's arrays

  GpuTimer clock;
  clock.Start();
  cudaStream_t stream = gbStream();
  ScratchLayout l;
  const size_t counters = l.place(BC_NCELLS*sizeof(unsigned long long));
  const size_t total = l.place(nn*sizeof(double));
  const size_t src = l.place(sources != NULL ? static_cast<size_t>(nsources)*sizeof(Index) : 0);
  const size_t seen = l.place(per_vertex*sizeof(unsigned int));
  const size_t fresh = l.place(2*per_vertex*sizeof(unsigned int));
  const size_t stamp0 = l.place(per_vertex*sizeof(unsigned long long));
  const size_t stamp1 = l.place(per_vertex*sizeof(unsigned long long));
  const size_t sigma = l.place(per_vertex*GB_BC_LANES*sizeof(double));
  const size_t delta = l.place(per_vertex*GB_BC_LANES*sizeof(double));
  const size_t level_start = l.place(batches > 0 ? (nn + 2)*sizeof(Index) : 0);
  const size_t list = l.place(batches > 0 ? entries*sizeof(int4) : 0);
  const size_t partial = l.place(slots*GB_BC_LANES*sizeof(double));
  const size_t ticket = l.place(slots*sizeof(int));
  const size_t zero_rows = l.place(batches > 0 ? GraphPattern::zeroRowBytes(S) : 0);
  const DeviceBlock block(gbMalloc(l.bytes));
  CUDA_CALL(cudaMemsetAsync(block.at<void>(counters), 0,
                            BC_NCELLS*sizeof(unsigned long long), stream));
  CUDA_CALL(cudaMemsetAsync(block.at<void>(total), 0, nn*sizeof(double), stream));
  if (batches > 0) {
    const GraphPattern g(S, block.at<Index>(zero_rows));
    CUDA_CALL(cudaMemsetAsync(block.at<void>(fresh), 0, 2*nn*sizeof(unsigned int), stream));
    CUDA_CALL(cudaMemsetAsync(block.at<void>(ticket), 0, slots*sizeof(int), stream));
    if (sources != NULL)
      CUDA_CALL(cudaMemcpyAsync(block.at<void>(src), sources,
                                static_cast<size_t>(nsources)*sizeof(Index),
                                cudaMemcpyHostToDevice, stream));
    BcArgs args;
    args.row_ptr = g.row_ptr;  args.row_ind = g.row_ind;
    args.in_ptr = g.in_ptr();
    args.in_ind = g.in_ind();
    args.n = n;
    args.sources = sources != NULL ? block.at<Index>(src) : NULL;
    args.seen = block.at<unsigned int>(seen);
    args.fresh[0] = block.at<unsigned int>(fresh);
    args.fresh[1] = args.fresh[0] + nn;
    args.stamp[0] = block.at<unsigned long long>(stamp0);
    args.stamp[1] = block.at<unsigned long long>(stamp1);
    args.sigma = block.at<double>(sigma);
    args.delta = block.at<double>(delta);
    args.total = block.at<double>(total);
    args.entries = block.at<int4>(list);
    args.level_start = block.at<Index>(level_start);
    args.partial = block.at<double>(partial);
    args.ticket = block.at<int>(ticket);
    args.counters = block.at<unsigned long long>(counters);
    for (Index b = 0; b < batches; ++b) {
      args.first = b*GB_BC_LANES;
      args.count = static_cast<int>(nsources - args.first < GB_BC_LANES ? nsources - args.first
                                                                        : GB_BC_LANES);
      CHECK((launchCooperative<bcKernel, GB_BC_NT>(stream, args)));
    }
  }
  CHECK(v->setStorage(GrB_DENSE));
  CHECK(v->dense_.allocateGpu());
  bcFinishKernel<<<gridFor(nn, 256), 256, 0, stream>>>(block.at<double>(total), n,
                                                       v->dense_.d_val_);
  GB_KERNEL_CHECK();
  clock.Stop();
  v->dense_.touched();
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_BC_HPP_
