// graphblast_b200 backend — host side of the greedy schedule
// (kernels/greedy_schedule.cuh): the scratch and the one cooperative launch that the
// graph colouring (color.hpp) and the maximal independent set (mis.hpp) share.
#ifndef GRAPHBLAS_BACKEND_CUDA_GREEDY_SCHEDULE_HPP_
#define GRAPHBLAS_BACKEND_CUDA_GREEDY_SCHEDULE_HPP_

#include "graphblas/backend/cuda/graph_input.hpp"
#include "graphblas/backend/cuda/kernels/greedy_schedule.cuh"

namespace graphblas {
namespace backend {

// One run of kernel K on an A that passed graphCheck (with its CSC): init(state,
// stream) sets the n-word state on the stream before v is touched, then v becomes dense
// with nrows(A) entries and K writes it; *count (when not NULL) = K's GREEDY_COUNT, 0
// when A has no rows; *ms (when not NULL) = the device time, from CUDA events.
// Scratch: the counter cells, five n-word arrays (state, waiting_on, resume, two lists)
// and the pattern's zero row pointers.
template <typename W, void (*K)(GreedyArgs, W*), typename a, typename Init>
Info greedyRun(Vector<W>* v, const SparseMatrix<a>* S, unsigned int seed, int* count,
               float* ms, Init init) {
  const Index n = S->nrows_;
  GpuTimer clock;
  clock.Start();
  if (count != NULL) *count = 0;
  if (n == 0) {
    CHECK(v->setStorage(GrB_DENSE));
    clock.Stop();
    if (ms != NULL) *ms = clock.ElapsedMillis();
    return GrB_SUCCESS;
  }
  cudaStream_t stream = gbStream();
  const size_t array = static_cast<size_t>(n)*sizeof(Index);   // bytes of an n-word array
  ScratchLayout l;
  const size_t counters = l.place(GREEDY_NCELLS*sizeof(unsigned long long));
  const size_t state = l.place(array), waiting_on = l.place(array), resume = l.place(array);
  const size_t list0 = l.place(array), list1 = l.place(array);
  const size_t zero_rows = l.place(GraphPattern::zeroRowBytes(*S));
  const DeviceBlock block(gbMalloc(l.bytes));
  const GraphPattern g(*S, block.at<Index>(zero_rows));
  GreedyArgs args;
  args.row_ptr = g.row_ptr;  args.row_ind = g.row_ind;
  args.col_ptr = g.col_ptr;  args.col_ind = g.col_ind;
  args.n = n;
  args.seed = seed;
  args.counters   = block.at<unsigned long long>(counters);
  args.state      = block.at<unsigned int>(state);
  args.waiting_on = block.at<Index>(waiting_on);
  args.resume     = block.at<Index>(resume);
  args.list[0]    = block.at<Index>(list0);
  args.list[1]    = block.at<Index>(list1);
  CUDA_CALL(cudaMemsetAsync(args.counters, 0, GREEDY_NCELLS*sizeof(unsigned long long),
                            stream));
  init(args.state, stream);

  CHECK(v->setStorage(GrB_DENSE));
  CHECK(v->dense_.allocateGpu());
  CHECK((launchCooperative<K, GB_GC_NT>(stream, args, v->dense_.d_val_)));
  clock.Stop();
  v->dense_.touched();
  if (count != NULL)
    *count = static_cast<int>(runtime().fetch(args.counters + GREEDY_COUNT));
  if (ms != NULL) *ms = clock.ElapsedMillis();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_GREEDY_SCHEDULE_HPP_
