// graphblast_b200 backend — host side of the fused BFS (kernels/bfs_fused.cuh):
// one cooperative launch (launchCooperative, util.hpp) per traversal.  Entered from
// algorithm::bfs of this project's frontend when the descriptor carries the BFS flags
// of the reference's benchmark script (run_bfs.sh:8-27: --struconly 1 --opreuse 1
// --earlyexit 1, --fusedmask 1); every other combination runs the operation-by-operation
// loop.
#ifndef GRAPHBLAS_BACKEND_CUDA_BFS_FUSED_HPP_
#define GRAPHBLAS_BACKEND_CUDA_BFS_FUSED_HPP_

#include "graphblas/backend/cuda/kernels/bfs_fused.cuh"

namespace graphblas {
namespace backend {

// True when the traversal described by desc is the one the fused kernel computes.
inline bool bfsFusedApplies(Descriptor* desc) {
  Desc_value mask_mode, outp, inp0, inp1;
  if (desc->get(GrB_MASK, &mask_mode) != GrB_SUCCESS) return false;
  desc->get(GrB_OUTP, &outp); desc->get(GrB_INP0, &inp0); desc->get(GrB_INP1, &inp1);
  return desc->struconly() && desc->opreuse() && desc->earlyexit() && desc->fusedmask() &&
         mask_mode == GrB_DEFAULT && outp == GrB_DEFAULT && inp0 == GrB_DEFAULT &&
         inp1 == GrB_DEFAULT && !desc->debug() && desc->timing_ != 1;
}

// GB200_BFS_TRACE=1: every fused traversal, single- or multi-GPU, prints its
// per-level times on stderr.  Read once per process.
inline bool bfsTrace() {
  static const bool on = getEnv("GB200_BFS_TRACE", 0) != 0;
  return on;
}

// Layout of GB_SCRATCH_BFS for a traversal of n vertices (ScratchLayout, util.hpp): the
// byte offset of each array of BfsFusedArgs, and the bytes of the slot.  The slot stays
// with the descriptor, not with the call: a traversal that was only enqueued still uses
// it after bfsFused returns.
struct BfsScratchLayout {
  size_t visited[2], frontier, next, counters, heavy, walk, walk_count, walk_chunks,
         level8, bytes;
};

inline BfsScratchLayout bfsScratchLayout(Index n) {
  const size_t nwords = (static_cast<size_t>(n) + 31)/32;
  const size_t nchunks = (nwords + 31)/32;
  BfsScratchLayout l;
  ScratchLayout at;
  l.visited[0]  = at.place(nwords*sizeof(unsigned int));
  l.visited[1]  = at.place(nwords*sizeof(unsigned int));
  l.frontier    = at.place(nwords*sizeof(unsigned int));
  l.next        = at.place(nwords*sizeof(unsigned int));
  l.counters    = at.place(GB_BFS_NCOUNTERS*sizeof(unsigned long long));
  l.heavy       = at.place(GB_BFS_HEAVY_CAP*sizeof(Index));
  l.walk        = at.place(nchunks*GB_BFS_CHUNK*sizeof(Index));
  l.walk_count  = at.place(nchunks*sizeof(int));
  l.walk_chunks = at.place(nchunks*sizeof(Index));
  l.level8      = at.place(static_cast<size_t>(n));
  l.bytes = at.bytes;
  return l;
}

// Work counters of the last fused traversal run with this descriptor: levels,
// entries inspected pulling, pull levels, vertices pushed, edges pushed, vertices
// discovered pushing.  Zeros when none has run.
inline void bfsFusedStats(Descriptor* desc, Index n, unsigned long long out[6]) {
  static_assert(GB_BFS_CELL_FOUND_PUSHING == GB_BFS_CELL_LEVELS + 5,
                "the six result cells are not consecutive");
  for (int i = 0; i < 6; ++i) out[i] = 0ull;
  const BfsScratchLayout l = bfsScratchLayout(n);
  const size_t cells = l.counters + GB_BFS_CELL_LEVELS*sizeof(unsigned long long);
  if (desc->scratchSize(GB_SCRATCH_BFS) < cells + 6*sizeof(unsigned long long)) return;
  unsigned char* base = reinterpret_cast<unsigned char*>(desc->scratch(GB_SCRATCH_BFS, 0));
  CUDA_CALL(cudaMemcpyAsync(out, base + cells, 6*sizeof(unsigned long long),
      cudaMemcpyDeviceToHost, gbStream()));
  runtime().sync();
}

// v = BFS levels of A from s (source 1, unreached 0).  *depth = levels executed.
template <typename a>
Info bfsFused(Vector<float>* v, const Matrix<a>* A, Index s, Descriptor* desc, int* depth) {
  SparseMatrix<a>* S = const_cast<SparseMatrix<a>*>(&A->sparse_);
  const Index n = S->nrows_;
  if (n != S->ncols_) return GrB_DIMENSION_MISMATCH;
  if (S->d_csrRowPtr_ == NULL || S->d_cscColPtr_ == NULL) return GrB_UNINITIALIZED_OBJECT;
  cudaStream_t stream = gbStream();
  CHECK(v->setStorage(GrB_DENSE));
  CHECK(v->dense_.allocateGpu());

  // highest-degree-neighbour summary of the pulled structure: the entry each open
  // row probes in the pull scan.  Built by the first traversal of a structure (2 nnz
  // gathers of the offsets) and kept with the matrix, 4(n + 1) + n/8 bytes.
  const int fw = 1;                                   // vxm pulls over the CSC
  const Index* probe = pullMaxDegreeNeighbours(S, fw, S->d_cscColPtr_, S->d_cscRowInd_, n);

  const BfsScratchLayout l = bfsScratchLayout(n);
  unsigned char* base =
      reinterpret_cast<unsigned char*>(desc->scratch(GB_SCRATCH_BFS, l.bytes));
  BfsFusedArgs args;
  args.push_ptr = S->d_csrRowPtr_;  args.push_ind = S->d_csrColInd_;
  args.pull_ptr = S->d_cscColPtr_;  args.pull_ind = S->d_cscRowInd_;
  args.pull_probe = probe;
  // Rows without in-neighbours may count as visited from the start only when they
  // have no out-neighbours either: a visited row is taken to have been expanded, so
  // in a directed graph one that points somewhere would let the pull discover what
  // it points at.  When the pulled structure is the pushed one, that is the same
  // bitmap; otherwise the pushed structure's empty rows are ANDed in.
  args.pull_empty = pullEmptyRowBits(probe, n);
  args.push_empty = S->sameStructure() ? NULL : pullEmptyRowBits(
      pullFirstNeighbours(S, 0, S->d_csrRowPtr_, S->d_csrColInd_, n), n);
  args.n = n;
  args.source = s;
  args.max_levels = desc->max_niter_;
  args.switchpoint = desc->switchpoint();
  args.mode = desc->mxvRoute();
  args.levels = v->dense_.d_val_;
  args.visited[0]  = reinterpret_cast<unsigned int*>(base + l.visited[0]);
  args.visited[1]  = reinterpret_cast<unsigned int*>(base + l.visited[1]);
  args.frontier    = reinterpret_cast<unsigned int*>(base + l.frontier);
  args.next        = reinterpret_cast<unsigned int*>(base + l.next);
  args.counters    = reinterpret_cast<unsigned long long*>(base + l.counters);
  args.heavy       = reinterpret_cast<Index*>(base + l.heavy);
  args.walk        = reinterpret_cast<Index*>(base + l.walk);
  args.walk_count  = reinterpret_cast<int*>(base + l.walk_count);
  args.walk_chunks = reinterpret_cast<Index*>(base + l.walk_chunks);
  // no fill: the kernel reads the byte of a row only when it wrote it in this traversal
  args.level8      = base + l.level8;

  args.trace = bfsTrace();
  args.prof_bytes = NULL;               // the kernel adds its bytes when profiling
  if (profiler().enabled) {
    profiler().ensureCells(gbStream());
    args.prof_bytes = profiler().d_cells + GB_PROF_PULL_BOOL;
  }

  // push-only traversals run the instantiation without the pull level, with more
  // warps per SM
  profiler().begin(GB_PROF_PULL_BOOL, stream);
  const Info launched = args.mode == 1
      ? launchCooperative<bfsFusedKernel<GB_BFS_PUSH_NT, GB_BFS_PUSH_MINB, false>,
                          GB_BFS_PUSH_NT>(stream, args)
      : launchCooperative<bfsFusedKernel<GB_BFS_NT, GB_BFS_MINB, true>, GB_BFS_NT>(stream, args);
  if (launched != GrB_SUCCESS) return launched;
  profiler().end(GB_PROF_PULL_BOOL, stream, 0.0);
  v->dense_.touched();
  if (args.trace) {                      // per-level times of this traversal
    unsigned long long cells[GB_BFS_NCOUNTERS];
    CUDA_CALL(cudaMemcpyAsync(cells, args.counters, sizeof(cells), cudaMemcpyDeviceToHost,
        stream));
    runtime().sync();
    const unsigned long long* const clock = cells + GB_BFS_CELL_LEVEL_CLOCK;
    const int levels = static_cast<int>(
        cells[GB_BFS_CELL_LEVELS] < GB_BFS_TIMED_LEVELS - 1 ? cells[GB_BFS_CELL_LEVELS]
                                                            : GB_BFS_TIMED_LEVELS - 1);
    fprintf(stderr, "bfs trace: set-up %.1fus",
            1e-3*static_cast<double>((clock[0] >> 2) - cells[GB_BFS_CELL_START_CLOCK]));
    int second_phases = 0;
    for (int l = 1; l <= levels; ++l) {
      const unsigned long long start = clock[l - 1] >> 2, end = clock[l] >> 2;
      const unsigned long long scan = cells[GB_BFS_CELL_SCAN_CLOCK + l];
      second_phases += static_cast<int>((clock[l] >> 1) & 1ull);
      // pull: scan, walk (0 without a second phase), rows walked, chunks listed
      if (clock[l] & 1ull)
        fprintf(stderr, " L%d pull %.1fus (scan %.1f walk %.1f, %llu walked, %llu listed)",
                l, 1e-3*static_cast<double>(end - start),
                1e-3*static_cast<double>(scan - start),
                1e-3*static_cast<double>(end - scan), cells[GB_BFS_CELL_WALKED + l],
                cells[GB_BFS_CELL_LISTED_CHUNKS + l]);
      else
        fprintf(stderr, " L%d push %.1fus", l, 1e-3*static_cast<double>(end - start));
    }
    fprintf(stderr, " end-pass %.1fus\n",
            1e-3*static_cast<double>(cells[GB_BFS_CELL_END_PASS_CLOCK] -
                                     cells[GB_BFS_CELL_LAST_LEVEL_CLOCK]));
    // Grid barriers: the set-up's, one per level and one per second phase.  Each level
    // marks in its clock cell whether it ran a second phase: a counter cell added to
    // after the barriers costs the push-only instantiation spill reloads.  Levels past
    // the traced ones are counted as if they ran none.
    fprintf(stderr, "bfs barriers: %llu (second phases %d%s)\n",
            1ull + cells[GB_BFS_CELL_LEVELS] + second_phases, second_phases,
            cells[GB_BFS_CELL_LEVELS] > static_cast<unsigned long long>(levels)
                ? ", later levels not traced" : "");
  }
  if (depth != NULL) {
    const unsigned long long levels = runtime().fetch(args.counters + GB_BFS_CELL_LEVELS);
    *depth = static_cast<int>(levels);
    desc->lastmxv_ = GrB_PULLONLY;
  }
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_BFS_FUSED_HPP_
