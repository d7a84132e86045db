// graphblast_b200 — breadth-first search as a loop of GraphBLAS operations.
//
// Operation sequence per level is the reference's (graphblas/algorithm/bfs.hpp:46-79):
//   assign(v<f1> = level) ; vxm(f2<!v> = f1 (||.&&) A) ; swap(f1,f2) ;
//   succ = reduce(+, f1) ; stop when succ == 0.
// With the flags of the reference's benchmark script (run_bfs.sh:8-27) that whole
// loop runs as ONE cooperative kernel (backend/cuda/bfs_fused.hpp): same levels,
// no launch or host round trip per level.  --timing 1 or any other flag
// combination takes the operation-by-operation loop below.
// Output convention: level of the source is 1, unreached vertices stay 0.
// Returns the device time of the loop in milliseconds ("tight" in the reference
// drivers), excluding the initial fill of v.  With timed = false the fused
// traversal is only enqueued: no events, no wait for it to end, and 0 is returned
// (back-to-back traversals then keep the GPU busy); the operation-by-operation
// loop reads frontier sizes on the host and is timed either way.
#ifndef GRAPHBLAS_ALGORITHM_BFS_HPP_
#define GRAPHBLAS_ALGORITHM_BFS_HPP_

#include <string>
#include <vector>

#include "graphblas/algorithm/common.hpp"

namespace graphblas {
namespace algorithm {

inline float bfs(Vector<float>* v, const Matrix<float>* A, Index s, Descriptor* desc,
                 bool timed = true) {
  Index n;
  GB_ALGO_STEP(A->nrows(&n));
  if (backend::bfsFusedApplies(&desc->descriptor_) && A->matrix_.isSparse()) {
    if (!timed) {
      if (backend::bfsFused(&v->vector_, &A->matrix_, s, &desc->descriptor_,
                            static_cast<int*>(NULL)) == GrB_SUCCESS)
        return 0.f;
    } else {
      backend::GpuTimer fused_clock;
      fused_clock.Start();
      const Info fused = backend::bfsFused(&v->vector_, &A->matrix_, s,
                                           &desc->descriptor_, static_cast<int*>(NULL));
      fused_clock.Stop();
      if (fused == GrB_SUCCESS) return fused_clock.ElapsedMillis();
    }
  }
  GB_ALGO_STEP(v->fill(0.f));

  Vector<float> frontier(n);
  Vector<float> next(n);

  Desc_value mxv_mode;
  GB_ALGO_STEP(desc->get(GrB_MXVMODE, &mxv_mode));
  if (mxv_mode == GrB_PULLONLY) {
    GB_ALGO_STEP(frontier.fill(0.f));
    GB_ALGO_STEP(frontier.setElement(1.f, s));
  } else {
    std::vector<Index> src_ind(1, s);
    std::vector<float> src_val(1, 1.f);
    GB_ALGO_STEP(frontier.build(&src_ind, &src_val, 1, GrB_NULL));
  }

  backend::Descriptor& d = desc->descriptor_;
  const bool verbose = (d.timing_ == 1);
  LoopTimer clock(verbose);
  float succ = 0.f;
  Index unvisited = n;
  clock.begin();

  for (int level = 1; level <= d.max_niter_; ++level) {
    unvisited -= static_cast<int>(succ);
    assign<float, float, float, Index>(v, &frontier, GrB_NULL,
        static_cast<float>(level), GrB_ALL, n, desc);
    GB_ALGO_STEP(desc->toggle(GrB_MASK));
    vxm<float, float, float, float>(&next, v, GrB_NULL,
        LogicalOrAndSemiring<float>(), &frontier, A, desc);
    GB_ALGO_STEP(desc->toggle(GrB_MASK));
    GB_ALGO_STEP(next.swap(&frontier));
    reduce<float, float>(&succ, GrB_NULL, PlusMonoid<float>(), &frontier, desc);

    if (verbose) {
      float ms = clock.lap();
      std::cout << level << ", " << succ << "/" << n << ", " << unvisited
                << ", " << (d.lastmxv_ == GrB_PUSHONLY ? "push" : "pull")
                << ", " << ms << "\n";
    }
    if (succ == 0) break;
  }
  return clock.finish();
}

}  // namespace algorithm
}  // namespace graphblas

#endif  // GRAPHBLAS_ALGORITHM_BFS_HPP_
