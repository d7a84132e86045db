// oracle/_ref/libgbref_lgc.so — the reference's OWN CPU checker of local graph
// clustering, compiled from the sources where they lie under the reference tree (never
// copied):
//   graphblas/algorithm/test_lgc.hpp   SimpleReferenceLgc<float>
// It is what the reference's lgc driver (example/glgc.cu) checks its result against.
// This file only adds an extern "C" entry point; tests/lgc_reference.py binds it.  It
// is its own small library (ref_lgc.mk) so that the other reference checkers'
// wrapper and recipe stay as they are.
//
// TEST INFRASTRUCTURE ONLY: used by tests/ and tools/bench_lgc.py.  Nothing in
// graphblast_b200/ links or loads it.
#define GRB_USE_CUDA
#define __host__
#define __device__

#include <fcntl.h>
#include <unistd.h>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <iostream>
#include <vector>

#include <boost/program_options.hpp>

#include "graphblas/backend.hpp"
#include "graphblas/mmio.hpp"
#include "graphblas/types.hpp"
#include "graphblas/util.hpp"
#include "graphblas/algorithm/test_lgc.hpp"

namespace {
// The checker prints its parameters, arrays and timing; keep the caller's stdout clean.
struct QuietStdout {
  int saved;
  QuietStdout() {
    fflush(stdout);
    std::cout.flush();
    saved = dup(1);
    int nul = open("/dev/null", O_WRONLY);
    dup2(nul, 1);
    close(nul);
  }
  ~QuietStdout() {
    fflush(stdout);
    std::cout.flush();
    dup2(saved, 1);
    close(saved);
  }
};
}  // namespace

#pragma GCC visibility push(default)
extern "C" {

// p[0..nrows) = SimpleReferenceLgc<float> of the CSR (rowptr, colind) from src, run for
// exactly max_niter rounds (its loop has no other stop).
void ref_lgc(int nrows, const int* rowptr, const int* colind, float* p, int src,
             double alpha, double eps, int max_niter) {
  QuietStdout q;
  graphblas::algorithm::SimpleReferenceLgc<float>(nrows, rowptr, colind,
      static_cast<const float*>(NULL), p, src, alpha, eps, max_niter);
}

}  // extern "C"
#pragma GCC visibility pop
