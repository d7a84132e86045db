// graphblast_b200 backend — index-driven vector operations used by the
// label-propagation style consumers of mxv (connected components, colouring):
//   scatter        w[(Index)u[i]] = val           for every stored value of u
//   assignScatter  w[(Index)ind[i]] = u[i]        i < nindices
//   extractGather  w[i] = u[(Index)ind[i]]        i < nindices
// Semantics follow reference graphblas/backend/cuda/scatter.hpp:11-138,
// gather.hpp:11-52 and their kernels (kernels/scatter.hpp:8-50, gather.hpp:9-35),
// including their guards: scatter skips targets <= 0 (kernels/scatter.hpp:16),
// assignScatter skips targets outside [0, size of w), and extractGather skips
// sources outside [0, length of u), leaving w[i] as it was.  The frontend refuses
// more indices than the vector indexed by position i (u for assignScatter, w for
// extractGather) holds.  Where several sources name the same target, which one
// lands is unspecified there and here.
// Grid-stride kernels on the backend stream instead of <<<n/nt, nt>>> on stream 0.
#ifndef GRAPHBLAS_BACKEND_CUDA_INDEXED_HPP_
#define GRAPHBLAS_BACKEND_CUDA_INDEXED_HPP_

#include <iostream>

#include "graphblas/backend/cuda/kernels/kernels.hpp"

namespace graphblas {
namespace backend {

template <typename W, typename U, typename T>
__global__ void scatterConstByValueKernel(W* __restrict__ w, Index w_size,
                                          const U* __restrict__ targets,
                                          Index ntargets, T val) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < ntargets; i += stride) {
    const Index at = static_cast<Index>(targets[i]);
    if (at > 0 && at < w_size) w[at] = static_cast<W>(val);
  }
}

template <typename W, typename I, typename U>
__global__ void scatterByIndexKernel(W* __restrict__ w, Index w_size,
                                     const I* __restrict__ index,
                                     const U* __restrict__ source, Index count) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < count; i += stride) {
    const Index at = static_cast<Index>(index[i]);
    if (at >= 0 && at < w_size) w[at] = static_cast<W>(source[i]);
  }
}

template <typename W, typename I, typename U>
__global__ void gatherByIndexKernel(W* __restrict__ w, Index limit,
                                    const I* __restrict__ index,
                                    const U* __restrict__ source, Index count) {
  Index i = blockIdx.x*blockDim.x + threadIdx.x;
  const Index stride = gridDim.x*blockDim.x;
  for (; i < count; i += stride) {
    const Index from = static_cast<Index>(index[i]);
    if (from >= 0 && from < limit) w[i] = static_cast<W>(source[from]);
  }
}

// The value array an operation reads: a dense vector's values or a sparse
// vector's stored values, after the storage of `vec` has been forced to `as`.
template <typename T>
const T* storedValues(const Vector<T>* vec, Storage as) {
  return as == GrB_DENSE ? vec->dense_.d_val_ : vec->sparse_.d_val_;
}

template <typename W, typename M, typename U, typename T>
Info scatterConstant(Vector<W>* w, const Vector<M>* mask, const Vector<U>* u, T val,
    Descriptor* desc) {
  if (mask != NULL) return GrB_NOT_IMPLEMENTED;
  Storage u_type;
  CHECK(u->getStorage(&u_type));
  if (u_type != GrB_DENSE && u_type != GrB_SPARSE) return GrB_UNINITIALIZED_OBJECT;
  CHECK(u->materialize());
  CHECK(w->setStorage(GrB_DENSE));
  CHECK(w->materialize());
  Index w_size;
  CHECK(w->dense_.nvals(&w_size));
  const Index ntargets = (u_type == GrB_DENSE) ? u->dense_.nvals_ : u->sparse_.nvals_;
  // the dense form bounds the targets by u's length (reference scatter.hpp:44)
  const Index bound = (u_type == GrB_DENSE) ? ntargets : w_size;
  if (ntargets > 0) {
    scatterConstByValueKernel<<<gridFor(ntargets, 256), 256, 0, gbStream()>>>(
        w->dense_.d_val_, bound, storedValues(u, u_type), ntargets, val);
    GB_KERNEL_CHECK();
  }
  w->dense_.touched();
  return GrB_SUCCESS;
}

// Shared front end of assignScatter / extractGather: u decides the storage the
// index vector and w are read in (reference operations.hpp:1171-1180, 1228-1237);
// only dense results exist.
template <bool Gather, typename W, typename U, typename M, typename I>
Info indexedMove(Vector<W>* w, const Vector<M>* mask, const Vector<U>* u,
    const Vector<I>* indices, Descriptor* desc) {
  if (mask != NULL) return GrB_NOT_IMPLEMENTED;
  Vector<I>* ind = const_cast<Vector<I>*>(indices);
  Index nindices;
  CHECK(ind->nvals(&nindices));
  Storage u_type;
  CHECK(u->getStorage(&u_type));
  if (u_type != GrB_DENSE && u_type != GrB_SPARSE) return GrB_UNINITIALIZED_OBJECT;
  CHECK(u->materialize());
  CHECK(ind->materialize());
  Storage ind_type;
  CHECK(ind->getStorage(&ind_type));
  if (ind_type != u_type) CHECK(ind->setStorage(u_type));
  Storage w_type;
  CHECK(w->getStorage(&w_type));
  if (w_type != u_type) CHECK(w->setStorage(u_type));
  CHECK(w->getStorage(&w_type));
  if (w_type != GrB_DENSE) {
    std::cout << "Error: indexed " << (Gather ? "gather" : "scatter")
              << " into a sparse vector is not implemented\n";
    return GrB_NOT_IMPLEMENTED;
  }
  CHECK(w->materialize());
  Index w_size;
  CHECK(w->dense_.nvals(&w_size));
  // the gather reads u's value array: its sources are bounded by that array
  const Index u_len = (u_type == GrB_DENSE) ? u->dense_.nvals_ : u->sparse_.nvals_;
  if (nindices > 0) {
    const int grid = gridFor(nindices, 256);
    if (Gather)
      gatherByIndexKernel<<<grid, 256, 0, gbStream()>>>(w->dense_.d_val_, u_len,
          storedValues(ind, u_type), storedValues(u, u_type), nindices);
    else
      scatterByIndexKernel<<<grid, 256, 0, gbStream()>>>(w->dense_.d_val_, w_size,
          storedValues(ind, u_type), storedValues(u, u_type), nindices);
    GB_KERNEL_CHECK();
  }
  w->dense_.touched();
  return GrB_SUCCESS;
}

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_INDEXED_HPP_
