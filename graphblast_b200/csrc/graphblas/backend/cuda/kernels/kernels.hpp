// graphblast_b200 backend — kernel umbrella (same role as reference
// graphblas/backend/cuda/kernels/kernels.hpp:1-16).
#ifndef GRAPHBLAS_BACKEND_CUDA_KERNELS_KERNELS_HPP_
#define GRAPHBLAS_BACKEND_CUDA_KERNELS_KERNELS_HPP_

#include "graphblas/backend/cuda/kernels/common.cuh"
#include "graphblas/backend/cuda/kernels/util.cuh"
#include "graphblas/backend/cuda/kernels/compact.cuh"
#include "graphblas/backend/cuda/kernels/elementwise.cuh"
#include "graphblas/backend/cuda/kernels/reduce.cuh"
#include "graphblas/backend/cuda/kernels/spmv_pull.cuh"
#include "graphblas/backend/cuda/kernels/spmspv_push.cuh"
#include "graphblas/backend/cuda/kernels/spgemm_masked.cuh"
#include "graphblas/backend/cuda/kernels/spgemm_hash.cuh"
#include "graphblas/backend/cuda/kernels/spgemm_unmasked.cuh"
#include "graphblas/backend/cuda/kernels/ewise_matrix.cuh"
#include "graphblas/backend/cuda/kernels/spmm.cuh"

#endif  // GRAPHBLAS_BACKEND_CUDA_KERNELS_KERNELS_HPP_
