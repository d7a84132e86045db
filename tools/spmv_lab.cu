// tools/spmv_lab.cu — kernel laboratory for the pull-direction merge-path SpMV.
// Generates an R-MAT graph on the device (same generator as gb200_rmat_edges),
// builds the CSR with thrust, and times configurations of spmvMergeKernelT plus
// two reference points (pure streaming of colind/val, streaming + gather without
// the merge).  Prints one line per variant: ms, algorithmic GB/s, fraction of the
// measured HBM peak.  Usage: spmv_lab [scale=22] [edgefactor=16] [reps=5]
#define GRB_USE_CUDA
#include <thrust/device_vector.h>
#include <thrust/sort.h>
#include <thrust/unique.h>
#include <thrust/remove.h>
#include <thrust/scan.h>
#include <thrust/binary_search.h>
#include <thrust/iterator/counting_iterator.h>
#include <boost/program_options.hpp>
#include "graphblas/graphblas.hpp"
#include "graphblas/backend/cuda/spmv_hub.hpp"

bool debug_;
bool memory_;

using graphblas::Index;
using namespace graphblas::backend;

__global__ void rmatKeys(int scale, long long nedges, unsigned long long seed,
                         unsigned long long* keys) {
  const unsigned int T1 = 2448131358u, T2 = 3264175144u, T3 = 4080218930u;
  long long e = (long long)blockIdx.x*blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x*blockDim.x;
  const unsigned long long n = 1ull << scale;
  for (; e < nedges; e += stride) {
    unsigned int s = 0, d = 0;
    for (int l = 0; l < scale; ++l) {
      unsigned long long z = ((seed << 48) ^ ((unsigned long long)e << 6) ^
          (unsigned long long)l) + 0x9E3779B97F4A7C15ull;
      z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
      z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
      z = z ^ (z >> 31);
      const unsigned int r = (unsigned int)(z >> 32);
      s = (s << 1) | ((r >= T2) ? 1u : 0u);
      d = (d << 1) | (((r >= T1 && r < T2) || r >= T3) ? 1u : 0u);
    }
    keys[2*e]     = (unsigned long long)s*n + d;
    keys[2*e + 1] = (unsigned long long)d*n + s;
  }
}

struct IsLoop {
  unsigned long long n;
  __host__ __device__ bool operator()(unsigned long long k) const {
    return (k / n) == (k % n);
  }
};

__global__ void splitKeys(const unsigned long long* keys, long long nnz,
                          unsigned long long n, int* rows, int* cols, float* val) {
  long long i = (long long)blockIdx.x*blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x*blockDim.x;
  for (; i < nnz; i += stride) {
    rows[i] = (int)(keys[i] / n);
    cols[i] = (int)(keys[i] % n);
    val[i]  = (float)(1 + (keys[i]*2654435761ull >> 40) % 64);
  }
}

// Reference point 1: stream colind + val with 256-bit loads, no gather.
template <int NT>
__global__ void __launch_bounds__(NT)
streamOnlyKernel(float* out, const int* colind, const float* val, long long nnz) {
  long long c = (long long)blockIdx.x*NT + threadIdx.x;
  const long long stride = (long long)gridDim.x*NT;
  float acc = 0.f;
  for (; (c + 1)*8 <= nnz; c += stride) {
    Word8 cw = ldStream256(colind + c*8);
    Word8 vw = ldStream256(val + c*8);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += __int_as_float(vw.w[j]) + (cw.w[j] & 1);
  }
  if (acc == 123.456f) out[0] = acc;
}

// Reference point 2: stream + gather u[col], no row reduction.
template <int NT>
__global__ void __launch_bounds__(NT)
streamGatherKernel(float* out, const int* colind, const float* val,
                   const float* u, long long nnz) {
  long long c = (long long)blockIdx.x*NT + threadIdx.x;
  const long long stride = (long long)gridDim.x*NT;
  const uint64_t pol = makeEvictLastPolicy();
  float acc = 0.f;
  for (; (c + 1)*8 <= nnz; c += stride) {
    Word8 cw = ldStream256(colind + c*8);
    Word8 vw = ldStream256(val + c*8);
    float uv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) uv[j] = ldGather(u + cw.w[j], pol);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fminf(acc, __int_as_float(vw.w[j]) + uv[j]);
  }
  if (acc == 123.456f) out[0] = acc;
}

// Reference point 3: same as 2 but every column is folded into a window of
// `mask`+1 elements: the gathers keep hitting distinct 128-byte lines (one L1
// wavefront each) while the L2 sector traffic disappears (window resident in L1).
template <int NT>
__global__ void __launch_bounds__(NT)
streamGatherWindowKernel(float* out, const int* colind, const float* val,
                         const float* u, long long nnz, int mask) {
  long long c = (long long)blockIdx.x*NT + threadIdx.x;
  const long long stride = (long long)gridDim.x*NT;
  const uint64_t pol = makeEvictLastPolicy();
  float acc = 0.f;
  for (; (c + 1)*8 <= nnz; c += stride) {
    Word8 cw = ldStream256(colind + c*8);
    Word8 vw = ldStream256(val + c*8);
    float uv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) uv[j] = ldGather(u + (cw.w[j] & mask), pol);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fminf(acc, __int_as_float(vw.w[j]) + uv[j]);
  }
  if (acc == 123.456f) out[0] = acc;
}

// Ceiling of the hub design: stream + (hub from shared memory | cold gather), no
// row reduction.  One persistent CTA per SM, K hub slots in dynamic shared memory.
template <int NT>
__global__ void __launch_bounds__(NT, 1)
streamGatherHubKernel(float* out, const int* enc, const float* val, const float* u,
                      const float* hub_vals, int K, long long nnz) {
  extern __shared__ float s_hubv[];
  for (int i = threadIdx.x; i < K; i += NT) s_hubv[i] = hub_vals[i];
  __syncthreads();
  long long c = (long long)blockIdx.x*NT + threadIdx.x;
  const long long stride = (long long)gridDim.x*NT;
  const uint64_t pol = makeEvictLastPolicy();
  float acc = 0.f;
  for (; (c + 1)*8 <= nnz; c += stride) {
    Word8 cw = ldStream256(enc + c*8);
    Word8 vw = ldStream256(val + c*8);
    float uv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (cw.w[j] >= 0)
        uv[j] = ldGather(u + cw.w[j], pol);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (cw.w[j] < 0) uv[j] = s_hubv[cw.w[j] & 0x7fffffff];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fminf(acc, __int_as_float(vw.w[j]) + uv[j]);
  }
  if (acc == 123.456f) out[0] = acc;
}

typedef graphblas::MinimumPlusSemiring<float> SR;

template <int GROUPS, int HUB_K>
float runHub(float* w, const HubIndex& h, const int* rowptr, const float* val,
             const float* u, int n, int nnz, int reps) {
  SR op;
  thrust::device_vector<int> crow(h.ntiles);
  thrust::device_vector<float> cval(h.ntiles);
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  float best = 1e30f;
  for (int r = 0; r < reps + 1; ++r) {
    cudaEventRecord(a, gbStream());
    spmvHubRun<GROUPS, HUB_K>(w, h, op, val, u, nnz,
        thrust::raw_pointer_cast(crow.data()), thrust::raw_pointer_cast(cval.data()),
        gbStream());
    cudaEventRecord(b, gbStream());
    cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    if (r > 0 && ms < best) best = ms;
  }
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) printf("CUDA error: %s\n", cudaGetErrorString(err));
  return best;
}

template <int NT, int IPT, bool LaneMajor>
float runMerge(float* w, const int* rowptr, const int* colind, const float* val,
               const float* u, int n, int nnz, int reps, int carveout) {
  SR op;
  const long long total = (long long)n + nnz;
  const int tile = NT*IPT;
  const int nctas = (int)((total + tile - 1)/tile);
  thrust::device_vector<int> tiles(nctas + 1), crow(nctas);
  thrust::device_vector<float> cval(nctas);
  spmvMergePartitionKernel<<<(nctas + 256)/256, 256>>>(
      thrust::raw_pointer_cast(tiles.data()), rowptr, n, nnz, nctas, tile);
  auto kern = spmvMergeKernelT<NT, IPT, LaneMajor, float, float, float,
      decltype(graphblas::extractMul(op)), decltype(graphblas::extractAdd(op))>;
  if (carveout >= 0)
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                         carveout);
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  float best = 1e30f;
  for (int r = 0; r < reps + 1; ++r) {
    cudaEventRecord(a);
    kern<<<nctas, NT>>>(w, thrust::raw_pointer_cast(tiles.data()),
        thrust::raw_pointer_cast(crow.data()),
        thrust::raw_pointer_cast(cval.data()), rowptr, colind, val, u, n, nnz,
        op.identity(), graphblas::extractMul(op), graphblas::extractAdd(op));
    spmvCarryFixupKernel<<<(nctas + 255)/256, 256>>>(w,
        thrust::raw_pointer_cast(crow.data()),
        thrust::raw_pointer_cast(cval.data()), nctas, graphblas::extractAdd(op));
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    if (r > 0 && ms < best) best = ms;
  }
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) printf("CUDA error: %s\n", cudaGetErrorString(err));
  return best;
}

int main(int argc, char** argv) {
  const int scale = argc > 1 ? atoi(argv[1]) : 22;
  const int ef    = argc > 2 ? atoi(argv[2]) : 16;
  const int reps  = argc > 3 ? atoi(argv[3]) : 5;
  const double peak = argc > 4 ? atof(argv[4]) : 6547.8;
  const unsigned long long n = 1ull << scale;
  const long long nedges = (long long)ef << scale;

  thrust::device_vector<unsigned long long> keys(2*nedges);
  rmatKeys<<<148*8, 256>>>(scale, nedges, 1ull, thrust::raw_pointer_cast(keys.data()));
  auto end1 = thrust::remove_if(keys.begin(), keys.end(), IsLoop{n});
  thrust::sort(keys.begin(), end1);
  auto end2 = thrust::unique(keys.begin(), end1);
  const long long nnz = end2 - keys.begin();
  thrust::device_vector<int> rows(nnz), cols(nnz), rowptr(n + 1);
  thrust::device_vector<float> val(nnz), u(n), w(n), w2(n);
  splitKeys<<<148*8, 256>>>(thrust::raw_pointer_cast(keys.data()), nnz, n,
      thrust::raw_pointer_cast(rows.data()), thrust::raw_pointer_cast(cols.data()),
      thrust::raw_pointer_cast(val.data()));
  thrust::lower_bound(rows.begin(), rows.end(), thrust::counting_iterator<int>(0),
      thrust::counting_iterator<int>((int)n + 1), rowptr.begin());
  keys.clear(); keys.shrink_to_fit();
  thrust::sequence(u.begin(), u.end());
  printf("scale %d: n=%llu nnz=%lld\n", scale, n, nnz);
  const int* rp = thrust::raw_pointer_cast(rowptr.data());
  const int* ci = thrust::raw_pointer_cast(cols.data());
  const float* va = thrust::raw_pointer_cast(val.data());
  const float* up = thrust::raw_pointer_cast(u.data());
  float* wp = thrust::raw_pointer_cast(w.data());
  const double alg = 8.0*nnz + 12.0*n + 4.0;
  auto report = [&](const char* name, float ms) {
    printf("%-44s %8.3f ms  %7.0f GB/s  %.3f of peak\n", name, ms,
           alg/1e6/ms, alg/1e6/ms/peak);
  };

  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  float ms, best;
  best = 1e30f;
  for (int r = 0; r < reps + 1; ++r) {
    cudaEventRecord(a);
    streamOnlyKernel<256><<<148*8, 256>>>(wp, ci, va, nnz);
    cudaEventRecord(b); cudaEventSynchronize(b); cudaEventElapsedTime(&ms, a, b);
    if (r > 0 && ms < best) best = ms;
  }
  report("stream colind+val only (no gather)", best);
  best = 1e30f;
  for (int r = 0; r < reps + 1; ++r) {
    cudaEventRecord(a);
    streamGatherKernel<256><<<148*8, 256>>>(wp, ci, va, up, nnz);
    cudaEventRecord(b); cudaEventSynchronize(b); cudaEventElapsedTime(&ms, a, b);
    if (r > 0 && ms < best) best = ms;
  }
  report("stream + gather (persistent 148x8x256)", best);
  best = 1e30f;
  for (int r = 0; r < reps + 1; ++r) {
    cudaEventRecord(a);
    streamGatherKernel<256><<<148*4, 256>>>(wp, ci, va, up, nnz);
    cudaEventRecord(b); cudaEventSynchronize(b); cudaEventElapsedTime(&ms, a, b);
    if (r > 0 && ms < best) best = ms;
  }
  report("stream + gather (persistent 148x4x256)", best);
  best = 1e30f;
  for (int r = 0; r < reps + 1; ++r) {
    cudaEventRecord(a);
    streamGatherKernel<256><<<(int)((nnz/8 + 255)/256), 256>>>(wp, ci, va, up, nnz);
    cudaEventRecord(b); cudaEventSynchronize(b); cudaEventElapsedTime(&ms, a, b);
    if (r > 0 && ms < best) best = ms;
  }
  report("stream + gather (one chunk per thread)", best);

#define LAB(NT, IPT, LM, CARVE)                                              \
  { char name[96];                                                           \
    snprintf(name, sizeof(name),                                             \
             "merge NT=%d IPT=%d lanemajor=%d carveout=%d",                  \
             NT, IPT, (int)LM, CARVE);                                       \
    report(name, runMerge<NT, IPT, LM>(wp, rp, ci, va, up, (int)n,           \
                                       (int)nnz, reps, CARVE)); }
  if (getenv("LAB_FULL")) {
  LAB(128, 7, false, 25)
  LAB(128, 9, false, 25)
  LAB(128, 11, false, 25)
  LAB(128, 15, false, 25)
  LAB(128, 15, false, 33)
  LAB(64, 11, false, 25)
  LAB(64, 15, false, 25)
  LAB(64, 19, false, 25)
  LAB(256, 7, false, 25)
  LAB(256, 9, false, 33)
  LAB(128, 9, true, 25)
  } else { LAB(128, 9, false, 25) }

  // wavefront vs sector: gathers folded into 4 KB / 64 KB / 1 MB windows
  for (int mask : {1023, 16383, 262143}) {
    best = 1e30f;
    for (int r = 0; r < reps + 1; ++r) {
      cudaEventRecord(a);
      streamGatherWindowKernel<256><<<148*8, 256>>>(wp, ci, va, up, nnz, mask);
      cudaEventRecord(b); cudaEventSynchronize(b); cudaEventElapsedTime(&ms, a, b);
      if (r > 0 && ms < best) best = ms;
    }
    char name[96];
    snprintf(name, sizeof(name), "stream + gather folded into %d floats", mask + 1);
    report(name, best);
  }

  // ---- ceiling of the hub design ------------------------------------------------
  for (int K : {40960}) {
    HubIndex h;
    buildHubIndex(&h, rp, ci, (Index)n, (Index)n, (Index)nnz, K > 0 ? K : 4);
    if (K == 0) cudaMemcpy(h.enc_ci, ci, nnz*sizeof(int), cudaMemcpyDeviceToDevice);
    hubPrepassKernel<<<(K + 255)/256 + 1, 256>>>((float*)h.hub_vals, up, h.hub_ids,
        K > 0 ? h.count : 0, K > 0 ? K : 4, 0.f, wp, (const Index*)NULL, 0, 0.f);
    for (int nt : {1024, 512}) {
      auto kern = nt == 1024 ? streamGatherHubKernel<1024> : streamGatherHubKernel<512>;
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200*1024);
      best = 1e30f;
      for (int r = 0; r < reps + 1; ++r) {
        cudaEventRecord(a);
        kern<<<148, nt, K*4 + 16>>>(wp, h.enc_ci, va, up, (float*)h.hub_vals, K, nnz);
        cudaEventRecord(b); cudaEventSynchronize(b); cudaEventElapsedTime(&ms, a, b);
        if (r > 0 && ms < best) best = ms;
      }
      char name[96];
      snprintf(name, sizeof(name), "ceiling K=%d cover=%.3f NT=%d", K,
               K > 0 ? h.coverage : 0.0, nt);
      report(name, best);
    }
    h.release();
  }
  if (getenv("LAB_CEILING_ONLY")) return 0;

  // ---- hub kernel -------------------------------------------------------------
  // reference result: the merge kernel
  runMerge<128, 9, false>(wp, rp, ci, va, up, (int)n, (int)nnz, 1, 25);
  std::vector<float> want(n), got(n);
  std::vector<int> h_rp(n + 1);
  cudaMemcpy(h_rp.data(), rp, (n + 1)*sizeof(int), cudaMemcpyDeviceToHost);
  cudaMemcpy(want.data(), wp, n*sizeof(float), cudaMemcpyDeviceToHost);
  float* w2p = thrust::raw_pointer_cast(w2.data());
  auto check = [&](const char* name) {
    cudaMemcpy(got.data(), w2p, n*sizeof(float), cudaMemcpyDeviceToHost);
    long long bad = 0; long long firstbad = -1;
    for (size_t i = 0; i < n; ++i)
      if (memcmp(&want[i], &got[i], 4) != 0) {
        if (bad < 4) printf("      row %zu want %g got %g deg %d\n", i, want[i], got[i], h_rp[i+1]-h_rp[i]);
        if (!bad) firstbad = i; ++bad; }
    printf("   %-40s %s (%lld mismatches, first %lld)\n", name,
           bad ? "MISMATCH" : "bit-exact", bad, firstbad);
    cudaMemset(w2p, 0xff, n*sizeof(float));
  };
#define HUBLAB(G, K)                                                           \
  { HubIndex h;                                                                \
    buildHubIndex(&h, rp, ci, (Index)n, (Index)n, (Index)nnz, K > 0 ? K : 4);  \
    if (K == 0) cudaMemcpy(h.enc_ci, ci, nnz*sizeof(int), cudaMemcpyDeviceToDevice); \
    char name[96];                                                             \
    snprintf(name, sizeof(name), "hub groups=%d K=%d cover=%.3f", G, K,         \
             K > 0 ? h.coverage : 0.0);                                        \
    report(name, runHub<G, K>(w2p, h, rp, va, up, (int)n, (int)nnz, reps));    \
    check(name);                                                               \
    h.release(); }
  HUBLAB(8, 32768)
  HUBLAB(8, 32768)
  HUBLAB(8, 40960)
  HUBLAB(7, 40960)
  HUBLAB(6, 40960)
  HUBLAB(8, 0)
  return 0;
}
