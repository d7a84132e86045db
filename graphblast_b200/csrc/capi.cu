// graphblast_b200 — C ABI implementation (include/graphblast_b200.h).
//
// One translation unit: includes the header-only frontend mirror (include/graphblas)
// and the sm_90a backend (graphblast_b200/csrc/graphblas/backend/cuda), and
// instantiates the operation templates for float vectors/matrices over the named
// semirings, and for int matrices on the triangle-counting path.  Every entry
// point forwards to the same frontend template a C++ user would call
// (reference graphblas/operations.hpp), so the C ABI and the drop-in C++ path
// execute identical code.
#define GRB_USE_CUDA

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <random>
#include <string>
#include <vector>

#include <boost/program_options.hpp>

#include "graphblas/graphblas.hpp"
#include "graphblas/algorithm/bfs.hpp"
#include "graphblas/algorithm/sssp.hpp"
#include "graphblas/algorithm/pr.hpp"
#include "graphblas/algorithm/tc.hpp"
#include "graphblas/algorithm/gc.hpp"
#include "graphblas/algorithm/mis.hpp"
#include "graphblas/algorithm/cc.hpp"
#include "graphblas/algorithm/lgc.hpp"

#include "graphblast_b200.h"
#include "graphblast_b200_lgc.h"

bool debug_;
bool memory_;

struct gb200_desc_s {
  graphblas::Descriptor desc;
};

struct gb200_vector_s {
  graphblas::Vector<float>* f;
};

// Exactly one of f and i is set: it names the handle's element type.
struct gb200_matrix_s {
  graphblas::Matrix<float>* f = NULL;
  graphblas::Matrix<int>*   i = NULL;
};

// Result of gb200_ingest_coo: a CSR in pool memory until exported / freed.
struct gb200_ingest_s {
  int nrows;
  graphblas::Index nnz;
  graphblas::Index* rowptr;
  graphblas::Index* colind;
  float* val;
};

namespace {

using graphblas::Info;
using graphblas::GrB_SUCCESS;

inline int rc(Info info) { return static_cast<int>(info); }

inline bool cudaOk() {
  int count = 0;
  cudaError_t err = cudaGetDeviceCount(&count);
  if (err != cudaSuccess || count == 0) {
    cudaGetLastError();
    return false;
  }
  return true;
}

// Loud failure: this library has no CPU path.
#define GB200_REQUIRE_DEVICE()                                                 \
  do {                                                                         \
    if (!cudaOk()) {                                                           \
      fprintf(stderr, "graphblast_b200: no CUDA device available; "            \
                      "this backend has no CPU fallback\n");                   \
      return rc(graphblas::GrB_PANIC);                                         \
    }                                                                          \
  } while (0)

// body(op) with the FP32 semiring of a GB200_* semiring id; GrB_INVALID_VALUE for
// an unknown id.
template <typename Body>
int withSemiring(int id, Body&& body) {
  using namespace graphblas;  // NOLINT(build/namespaces)
  switch (id) {
    case GB200_LOGICAL_OR_AND:        return body(LogicalOrAndSemiring<float>());
    case GB200_PLUS_MULTIPLIES:       return body(PlusMultipliesSemiring<float>());
    case GB200_MINIMUM_PLUS:          return body(MinimumPlusSemiring<float>());
    case GB200_MAXIMUM_MULTIPLIES:    return body(MaximumMultipliesSemiring<float>());
    case GB200_PLUS_DIVIDES:          return body(PlusDividesSemiring<float>());
    case GB200_PLUS_GREATER:          return body(PlusGreaterSemiring<float>());
    case GB200_GREATER_PLUS:          return body(GreaterPlusSemiring<float>());
    case GB200_PLUS_MINUS:            return body(PlusMinusSemiring<float>());
    case GB200_PLUS_LESS:             return body(PlusLessSemiring<float>());
    case GB200_CUSTOM_LESS_PLUS:      return body(CustomLessPlusSemiring<float>());
    case GB200_MINIMUM_MULTIPLIES:    return body(MinimumMultipliesSemiring<float>());
    case GB200_MULTIPLIES_MULTIPLIES: return body(MultipliesMultipliesSemiring<float>());
    case GB200_NOT_EQUAL_TO_PLUS:     return body(NotEqualToPlusSemiring<float>());
    case GB200_MINIMUM_SELECT_SECOND: return body(MinimumSelectSecondSemiring<float>());
    case GB200_PLUS_NOT_EQUAL_TO:     return body(PlusNotEqualToSemiring<float>());
    case GB200_CUSTOM_LESS_LESS:      return body(CustomLessLessSemiring<float>());
    case GB200_MINIMUM_NOT_EQUAL_TO:  return body(MinimumNotEqualToSemiring<float>());
    default: return rc(GrB_INVALID_VALUE);
  }
}

// body(op) with the monoid over T of a GB200_*_MONOID id; GrB_INVALID_VALUE for an
// unknown id.
template <typename T, typename Body>
int withMonoid(int id, Body&& body) {
  using namespace graphblas;  // NOLINT(build/namespaces)
  switch (id) {
    case GB200_PLUS_MONOID:         return body(PlusMonoid<T>());
    case GB200_MULTIPLIES_MONOID:   return body(MultipliesMonoid<T>());
    case GB200_MINIMUM_MONOID:      return body(MinimumMonoid<T>());
    case GB200_MAXIMUM_MONOID:      return body(MaximumMonoid<T>());
    case GB200_LOGICAL_OR_MONOID:   return body(LogicalOrMonoid<T>());
    case GB200_LOGICAL_AND_MONOID:  return body(LogicalAndMonoid<T>());
    case GB200_GREATER_MONOID:      return body(GreaterMonoid<T>());
    case GB200_CUSTOM_LESS_MONOID:  return body(CustomLessMonoid<T>());
    case GB200_NOT_EQUAL_TO_MONOID: return body(NotEqualToMonoid<T>());
    default: return rc(GrB_INVALID_VALUE);
  }
}

graphblas::Vector<float>* vec(gb200_vector_t v) { return v ? v->f : NULL; }

// The element type T of a graphblas::Matrix<T>* M: decltype(elementOf(M)).
template <typename T> T elementOf(const graphblas::Matrix<T>*);

// f(M) with A's typed matrix M, a graphblas::Matrix<float>* or Matrix<int>*.
template <typename F>
auto onMatrix(gb200_matrix_t A, F&& f) { return A->f != NULL ? f(A->f) : f(A->i); }

// Every given handle holds FP32 (allFp32) or INT32 (allInt32) values; NULL, an
// absent mask, matches either.
template <typename... M>
bool allFp32(M... m) { return ((m == NULL || m->f != NULL) && ...); }
template <typename... M>
bool allInt32(M... m) { return ((m == NULL || m->i != NULL) && ...); }

// *out = a new handle of element type dtype, its matrix M (a Matrix<float>*& or
// Matrix<int>*&) set by make(M); GrB_DOMAIN_MISMATCH for an unknown dtype.
template <typename Make>
int newMatrix(gb200_matrix_t* out, int dtype, Make&& make) {
  gb200_matrix_s* m = new gb200_matrix_s();
  const Info info = dtype == GB200_FP32  ? make(m->f)
                  : dtype == GB200_INT32 ? make(m->i) : graphblas::GrB_DOMAIN_MISMATCH;
  if (info != GrB_SUCCESS) {
    delete m;
    return rc(info);
  }
  *out = m;
  return 0;
}

// An algorithm driver run(): it returns the device time of its loop in ms, or a
// negative time with the failing status left in algorithm::lastStatus().  The time
// goes to *tight_ms when asked for.
template <typename Run>
int runAlgorithm(float* tight_ms, Run&& run) {
  graphblas::algorithm::lastStatus() = GrB_SUCCESS;
  const float ms = run();
  if (ms < 0.f) return rc(graphblas::algorithm::lastStatus());
  if (tight_ms) *tight_ms = ms;
  return 0;
}

template <typename T>
Info buildCoo(graphblas::Matrix<T>* M, const int* rows, const int* cols,
              const void* vals, int nvals, int undirected) {
  std::vector<graphblas::Index> r(rows, rows + nvals);
  std::vector<graphblas::Index> c(cols, cols + nvals);
  std::vector<T> v(nvals, static_cast<T>(1));
  if (vals != NULL) {
    const T* tv = static_cast<const T*>(vals);
    v.assign(tv, tv + nvals);
  }
  // The backend keys CSR/CSC aliasing on the ".ud." marker of the cache name
  // (reference sparse_matrix.hpp:300-306); pass the marker without a cache file.
  M->matrix_.sparse_.symmetric_ = (undirected != 0);
  Info info = M->build(&r, &c, &v, nvals, GrB_NULL);
  return info;
}

// Matrix Market file -> matrix: the text is parsed on the host (MtxFile), the raw
// tuples go to the device, and symmetrising, ordering and the removal of
// self-loops / repeated pairs run there (backend/cuda/ingest.hpp) with the
// semantics of the reference's readMtx (graphblas/util.hpp:264-329, 364-430).
template <typename T>
Info loadMtx(graphblas::Matrix<T>** out, const char* path, int directed) {
  using namespace graphblas::backend;
  MtxFile file(path);
  if (!file.ok) return graphblas::GrB_INVALID_VALUE;
  std::vector<graphblas::Index> rows, cols;
  std::vector<T> vals;
  file.tuples<T>(&rows, &cols, &vals);
  const bool undirected = directed != 1 && (file.symmetric() || directed == 2);
  const bool drop_loops = getEnv("GRB_UTIL_REMOVE_SELFLOOP", true);
  graphblas::Matrix<T>* M = new graphblas::Matrix<T>(file.nrows, file.ncols);
  const size_t m = rows.size();
  const size_t alloc = m > 0 ? m : 1;
  graphblas::Index* d_r = reinterpret_cast<graphblas::Index*>(gbMalloc(alloc*sizeof(graphblas::Index)));
  graphblas::Index* d_c = reinterpret_cast<graphblas::Index*>(gbMalloc(alloc*sizeof(graphblas::Index)));
  T* d_v = reinterpret_cast<T*>(gbMalloc(alloc*sizeof(T)));
  if (m > 0) {
    CUDA_CALL(cudaMemcpyAsync(d_r, rows.data(), m*sizeof(graphblas::Index), cudaMemcpyHostToDevice, gbStream()));
    CUDA_CALL(cudaMemcpyAsync(d_c, cols.data(), m*sizeof(graphblas::Index), cudaMemcpyHostToDevice, gbStream()));
    CUDA_CALL(cudaMemcpyAsync(d_v, vals.data(), m*sizeof(T), cudaMemcpyHostToDevice, gbStream()));
    runtime().sync();
  }
  const int mode = (undirected ? GB_INGEST_SYMMETRIZE : 0) |
                   (drop_loops ? GB_INGEST_DROP_LOOPS : 0) | GB_INGEST_DEDUP;
  M->matrix_.mat_type_ = graphblas::GrB_SPARSE;
  Info info = M->matrix_.sparse_.buildFromDeviceTuples(d_r, d_c, d_v,
      static_cast<long long>(m), mode, undirected);
  gbFree(d_v); gbFree(d_c); gbFree(d_r);
  if (info != GrB_SUCCESS) {
    delete M;
    return info;
  }
  *out = M;
  return GrB_SUCCESS;
}

template <typename T>
Info extractCsr(graphblas::Matrix<T>* M, int* rowptr, int* colind, void* val) {
  if (!M->matrix_.isSparse()) return graphblas::GrB_UNINITIALIZED_OBJECT;
  graphblas::backend::SparseMatrix<T>& S = M->matrix_.sparse_;
  CHECK(S.gpuToCpu());
  memcpy(rowptr, S.h_csrRowPtr_, (S.nrows_ + 1)*sizeof(int));
  memcpy(colind, S.h_csrColInd_, static_cast<size_t>(S.nvals_)*sizeof(int));
  if (val != NULL)
    memcpy(val, S.h_csrVal_, static_cast<size_t>(S.nvals_)*sizeof(T));
  return GrB_SUCCESS;
}

// C = A (+) B (IsAdd) or A (x) B of two matrices: FP32 over every semiring,
// INT32 over PlusMultiplies only, no mixing.
template <bool IsAdd>
int ewiseMatrix(gb200_matrix_t C, gb200_matrix_t mask, int semiring, gb200_matrix_t A,
                gb200_matrix_t B, gb200_desc_t desc) {
  if (C == NULL || A == NULL || B == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (allFp32(C, A, B, mask)) {
    GB200_REQUIRE_DEVICE();
    return withSemiring(semiring, [&](auto op) {
      if constexpr (IsAdd)
        return rc((graphblas::eWiseAdd<float, float, float, float>(C->f,
            mask != NULL ? mask->f : NULL, GrB_NULL, op, A->f, B->f, &desc->desc)));
      else
        return rc((graphblas::eWiseMult<float, float, float, float>(C->f,
            mask != NULL ? mask->f : NULL, GrB_NULL, op, A->f, B->f, &desc->desc)));
    });
  }
  if (!allInt32(C, A, B, mask)) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  if (semiring != GB200_PLUS_MULTIPLIES) return rc(graphblas::GrB_NOT_IMPLEMENTED);
  GB200_REQUIRE_DEVICE();
  if constexpr (IsAdd)
    return rc((graphblas::eWiseAdd<int, int, int, int>(C->i, mask ? mask->i : NULL,
        GrB_NULL, graphblas::PlusMultipliesSemiring<int>(), A->i, B->i, &desc->desc)));
  else
    return rc((graphblas::eWiseMult<int, int, int, int>(C->i, mask ? mask->i : NULL,
        GrB_NULL, graphblas::PlusMultipliesSemiring<int>(), A->i, B->i, &desc->desc)));
}

__global__ void rmatEdgesKernel(int scale, long long nedges,
                                unsigned long long seed, long long first_edge,
                                int* __restrict__ src, int* __restrict__ dst) {
  const unsigned int T1 = 2448131358u, T2 = 3264175144u, T3 = 4080218930u;
  long long e = static_cast<long long>(blockIdx.x)*blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x)*blockDim.x;
  for (; e < nedges; e += stride) {
    const unsigned long long ge = static_cast<unsigned long long>(first_edge + e);
    unsigned int s = 0, d = 0;
    for (int l = 0; l < scale; ++l) {
      unsigned long long z = ((seed << 48) ^ (ge << 6) ^
          static_cast<unsigned long long>(l)) + 0x9E3779B97F4A7C15ull;
      z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
      z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
      z = z ^ (z >> 31);
      const unsigned int r = static_cast<unsigned int>(z >> 32);
      const unsigned int sb = (r >= T2) ? 1u : 0u;
      const unsigned int db = ((r >= T1 && r < T2) || r >= T3) ? 1u : 0u;
      s = (s << 1) | sb;
      d = (d << 1) | db;
    }
    src[e] = static_cast<int>(s);
    dst[e] = static_cast<int>(d);
  }
}

}  // namespace

extern "C" {

// ---- runtime ---------------------------------------------------------------

int gb200_init(int device) {
  GB200_REQUIRE_DEVICE();
  if (cudaSetDevice(device) != cudaSuccess) return rc(graphblas::GrB_PANIC);
  graphblas::backend::runtime();
  return 0;
}

int gb200_set_stream(void* cuda_stream) {
  GB200_REQUIRE_DEVICE();
  // Work already queued on the old stream must not be overtaken by work on the
  // new one (pool frees, cached tiles, scratch arenas are all stream-ordered).
  graphblas::backend::Runtime& rt = graphblas::backend::runtime();
  cudaStream_t next = static_cast<cudaStream_t>(cuda_stream);
  if (next != rt.stream) {
    if (cudaStreamSynchronize(rt.stream) != cudaSuccess) return rc(graphblas::GrB_PANIC);
    rt.stream = next;
  }
  return 0;
}

int gb200_sync(void) {
  GB200_REQUIRE_DEVICE();
  graphblas::backend::runtime().sync();
  return 0;
}

int gb200_sm_count(int* out) {
  GB200_REQUIRE_DEVICE();
  *out = graphblas::backend::runtime().sm_count;
  return 0;
}

const char* gb200_version(void) { return "graphblast_b200 0.1 (sm_90a)"; }

// ---- Descriptor -------------------------------------------------------------

int gb200_desc_new(gb200_desc_t* out) {
  if (out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  gb200_desc_s* d = new gb200_desc_s();
  // Start from the parseArgs() defaults (reference graphblas/util.hpp:39-132).
  po::variables_map vm;
  char  prog[] = "gb200";
  char* argv[] = { prog };
  parseArgs(1, argv, &vm);
  Info info = d->desc.loadArgs(vm);
  if (info != GrB_SUCCESS) {
    delete d;
    return rc(info);
  }
  d->desc.descriptor_.timing_ = 0;
  *out = d;
  return 0;
}

int gb200_desc_free(gb200_desc_t desc) {
  delete desc;
  return 0;
}

int gb200_desc_set(gb200_desc_t desc, int field, int value) {
  if (desc == NULL) return rc(graphblas::GrB_NULL_POINTER);
  if (field < 0 || field >= graphblas::GrB_NDESCFIELD)
    return rc(graphblas::GrB_INVALID_VALUE);
  return rc(desc->desc.set(static_cast<graphblas::Desc_field>(field), value));
}

int gb200_desc_get(gb200_desc_t desc, int field, int* value) {
  if (desc == NULL || value == NULL) return rc(graphblas::GrB_NULL_POINTER);
  if (field < 0 || field >= graphblas::GrB_NDESCFIELD)
    return rc(graphblas::GrB_INVALID_VALUE);
  graphblas::Desc_value v;
  Info info = desc->desc.get(static_cast<graphblas::Desc_field>(field), &v);
  *value = static_cast<int>(v);
  return rc(info);
}

int gb200_desc_toggle(gb200_desc_t desc, int field) {
  if (desc == NULL) return rc(graphblas::GrB_NULL_POINTER);
  if (field < 0 || field >= graphblas::GrB_NDESCFIELD)
    return rc(graphblas::GrB_INVALID_VALUE);
  return rc(desc->desc.toggle(static_cast<graphblas::Desc_field>(field)));
}

int gb200_desc_set_knob(gb200_desc_t desc, const char* name, double value) {
  if (desc == NULL || name == NULL) return rc(graphblas::GrB_NULL_POINTER);
  return rc(desc->desc.descriptor_.setKnob(name, value));
}

int gb200_desc_get_knob(gb200_desc_t desc, const char* name, double* value) {
  if (desc == NULL || name == NULL || value == NULL)
    return rc(graphblas::GrB_NULL_POINTER);
  return rc(desc->desc.descriptor_.getKnob(name, value));
}

// ---- Matrix -----------------------------------------------------------------

int gb200_matrix_new(gb200_matrix_t* out, int dtype, int nrows, int ncols) {
  if (out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  if (nrows <= 0 || ncols <= 0) return rc(graphblas::GrB_INVALID_VALUE);
  GB200_REQUIRE_DEVICE();
  return newMatrix(out, dtype, [&](auto& M) {
    M = new graphblas::Matrix<decltype(elementOf(M))>(nrows, ncols);
    return GrB_SUCCESS;
  });
}

int gb200_matrix_free(gb200_matrix_t A) {
  if (A == NULL) return 0;
  delete A->f;
  delete A->i;
  delete A;
  return 0;
}

int gb200_matrix_build_coo(gb200_matrix_t A, const int* h_rows,
                           const int* h_cols, const void* h_vals, int nvals,
                           int undirected) {
  if (A == NULL || h_rows == NULL || h_cols == NULL)
    return rc(graphblas::GrB_NULL_POINTER);
  if (nvals <= 0) return rc(graphblas::GrB_NO_VALUE);
  GB200_REQUIRE_DEVICE();
  return rc(onMatrix(A, [&](auto M) {
    return buildCoo(M, h_rows, h_cols, h_vals, nvals, undirected);
  }));
}

int gb200_matrix_load_mtx(gb200_matrix_t* out, int dtype, const char* path,
                          int directed) {
  if (out == NULL || path == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  FILE* probe = fopen(path, "r");
  if (probe == NULL) return rc(graphblas::GrB_INVALID_VALUE);
  fclose(probe);
  return newMatrix(out, dtype, [&](auto& M) { return loadMtx(&M, path, directed); });
}

int gb200_matrix_build_coo_device(gb200_matrix_t A, const int* d_rows,
                                  const int* d_cols, const void* d_vals,
                                  long long ntuples, int flags) {
  if (A == NULL || (ntuples > 0 && (d_rows == NULL || d_cols == NULL)))
    return rc(graphblas::GrB_NULL_POINTER);
  if (ntuples < 0) return rc(graphblas::GrB_INVALID_VALUE);
  GB200_REQUIRE_DEVICE();
  const int mode = flags & 7;
  const bool symmetric = (flags & GB200_INGEST_SYMMETRIC_STRUCTURE) != 0;
  return rc(onMatrix(A, [&](auto M) {
    using T = decltype(elementOf(M));
    CHECK(M->matrix_.setStorage(graphblas::GrB_SPARSE));
    return M->matrix_.sparse_.buildFromDeviceTuples(d_rows, d_cols,
        static_cast<const T*>(d_vals), ntuples, mode, symmetric);
  }));
}

int gb200_ingest_coo(int nrows, int ncols, const int* d_rows, const int* d_cols,
                     const float* d_vals, long long ntuples, int flags,
                     gb200_ingest_t* out, long long* nnz) {
  if (out == NULL || nnz == NULL || (ntuples > 0 && (d_rows == NULL || d_cols == NULL)))
    return rc(graphblas::GrB_NULL_POINTER);
  if (nrows <= 0 || ncols <= 0 || ntuples < 0) return rc(graphblas::GrB_INVALID_VALUE);
  GB200_REQUIRE_DEVICE();
  gb200_ingest_s* h = new gb200_ingest_s();
  h->nrows = nrows;
  h->nnz = graphblas::backend::ingestCooToCsr<float>(nrows, ncols, d_rows, d_cols,
      d_vals, ntuples, flags & 7, &h->rowptr, &h->colind, &h->val);
  *out = h;
  *nnz = h->nnz;
  return 0;
}

int gb200_ingest_export(gb200_ingest_t h, int* d_rowptr, int* d_colind, float* d_val) {
  if (h == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  using namespace graphblas::backend;
  copyAsync(d_rowptr, h->rowptr, static_cast<size_t>(h->nrows) + 1, cudaMemcpyDeviceToDevice);
  copyAsync(d_colind, h->colind, static_cast<size_t>(h->nnz), cudaMemcpyDeviceToDevice);
  copyAsync(d_val, h->val, static_cast<size_t>(h->nnz), cudaMemcpyDeviceToDevice);
  runtime().sync();
  return 0;
}

int gb200_ingest_free(gb200_ingest_t h) {
  if (h == NULL) return 0;
  graphblas::backend::gbFree(h->val);
  graphblas::backend::gbFree(h->colind);
  graphblas::backend::gbFree(h->rowptr);
  delete h;
  return 0;
}

int gb200_csr_transpose_values(int nrows, int ncols, int nnz, const int* d_rowptr,
                               const int* d_colind, const float* d_val,
                               int* d_colptr_out, int* d_rowind_out,
                               float* d_cscval_out) {
  if (d_rowptr == NULL || d_colind == NULL || d_val == NULL)
    return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  using namespace graphblas::backend;
  graphblas::Index* colptr = NULL; graphblas::Index* rowind = NULL; float* cval = NULL;
  ingestCsrToCsc<float>(nrows, ncols, nnz, d_rowptr, d_colind, d_val,
      d_colptr_out != NULL ? &colptr : NULL, d_rowind_out != NULL ? &rowind : NULL,
      d_cscval_out != NULL ? &cval : NULL);
  const size_t nvals = nnz > 0 ? static_cast<size_t>(nnz) : 0;
  copyAsync(d_colptr_out, colptr, static_cast<size_t>(ncols) + 1, cudaMemcpyDeviceToDevice);
  copyAsync(d_rowind_out, rowind, nvals, cudaMemcpyDeviceToDevice);
  copyAsync(d_cscval_out, cval, nvals, cudaMemcpyDeviceToDevice);
  gbFree(colptr); gbFree(rowind); gbFree(cval);
  runtime().sync();
  return 0;
}

int gb200_sort_pairs_u64(unsigned long long* d_keys, unsigned int* d_payload,
                         long long n, int bits) {
  if (d_keys == NULL) return rc(graphblas::GrB_NULL_POINTER);
  if (n < 0 || bits < 1 || bits > 64) return rc(graphblas::GrB_INVALID_VALUE);
  GB200_REQUIRE_DEVICE();
  using namespace graphblas::backend;
  const size_t alloc = n > 0 ? static_cast<size_t>(n) : 1;
  unsigned long long* keys = d_keys;
  unsigned int* pay = d_payload;
  unsigned long long* keys_tmp = reinterpret_cast<unsigned long long*>(gbMalloc(alloc*8));
  unsigned int* pay_tmp = d_payload != NULL
      ? reinterpret_cast<unsigned int*>(gbMalloc(alloc*4)) : NULL;
  radixSortPairs(&keys, d_payload != NULL ? &pay : NULL, &keys_tmp,
      d_payload != NULL ? &pay_tmp : NULL, n, bits);
  if (keys != d_keys) {              // an odd number of passes left the result in the temporaries
    copyAsync(d_keys, keys, alloc, cudaMemcpyDeviceToDevice);
    copyAsync(d_payload, pay, alloc, cudaMemcpyDeviceToDevice);
    runtime().sync();
    gbFree(keys);
    if (pay != NULL && pay != d_payload) gbFree(pay);
  } else {
    runtime().sync();
    gbFree(keys_tmp);
    if (pay_tmp != NULL) gbFree(pay_tmp);
  }
  return 0;
}

int gb200_matrix_adopt_csr(gb200_matrix_t A, int* d_rowptr, int* d_colind,
                           void* d_val, int nvals) {
  if (A == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(onMatrix(A, [&](auto M) {
    using T = decltype(elementOf(M));
    return M->build(d_rowptr, d_colind, static_cast<T*>(d_val), nvals);
  }));
}

int gb200_matrix_adopt_csc(gb200_matrix_t A, int* d_colptr, int* d_rowind,
                           void* d_val, int symmetric) {
  if (A == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(onMatrix(A, [&](auto M) {
    using T = decltype(elementOf(M));
    return M->matrix_.sparse_.adoptCsc(d_colptr, d_rowind, static_cast<T*>(d_val),
                                       symmetric != 0);
  }));
}

int gb200_matrix_nrows(gb200_matrix_t A, int* out) {
  if (A == NULL || out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  return rc(onMatrix(A, [&](auto M) { return M->nrows(out); }));
}

int gb200_matrix_ncols(gb200_matrix_t A, int* out) {
  if (A == NULL || out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  return rc(onMatrix(A, [&](auto M) { return M->ncols(out); }));
}

int gb200_matrix_nvals(gb200_matrix_t A, int* out) {
  if (A == NULL || out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  return rc(onMatrix(A, [&](auto M) { return M->nvals(out); }));
}

int gb200_matrix_extract_csr(gb200_matrix_t A, int* h_rowptr, int* h_colind,
                             void* h_val) {
  if (A == NULL || h_rowptr == NULL || h_colind == NULL)
    return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(onMatrix(A, [&](auto M) { return extractCsr(M, h_rowptr, h_colind, h_val); }));
}

int gb200_matrix_build_dense(gb200_matrix_t A, const void* h_vals, long long nvals) {
  if (A == NULL || (h_vals == NULL && nvals > 0)) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  if (A->f == NULL) return rc(graphblas::GrB_NOT_IMPLEMENTED);
  return rc(A->f->matrix_.buildDense(static_cast<const float*>(h_vals), nvals));
}

int gb200_matrix_adopt_dense(gb200_matrix_t A, void* d_vals) {
  if (A == NULL || d_vals == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  if (A->f == NULL) return rc(graphblas::GrB_NOT_IMPLEMENTED);
  return rc(A->f->adoptDense(static_cast<float*>(d_vals)));
}

int gb200_matrix_extract_dense(gb200_matrix_t A, void* h_out, long long n) {
  if (A == NULL || h_out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  if (A->f == NULL || !A->f->matrix_.isDense())
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  return rc(A->f->matrix_.dense_.extract(static_cast<float*>(h_out), n, NULL));
}

int gb200_matrix_dense_ptr(gb200_matrix_t A, void** d_vals) {
  if (A == NULL || d_vals == NULL) return rc(graphblas::GrB_NULL_POINTER);
  if (A->f == NULL || !A->f->matrix_.isDense() || A->f->matrix_.dense_.d_val_ == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  *d_vals = A->f->matrix_.dense_.d_val_;
  return 0;
}

int gb200_matrix_storage(gb200_matrix_t A, int* out) {
  if (A == NULL || out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  graphblas::Storage s;
  Info info = onMatrix(A, [&](auto M) { return M->getStorage(&s); });
  *out = static_cast<int>(s);
  return rc(info);
}

int gb200_matrix_tril(gb200_matrix_t A, gb200_desc_t desc) {
  if (A == NULL || desc == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  Info info = desc->desc.set(graphblas::GrB_BACKEND, graphblas::GrB_SEQUENTIAL);
  if (info == GrB_SUCCESS) {
    info = onMatrix(A, [&](auto M) {
      using T = decltype(elementOf(M));
      return graphblas::tril<T, T>(M, M, &desc->desc);
    });
  }
  desc->desc.set(graphblas::GrB_BACKEND, graphblas::GrB_CUDA);
  return rc(info);
}

int gb200_matrix_apply_uniform_random(gb200_matrix_t A, gb200_desc_t desc,
                                      int seed, int lo, int hi) {
  if (A == NULL || desc == NULL) return rc(graphblas::GrB_NULL_POINTER);
  if (A->f == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  desc->desc.set(graphblas::GrB_BACKEND, graphblas::GrB_SEQUENTIAL);
  Info info = graphblas::apply<float, float, float>(A->f, GrB_NULL, GrB_NULL,
      graphblas::set_uniform_random<float>(seed, lo, hi), A->f, &desc->desc);
  desc->desc.set(graphblas::GrB_BACKEND, graphblas::GrB_CUDA);
  return rc(info);
}

int gb200_host_uniform_weights(int seed, int lo, int hi, long long n,
                               float* h_out) {
  if (h_out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  graphblas::set_uniform_random<float> gen(seed, lo, hi);
  for (long long k = 0; k < n; ++k) h_out[k] = gen(0.f);
  return 0;
}

int gb200_pr_normalize(gb200_matrix_t A, float alpha, gb200_desc_t desc) {
  if (A == NULL || desc == NULL) return rc(graphblas::GrB_NULL_POINTER);
  if (A->f == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  return rc(graphblas::algorithm::prNormalize(A->f, alpha, &desc->desc));
}

// ---- Vector -----------------------------------------------------------------

int gb200_vector_new(gb200_vector_t* out, int dtype, int size) {
  if (out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  if (dtype != GB200_FP32) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  if (size <= 0) return rc(graphblas::GrB_INVALID_VALUE);
  GB200_REQUIRE_DEVICE();
  gb200_vector_s* v = new gb200_vector_s();
  v->f = new graphblas::Vector<float>(size);
  *out = v;
  return 0;
}

int gb200_vector_free(gb200_vector_t v) {
  if (v == NULL) return 0;
  delete v->f;
  delete v;
  return 0;
}

int gb200_vector_fill(gb200_vector_t v, double val) {
  if (v == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(v->f->fill(static_cast<float>(val)));
}

int gb200_vector_build_sparse(gb200_vector_t v, const int* h_ind,
                              const void* h_val, int nvals) {
  if (v == NULL || h_ind == NULL || h_val == NULL)
    return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  std::vector<graphblas::Index> ind(h_ind, h_ind + nvals);
  const float* fv = static_cast<const float*>(h_val);
  std::vector<float> val(fv, fv + nvals);
  return rc(v->f->build(&ind, &val, nvals, GrB_NULL));
}

int gb200_vector_build_dense(gb200_vector_t v, const void* h_val, int n) {
  if (v == NULL || h_val == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  const float* fv = static_cast<const float*>(h_val);
  std::vector<float> val(fv, fv + n);
  Info info = v->f->setStorage(graphblas::GrB_DENSE);
  if (info != GrB_SUCCESS) return rc(info);
  return rc(v->f->build(&val, n));
}

int gb200_vector_adopt_dense(gb200_vector_t v, void* d_val, int n) {
  if (v == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(v->f->build(static_cast<float*>(d_val), n));
}

int gb200_vector_adopt_sparse(gb200_vector_t v, int* d_ind, void* d_val,
                              int nvals) {
  if (v == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(v->f->build(d_ind, static_cast<float*>(d_val), nvals));
}

int gb200_vector_set_element(gb200_vector_t v, double val, int index) {
  if (v == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(v->f->setElement(static_cast<float>(val), index));
}

int gb200_vector_size(gb200_vector_t v, int* out) {
  if (v == NULL || out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  return rc(v->f->size(out));
}

int gb200_vector_nvals(gb200_vector_t v, int* out) {
  if (v == NULL || out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  return rc(v->f->nvals(out));
}

int gb200_vector_storage(gb200_vector_t v, int* out) {
  if (v == NULL || out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  graphblas::Storage s;
  Info info = v->f->getStorage(&s);
  *out = static_cast<int>(s);
  return rc(info);
}

int gb200_vector_extract_dense(gb200_vector_t v, void* h_out, int n) {
  if (v == NULL || h_out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  graphblas::backend::Vector<float>& b = v->f->vector_;
  if (b.vec_type_ == graphblas::GrB_SPARSE) {
    Info info = b.sparse2dense(0.f);
    if (info != GrB_SUCCESS) return rc(info);
  } else if (b.vec_type_ != graphblas::GrB_DENSE) {
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  }
  return rc(b.dense_.extractRaw(static_cast<float*>(h_out), n));
}

int gb200_vector_extract_sparse(gb200_vector_t v, int* h_ind, void* h_val,
                                int* n_inout) {
  if (v == NULL || h_ind == NULL || h_val == NULL || n_inout == NULL)
    return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  graphblas::backend::Vector<float>& b = v->f->vector_;
  if (b.vec_type_ != graphblas::GrB_SPARSE)
    return rc(graphblas::GrB_INVALID_OBJECT);
  int count = b.sparse_.nvals_;
  if (count > *n_inout) return rc(graphblas::GrB_INSUFFICIENT_SPACE);
  std::vector<graphblas::Index> ind;
  std::vector<float> val;
  Info info = b.sparse_.extractTuples(&ind, &val, &count);
  if (info != GrB_SUCCESS) return rc(info);
  memcpy(h_ind, ind.data(), count*sizeof(int));
  memcpy(h_val, val.data(), count*sizeof(float));
  *n_inout = count;
  return 0;
}

int gb200_vector_swap(gb200_vector_t a, gb200_vector_t b) {
  if (a == NULL || b == NULL) return rc(graphblas::GrB_NULL_POINTER);
  return rc(a->f->swap(b->f));
}

int gb200_vector_dup(gb200_vector_t dst, gb200_vector_t src) {
  if (dst == NULL || src == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(dst->f->dup(src->f));
}

int gb200_vector_clear(gb200_vector_t v) {
  if (v == NULL) return rc(graphblas::GrB_NULL_POINTER);
  return rc(v->f->clear());
}

int gb200_vector_sparse2dense(gb200_vector_t v, double identity,
                              gb200_desc_t desc) {
  if (v == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(v->f->sparse2dense(static_cast<float>(identity),
      desc ? &desc->desc : NULL));
}

int gb200_vector_dense2sparse(gb200_vector_t v, double identity,
                              gb200_desc_t desc) {
  if (v == NULL || desc == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(v->f->dense2sparse(static_cast<float>(identity), &desc->desc));
}

int gb200_vector_device_ptr(gb200_vector_t v, void** d_val) {
  if (v == NULL || d_val == NULL) return rc(graphblas::GrB_NULL_POINTER);
  graphblas::backend::Vector<float>& b = v->f->vector_;
  if (b.vec_type_ != graphblas::GrB_DENSE)
    return rc(graphblas::GrB_INVALID_OBJECT);
  graphblas::Info info = b.dense_.allocateGpu();
  if (info == graphblas::GrB_SUCCESS) info = b.dense_.materialize();
  if (info != graphblas::GrB_SUCCESS) return rc(info);
  *d_val = b.dense_.d_val_;
  return 0;
}

// ---- Operations -------------------------------------------------------------

int gb200_vxm(gb200_vector_t w, gb200_vector_t mask, int use_accum,
              int semiring, gb200_vector_t u, gb200_matrix_t A,
              gb200_desc_t desc) {
  if (w == NULL || u == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  return withSemiring(semiring, [&](auto op) {
    if (use_accum)
      return rc((graphblas::vxm<float, float, float, float>(vec(w), vec(mask),
          graphblas::plus<float>(), op, vec(u), A->f, &desc->desc)));
    return rc((graphblas::vxm<float, float, float, float>(vec(w), vec(mask),
        GrB_NULL, op, vec(u), A->f, &desc->desc)));
  });
}

int gb200_mxv(gb200_vector_t w, gb200_vector_t mask, int use_accum,
              int semiring, gb200_matrix_t A, gb200_vector_t u,
              gb200_desc_t desc) {
  if (w == NULL || u == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  return withSemiring(semiring, [&](auto op) {
    if (use_accum)
      return rc((graphblas::mxv<float, float, float, float>(vec(w), vec(mask),
          graphblas::plus<float>(), op, A->f, vec(u), &desc->desc)));
    return rc((graphblas::mxv<float, float, float, float>(vec(w), vec(mask),
        GrB_NULL, op, A->f, vec(u), &desc->desc)));
  });
}

int gb200_mxm(gb200_matrix_t C, gb200_matrix_t mask, int semiring,
              gb200_matrix_t A, gb200_matrix_t B, gb200_desc_t desc) {
  if (C == NULL || A == NULL || B == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  // a float mask only reaches the backend beside a dense operand, which refuses it
  if (allFp32(C, A, B, mask) &&
      (mask == NULL || A->f->matrix_.isDense() || B->f->matrix_.isDense())) {
    GB200_REQUIRE_DEVICE();
    return withSemiring(semiring, [&](auto op) {
      return rc((graphblas::mxm<float, float, float, float>(C->f,
          mask != NULL ? mask->f : NULL, GrB_NULL, op, A->f, B->f, &desc->desc)));
    });
  }
  if (!allInt32(C, A, B, mask)) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  if (semiring != GB200_PLUS_MULTIPLIES)
    return rc(graphblas::GrB_NOT_IMPLEMENTED);
  GB200_REQUIRE_DEVICE();
  return rc((graphblas::mxm<int, int, int, int>(C->i, mask ? mask->i : NULL,
      GrB_NULL, graphblas::PlusMultipliesSemiring<int>(), A->i, B->i,
      &desc->desc)));
}

int gb200_ewise_add_matrix(gb200_matrix_t C, gb200_matrix_t mask, int semiring,
                           gb200_matrix_t A, gb200_matrix_t B, gb200_desc_t desc) {
  return ewiseMatrix<true>(C, mask, semiring, A, B, desc);
}

int gb200_ewise_mult_matrix(gb200_matrix_t C, gb200_matrix_t mask, int semiring,
                            gb200_matrix_t A, gb200_matrix_t B, gb200_desc_t desc) {
  return ewiseMatrix<false>(C, mask, semiring, A, B, desc);
}

int gb200_transpose(gb200_matrix_t C, gb200_matrix_t mask, gb200_matrix_t A,
                    gb200_desc_t desc) {
  if (C == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (allFp32(C, A, mask)) {
    GB200_REQUIRE_DEVICE();
    return rc((graphblas::transpose<float, float, float>(C->f,
        mask != NULL ? mask->f : NULL, GrB_NULL, A->f, &desc->desc)));
  }
  if (!allInt32(C, A, mask)) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  return rc((graphblas::transpose<int, int, int>(C->i, mask ? mask->i : NULL, GrB_NULL,
      A->i, &desc->desc)));
}

int gb200_ewise_add(gb200_vector_t w, gb200_vector_t mask, int semiring,
                    gb200_vector_t u, gb200_vector_t v, gb200_desc_t desc) {
  if (w == NULL || u == NULL || v == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  GB200_REQUIRE_DEVICE();
  return withSemiring(semiring, [&](auto op) {
    return rc((graphblas::eWiseAdd<float, float, float, float>(vec(w),
        vec(mask), GrB_NULL, op, vec(u), vec(v), &desc->desc)));
  });
}

int gb200_ewise_add_scalar(gb200_vector_t w, gb200_vector_t mask, int semiring,
                           gb200_vector_t u, double val, gb200_desc_t desc) {
  if (w == NULL || u == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  GB200_REQUIRE_DEVICE();
  return withSemiring(semiring, [&](auto op) {
    return rc((graphblas::eWiseAdd<float, float, float, float>(vec(w),
        vec(mask), GrB_NULL, op, vec(u), static_cast<float>(val),
        &desc->desc)));
  });
}

int gb200_ewise_mult(gb200_vector_t w, gb200_vector_t mask, int semiring,
                     gb200_vector_t u, gb200_vector_t v, gb200_desc_t desc) {
  if (w == NULL || u == NULL || v == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  GB200_REQUIRE_DEVICE();
  return withSemiring(semiring, [&](auto op) {
    return rc((graphblas::eWiseMult<float, float, float, float>(vec(w),
        vec(mask), GrB_NULL, op, vec(u), vec(v), &desc->desc)));
  });
}

int gb200_assign_scalar(gb200_vector_t w, gb200_vector_t mask, double val,
                        gb200_desc_t desc) {
  if (w == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  GB200_REQUIRE_DEVICE();
  int n = 0;
  w->f->size(&n);
  return rc((graphblas::assign<float, float, float, graphblas::Index>(vec(w),
      vec(mask), GrB_NULL, static_cast<float>(val), GrB_ALL, n, &desc->desc)));
}

int gb200_reduce_vector(double* out, int monoid, gb200_vector_t u,
                        gb200_desc_t desc) {
  if (out == NULL || u == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  GB200_REQUIRE_DEVICE();
  return withMonoid<float>(monoid, [&](auto op) {
    float val = 0.f;
    Info info = graphblas::reduce<float, float>(&val, GrB_NULL, op, vec(u),
        &desc->desc);
    *out = val;
    return rc(info);
  });
}

int gb200_reduce_matrix(double* out, int monoid, gb200_matrix_t A,
                        gb200_desc_t desc) {
  if (out == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  GB200_REQUIRE_DEVICE();
  if (A->f != NULL) {
    return withMonoid<float>(monoid, [&](auto op) {
      float val = 0.f;
      Info info = graphblas::reduce<float, float>(&val, GrB_NULL, op, A->f,
          &desc->desc);
      *out = val;
      return rc(info);
    });
  }
  if (monoid != GB200_PLUS_MONOID) return rc(graphblas::GrB_NOT_IMPLEMENTED);
  int val = 0;
  Info info = graphblas::reduce<int, int>(&val, GrB_NULL,
      graphblas::PlusMonoid<int>(), A->i, &desc->desc);
  *out = val;
  return rc(info);
}

int gb200_reduce_matrix_rows(gb200_vector_t w, int monoid, gb200_matrix_t A,
                             gb200_desc_t desc) {
  if (w == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  return withMonoid<float>(monoid, [&](auto op) {
    return rc((graphblas::reduce<float, float, float>(vec(w), GrB_NULL,
        GrB_NULL, op, A->f, &desc->desc)));
  });
}

// ---- Algorithms ---------------------------------------------------------------

int gb200_bfs(gb200_vector_t v, gb200_matrix_t A, int source, gb200_desc_t desc,
              float* tight_ms) {
  if (v == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  int n = 0;
  A->f->nrows(&n);
  if (source < 0 || source >= n) return rc(graphblas::GrB_INVALID_INDEX);
  GB200_REQUIRE_DEVICE();
  return runAlgorithm(tight_ms, [&] {
    return graphblas::algorithm::bfs(v->f, A->f, source, &desc->desc, tight_ms != NULL);
  });
}

// scatter / assignScatter / extractGather (reference graphblas/operations.hpp:
// scatter :771, assignScatter :806, extractGather :839) on float vectors; index
// values are truncated to integers as in the reference kernels.
int gb200_scatter(gb200_vector_t w, gb200_vector_t u, float val, gb200_desc_t desc) {
  if (w == NULL || u == NULL || desc == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(graphblas::scatter<float, float, float, float>(w->f, GrB_NULL, u->f, val,
      &desc->desc));
}

int gb200_assign_scatter(gb200_vector_t w, gb200_vector_t u, gb200_vector_t indices,
                         gb200_desc_t desc) {
  if (w == NULL || u == NULL || indices == NULL || desc == NULL)
    return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(graphblas::assignScatter<float, float, float, float>(w->f, GrB_NULL, GrB_NULL,
      u->f, indices->f, &desc->desc));
}

int gb200_extract_gather(gb200_vector_t w, gb200_vector_t u, gb200_vector_t indices,
                         gb200_desc_t desc) {
  if (w == NULL || u == NULL || indices == NULL || desc == NULL)
    return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  return rc(graphblas::extractGather<float, float, float, float>(w->f, GrB_NULL, GrB_NULL,
      u->f, indices->f, &desc->desc));
}

int gb200_bfs_stats(gb200_desc_t desc, int n, unsigned long long* out6) {
  if (desc == NULL || out6 == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  graphblas::backend::bfsFusedStats(&desc->desc.descriptor_, n, out6);
  return 0;
}

int gb200_sssp(gb200_vector_t v, gb200_matrix_t A, int source,
               gb200_desc_t desc, float* tight_ms) {
  if (v == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  int n = 0;
  A->f->nrows(&n);
  if (source < 0 || source >= n) return rc(graphblas::GrB_INVALID_INDEX);
  GB200_REQUIRE_DEVICE();
  return runAlgorithm(tight_ms, [&] {
    return graphblas::algorithm::sssp(v->f, A->f, source, &desc->desc);
  });
}

int gb200_gc(gb200_vector_t v, gb200_matrix_t A, int seed, gb200_desc_t desc,
             int* ncolors, float* tight_ms) {
  if (v == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL && A->i == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  int count = 0;
  const int info = runAlgorithm(tight_ms, [&] {
    return onMatrix(A, [&](auto M) {
      return graphblas::algorithm::gc(v->f, M, seed, &desc->desc, &count);
    });
  });
  if (info == 0 && ncolors) *ncolors = count;
  return info;
}

int gb200_mis(gb200_vector_t v, gb200_matrix_t A, int seed, gb200_vector_t candidates,
              gb200_desc_t desc, int* nmembers, float* tight_ms) {
  if (v == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL && A->i == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  int count = 0;
  const graphblas::Vector<float>* cand = candidates != NULL ? candidates->f : NULL;
  const int info = runAlgorithm(tight_ms, [&] {
    return onMatrix(A, [&](auto M) {
      return graphblas::algorithm::mis(v->f, M, seed, &desc->desc, &count, cand);
    });
  });
  if (info == 0 && nmembers) *nmembers = count;
  return info;
}

int gb200_cc(gb200_vector_t v, gb200_matrix_t A, gb200_desc_t desc, int* ncomponents,
             float* tight_ms) {
  if (v == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL && A->i == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  int count = 0;
  const int info = runAlgorithm(tight_ms, [&] {
    return onMatrix(A, [&](auto M) {
      return graphblas::algorithm::cc(v->f, M, &desc->desc, &count);
    });
  });
  if (info == 0 && ncomponents) *ncomponents = count;
  return info;
}

int gb200_lgc(gb200_vector_t p, gb200_vector_t r, gb200_matrix_t A, int source,
              double alpha, double eps, gb200_desc_t desc, int* rounds, float* tight_ms) {
  if (p == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL && A->i == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  int n = 0;
  onMatrix(A, [&](auto M) { return M->nrows(&n); });
  if (source < 0 || source >= n) return rc(graphblas::GrB_INVALID_INDEX);
  if (!(alpha > 0.0 && alpha <= 1.0) || !(eps > 0.0)) return rc(graphblas::GrB_INVALID_VALUE);
  GB200_REQUIRE_DEVICE();
  int count = 0;
  const int info = runAlgorithm(tight_ms, [&] {
    return onMatrix(A, [&](auto M) {
      return graphblas::algorithm::lgc(p->f, vec(r), M, source, alpha, eps, &desc->desc,
                                       &count);
    });
  });
  if (info == 0 && rounds) *rounds = count;
  return info;
}

int gb200_lgc_sweep(gb200_vector_t cluster, gb200_vector_t p, gb200_matrix_t A,
                    gb200_desc_t desc, int* size, double* conductance, float* tight_ms) {
  if (cluster == NULL || p == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL && A->i == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  int members = 0;
  double phi = 0.0;
  const int info = runAlgorithm(tight_ms, [&] {
    return onMatrix(A, [&](auto M) {
      return graphblas::algorithm::lgcSweep(cluster->f, p->f, M, &desc->desc, &members,
                                            &phi);
    });
  });
  if (info == 0 && size) *size = members;
  if (info == 0 && conductance) *conductance = phi;
  return info;
}

int gb200_pr(gb200_vector_t p, gb200_matrix_t A, float alpha, float eps,
             gb200_desc_t desc, float* tight_ms) {
  if (p == NULL || A == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (A->f == NULL) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  return runAlgorithm(tight_ms, [&] {
    return graphblas::algorithm::pr(p->f, A->f, alpha, eps, &desc->desc);
  });
}

int gb200_tc(long long* ntris, gb200_matrix_t A, gb200_matrix_t B,
             gb200_desc_t desc, float* tight_ms) {
  if (ntris == NULL || A == NULL || B == NULL || desc == NULL)
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  if (!allInt32(A, B)) return rc(graphblas::GrB_DOMAIN_MISMATCH);
  GB200_REQUIRE_DEVICE();
  int count = 0;
  const int info = runAlgorithm(tight_ms, [&] {
    return graphblas::algorithm::tc(&count, A->i, B->i, &desc->desc);
  });
  if (info == 0) *ntris = count;
  return info;
}

// ---- Vector as a bitmap ---------------------------------------------------------

int gb200_vector_export_bits(gb200_vector_t v, uint32_t* d_bits,
                             long long* count_out) {
  if (v == NULL || d_bits == NULL) return rc(graphblas::GrB_NULL_POINTER);
  GB200_REQUIRE_DEVICE();
  using namespace graphblas::backend;
  graphblas::backend::Vector<float>& b = v->f->vector_;
  cudaStream_t s = gbStream();
  const size_t nwords = (static_cast<size_t>(b.nsize_) + 31)/32;
  if (b.vec_type_ == graphblas::GrB_DENSE) {
    const unsigned int* bits = b.dense_.ensureBits();
    CUDA_CALL(cudaMemcpyAsync(d_bits, bits, nwords*sizeof(unsigned int),
        cudaMemcpyDeviceToDevice, s));
  } else if (b.vec_type_ == graphblas::GrB_SPARSE) {
    CUDA_CALL(cudaMemsetAsync(d_bits, 0, nwords*sizeof(unsigned int), s));
    if (b.sparse_.nvals_ > 0) {
      scatterBitsKernel<<<gridFor(b.sparse_.nvals_, 256), 256, 0, s>>>(d_bits,
          b.sparse_.d_ind_, b.sparse_.nvals_);
      GB_KERNEL_CHECK();
    }
  } else {
    return rc(graphblas::GrB_UNINITIALIZED_OBJECT);
  }
  if (count_out != NULL) {
    if (b.vec_type_ == graphblas::GrB_SPARSE) {
      *count_out = b.sparse_.nvals_;
    } else {
      static unsigned long long* cell = NULL;
      if (cell == NULL) CUDA_CALL(cudaMalloc(&cell, sizeof(unsigned long long)));
      CUDA_CALL(cudaMemsetAsync(cell, 0, sizeof(unsigned long long), s));
      popcountKernel<<<gridFor(nwords, 256), 256, 0, s>>>(cell, d_bits,
          static_cast<graphblas::Index>(nwords));
      GB_KERNEL_CHECK();
      *count_out = static_cast<long long>(runtime().fetch(cell));
    }
  }
  return 0;
}

// ---- Measurement hooks --------------------------------------------------------

int gb200_profile_enable(int on) {
  GB200_REQUIRE_DEVICE();
  graphblas::backend::profiler().enabled = (on != 0);
  if (on) graphblas::backend::profiler().ensureCells();
  return 0;
}

int gb200_profile_reset(void) {
  GB200_REQUIRE_DEVICE();
  graphblas::backend::profiler().reset(graphblas::backend::gbStream());
  return 0;
}

int gb200_profile_read(int kind, double* ms, long long* launches,
                       double* bytes) {
  if (ms == NULL || launches == NULL || bytes == NULL)
    return rc(graphblas::GrB_NULL_POINTER);
  if (kind < 0 || kind >= GB_PROF_NKINDS)
    return rc(graphblas::GrB_INVALID_VALUE);
  GB200_REQUIRE_DEVICE();
  graphblas::backend::profiler().read(kind, graphblas::backend::gbStream(), ms,
      launches, bytes);
  return 0;
}

int gb200_launch_count(unsigned long long* out) {
  if (out == NULL) return rc(graphblas::GrB_NULL_POINTER);
  *out = graphblas::backend::launchCounter();
  return 0;
}

// ---- Graph ingest -------------------------------------------------------------

int gb200_rmat_edges(int scale, long long nedges, unsigned long long seed,
                     long long first_edge, int* d_src, int* d_dst) {
  if (d_src == NULL || d_dst == NULL) return rc(graphblas::GrB_NULL_POINTER);
  if (scale < 1 || scale > 30 || nedges < 0)
    return rc(graphblas::GrB_INVALID_VALUE);
  GB200_REQUIRE_DEVICE();
  if (nedges == 0) return 0;
  const int grid = graphblas::backend::runtime().sm_count*8;
  rmatEdgesKernel<<<grid, 256, 0, graphblas::backend::gbStream()>>>(scale,
      nedges, seed, first_edge, d_src, d_dst);
  if (cudaGetLastError() != cudaSuccess) return rc(graphblas::GrB_PANIC);
  ++graphblas::backend::launchCounter();
  return 0;
}

}  // extern "C"

#include "dist_exchange.cuh"
#include "dist_bfs_fused.cuh"
