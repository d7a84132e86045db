// graphblast_b200 backend — error macros, debug printing, GpuTimer and the
// per-process runtime context (stream, SM count, pinned staging).
//
// Replaces reference graphblas/backend/cuda/util.hpp:4-120.  Algorithm headers
// include this file by literal path (reference graphblas/algorithm/bfs.hpp:8)
// and use backend::GpuTimer {Start, Stop, ElapsedMillis}.
//
// Difference from the reference by design: CUDA_CALL checks the API status but
// does NOT cudaThreadSynchronize() after every call (reference util.hpp:12-19);
// the backend synchronises only where the host consumes a device result.
#ifndef GRAPHBLAS_BACKEND_CUDA_UTIL_HPP_
#define GRAPHBLAS_BACKEND_CUDA_UTIL_HPP_

#include <cuda_runtime.h>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <utility>
#include <vector>

#define CUDA_SAFE_CALL_NO_SYNC(call) do {                                    \
  cudaError_t gb_err__ = (call);                                             \
  if (cudaSuccess != gb_err__) {                                             \
    fprintf(stderr, "Cuda error in file '%s' in line %i : %s.\n",            \
            __FILE__, __LINE__, cudaGetErrorString(gb_err__));               \
    exit(EXIT_FAILURE);                                                      \
  } } while (0)

#define CUDA_CALL(call) CUDA_SAFE_CALL_NO_SYNC(call)

// After a kernel launch: catches launch-configuration errors immediately and
// counts the launch (bench.py reports gpu_launches from this counter).
#define GB_KERNEL_CHECK() do {                                               \
  CUDA_SAFE_CALL_NO_SYNC(cudaGetLastError());                                \
  ++graphblas::backend::launchCounter();                                     \
} while (0)

// Hot-kernel kinds timed by the optional profiler (gb200_profile_*).
#define GB_PROF_SPMV_MERGE 0
#define GB_PROF_PULL_BOOL  1
#define GB_PROF_PUSH       2
#define GB_PROF_SPGEMM     3
#define GB_PROF_SPMM       4
#define GB_PROF_NKINDS     5

namespace graphblas {
namespace backend {

inline unsigned long long& launchCounter() {
  static unsigned long long count = 0;
  return count;
}

// ---------------------------------------------------------------------------
// Optional hot-kernel profiler.  When enabled, every launch of a hot kernel is
// bracketed by two cudaEvents on the launching stream; reading a kind sums the
// elapsed times.  Algorithmic bytes that are only known on the device (edges
// inspected by the early-exit pull, edges expanded by the push) are accumulated
// by the kernels themselves into d_cells.  Off by default: no events, and the
// kernels' accumulation is one atomic per CTA.
// ---------------------------------------------------------------------------
struct Profiler {
  bool enabled;
  std::vector<cudaEvent_t> start[GB_PROF_NKINDS];
  std::vector<cudaEvent_t> stop[GB_PROF_NKINDS];
  size_t used[GB_PROF_NKINDS];
  double host_bytes[GB_PROF_NKINDS];       // algorithmic bytes known on the host
  unsigned long long* d_cells;             // [kind] device-side byte/edge counters

  Profiler() : enabled(false), d_cells(NULL) {
    for (int k = 0; k < GB_PROF_NKINDS; ++k) { used[k] = 0; host_bytes[k] = 0; }
  }

  // The cells are cleared on the stream whose kernels add into them: a clear on the
  // legacy stream would be unordered with those kernels under a non-blocking stream.
  void ensureCells(cudaStream_t s) {
    if (d_cells == NULL) {
      CUDA_CALL(cudaMalloc(&d_cells, GB_PROF_NKINDS*sizeof(unsigned long long)));
      CUDA_CALL(cudaMemsetAsync(d_cells, 0, GB_PROF_NKINDS*sizeof(unsigned long long), s));
    }
  }

  void begin(int kind, cudaStream_t s) {
    if (!enabled) return;
    if (used[kind] == start[kind].size()) {
      cudaEvent_t a, b;
      CUDA_CALL(cudaEventCreate(&a));
      CUDA_CALL(cudaEventCreate(&b));
      start[kind].push_back(a);
      stop[kind].push_back(b);
    }
    CUDA_CALL(cudaEventRecord(start[kind][used[kind]], s));
  }

  void end(int kind, cudaStream_t s, double bytes) {
    if (!enabled) return;
    CUDA_CALL(cudaEventRecord(stop[kind][used[kind]], s));
    ++used[kind];
    host_bytes[kind] += bytes;
  }

  void reset(cudaStream_t s) {
    ensureCells(s);
    for (int k = 0; k < GB_PROF_NKINDS; ++k) { used[k] = 0; host_bytes[k] = 0; }
    CUDA_CALL(cudaMemsetAsync(d_cells, 0, GB_PROF_NKINDS*sizeof(unsigned long long), s));
  }

  // Total milliseconds, launches and bytes of one kind (synchronises).
  void read(int kind, cudaStream_t s, double* ms, long long* launches, double* bytes) {
    ensureCells(s);
    unsigned long long cell = 0;
    CUDA_CALL(cudaMemcpyAsync(&cell, d_cells + kind, sizeof(cell), cudaMemcpyDeviceToHost, s));
    CUDA_CALL(cudaStreamSynchronize(s));
    double total = 0;
    for (size_t i = 0; i < used[kind]; ++i) {
      float t = 0.f;
      CUDA_CALL(cudaEventElapsedTime(&t, start[kind][i], stop[kind][i]));
      total += t;
    }
    *ms = total;
    *launches = static_cast<long long>(used[kind]);
    *bytes = host_bytes[kind] + static_cast<double>(cell);
  }
};

inline Profiler& profiler() {
  static Profiler p;
  return p;
}

// ---------------------------------------------------------------------------
// Runtime context: one per process (one process per GPU).
// ---------------------------------------------------------------------------
struct Runtime {
  cudaStream_t stream;      // every backend kernel / copy is issued here
  int          device;
  int          sm_count;
  void*        h_pinned;    // pinned staging for small D2H results
  size_t       h_pinned_bytes;
  bool         ready;

  Runtime() : stream(0), device(0), sm_count(132), h_pinned(NULL),
              h_pinned_bytes(0), ready(false), h_mail(NULL), d_mail(NULL),
              mail_seq(0) {}

  void init() {
    if (ready) return;
    CUDA_CALL(cudaGetDevice(&device));
    cudaDeviceProp prop;
    CUDA_CALL(cudaGetDeviceProperties(&prop, device));
    sm_count = prop.multiProcessorCount;
    h_pinned_bytes = 4096;
    CUDA_CALL(cudaMallocHost(&h_pinned, h_pinned_bytes));
    ready = true;
  }

  // Blocking read of a small device value through pinned memory.
  template <typename T>
  T fetch(const T* d_ptr) {
    init();
    CUDA_CALL(cudaMemcpyAsync(h_pinned, d_ptr, sizeof(T), cudaMemcpyDeviceToHost, stream));
    CUDA_CALL(cudaStreamSynchronize(stream));
    return *reinterpret_cast<T*>(h_pinned);
  }

  template <typename T>
  void fetch2(const T* d_ptr, T* a, T* b) {
    init();
    CUDA_CALL(cudaMemcpyAsync(h_pinned, d_ptr, 2*sizeof(T), cudaMemcpyDeviceToHost, stream));
    CUDA_CALL(cudaStreamSynchronize(stream));
    *a = reinterpret_cast<T*>(h_pinned)[0];
    *b = reinterpret_cast<T*>(h_pinned)[1];
  }

  void sync() { CUDA_CALL(cudaStreamSynchronize(stream)); }

  // ---- mailbox: small results a kernel posts straight into host memory ---------
  // A per-level count (compaction total, discovered rows) decides what the host
  // launches next.  Reading it with cudaMemcpyAsync + cudaStreamSynchronize
  // waits for EVERYTHING queued on the stream and costs ~10 us of idle GPU per
  // level; instead the kernel that knows the value stores (ticket << 40 | value)
  // into mapped pinned memory (mailPost, kernels/util.cuh) and the host polls that
  // word (mailWait), so it goes on once the producing kernel is done, while later
  // kernels still run.  Slots: 0 compaction, 1 Boolean pull, 2 reduce, 4 push edges.
  unsigned long long* h_mail;     // pinned + mapped, 8 slots
  unsigned long long* d_mail;
  unsigned long long  mail_seq;

  void mailInit() {
    if (h_mail != NULL) return;
    CUDA_CALL(cudaHostAlloc(reinterpret_cast<void**>(&h_mail), 8*sizeof(unsigned long long), cudaHostAllocMapped));
    for (int i = 0; i < 8; ++i) h_mail[i] = 0ull;
    CUDA_CALL(cudaHostGetDevicePointer(reinterpret_cast<void**>(&d_mail), h_mail, 0));
    mail_seq = 0;
  }
  // Ticket for the next post (24 bits, never 0) and where the kernel writes it.
  unsigned long long mailTicket() { mailInit(); mail_seq = (mail_seq % 0xfffffeull) + 1; return mail_seq; }
  unsigned long long* mailSlot(int slot) { mailInit(); return d_mail + slot; }
  // The 40-bit value posted under `ticket`; false if the slot was reused by a later
  // post or nothing arrives (the caller then reads its own cell stream-ordered).
  bool mailWait(int slot, unsigned long long ticket, unsigned long long* value) {
    volatile unsigned long long* p = h_mail + slot;
    const auto t0 = std::chrono::steady_clock::now();
    for (unsigned long long spin = 0;; ++spin) {
      const unsigned long long v = *p;
      const unsigned long long got = v >> 40;
      if (got == ticket) { *value = v & ((1ull << 40) - 1ull); return true; }
      if (got != 0 && ((got - ticket) & 0xffffffull) < 0x800000ull)
        return false;                           // overwritten by a later post
      if ((spin & 0x3ff) == 0x3ff &&
          std::chrono::steady_clock::now() - t0 > std::chrono::seconds(2))
        return false;
    }
  }
};

inline Runtime& runtime() {
  static Runtime rt;
  if (!rt.ready) rt.init();
  return rt;
}

inline cudaStream_t gbStream() { return runtime().stream; }

// Stream-ordered device allocation (cudaMallocAsync on the backend stream, pool
// release threshold raised so freed blocks are reused without a device sync).
// The reference allocates with cudaMalloc/cudaFree inside every algorithm call
// (frontier vectors in algorithm/bfs.hpp:25-26); here that costs microseconds.
inline void* gbMalloc(size_t bytes) {
  static bool pool_ready = false;
  Runtime& rt = runtime();
  if (!pool_ready) {
    cudaMemPool_t pool;
    CUDA_CALL(cudaDeviceGetDefaultMemPool(&pool, rt.device));
    unsigned long long threshold = ~0ull;
    CUDA_CALL(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold));
    pool_ready = true;
  }
  void* p = NULL;
  if (bytes == 0) bytes = 16;
  CUDA_CALL(cudaMallocAsync(&p, bytes, rt.stream));
  return p;
}

inline void gbFree(void* p) {
  // Errors ignored on purpose: destructors may run during context teardown.
  if (p != NULL) (void)cudaFreeAsync(p, runtime().stream);
}

// Owner of one gbMalloc block (or of NULL): gbFree'd when the owner goes out of scope,
// on every return path.
class DeviceBlock {
 public:
  explicit DeviceBlock(void* p) : p_(static_cast<unsigned char*>(p)) {}
  ~DeviceBlock() { gbFree(p_); }
  DeviceBlock(const DeviceBlock&) = delete;
  DeviceBlock& operator=(const DeviceBlock&) = delete;
  // The array at byte offset `off` of the block.
  template <typename T> T* at(size_t off = 0) const { return reinterpret_cast<T*>(p_ + off); }
  void swap(DeviceBlock& other) { std::swap(p_, other.p_); }   // exchanges the blocks

 private:
  unsigned char* p_;
};

// Arrays placed one after another in one device block, each on a 256-byte boundary:
// place() returns an array's byte offset, `bytes` is the size of the block so far.
struct ScratchLayout {
  size_t bytes = 0;
  size_t place(size_t array_bytes) {
    const size_t off = bytes;
    bytes += (array_bytes + 255)/256*256;
    return off;
  }
};

// Copy of count elements on the backend stream; none for an empty count, a NULL
// end or a copy of an array onto itself.
template <typename X>
void copyAsync(X* dst, const X* src, size_t count, cudaMemcpyKind kind) {
  if (count > 0 && dst != NULL && src != NULL && dst != src)
    CUDA_CALL(cudaMemcpyAsync(dst, src, count*sizeof(X), kind, gbStream()));
}

// One cooperative launch of kernel K, CTAs of NT threads, with K's arguments, on
// `stream`.  The grid is every CTA of K that fits on the device at once; the occupancy
// query runs on K's first launch and is cached.  GrB_PANIC when no CTA fits.
template <auto K, int NT, typename... Args>
Info launchCooperative(cudaStream_t stream, Args... args) {
  static_assert(std::is_same<decltype(K), void (*)(Args...)>::value,
                "the arguments must have the kernel's parameter types");
  static int resident = 0;
  if (resident == 0) {
    int per_sm = 0;
    CUDA_CALL(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, K, NT, 0));
    resident = per_sm*runtime().sm_count;
  }
  if (resident < 1) return GrB_PANIC;
  void* params[] = { &args... };
  CUDA_CALL(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(K), dim3(resident), dim3(NT),
                                        params, 0, stream));
  GB_KERNEL_CHECK();
  return GrB_SUCCESS;
}

// Grid sizing helper: a grid-stride launch sized in whole waves of the SM count.
inline int gridFor(size_t work_items, int threads, int ctas_per_sm = 8) {
  size_t want = (work_items + threads - 1) / threads;
  size_t cap  = static_cast<size_t>(runtime().sm_count) * ctas_per_sm;
  if (want < 1) want = 1;
  return static_cast<int>(want < cap ? want : cap);
}

inline void printMemory(const char* str) {
  size_t free_b, total_b;
  if (GrB_MEMORY) {
    CUDA_CALL(cudaMemGetInfo(&free_b, &total_b));
    std::cout << str << ": " << free_b << " bytes left out of " << total_b
              << " bytes\n";
  }
}

template <typename T>
void printDevice(const char* str, const T* array, int length = 40, bool limit = true) {
  if (limit && length > 40) length = 40;
  if (length <= 0 || array == NULL) {
    std::cout << str << ": (empty)\n";
    return;
  }
  T* temp = reinterpret_cast<T*>(malloc(length*sizeof(T)));
  CUDA_CALL(cudaMemcpyAsync(temp, array, length*sizeof(T), cudaMemcpyDeviceToHost, gbStream()));
  runtime().sync();
  printArray(str, temp, length, limit);
  if (temp) free(temp);
}

inline void printState(bool use_mask, bool use_accum, bool use_scmp, bool use_repl,
    bool use_tran) {
  std::cout << "Mask: " << use_mask  << std::endl;
  std::cout << "Accum:" << use_accum << std::endl;
  std::cout << "SCMP: " << use_scmp  << std::endl;
  std::cout << "Repl: " << use_repl  << std::endl;
  std::cout << "Tran: " << use_tran  << std::endl;
}

template <typename T> constexpr
T const& min(T const& a, T const& b) {
  return a < b ? a : b;
}

template <typename T> constexpr
T const& max(T const& a, T const& b) {  // NOLINT(build/include_what_you_use)
  return a > b ? a : b;
}

// "accum is GrB_NULL" test.  The reference decides this at run time from
// typeid(accum).name().size() > 1 (reference spmv.hpp:34-40): GrB_NULL is NULL,
// whose type mangles to a single character.  Same rule, decided at compile time.
template <typename BinaryOpT>
struct AccumIsNull {
  static const bool value = std::is_integral<BinaryOpT>::value ||
                            std::is_pointer<BinaryOpT>::value ||
                            std::is_same<BinaryOpT, std::nullptr_t>::value;
};

struct GpuTimer {
  cudaEvent_t start;
  cudaEvent_t stop;

  GpuTimer() {
    cudaEventCreate(&start);
    cudaEventCreate(&stop);
  }

  ~GpuTimer() {
    cudaEventDestroy(start);
    cudaEventDestroy(stop);
  }

  void Start() { cudaEventRecord(start, gbStream()); }
  void Stop()  { cudaEventRecord(stop,  gbStream()); }

  float ElapsedMillis() {
    float elapsed;
    cudaEventSynchronize(stop);
    cudaEventElapsedTime(&elapsed, start, stop);
    return elapsed;
  }
};

}  // namespace backend
}  // namespace graphblas

#endif  // GRAPHBLAS_BACKEND_CUDA_UTIL_HPP_
