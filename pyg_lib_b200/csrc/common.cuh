// Shared helpers for libpyg_b200.so (error reporting, launch accounting, tiny device utilities).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "pyg_b200.h"

typedef unsigned long long u64;
typedef long long i64;
typedef unsigned int u32;

namespace pygb200 {

void set_error(const std::string& msg);  // thread-local, read by pygb200_last_error()
void count_launch(int n = 1);            // process-wide kernel launch counter

// Optional per-kernel device timing (pygb200_profile_enable): CUDA events on the launching stream
// around selected launches, accumulated per name.  Off by default (zero overhead besides a branch).
bool prof_enabled();
void* prof_begin(cudaStream_t st);                                   // returns an opaque token (or null)
void prof_end(void* token, const char* name, cudaStream_t st, long long work);

#define PYGB_CUDA(expr)                                                                          \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      ::pygb200::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ + \
                           ":" + std::to_string(__LINE__) + ")");                                \
      return PYGB200_ERR_CUDA;                                                                   \
    }                                                                                            \
  } while (0)

#define PYGB_CHECK(cond, code, msg)  \
  do {                               \
    if (!(cond)) {                   \
      ::pygb200::set_error(msg);     \
      return (code);                 \
    }                                \
  } while (0)

#define PYGB_LAUNCH_CHECK()              \
  do {                                   \
    ::pygb200::count_launch();           \
    PYGB_CUDA(cudaGetLastError());       \
  } while (0)

// Device buffer that only ever grows (persistent workspace).  `ensure` keeps the first
// `preserve_bytes` bytes when it has to reallocate.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes, size_t preserve_bytes, cudaStream_t stream) {
    if (bytes <= cap) return PYGB200_OK;
    size_t ncap = cap ? cap : 4096;
    while (ncap < bytes) ncap *= 2;
    void* np = nullptr;
    PYGB_CUDA(cudaMalloc(&np, ncap));
    if (p && preserve_bytes) PYGB_CUDA(cudaMemcpyAsync(np, p, preserve_bytes, cudaMemcpyDeviceToDevice, stream));
    if (p) {
      PYGB_CUDA(cudaStreamSynchronize(stream));
      PYGB_CUDA(cudaFree(p));
    }
    p = np;
    cap = ncap;
    return PYGB200_OK;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

// The stream-ordered allocator's default pool hands memory back to the OS at every synchronisation point, which made
// matmul run times jump between 2 and 9 ms; keep what it has.
inline void keep_pool_memory() {
  static bool done = false;
  if (done) return;
  done = true;
  int dev = 0;
  cudaMemPool_t pool;
  if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
    unsigned long long thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
}

// Stream-ordered scratch (problem lists, split-K partials) that is returned to the pool on every exit path (the PYGB_*
// macros return early on errors).
struct AsyncScratch {
  void* p = nullptr;
  cudaStream_t st = nullptr;
  int alloc(size_t bytes, cudaStream_t stream) {
    st = stream;
    keep_pool_memory();
    PYGB_CUDA(cudaMallocAsync(&p, bytes, stream));
    return PYGB200_OK;
  }
  ~AsyncScratch() { if (p) cudaFreeAsync(p, st); }
  AsyncScratch() = default;
  AsyncScratch(const AsyncScratch&) = delete;
  AsyncScratch& operator=(const AsyncScratch&) = delete;
};

__host__ __device__ inline i64 ceil_div(i64 a, i64 b) { return (a + b - 1) / b; }

// Asynchronous argument errors (matmul.cu): a kernel that finds invalid input raises its slot's flag instead of touching
// memory, and the next call of that family reports it.  async_error_flag_dev may return null (no mapped memory).
enum { ASYNC_ERR_MATMUL = 0, ASYNC_ERR_RANDOM_WALK = 1, ASYNC_ERR_SLOTS = 2 };
int* async_error_flag_dev(int slot);
bool take_async_error(int slot);   // reads and clears the slot's flag

}  // namespace pygb200
