// Shared helpers for the shapy_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <string>
#include <vector>

#include "../../include/shapy_b200.h"

namespace shapy {

void set_error(const char *fmt, ...);
void count_launch(int n = 1);

#define SHAPY_CUDA_TRY(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      shapy::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return (int)_e;                                                                     \
    }                                                                                     \
  } while (0)

#define SHAPY_LAUNCH_CHECK()                                                              \
  do {                                                                                    \
    shapy::count_launch();                                                                \
    cudaError_t _e = cudaGetLastError();                                                  \
    if (_e != cudaSuccess) {                                                              \
      shapy::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return (int)_e;                                                                     \
    }                                                                                     \
  } while (0)

#define SHAPY_REQUIRE(cond, ...)                                                          \
  do {                                                                                    \
    if (!(cond)) {                                                                        \
      shapy::set_error(__VA_ARGS__);                                                      \
      return SHAPY_ERR_ARG;                                                               \
    }                                                                                     \
  } while (0)

// cudaFuncSetAttribute applies to the CURRENT device only: a process that drives several GPUs must configure the
// kernel once per device, so the "already done" state is a per-device bit, not a process-wide flag.
template <typename Kernel>
static inline cudaError_t set_max_dynamic_smem(Kernel kernel, int bytes, std::atomic<unsigned long long> &done_mask) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const unsigned long long bit = 1ull << (dev & 63);
  if (done_mask.load(std::memory_order_acquire) & bit) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done_mask.fetch_or(bit, std::memory_order_release);
  return e;
}

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// RAII-less device buffer owned by long-lived objects (model constants).
template <typename T>
struct DevBuf {
  T *ptr = nullptr;
  size_t n = 0;
  cudaError_t upload(const std::vector<T> &h) {
    n = h.size();
    cudaError_t e = cudaMalloc((void **)&ptr, std::max<size_t>(n, 1) * sizeof(T));
    if (e != cudaSuccess) return e;
    if (n) e = cudaMemcpy(ptr, h.data(), n * sizeof(T), cudaMemcpyHostToDevice);
    return e;
  }
  cudaError_t alloc(size_t count) {
    n = count;
    return cudaMalloc((void **)&ptr, std::max<size_t>(n, 1) * sizeof(T));
  }
  void release() {
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    n = 0;
  }
};

}  // namespace shapy
