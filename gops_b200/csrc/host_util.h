// Host-side helpers shared by every translation unit of the library: the thread-local last error
// (gops_b200_last_error), the launch counter (gops_b200_launch_count), CUDA error checks, device guards, grow-only
// device buffers and the once-per-device shared-memory opt-in of a kernel.
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>

#include <atomic>
#include <string>

namespace gops {

extern std::atomic<long long> g_launches;   // kernels launched by this library

int fail(const std::string& msg);           // records msg as the calling thread's last error; returns 1
const char* last_error();

// CUDA_OK(expr) fails with "<expr>: <CUDA error>", CUDA_OK(expr, label) with "<label>: <CUDA error>".
#define GOPS_CUDA_OK2(expr, label)                                                                 \
  do {                                                                                             \
    const cudaError_t e__ = (expr);                                                                \
    if (e__ != cudaSuccess) return ::gops::fail(std::string(label) + ": " + cudaGetErrorString(e__)); \
  } while (0)
#define GOPS_CUDA_OK1(expr) GOPS_CUDA_OK2(expr, #expr)
#define GOPS_CUDA_OK_PICK(_1, _2, NAME, ...) NAME
#define CUDA_OK(...) GOPS_CUDA_OK_PICK(__VA_ARGS__, GOPS_CUDA_OK2, GOPS_CUDA_OK1, )(__VA_ARGS__)

// A CUDA error left behind by an earlier (possibly foreign) call must not be blamed on the next launch.
#define ENTRY()                                                                                    \
  do {                                                                                             \
    const cudaError_t e0__ = cudaGetLastError();                                                   \
    if (e0__ != cudaSuccess && getenv("GOPS_B200_DEBUG"))                                          \
      fprintf(stderr, "[gops_b200] stale CUDA error at entry of %s: %s\n", __func__, cudaGetErrorString(e0__)); \
  } while (0)

// Device that owns p; the current device when p is not device memory.
int device_of(const void* p);

// Every entry point runs on the device that owns its plan / buffers, whatever the caller's current device is
// (networks on cuda:1 while cuda:0 is current must not put scratch on one GPU and the launch on the other).
struct DevGuard {
  int prev = -1;
  bool switched = false;
  explicit DevGuard(int dev) {
    if (dev >= 0 && cudaGetDevice(&prev) == cudaSuccess && prev != dev) switched = cudaSetDevice(dev) == cudaSuccess;
  }
  explicit DevGuard(const void* p) : DevGuard(device_of(p)) {}
  ~DevGuard() {
    if (switched) cudaSetDevice(prev);
  }
  DevGuard(const DevGuard&) = delete;
  DevGuard& operator=(const DevGuard&) = delete;
};

// Grow-only float buffer in device memory, freed with its owner.
struct DevBuf {
  float* p = nullptr;
  size_t n = 0;   // floats
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  // at least `floats` floats; a new allocation is zero-filled when zero_fill is set
  int ensure(size_t floats, bool zero_fill = false);
  void release();   // a failed cudaFree is reported on stderr under GOPS_B200_DEBUG
};

// cudaFuncAttributeMaxDynamicSharedMemorySize = bytes for kernel fn on device dev, set once per (kernel, device).
int allow_smem(const void* fn, int dev, int bytes);

}  // namespace gops
