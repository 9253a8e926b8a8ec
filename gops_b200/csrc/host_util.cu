// Host-side helpers shared by every translation unit of the library (host_util.h).
#include "host_util.h"

#include <mutex>
#include <set>
#include <utility>

namespace gops {

std::atomic<long long> g_launches{0};

namespace {
thread_local std::string g_err;
}  // namespace

int fail(const std::string& msg) {
  g_err = msg;
  return 1;
}
const char* last_error() { return g_err.c_str(); }

int device_of(const void* p) {
  cudaPointerAttributes a;
  if (p && cudaPointerGetAttributes(&a, p) == cudaSuccess && a.type == cudaMemoryTypeDevice) return a.device;
  (void)cudaGetLastError();
  int d = 0;
  cudaGetDevice(&d);
  return d;
}

int DevBuf::ensure(size_t floats, bool zero_fill) {
  if (floats <= n) return 0;
  release();
  CUDA_OK(cudaMalloc(&p, floats * sizeof(float)));
  n = floats;
  if (zero_fill) CUDA_OK(cudaMemset(p, 0, floats * sizeof(float)));
  return 0;
}

void DevBuf::release() {
  if (p) {
    const cudaError_t e = cudaFree(p);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      if (getenv("GOPS_B200_DEBUG")) fprintf(stderr, "[gops_b200] cudaFree(%p) failed: %s\n", (void*)p, cudaGetErrorString(e));
    }
  }
  p = nullptr;
  n = 0;
}

int allow_smem(const void* fn, int dev, int bytes) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;
  std::lock_guard<std::mutex> lock(mu);
  if (done.count({fn, dev})) return 0;
  CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.insert({fn, dev});
  return 0;
}

}  // namespace gops
