// Data-parallel gradient exchange over NVLink peer memory, fused with the optimizer step.
//
// The reference trains its replicas with one gradient exchange per update (gops/trainer/off_sync_trainer.py: every
// worker's `get_remote_update_info` gradient is applied by `remote_update`); here every rank holds the flat vector
// [gradient | loss | critic mean | #done] of its shard and needs the SUM over ranks followed by Adam.  The vector is a
// few thousand floats, so the exchange is latency, not bandwidth: instead of reduce kernel -> NCCL all-reduce -> Adam
// kernel, ONE kernel per rank
//   1. pushes its chunk of the vector into a slot of every peer's exchange buffer (plain stores through NVLink),
//   2. publishes a per-(CTA, source rank) sequence flag with release semantics at system scope,
//   3. waits for the flags of all peers on its OWN buffer, sums the slots in rank order (bit-identical on every rank),
//   4. applies torch.optim.Adam to its chunk of the parameters (optional).
// Slots and flags are double-buffered on the parity of the call number: a rank can only reach call s+2 after every
// peer has published call s+1, i.e. after every peer has finished reading call s.  Exchange buffers are plain
// cudaMalloc regions shared with cudaIpc handles (one process per GPU) or wired directly (one process, several
// streams / devices: gops_b200_peer_connect_local, also what the single-GPU protocol test uses).
#include "gops_b200.h"
#include "adam_math.cuh"

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <new>
#include <string>

#include "host_util.h"

using gops::DevGuard;
using gops::fail;

namespace {

constexpr int kMaxWorld = 16;
constexpr int kBlocks = 8;                 // CTAs per call; each owns a contiguous chunk and its own flags
constexpr int kThreads = 256;
constexpr long long kSpinLimitNs = 60000000000ll;    // 60 s: a peer that never arrives must not hang the GPU for good

struct PeerArgs {
  int world, rank;
  long long cap;                 // floats per slot
  unsigned seq;                  // call number (>= 1)
  float* base[kMaxWorld];        // exchange regions, base[rank] is the local one
  float* buf;                    // in: this rank's vector, out: the sum
  long long n;
  unsigned* err;                 // local error word (set when a peer did not arrive in time)
  // Adam (params == nullptr: plain all-reduce)
  float *params, *m, *v;
  long long nparam;
  float one_minus_b1, b2, one_minus_b2, eps, step_size, bc2_sqrt;
};

__host__ __device__ inline size_t flags_offset_floats(int world, long long cap) { return (size_t)2 * world * cap; }
__device__ __forceinline__ float* slot(float* base, int world, long long cap, unsigned parity, int src) {
  return base + ((size_t)parity * world + src) * cap;
}
__device__ __forceinline__ unsigned* flag(float* base, int world, long long cap, unsigned parity, int blk, int src) {
  return reinterpret_cast<unsigned*>(base + flags_offset_floats(world, cap)) + ((size_t)parity * kBlocks + blk) * kMaxWorld + src;
}
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ long long globaltimer_ns() {
  long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

__global__ void __launch_bounds__(kThreads) peer_allreduce_kernel(PeerArgs a) {
  const int blk = blockIdx.x, tid = threadIdx.x;
  const unsigned parity = a.seq & 1u;
  long long chunk = (a.n + kBlocks - 1) / kBlocks;
  chunk = (chunk + 3) / 4 * 4;
  const long long i0 = (long long)blk * chunk, i1 = i0 + chunk < a.n ? i0 + chunk : a.n;
  float* local = a.base[a.rank];
  // 1. push this chunk into slot [parity][rank] of every peer, nearest neighbour first so the links are used evenly
  for (int d = 1; d < a.world; ++d) {
    const int dst = (a.rank + d) % a.world;
    float* s = slot(a.base[dst], a.world, a.cap, parity, a.rank);
    for (long long i = i0 + tid; i < i1; i += kThreads) s[i] = a.buf[i];
  }
  __threadfence_system();
  __syncthreads();
  // 2. publish, 3. wait: one thread per peer
  __shared__ int timed_out;
  if (tid == 0) timed_out = 0;
  __syncthreads();
  if (tid < a.world && tid != a.rank) {
    st_release_sys(flag(a.base[tid], a.world, a.cap, parity, blk, a.rank), a.seq);
    const unsigned* f = flag(local, a.world, a.cap, parity, blk, tid);
    const long long t0 = globaltimer_ns();
    while (ld_acquire_sys(f) != a.seq) {
      if (globaltimer_ns() - t0 > kSpinLimitNs) { timed_out = 1; break; }
    }
  }
  __syncthreads();
  if (timed_out) {
    if (tid == 0) atomicExch(a.err, 1u);
    for (long long i = i0 + tid; i < i1; i += kThreads) a.buf[i] = nanf("");     // never a silently partial sum
    return;
  }
  // sum in rank order: every rank adds the same numbers in the same order
  for (long long i = i0 + tid; i < i1; i += kThreads) {
    float s = 0.f;
    for (int r = 0; r < a.world; ++r)
      s += r == a.rank ? a.buf[i] : __ldcg(slot(local, a.world, a.cap, parity, r) + i);
    a.buf[i] = s;
    if (a.params && i < a.nparam) {       // the arithmetic of adam_kernel (adam_math.cuh)
      float pi = a.params[i], mi = a.m[i], vi = a.v[i];
      gops::adam_update(s, pi, mi, vi, a.one_minus_b1, a.b2, a.one_minus_b2, a.eps, a.step_size, a.bc2_sqrt);
      a.params[i] = pi;
      a.m[i] = mi;
      a.v[i] = vi;
    }
  }
}

}  // namespace

struct gops_b200_peer {
  int world = 0, rank = 0, device = -1;
  long long cap = 0;
  float* base[kMaxWorld] = {};
  bool ipc_opened[kMaxWorld] = {};
  bool connected = false;
  unsigned seq = 0;
  unsigned* err = nullptr;
  size_t region_bytes = 0;
};

extern "C" {

int gops_b200_peer_create(int32_t world, int32_t rank, int64_t max_floats, gops_b200_peer** out) {
  if (!out) return fail("peer_create: null out");
  *out = nullptr;
  if (world < 1 || world > kMaxWorld || rank < 0 || rank >= world) return fail("peer_create: world must be 1..16, 0 <= rank < world");
  if (max_floats < 1) return fail("peer_create: max_floats must be positive");
  gops_b200_peer* p = new (std::nothrow) gops_b200_peer();
  if (!p) return fail("out of host memory");
  p->world = world;
  p->rank = rank;
  p->cap = (max_floats + 3) / 4 * 4;
  if (cudaGetDevice(&p->device) != cudaSuccess) { delete p; return fail("no CUDA device"); }
  p->region_bytes = flags_offset_floats(world, p->cap) * sizeof(float) + (size_t)2 * kBlocks * kMaxWorld * sizeof(unsigned) + 16;
  void* q = nullptr;
  if (cudaMalloc(&q, p->region_bytes) != cudaSuccess || cudaMemset(q, 0, p->region_bytes) != cudaSuccess) {
    cudaFree(q);
    delete p;
    return fail("peer_create: cudaMalloc of the exchange region failed");
  }
  p->base[rank] = static_cast<float*>(q);
  // the error word lives behind the flags
  p->err = reinterpret_cast<unsigned*>(static_cast<char*>(q) + p->region_bytes - 16);
  p->connected = world == 1;
  cudaDeviceSynchronize();
  *out = p;
  return 0;
}

int gops_b200_peer_region_bytes(const gops_b200_peer* p, int64_t* bytes) {
  if (!p || !bytes) return fail("null argument");
  *bytes = (int64_t)p->region_bytes;
  return 0;
}

int gops_b200_peer_export(gops_b200_peer* p, void* handle64) {
  if (!p || !handle64) return fail("null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == GOPS_B200_IPC_HANDLE_BYTES, "handle size");
  DevGuard g(p->device);
  cudaIpcMemHandle_t h;
  CUDA_OK(cudaIpcGetMemHandle(&h, p->base[p->rank]));
  memcpy(handle64, &h, sizeof(h));
  return 0;
}

int gops_b200_peer_connect(gops_b200_peer* p, const void* handles) {
  if (!p || !handles) return fail("null argument");
  DevGuard g(p->device);
  for (int r = 0; r < p->world; ++r) {
    if (r == p->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, static_cast<const char*>(handles) + (size_t)r * GOPS_B200_IPC_HANDLE_BYTES, sizeof(h));
    void* q = nullptr;
    CUDA_OK(cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess));
    p->base[r] = static_cast<float*>(q);
    p->ipc_opened[r] = true;
  }
  p->connected = true;
  return 0;
}

int gops_b200_peer_local_base(gops_b200_peer* p, void** base) {
  if (!p || !base) return fail("null argument");
  *base = p->base[p->rank];
  return 0;
}

int gops_b200_peer_connect_local(gops_b200_peer* p, void* const* bases) {
  if (!p || !bases) return fail("null argument");
  DevGuard g(p->device);
  for (int r = 0; r < p->world; ++r) {
    if (r == p->rank) continue;
    if (!bases[r]) return fail("peer_connect_local: null region");
    cudaPointerAttributes at;
    CUDA_OK(cudaPointerGetAttributes(&at, bases[r]));
    if (at.type != cudaMemoryTypeDevice) return fail("peer_connect_local: not a device pointer");
    if (at.device != p->device) {
      int can = 0;
      CUDA_OK(cudaDeviceCanAccessPeer(&can, p->device, at.device));
      if (!can) return fail("peer_connect_local: no peer access between the devices");
      const cudaError_t e = cudaDeviceEnablePeerAccess(at.device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
      (void)cudaGetLastError();
    }
    p->base[r] = static_cast<float*>(bases[r]);
  }
  p->connected = true;
  return 0;
}

int gops_b200_peer_allreduce(gops_b200_peer* p, float* buf, int64_t n, float* params, float* exp_avg, float* exp_avg_sq,
                             int64_t nparam, int32_t step, double lr, double beta1, double beta2, double eps, void* stream) {
  if (!p || !buf) return fail("null argument");
  if (!p->connected) return fail("peer_allreduce: peers are not connected");
  if (n < 1 || n > p->cap) return fail("peer_allreduce: vector longer than the exchange slots");
  if (params && (!exp_avg || !exp_avg_sq || nparam < 1 || nparam > n || step < 1)) return fail("peer_allreduce: bad Adam arguments");
  DevGuard g(p->device);
  PeerArgs a;
  memset(&a, 0, sizeof(a));
  a.world = p->world; a.rank = p->rank; a.cap = p->cap; a.seq = ++p->seq;
  for (int r = 0; r < p->world; ++r) a.base[r] = p->base[r];
  a.buf = buf; a.n = n; a.err = p->err;
  a.params = params; a.m = exp_avg; a.v = exp_avg_sq; a.nparam = params ? nparam : 0;
  if (params) {
    const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
    a.one_minus_b1 = (float)(1.0 - beta1); a.b2 = (float)beta2; a.one_minus_b2 = (float)(1.0 - beta2); a.eps = (float)eps;
    a.step_size = (float)(lr / bc1); a.bc2_sqrt = (float)sqrt(bc2);
  }
  peer_allreduce_kernel<<<kBlocks, kThreads, 0, (cudaStream_t)stream>>>(a);
  gops::g_launches += 1;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int gops_b200_peer_error(gops_b200_peer* p, int32_t* err) {
  if (!p || !err) return fail("null argument");
  DevGuard g(p->device);
  unsigned e = 0;
  CUDA_OK(cudaMemcpy(&e, p->err, sizeof(e), cudaMemcpyDeviceToHost));
  *err = (int32_t)e;
  return 0;
}

int gops_b200_peer_destroy(gops_b200_peer* p) {
  if (!p) return 0;
  DevGuard g(p->device);
  cudaDeviceSynchronize();
  for (int r = 0; r < p->world; ++r)
    if (p->ipc_opened[r]) cudaIpcCloseMemHandle(p->base[r]);
  cudaFree(p->base[p->rank]);
  (void)cudaGetLastError();
  delete p;
  return 0;
}

}  // extern "C"
