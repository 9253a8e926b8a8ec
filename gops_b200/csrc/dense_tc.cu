// C ABI of the generic wgmma dense-layer path (include/gops_b200.h, section "layer-wise MLP"): a trainable MLP of
// any depth (widths <= 256 per layer) evaluated layer by layer with the kernels of dense_tc.cuh.  Used by the wide-net
// FHADP path, DSAC and FHADP2; the fused rollout kernels remain the path for 64-wide nets with small inputs.
#include "gops_b200.h"

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <new>
#include <string>

#include "dense_tc.cuh"

using namespace gops;

namespace gops {
int dense_fail(const std::string& msg);       // defined in gops_b200.cu (thread-local last error)
void dense_count_launch(int n);
}  // namespace gops

#define DCUDA(expr)                                                                              \
  do {                                                                                           \
    cudaError_t e__ = (expr);                                                                    \
    if (e__ != cudaSuccess) return gops::dense_fail(std::string(#expr) + ": " + cudaGetErrorString(e__)); \
  } while (0)

constexpr int kMaxLayers = 8, kMaxSlots = 128, kMaxWidth = 256;

struct gops_b200_mlpnet {
  int device = 0, sm_count = 148, max_smem = 0;
  int nl = 0, sizes[kMaxLayers + 1] = {}, act = 0, slots = 1;
  int64_t max_batch = 0;
  int w_off[kMaxLayers] = {}, b_off[kMaxLayers] = {}, nparam = 0;
  unsigned char* fwd_img[kMaxLayers] = {};
  unsigned char* bwd_img[kMaxLayers] = {};
  // per hidden layer ONE buffer [slots][max_batch][width] (slot s = offset s * max_batch rows): the slots of a rollout
  // form one tall matrix for the weight-gradient contraction over all steps (mlpnet_wgrad_slots)
  float* hbuf[kMaxLayers] = {};               // post-activation outputs of the hidden layers
  float* dbuf[kMaxLayers] = {};               // act'(pre) of the hidden layers
  float* gbuf[kMaxLayers] = {};               // dL/d(output of hidden layer l) after the act' factor (saved deltas)
  float* h[kMaxSlots][kMaxLayers] = {};
  float* d[kMaxSlots][kMaxLayers] = {};
  float* gl[kMaxSlots][kMaxLayers] = {};
  const float* xin[kMaxSlots] = {};
  int ldx[kMaxSlots] = {};
  bool keep_deltas = false;
  const float* params = nullptr;              // flat parameters of the last pack (biases are read from here)
  float* delta[2] = {};
  float* wpart = nullptr;
  float* bpart = nullptr;
  int wchunks = 1;
  bool attr_set = false;
};

namespace {

struct DevGuard2 {
  int prev = -1;
  bool sw = false;
  explicit DevGuard2(int dev) {
    if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) sw = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DevGuard2() {
    if (sw) cudaSetDevice(prev);
  }
};

template <int EPI, bool GRAD>
int launch_gemm(gops_b200_mlpnet* net, const dense::GemmArgs& a, cudaStream_t st) {
  const size_t smem = dense::gemm_smem(a.n, GRAD);
  static bool attr_of[64] = {};        // per template instantiation and device: the widest tile (N = 128)
  bool& attr = attr_of[net->device & 63];
  if (!attr) {
    DCUDA(cudaFuncSetAttribute(dense::dense_gemm_kernel<EPI, GRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)dense::gemm_smem(dense::NCMAX, GRAD)));
    attr = true;
  }
  dim3 grid((unsigned)((a.rows + dense::TM - 1) / dense::TM), (unsigned)dense::splits_of(a.n));
  dense::dense_gemm_kernel<EPI, GRAD><<<grid, dense::NTH, smem, st>>>(a);
  gops::dense_count_launch(1);
  DCUDA(cudaGetLastError());
  (void)net;
  return 0;
}

}  // namespace

extern "C" {

int gops_b200_mlpnet_create(const int32_t* sizes, int32_t n_sizes, int32_t hidden_act, int64_t max_batch, int32_t slots,
                            gops_b200_mlpnet** out) {
  if (!sizes || !out || n_sizes < 2 || n_sizes > kMaxLayers + 1) return dense_fail("mlpnet: 1..8 layers");
  if (max_batch < 1 || slots < 1 || slots > kMaxSlots) return dense_fail("mlpnet: bad max_batch / slots");
  if (hidden_act < 0 || hidden_act > GOPS_ACT_LINEAR) return dense_fail("mlpnet: bad activation");
  for (int i = 0; i < n_sizes; ++i)
    if (sizes[i] < 1 || sizes[i] > kMaxWidth) return dense_fail("mlpnet: layer widths must be in 1..256");
  *out = nullptr;
  gops_b200_mlpnet* net = new (std::nothrow) gops_b200_mlpnet();
  if (!net) return dense_fail("out of host memory");
  cudaDeviceProp prop;
  if (cudaGetDevice(&net->device) != cudaSuccess || cudaGetDeviceProperties(&prop, net->device) != cudaSuccess) {
    delete net;
    return dense_fail("no CUDA device");
  }
  if (prop.major != 9 || prop.minor != 0) { delete net; return dense_fail("gops_b200 is built for sm_90a and needs an H100-class (sm_90) device"); }
  net->sm_count = prop.multiProcessorCount;
  net->max_smem = (int)prop.sharedMemPerBlockOptin;
  net->nl = n_sizes - 1;
  net->act = hidden_act;
  net->slots = slots;
  net->max_batch = max_batch;
  int off = 0, maxw = 0;
  for (int l = 0; l <= net->nl; ++l) { net->sizes[l] = sizes[l]; maxw = sizes[l] > maxw ? sizes[l] : maxw; }
  for (int l = 0; l < net->nl; ++l) {
    net->w_off[l] = off; off += sizes[l + 1] * sizes[l];
    net->b_off[l] = off; off += sizes[l + 1];
  }
  net->nparam = off;
  bool ok = true;
  for (int l = 0; l < net->nl && ok; ++l) {
    ok = cudaMalloc(&net->fwd_img[l], dense::packed_bytes(sizes[l + 1], sizes[l])) == cudaSuccess &&
         cudaMalloc(&net->bwd_img[l], dense::packed_bytes(sizes[l], sizes[l + 1])) == cudaSuccess;
  }
  for (int l = 0; l + 1 < net->nl && ok; ++l) {
    const size_t per = (size_t)max_batch * sizes[l + 1];
    ok = cudaMalloc(&net->hbuf[l], per * slots * sizeof(float)) == cudaSuccess &&
         cudaMalloc(&net->dbuf[l], per * slots * sizeof(float)) == cudaSuccess;
    for (int s = 0; s < slots && ok; ++s) { net->h[s][l] = net->hbuf[l] + per * s; net->d[s][l] = net->dbuf[l] + per * s; }
  }
  const int64_t tiles = (max_batch + dense::TM - 1) / dense::TM;
  net->wchunks = (int)(tiles < 32 ? tiles : 32);
  ok = ok && cudaMalloc(&net->delta[0], (size_t)max_batch * maxw * sizeof(float)) == cudaSuccess &&
       cudaMalloc(&net->delta[1], (size_t)max_batch * maxw * sizeof(float)) == cudaSuccess &&
       cudaMalloc(&net->wpart, (size_t)net->wchunks * maxw * maxw * sizeof(float)) == cudaSuccess &&
       cudaMalloc(&net->bpart, (size_t)64 * maxw * sizeof(float)) == cudaSuccess;
  if (!ok) {
    gops_b200_mlpnet_destroy(net);
    return dense_fail("mlpnet: cudaMalloc failed");
  }
  *out = net;
  return 0;
}

int gops_b200_mlpnet_destroy(gops_b200_mlpnet* net) {
  if (!net) return 0;
  DevGuard2 dg(net->device);
  for (int l = 0; l < kMaxLayers; ++l) { cudaFree(net->fwd_img[l]); cudaFree(net->bwd_img[l]); }
  for (int l = 0; l < kMaxLayers; ++l) { cudaFree(net->hbuf[l]); cudaFree(net->dbuf[l]); cudaFree(net->gbuf[l]); }
  cudaFree(net->delta[0]); cudaFree(net->delta[1]); cudaFree(net->wpart); cudaFree(net->bpart);
  (void)cudaGetLastError();
  delete net;
  return 0;
}

int64_t gops_b200_mlpnet_param_count(const gops_b200_mlpnet* net) { return net ? net->nparam : -1; }

int gops_b200_mlpnet_pack(gops_b200_mlpnet* net, const float* params, void* stream) {
  if (!net || !params) return dense_fail("null argument");
  DevGuard2 dg(net->device);
  cudaStream_t st = (cudaStream_t)stream;
  for (int l = 0; l < net->nl; ++l) {
    dense::pack_dense_kernel<<<64, 256, 0, st>>>(params + net->w_off[l], net->sizes[l + 1], net->sizes[l], net->fwd_img[l],
                                                 net->bwd_img[l]);
    gops::dense_count_launch(1);
  }
  DCUDA(cudaGetLastError());
  net->params = params;
  return 0;
}

int gops_b200_mlpnet_forward(gops_b200_mlpnet* net, const float* x, int32_t ldx, int64_t batch, int32_t slot, int32_t train,
                             float* y, int32_t ldy, void* stream) {
  if (!net || !x || !y) return dense_fail("null argument");
  if (!net->params) return dense_fail("mlpnet_forward before mlpnet_pack");
  if (batch < 1 || batch > net->max_batch || slot < 0 || slot >= net->slots) return dense_fail("mlpnet_forward: bad batch / slot");
  DevGuard2 dg(net->device);
  cudaStream_t st = (cudaStream_t)stream;
  net->xin[slot] = x;
  net->ldx[slot] = ldx;
  for (int l = 0; l < net->nl; ++l) {
    dense::GemmArgs a;
    memset(&a, 0, sizeof(a));
    a.A = l == 0 ? x : net->h[slot][l - 1];
    a.lda = l == 0 ? ldx : net->sizes[l];
    a.rows = batch;
    a.k = net->sizes[l];
    a.Bimg = net->fwd_img[l];
    a.n = net->sizes[l + 1];
    a.bias = net->params + net->b_off[l];
    a.act = net->act;
    if (l + 1 < net->nl) {
      a.Y = net->h[slot][l]; a.ldy = a.n;
      a.D = train ? net->d[slot][l] : nullptr; a.ldd = a.n;
      if (launch_gemm<dense::EPI_ACT, false>(net, a, st)) return 1;
    } else {
      a.Y = y; a.ldy = ldy;
      if (launch_gemm<dense::EPI_LINEAR, false>(net, a, st)) return 1;
    }
  }
  return 0;
}

int gops_b200_mlpnet_backward(gops_b200_mlpnet* net, const float* dy, int32_t lddy, int64_t batch, int32_t slot,
                              float* grad_flat, int32_t accumulate, float* dx, int32_t lddx, void* stream) {
  if (!net || !dy) return dense_fail("null argument");
  if (batch < 1 || batch > net->max_batch || slot < 0 || slot >= net->slots || !net->xin[slot])
    return dense_fail("mlpnet_backward: no forward pass recorded in this slot");
  DevGuard2 dg(net->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (!net->attr_set) {
    DCUDA(cudaFuncSetAttribute(dense::dense_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dense::wgrad_smem()));
    net->attr_set = true;
  }
  const float* delta = dy;
  int ldd = lddy;
  for (int l = net->nl - 1; l >= 0; --l) {
    const int n = net->sizes[l + 1], k = net->sizes[l];
    const float* in = l == 0 ? net->xin[slot] : net->h[slot][l - 1];
    const int ldin = l == 0 ? net->ldx[slot] : k;
    if (grad_flat) {
      dense::WgradArgs w;
      w.dY = delta; w.ldy = ldd; w.X = in; w.ldx = ldin; w.rows = batch; w.n = n; w.k = k;
      w.partial = net->wpart;
      const int64_t tiles = (batch + dense::TM - 1) / dense::TM;
      const int chunks = (int)(tiles < net->wchunks ? tiles : net->wchunks);
      w.tiles_per_chunk = (int)((tiles + chunks - 1) / chunks);
      w.nslots = 1; w.sy = 0; w.sx = 0;
      dim3 grid((unsigned)(((n + 127) / 128) * ((k + 127) / 128)), (unsigned)chunks);
      dense::dense_wgrad_kernel<<<grid, dense::NTH, dense::wgrad_smem(), st>>>(w);
      const long long nk = (long long)n * k;
      dense::dense_reduce_kernel<<<(unsigned)((nk + 255) / 256), 256, 0, st>>>(net->wpart, chunks, nk, grad_flat + net->w_off[l],
                                                                             accumulate);
      const int brows = 64;
      const long long rpb = (batch + brows - 1) / brows;
      dense::dense_colsum_kernel<<<dim3((unsigned)((n + 31) / 32), (unsigned)brows), dim3(32, 8), 0, st>>>(delta, ldd, batch, n,
                                                                                                     net->bpart, rpb, 1, 0);
      dense::dense_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(net->bpart, brows, n, grad_flat + net->b_off[l],
                                                                            accumulate);
      gops::dense_count_launch(4);
      DCUDA(cudaGetLastError());
    }
    if (l > 0 || dx) {
      dense::GemmArgs a;
      memset(&a, 0, sizeof(a));
      a.A = delta; a.lda = ldd; a.rows = batch; a.k = n;      // contraction over the layer's outputs
      a.Bimg = net->bwd_img[l];
      a.n = k;
      if (l > 0) {
        float* outb = net->keep_deltas ? net->gl[slot][l - 1] : net->delta[(net->nl - l) & 1];
        a.mul = net->d[slot][l - 1]; a.ldm = k;
        a.Y = outb; a.ldy = k;
        if (launch_gemm<dense::EPI_MUL, true>(net, a, st)) return 1;
        delta = outb;
        ldd = k;
      } else {
        a.Y = dx; a.ldy = lddx;
        if (launch_gemm<dense::EPI_PLAIN, true>(net, a, st)) return 1;
      }
    }
  }
  return 0;
}

/* Keep the per-layer deltas of every backward pass in its slot (memory: slots x max_batch x width per hidden layer) so
 * that mlpnet_wgrad_slots can contract the weight gradients over ALL slots at once. */
int gops_b200_mlpnet_keep_deltas(gops_b200_mlpnet* net, int32_t enable) {
  if (!net) return dense_fail("null argument");
  DevGuard2 dg(net->device);
  if (enable && !net->gbuf[0]) {
    for (int l = 0; l + 1 < net->nl; ++l) {
      const size_t per = (size_t)net->max_batch * net->sizes[l + 1];
      DCUDA(cudaMalloc(&net->gbuf[l], per * net->slots * sizeof(float)));
      for (int s = 0; s < net->slots; ++s) net->gl[s][l] = net->gbuf[l] + per * s;
    }
  }
  net->keep_deltas = enable != 0;
  return 0;
}

/* Weight gradients of `nslots` backward passes (slots slot0 .. slot0 + nslots - 1, each of `batch` rows, run with
 * grad_flat = NULL and keep_deltas on) in ONE contraction per layer.  x / dy: the first slot's network input / output
 * adjoint; slot s of them starts x_stride / dy_stride ROWS further. */
int gops_b200_mlpnet_wgrad_slots(gops_b200_mlpnet* net, int32_t slot0, int32_t nslots, int64_t batch, const float* x,
                                 int32_t ldx, int64_t x_stride, const float* dy, int32_t lddy, int64_t dy_stride,
                                 float* grad_flat, int32_t accumulate, void* stream) {
  if (!net || !x || !dy || !grad_flat) return dense_fail("null argument");
  if (!net->keep_deltas) return dense_fail("mlpnet_wgrad_slots needs mlpnet_keep_deltas(1)");
  if (slot0 < 0 || nslots < 1 || slot0 + nslots > net->slots || batch < 1 || batch > net->max_batch)
    return dense_fail("mlpnet_wgrad_slots: bad slot range / batch");
  DevGuard2 dg(net->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (!net->attr_set) {
    DCUDA(cudaFuncSetAttribute(dense::dense_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dense::wgrad_smem()));
    net->attr_set = true;
  }
  for (int l = net->nl - 1; l >= 0; --l) {
    const int n = net->sizes[l + 1], k = net->sizes[l];
    dense::WgradArgs w;
    w.dY = l == net->nl - 1 ? dy : net->gl[slot0][l]; w.ldy = l == net->nl - 1 ? lddy : n;
    w.sy = l == net->nl - 1 ? dy_stride : net->max_batch;
    w.X = l == 0 ? x : net->h[slot0][l - 1]; w.ldx = l == 0 ? ldx : k;
    w.sx = l == 0 ? x_stride : net->max_batch;
    w.rows = batch; w.n = n; w.k = k; w.nslots = nslots;
    w.partial = net->wpart;
    const int64_t tiles = (batch + dense::TM - 1) / dense::TM * nslots;
    const int chunks = (int)(tiles < net->wchunks ? tiles : net->wchunks);
    w.tiles_per_chunk = (int)((tiles + chunks - 1) / chunks);
    dim3 grid((unsigned)(((n + 127) / 128) * ((k + 127) / 128)), (unsigned)chunks);
    dense::dense_wgrad_kernel<<<grid, dense::NTH, dense::wgrad_smem(), st>>>(w);
    const long long nk = (long long)n * k;
    dense::dense_reduce_kernel<<<(unsigned)((nk + 255) / 256), 256, 0, st>>>(net->wpart, chunks, nk, grad_flat + net->w_off[l],
                                                                           accumulate);
    const int brows = 64;
    const long long rpb = (batch + brows - 1) / brows;
    dense::dense_colsum_kernel<<<dim3((unsigned)((n + 31) / 32), (unsigned)brows), dim3(32, 8), 0, st>>>(w.dY, w.ldy, batch, n,
                                                                                                   net->bpart, rpb, nslots, w.sy);
    dense::dense_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(net->bpart, brows, n, grad_flat + net->b_off[l],
                                                                          accumulate);
    gops::dense_count_launch(4);
    DCUDA(cudaGetLastError());
  }
  return 0;
}

}  // extern "C"
