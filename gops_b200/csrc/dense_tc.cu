// C ABI of the generic wgmma dense-layer path (include/gops_b200.h, section "layer-wise MLP"): a trainable MLP of
// any depth (widths <= 256 per layer) evaluated layer by layer with the kernels of dense_tc.cuh.  Used by the wide-net
// FHADP path, DSAC, DSAC-T (paired twin-critic passes) and FHADP2; the fused rollout kernels remain the path for 64-wide
// nets with small inputs.
#include "gops_b200.h"

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <string>

#include "dense_tc.cuh"
#include "host_util.h"

using namespace gops;

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
};

namespace {

template <int EPI, bool GRAD>
int launch_gemm(gops_b200_mlpnet* net, const dense::GemmArgs& a, cudaStream_t st) {
  const size_t smem = dense::gemm_smem(a.n, GRAD);
  // the widest tile (N = 128)
  if (allow_smem((const void*)dense::dense_gemm_kernel<EPI, GRAD>, net->device, (int)dense::gemm_smem(dense::NCMAX, GRAD)))
    return 1;
  dim3 grid((unsigned)((a.rows + dense::TM - 1) / dense::TM), (unsigned)dense::splits_of(a.n));
  dense::dense_gemm_kernel<EPI, GRAD><<<grid, dense::NTH, smem, st>>>(a);
  g_launches += 1;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// One GEMM for `nn` networks of identical shape: the single-network kernel, or both networks of a pair in ONE launch
// (blockIdx.z = network, same grid x / y and tiles as the single launch).
template <int EPI, bool GRAD>
int launch_gemm_n(gops_b200_mlpnet* const* nets, int nn, const dense::GemmArgs* a, cudaStream_t st) {
  if (nn == 1) return launch_gemm<EPI, GRAD>(nets[0], a[0], st);
  const size_t smem = dense::gemm_smem(a[0].n, GRAD);
  if (allow_smem((const void*)dense::dense_gemm_pair_kernel<EPI, GRAD>, nets[0]->device,
                 (int)dense::gemm_smem(dense::NCMAX, GRAD)))
    return 1;
  dense::GemmPair p;
  p.g[0] = a[0];
  p.g[1] = a[1];
  dim3 grid((unsigned)((a[0].rows + dense::TM - 1) / dense::TM), (unsigned)dense::splits_of(a[0].n), 2u);
  dense::dense_gemm_pair_kernel<EPI, GRAD><<<grid, dense::NTH, smem, st>>>(p);
  g_launches += 1;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int set_wgrad_attr(gops_b200_mlpnet* const* nets, int nn) {
  return allow_smem(nn == 1 ? (const void*)dense::dense_wgrad_kernel : (const void*)dense::dense_wgrad_pair_kernel,
                    nets[0]->device, (int)dense::wgrad_smem());
}

// Forward pass of `nn` (1 or 2) networks of identical shape on the same input x; network i writes y[i].
int forward_n(gops_b200_mlpnet* const* nets, int nn, const float* x, int32_t ldx, int64_t batch, int32_t slot, int32_t train,
              float* const* y, int32_t ldy, cudaStream_t st) {
  for (int i = 0; i < nn; ++i) {
    nets[i]->xin[slot] = x;
    nets[i]->ldx[slot] = ldx;
  }
  const gops_b200_mlpnet* n0 = nets[0];
  for (int l = 0; l < n0->nl; ++l) {
    dense::GemmArgs a[2];
    for (int i = 0; i < nn; ++i) {
      gops_b200_mlpnet* net = nets[i];
      memset(&a[i], 0, sizeof(a[i]));
      a[i].A = l == 0 ? x : net->h[slot][l - 1];
      a[i].lda = l == 0 ? ldx : net->sizes[l];
      a[i].rows = batch;
      a[i].k = net->sizes[l];
      a[i].Bimg = net->fwd_img[l];
      a[i].n = net->sizes[l + 1];
      a[i].bias = net->params + net->b_off[l];
      a[i].act = net->act;
      if (l + 1 < net->nl) {
        a[i].Y = net->h[slot][l]; a[i].ldy = a[i].n;
        a[i].D = train ? net->d[slot][l] : nullptr; a[i].ldd = a[i].n;
      } else {
        a[i].Y = y[i]; a[i].ldy = ldy;
      }
    }
    if (l + 1 < n0->nl) {
      if (launch_gemm_n<dense::EPI_ACT, false>(nets, nn, a, st)) return 1;
    } else {
      if (launch_gemm_n<dense::EPI_LINEAR, false>(nets, nn, a, st)) return 1;
    }
  }
  return 0;
}

// Backward pass of `nn` (1 or 2) networks of identical shape: network i takes dy[i] and writes grad[i] / dx[i]
// (grad / dx are all NULL or all set).  Every weight-gradient contraction, column sum, reduction and dgrad GEMM is ONE
// launch for all networks.
int backward_n(gops_b200_mlpnet* const* nets, int nn, const float* const* dy, int32_t lddy, int64_t batch, int32_t slot,
               float* const* grad, int32_t accumulate, float* const* dx, int32_t lddx, cudaStream_t st) {
  if (set_wgrad_attr(nets, nn)) return 1;
  const gops_b200_mlpnet* n0 = nets[0];
  const float* delta[2] = {dy[0], nn > 1 ? dy[1] : nullptr};
  int ldd = lddy;
  for (int l = n0->nl - 1; l >= 0; --l) {
    const int n = n0->sizes[l + 1], k = n0->sizes[l];
    if (grad[0]) {
      const int64_t tiles = (batch + dense::TM - 1) / dense::TM;
      const int chunks = (int)(tiles < n0->wchunks ? tiles : n0->wchunks);
      dense::WgradArgs w[2];
      for (int i = 0; i < nn; ++i) {
        const gops_b200_mlpnet* net = nets[i];
        w[i].dY = delta[i]; w[i].ldy = ldd;
        w[i].X = l == 0 ? net->xin[slot] : net->h[slot][l - 1]; w[i].ldx = l == 0 ? net->ldx[slot] : k;
        w[i].rows = batch; w[i].n = n; w[i].k = k;
        w[i].partial = net->wpart;
        w[i].tiles_per_chunk = (int)((tiles + chunks - 1) / chunks);
        w[i].nslots = 1; w[i].sy = 0; w[i].sx = 0;
      }
      const long long nk = (long long)n * k;
      const int brows = 64;
      const long long rpb = (batch + brows - 1) / brows;
      const unsigned wblocks = (unsigned)(((n + 127) / 128) * ((k + 127) / 128));
      if (nn == 1) {
        gops_b200_mlpnet* net = nets[0];
        dense::dense_wgrad_kernel<<<dim3(wblocks, (unsigned)chunks), dense::NTH, dense::wgrad_smem(), st>>>(w[0]);
        dense::dense_reduce_kernel<<<(unsigned)((nk + 255) / 256), 256, 0, st>>>(net->wpart, chunks, nk,
                                                                               grad[0] + net->w_off[l], accumulate);
        dense::dense_colsum_kernel<<<dim3((unsigned)((n + 31) / 32), (unsigned)brows), dim3(32, 8), 0, st>>>(
            delta[0], ldd, batch, n, net->bpart, rpb, 1, 0);
        dense::dense_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(net->bpart, brows, n,
                                                                              grad[0] + net->b_off[l], accumulate);
      } else {
        const gops_b200_mlpnet* a = nets[0];
        const gops_b200_mlpnet* b = nets[1];
        dense::WgradPair wp;
        wp.g[0] = w[0];
        wp.g[1] = w[1];
        dense::dense_wgrad_pair_kernel<<<dim3(wblocks, (unsigned)chunks, 2u), dense::NTH, dense::wgrad_smem(), st>>>(wp);
        dense::dense_reduce_pair_kernel<<<dim3((unsigned)((nk + 255) / 256), 1u, 2u), 256, 0, st>>>(
            a->wpart, b->wpart, chunks, nk, grad[0] + a->w_off[l], grad[1] + b->w_off[l], accumulate);
        dense::dense_colsum_pair_kernel<<<dim3((unsigned)((n + 31) / 32), (unsigned)brows, 2u), dim3(32, 8), 0, st>>>(
            delta[0], delta[1], ldd, batch, n, a->bpart, b->bpart, rpb);
        dense::dense_reduce_pair_kernel<<<dim3((unsigned)((n + 255) / 256), 1u, 2u), 256, 0, st>>>(
            a->bpart, b->bpart, brows, n, grad[0] + a->b_off[l], grad[1] + b->b_off[l], accumulate);
      }
      g_launches += 4;
      CUDA_OK(cudaGetLastError());
    }
    if (l > 0 || dx[0]) {
      dense::GemmArgs a[2];
      float* outb[2] = {};
      for (int i = 0; i < nn; ++i) {
        gops_b200_mlpnet* net = nets[i];
        memset(&a[i], 0, sizeof(a[i]));
        a[i].A = delta[i]; a[i].lda = ldd; a[i].rows = batch; a[i].k = n;      // contraction over the layer's outputs
        a[i].Bimg = net->bwd_img[l];
        a[i].n = k;
        if (l > 0) {
          outb[i] = net->keep_deltas ? net->gl[slot][l - 1] : net->delta[(net->nl - l) & 1];
          a[i].mul = net->d[slot][l - 1]; a[i].ldm = k;
          a[i].Y = outb[i]; a[i].ldy = k;
        } else {
          a[i].Y = dx[i]; a[i].ldy = lddx;
        }
      }
      if (l > 0) {
        if (launch_gemm_n<dense::EPI_MUL, true>(nets, nn, a, st)) return 1;
        for (int i = 0; i < nn; ++i) delta[i] = outb[i];
        ldd = k;
      } else {
        if (launch_gemm_n<dense::EPI_PLAIN, true>(nets, nn, a, st)) return 1;
      }
    }
  }
  return 0;
}

// Two handles may run as a pair when their shapes, activation, max_batch and slots agree and both are packed on
// the same device.
int check_pair(const gops_b200_mlpnet* a, const gops_b200_mlpnet* b, const char* fn) {
  if (!a || !b) return fail(std::string(fn) + ": null network handle");
  if (a == b) return fail(std::string(fn) + ": the two networks of a pair must be distinct handles");
  bool same = a->nl == b->nl && a->act == b->act && a->max_batch == b->max_batch && a->slots == b->slots &&
              a->device == b->device;
  for (int l = 0; same && l <= a->nl; ++l) same = a->sizes[l] == b->sizes[l];
  if (!same)
    return fail(std::string(fn) + ": the two networks differ in layer sizes, activation, max_batch, slots or device");
  if (!a->params || !b->params) return fail(std::string(fn) + " before mlpnet_pack of both networks");
  return 0;
}

}  // namespace

extern "C" {

int gops_b200_mlpnet_create(const int32_t* sizes, int32_t n_sizes, int32_t hidden_act, int64_t max_batch, int32_t slots,
                            gops_b200_mlpnet** out) {
  if (!sizes || !out || n_sizes < 2 || n_sizes > kMaxLayers + 1) return fail("mlpnet: 1..8 layers");
  if (max_batch < 1 || slots < 1 || slots > kMaxSlots) return fail("mlpnet: bad max_batch / slots");
  if (hidden_act < 0 || hidden_act > GOPS_ACT_LINEAR) return fail("mlpnet: bad activation");
  for (int i = 0; i < n_sizes; ++i)
    if (sizes[i] < 1 || sizes[i] > kMaxWidth) return fail("mlpnet: layer widths must be in 1..256");
  *out = nullptr;
  gops_b200_mlpnet* net = new (std::nothrow) gops_b200_mlpnet();
  if (!net) return fail("out of host memory");
  cudaDeviceProp prop;
  if (cudaGetDevice(&net->device) != cudaSuccess || cudaGetDeviceProperties(&prop, net->device) != cudaSuccess) {
    delete net;
    return fail("no CUDA device");
  }
  if (prop.major != 9 || prop.minor != 0) { delete net; return fail("gops_b200 is built for sm_90a and needs an H100-class (sm_90) device"); }
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
    return fail("mlpnet: cudaMalloc failed");
  }
  *out = net;
  return 0;
}

int gops_b200_mlpnet_destroy(gops_b200_mlpnet* net) {
  if (!net) return 0;
  DevGuard dg(net->device);
  for (int l = 0; l < kMaxLayers; ++l) { cudaFree(net->fwd_img[l]); cudaFree(net->bwd_img[l]); }
  for (int l = 0; l < kMaxLayers; ++l) { cudaFree(net->hbuf[l]); cudaFree(net->dbuf[l]); cudaFree(net->gbuf[l]); }
  cudaFree(net->delta[0]); cudaFree(net->delta[1]); cudaFree(net->wpart); cudaFree(net->bpart);
  (void)cudaGetLastError();
  delete net;
  return 0;
}

int64_t gops_b200_mlpnet_param_count(const gops_b200_mlpnet* net) { return net ? net->nparam : -1; }

int gops_b200_mlpnet_pack(gops_b200_mlpnet* net, const float* params, void* stream) {
  if (!net || !params) return fail("null argument");
  DevGuard dg(net->device);
  cudaStream_t st = (cudaStream_t)stream;
  for (int l = 0; l < net->nl; ++l) {
    dense::pack_dense_kernel<<<64, 256, 0, st>>>(params + net->w_off[l], net->sizes[l + 1], net->sizes[l], net->fwd_img[l],
                                                 net->bwd_img[l]);
    g_launches += 1;
  }
  CUDA_OK(cudaGetLastError());
  net->params = params;
  return 0;
}

int gops_b200_mlpnet_forward(gops_b200_mlpnet* net, const float* x, int32_t ldx, int64_t batch, int32_t slot, int32_t train,
                             float* y, int32_t ldy, void* stream) {
  if (!net || !x || !y) return fail("null argument");
  if (!net->params) return fail("mlpnet_forward before mlpnet_pack");
  if (batch < 1 || batch > net->max_batch || slot < 0 || slot >= net->slots) return fail("mlpnet_forward: bad batch / slot");
  DevGuard dg(net->device);
  return forward_n(&net, 1, x, ldx, batch, slot, train, &y, ldy, (cudaStream_t)stream);
}

int gops_b200_mlpnet_backward(gops_b200_mlpnet* net, const float* dy, int32_t lddy, int64_t batch, int32_t slot,
                              float* grad_flat, int32_t accumulate, float* dx, int32_t lddx, void* stream) {
  if (!net || !dy) return fail("null argument");
  if (batch < 1 || batch > net->max_batch || slot < 0 || slot >= net->slots || !net->xin[slot])
    return fail("mlpnet_backward: no forward pass recorded in this slot");
  DevGuard dg(net->device);
  return backward_n(&net, 1, &dy, lddy, batch, slot, &grad_flat, accumulate, &dx, lddx, (cudaStream_t)stream);
}

int gops_b200_mlpnet_pair_forward(gops_b200_mlpnet* net_a, gops_b200_mlpnet* net_b, const float* x, int32_t ldx,
                                  int64_t batch, int32_t slot, int32_t train, float* y_a, float* y_b, int32_t ldy,
                                  void* stream) {
  if (check_pair(net_a, net_b, "mlpnet_pair_forward")) return 1;
  if (!x || !y_a || !y_b) return fail("mlpnet_pair_forward: null argument");
  if (batch < 1 || batch > net_a->max_batch || slot < 0 || slot >= net_a->slots)
    return fail("mlpnet_pair_forward: bad batch / slot");
  DevGuard dg(net_a->device);
  gops_b200_mlpnet* nets[2] = {net_a, net_b};
  float* ys[2] = {y_a, y_b};
  return forward_n(nets, 2, x, ldx, batch, slot, train, ys, ldy, (cudaStream_t)stream);
}

int gops_b200_mlpnet_pair_backward(gops_b200_mlpnet* net_a, gops_b200_mlpnet* net_b, const float* dy_a, const float* dy_b,
                                   int32_t lddy, int64_t batch, int32_t slot, float* grad_a, float* grad_b,
                                   int32_t accumulate, float* dx_a, float* dx_b, int32_t lddx, void* stream) {
  if (check_pair(net_a, net_b, "mlpnet_pair_backward")) return 1;
  if (!dy_a || !dy_b) return fail("mlpnet_pair_backward: null argument");
  if (!grad_a != !grad_b || !dx_a != !dx_b)
    return fail("mlpnet_pair_backward: grad_a / grad_b and dx_a / dx_b must both be set or both be NULL");
  if (batch < 1 || batch > net_a->max_batch || slot < 0 || slot >= net_a->slots || !net_a->xin[slot] || !net_b->xin[slot])
    return fail("mlpnet_pair_backward: no forward pass recorded in this slot");
  DevGuard dg(net_a->device);
  gops_b200_mlpnet* nets[2] = {net_a, net_b};
  const float* dys[2] = {dy_a, dy_b};
  float* grads[2] = {grad_a, grad_b};
  float* dxs[2] = {dx_a, dx_b};
  return backward_n(nets, 2, dys, lddy, batch, slot, grads, accumulate, dxs, lddx, (cudaStream_t)stream);
}

/* Keep the per-layer deltas of every backward pass in its slot (memory: slots x max_batch x width per hidden layer) so
 * that mlpnet_wgrad_slots can contract the weight gradients over ALL slots at once. */
int gops_b200_mlpnet_keep_deltas(gops_b200_mlpnet* net, int32_t enable) {
  if (!net) return fail("null argument");
  DevGuard dg(net->device);
  if (enable && !net->gbuf[0]) {
    for (int l = 0; l + 1 < net->nl; ++l) {
      const size_t per = (size_t)net->max_batch * net->sizes[l + 1];
      CUDA_OK(cudaMalloc(&net->gbuf[l], per * net->slots * sizeof(float)));
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
  if (!net || !x || !dy || !grad_flat) return fail("null argument");
  if (!net->keep_deltas) return fail("mlpnet_wgrad_slots needs mlpnet_keep_deltas(1)");
  if (slot0 < 0 || nslots < 1 || slot0 + nslots > net->slots || batch < 1 || batch > net->max_batch)
    return fail("mlpnet_wgrad_slots: bad slot range / batch");
  DevGuard dg(net->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (set_wgrad_attr(&net, 1)) return 1;
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
    g_launches += 4;
    CUDA_OK(cudaGetLastError());
  }
  return 0;
}

}  // extern "C"
