// Warpgroup tensor-core path of the 64-wide MLP (gops/apprfunc/mlp.py:73-77,103-111,327-329): batched inference with
// the two hidden-layer GEMMs on wgmma.
//
//   per 64-sample tile, one warpgroup:
//     X planes (hi | lo, chunk-major, see wgmma.cuh) <- observation rows (+ time column)
//     acc[64 x 64] (registers) = Xl.W1h^T + Xh.W1l^T + Xh.W1h^T      3xTF32, wgmma m64n64k8 .tf32
//     + b1 -> activation -> H1 planes (hi | lo)
//     acc = H1l.W2h^T + H1h.W2l^T + H1h.W2h^T
//     + b2 -> activation -> output layer (dot with W3 over the thread's columns, summed over the 4 lanes of a row)
//     -> squash -> global
//   weights: packed once per call into chunk-major hi / lo planes (pack_params_tc_kernel), staged by TMA bulk copy.
// Two warpgroups per CTA run independent tiles so that one's MMA round trip overlaps the other's epilogue.
#pragma once
#include "rollout.cuh"
#include "wgmma.cuh"

namespace gops {

struct TcNet {
  int in, obs, out, hact, time_input, k1;          // k1 = in rounded up to 8
  int g_w1, g_b1, g_w2, g_b2, g_w3, g_b3;          // torch flat offsets
  int o_w1h, o_w1l, o_w2h, o_w2l, o_w3, o_b1, o_b2, o_b3, blob;   // packed blob offsets (floats)
  int squash;
  float half[MAXA], mid[MAXA];
};

constexpr int TC_TILE = 64;       // samples per tile = wgmma M

// WGS = warpgroups per CTA (2 when the planes fit, 1 for wide observations)
inline __host__ size_t tc_infer_smem_bytes(const TcNet& T, int WGS) {
  // 128 B header (mbarrier) | weight blob | per warpgroup: X planes (2 * k1 * 64) + H1 planes (2 * 64 * 64)
  return 128 + sizeof(float) * ((size_t)T.blob + (size_t)WGS * (2 * T.k1 * TC_TILE + 2 * 64 * TC_TILE));
}

// torch-layout flat parameters -> chunk-major hi / lo planes  plane[kc][n][4] (n = output feature, kc = k / 4)
__global__ void pack_params_tc_kernel(const float* __restrict__ flat, TcNet T, float* __restrict__ blob) {
  const int n = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
  for (int i = t0; i < 64 * T.k1; i += n) {
    const int kc = i / 256, o = (i >> 2) & 63, k = 4 * kc + (i & 3);
    const float w = k < T.in ? flat[T.g_w1 + o * T.in + k] : 0.f;
    float hi, lo;
    wg::split(w, hi, lo);
    blob[T.o_w1h + i] = hi;
    blob[T.o_w1l + i] = lo;
  }
  for (int i = t0; i < 64 * 64; i += n) {
    const int kc = i / 256, o = (i >> 2) & 63, k = 4 * kc + (i & 3);
    float hi, lo;
    wg::split(flat[T.g_w2 + o * 64 + k], hi, lo);
    blob[T.o_w2h + i] = hi;
    blob[T.o_w2l + i] = lo;
  }
  for (int i = t0; i < T.out * 64; i += n) blob[T.o_w3 + i] = flat[T.g_w3 + i];
  for (int i = t0; i < 64; i += n) {
    blob[T.o_b1 + i] = flat[T.g_b1 + i];
    blob[T.o_b2 + i] = flat[T.g_b2 + i];
  }
  for (int i = t0; i < 4; i += n) blob[T.o_b3 + i] = i < T.out ? flat[T.g_b3 + i] : 0.f;
}

// The warpgroup's D = A.B^T in 3xTF32 over `ksteps` K-steps of 8 (small terms first, the dominant hi.hi last).
// A planes are chunk-major with TC_TILE rows, B planes with 64 rows.
__device__ __forceinline__ void issue_3xtf32(float* acc, const float* Ah, const float* Al, const float* Bh,
                                             const float* Bl, int ksteps) {
  constexpr uint32_t LBO_A = TC_TILE * 16, LBO_B = 64 * 16, SBO = 128;
  const uint32_t ah = smem_u32(Ah), al = smem_u32(Al), bh = smem_u32(Bh), bl = smem_u32(Bl);
  wg::fence();
  uint32_t first = 0;
  for (int ks = 0; ks < ksteps; ++ks, first = 1)
    wg::mma_tf32_n64(acc, wg::smem_desc(al + ks * 2 * LBO_A, LBO_A, SBO), wg::smem_desc(bh + ks * 2 * LBO_B, LBO_B, SBO), first);
  for (int ks = 0; ks < ksteps; ++ks)
    wg::mma_tf32_n64(acc, wg::smem_desc(ah + ks * 2 * LBO_A, LBO_A, SBO), wg::smem_desc(bl + ks * 2 * LBO_B, LBO_B, SBO), 1);
  for (int ks = 0; ks < ksteps; ++ks)
    wg::mma_tf32_n64(acc, wg::smem_desc(ah + ks * 2 * LBO_A, LBO_A, SBO), wg::smem_desc(bh + ks * 2 * LBO_B, LBO_B, SBO), 1);
  wg::commit();
  wg::wait<0>();
  wg::reg_fence<32>(acc);
}

// Hidden-layer epilogue of one thread: its 32 accumulator elements -> + bias -> activation -> hi / lo planes of the next
// GEMM's A operand (column pairs (c, c + 1) share one 16-byte chunk).  ACT is a compile-time constant.
template <int ACT>
__device__ __forceinline__ void tc_epilogue_hidden(const float* acc, const float* __restrict__ bias, float* __restrict__ Hh,
                                                   float* __restrict__ Hl, int t) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int row = wg::frag_row(t, i), col = wg::frag_col(t, i);
    float2 h, l;
    wg::split(act_fwd_t<ACT>(acc[i] + bias[col]), h.x, l.x);
    wg::split(act_fwd_t<ACT>(acc[i + 1] + bias[col + 1]), h.y, l.y);
    const int o = (col >> 2) * (TC_TILE * 4) + row * 4 + (col & 3);
    *reinterpret_cast<float2*>(Hh + o) = h;
    *reinterpret_cast<float2*>(Hl + o) = l;
  }
}
// Last hidden layer + output layer: z[q][a] = sum over this thread's columns of W3[a][j] * act(acc[j] + b2[j]) for its two
// rows (q = 0: row, q = 1: row + 8); the caller sums the four lanes of a row
template <int ACT>
__device__ __forceinline__ void tc_epilogue_out(const float* acc, const float* __restrict__ bias, const float* __restrict__ W3,
                                                int out, int t, float (*z)[MAXA]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int col = wg::frag_col(t, i), q = (i >> 1) & 1;
    const float h = act_fwd_t<ACT>(acc[i] + bias[col]);
#pragma unroll
    for (int a = 0; a < MAXA; ++a)
      if (a < out) z[q][a] = fmaf(W3[a * 64 + col], h, z[q][a]);
  }
}

template <int TC_WGS>
__global__ void __launch_bounds__(128 * TC_WGS, 1)
    mlp_infer_tc_kernel(const __grid_constant__ TcNet T, const float* __restrict__ blob, const float* __restrict__ obs,
                        long long B, float virtual_t, float* __restrict__ out) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint64_t* wbar = reinterpret_cast<uint64_t*>(smem_raw);            // weights landed
  float* W = reinterpret_cast<float*>(smem_raw + 128);
  const int tid = threadIdx.x, wgi = tid >> 7, t = tid & 127;
  float* Xh = W + T.blob + (size_t)wgi * (2 * T.k1 * TC_TILE + 2 * 64 * TC_TILE);
  float* Xl = Xh + T.k1 * TC_TILE;
  float* Hh = Xl + T.k1 * TC_TILE;
  float* Hl = Hh + 64 * TC_TILE;

  if (tid == 0) {
    mbar_init(wbar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    const uint32_t bytes = (uint32_t)T.blob * 4u;
    mbar_expect_tx(wbar, bytes);
    for (uint32_t off = 0; off < bytes; off += 32768u) {
      const uint32_t nb = bytes - off < 32768u ? bytes - off : 32768u;
      tma_bulk_g2s(reinterpret_cast<char*>(W) + off, reinterpret_cast<const char*>(blob) + off, nb, wbar);
    }
  }
  mbar_wait(wbar, 0);

  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  const long long n_tiles = (B + TC_TILE - 1) / TC_TILE;
  const int nchunk = T.k1 / 4;
  for (long long tile = (long long)blockIdx.x * TC_WGS + wgi; tile < n_tiles; tile += (long long)gridDim.x * TC_WGS) {
    // ---- observation rows -> X planes (thread = (chunk, row)); the previous tile's MMAs have retired
    for (int idx = t; idx < nchunk * TC_TILE; idx += 128) {
      const int kc = idx / TC_TILE, r = idx % TC_TILE;
      const long long s = tile * TC_TILE + r;
      float4 h, l;
      float x[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int f = 4 * kc + q;
        x[q] = s >= B ? 0.f : f < T.obs ? obs[s * T.obs + f] : (f < T.in ? virtual_t : 0.f);
      }
      wg::split(x[0], h.x, l.x); wg::split(x[1], h.y, l.y);
      wg::split(x[2], h.z, l.z); wg::split(x[3], h.w, l.w);
      reinterpret_cast<float4*>(Xh)[kc * TC_TILE + r] = h;
      reinterpret_cast<float4*>(Xl)[kc * TC_TILE + r] = l;
    }
    fence_proxy_async();            // generic-proxy smem writes -> visible to the tensor core (async proxy)
    wg::wg_sync(wgi);
    issue_3xtf32(acc, Xh, Xl, W + T.o_w1h, W + T.o_w1l, T.k1 / 8);
    // ---- layer-1 epilogue: + b1, activation, split, H1 planes
#define GOPS_TC_EPI1(A) tc_epilogue_hidden<A>(acc, W + T.o_b1, Hh, Hl, t)
    GOPS_ACT_SWITCH(T.hact, GOPS_TC_EPI1)
#undef GOPS_TC_EPI1
    fence_proxy_async();
    wg::wg_sync(wgi);
    issue_3xtf32(acc, Hh, Hl, W + T.o_w2h, W + T.o_w2l, 8);
    // ---- layer-2 epilogue + output layer
    float z[2][MAXA];
#pragma unroll
    for (int a = 0; a < MAXA; ++a) z[0][a] = z[1][a] = 0.f;
#define GOPS_TC_EPI2(A) tc_epilogue_out<A>(acc, W + T.o_b2, W + T.o_w3, T.out, t, z)
    GOPS_ACT_SWITCH(T.hact, GOPS_TC_EPI2)
#undef GOPS_TC_EPI2
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
      for (int a = 0; a < MAXA; ++a) {
        z[q][a] += __shfl_xor_sync(0xffffffffu, z[q][a], 1);
        z[q][a] += __shfl_xor_sync(0xffffffffu, z[q][a], 2);
      }
    if ((t & 3) == 0) {
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const long long s = tile * TC_TILE + wg::frag_row(t, 2 * q);
        if (s < B) {
#pragma unroll
          for (int a = 0; a < MAXA; ++a)
            if (a < T.out) {
              float y = W[T.o_b3 + a] + z[q][a];
              if (T.squash) y = __fadd_rn(__fmul_rn(T.half[a], tanhf(y)), T.mid[a]);
              out[s * T.out + a] = y;
            }
        }
      }
    }
    wg::wg_sync(wgi);               // every thread's layer-2 operand reads retired before the next tile's planes
  }
}

}  // namespace gops
