// Tensor-core versions of the three dense primitives (hidden width 64 path): warp-level
// mma.sync.m16n8k8 TF32 with the 3xTF32 error-compensated split (hi*hi + hi*lo + lo*hi, FP32 accumulate).
// SURVEY F8: plain TF32 operands break the 1e-4 loss budget (8e-4 .. 5e-3), the split keeps ~2e-6.
//
// Operand roles (g = lane >> 2, t = lane & 3):
//   A (16 x 8, row)  a0 = A[g][t]      a1 = A[g+8][t]    a2 = A[g][t+4]   a3 = A[g+8][t+4]
//   B ( 8 x 8, col)  b0 = B[t][g]      b1 = B[t+4][g]
//   C (16 x 8)       c0 = C[g][2t]     c1 = C[g][2t+1]   c2 = C[g+8][2t]  c3 = C[g+8][2t+1]
// Activations are [feature][sample] tiles, so "row of A" = sample and k = feature for the layer GEMMs, and
// k = sample for the weight-gradient GEMM.  Weights are pre-split into hi / lo planes by pack_params_kernel.
#pragma once
#include "common.cuh"

namespace gops {

__device__ __forceinline__ void mma_tf32(float* d, const uint32_t* a, const uint32_t* b) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// x = hi + lo exactly; hi carries the top 11 mantissa bits (round-to-nearest, ties away: integer add of half an ulp,
// then mask -- 2 instructions; cvt.rna.tf32.f32 takes more instructions because it also screens Inf/NaN, which
// poison the result either way here), the tensor core truncates lo
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = (__float_as_uint(x) + 0x1000u) & 0xffffe000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}
// d += a * b with the three significant partial products (small ones first)
__device__ __forceinline__ void mma_3xtf32(float* d, const uint32_t* ah, const uint32_t* al, const uint32_t* bh,
                                           const uint32_t* bl) {
  mma_tf32(d, al, bh);
  mma_tf32(d, ah, bl);
  mma_tf32(d, ah, bh);
}

// Warp tiling of a [S samples x 64 features] layer output: warp w -> 16 samples (w >> 1) x 32 features (w & 1).
template <int S, int NT>
struct MmaMap {
  static_assert(NT == 4 * S, "layer-GEMM warp tiling assumes NT = 4 S (two warps per 16-sample stripe)");
  int s0, m0, g, t;
  __device__ __forceinline__ MmaMap() {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    s0 = (w >> 1) * 16;
    m0 = (w & 1) * 32;
    g = l >> 2;
    t = l & 3;
  }
};

// ---------------------------------------------------------------------------------------------
// P[m][s] = bias[m] + sum_k W[k][m] * B[k][s]      (hidden-layer pre-activations), K8 = K rounded up to 8
// (rows K..K8-1 of B and of the weight planes are zero).  Whi/Wlo: [K8][HP] planes, B: [K8][ldb].
// The fragment owners store P, then `act_pass_frag` re-reads exactly the same elements (no barrier).
// ---------------------------------------------------------------------------------------------
template <int S, int NT, int HP>
__device__ __noinline__ void gemm_fwd_mma(const float* __restrict__ Whi, const float* __restrict__ Wlo,
                                          const float* __restrict__ Bm, int ldb, int K8,
                                          const float* __restrict__ bias, float* __restrict__ P, bool swz_b) {
  constexpr int SP = S + 4;
  const MmaMap<S, NT> mp;
  float c[4][4];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const float b0 = bias[mp.m0 + 8 * nt + 2 * mp.t], b1 = bias[mp.m0 + 8 * nt + 2 * mp.t + 1];
    c[nt][0] = b0; c[nt][1] = b1; c[nt][2] = b0; c[nt][3] = b1;
  }
  // activation tiles are stored with column ^= (row & 1) << 3: rows k0+t / k0+4+t have parity t & 1
  const int sw = swz_b ? (mp.t & 1) << 3 : 0;
  const float* ap = Bm + mp.t * ldb + mp.s0 + (mp.g ^ sw);
  const float* ap8 = Bm + mp.t * ldb + mp.s0 + ((mp.g + 8) ^ sw);
  // weight planes are stored with column ^= ((row >> 2) & 1) << 2 (bank swizzle that makes BOTH this k-major read
  // and the transposed read of the backward GEMMs conflict-free): rows k0+t keep their columns, rows k0+4+t flip bit 2
  const float* wh = Whi + mp.t * HP + mp.m0 + mp.g;
  const float* wl = Wlo + mp.t * HP + mp.m0 + mp.g;
  const float* wh4 = Whi + (mp.t + 4) * HP + mp.m0 + (mp.g ^ 4);
  const float* wl4 = Wlo + (mp.t + 4) * HP + mp.m0 + (mp.g ^ 4);
#pragma unroll 2
  for (int k0 = 0; k0 < K8; k0 += 8) {
    uint32_t ah[4], al[4];
    split_tf32(ap[k0 * ldb], ah[0], al[0]);
    split_tf32(ap8[k0 * ldb], ah[1], al[1]);
    split_tf32(ap[(k0 + 4) * ldb], ah[2], al[2]);
    split_tf32(ap8[(k0 + 4) * ldb], ah[3], al[3]);
    uint32_t bh[4][2], bl[4][2];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      bh[nt][0] = __float_as_uint(wh[k0 * HP + 8 * nt]);
      bh[nt][1] = __float_as_uint(wh4[k0 * HP + 8 * nt]);
      bl[nt][0] = __float_as_uint(wl[k0 * HP + 8 * nt]);
      bl[nt][1] = __float_as_uint(wl4[k0 * HP + 8 * nt]);
    }
    // three passes over the four independent accumulators: no back-to-back dependent HMMA
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) mma_tf32(c[nt], al, bh[nt]);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) mma_tf32(c[nt], ah, bl[nt]);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) mma_tf32(c[nt], ah, bh[nt]);
  }
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    float* p = P + (mp.m0 + 8 * nt + 2 * mp.t) * SP + mp.s0 + mp.g;
    p[0] = c[nt][0]; p[SP + 8] = c[nt][1]; p[8] = c[nt][2]; p[SP] = c[nt][3];   // odd feature row: column ^ 8
  }
}

// 64-thread named barrier of the warp pair that owns one 16-sample stripe (ids 1..NT/64; id 0 = __syncthreads)
__device__ __forceinline__ void pair_sync() {
  asm volatile("bar.sync %0, 64;" ::"r"(1 + (int)(threadIdx.x >> 6)) : "memory");
}

// In-place activation with the SAME element ownership as gemm_fwd_mma's epilogue: H <- act(P), D <- act'(P).
// If W3 != nullptr the output layer is fused: every thread dots its 8 features x 2 samples with W3, the quad
// (4 lanes, 32 features) is reduced by shuffles and lane t == 0 stores the half-stripe partial
//   Zout[(4 * half + a) * ldz + s]   (half 0 also adds the bias b3[a]); consumers add the two halves.
// ACT / FULL are compile-time so that the four independent elements of an iteration interleave (a per-element
// `switch (act)` is a branch region per element and serialises their dependent chains).
template <int S, int NT, int ACT, bool FULL>
__device__ __noinline__ void act_pass_frag_t(float* __restrict__ H, float* __restrict__ D,
                                             const float* __restrict__ W3, const float* __restrict__ b3, int out,
                                             float* __restrict__ Zout, int ldz) {
  constexpr int SP = S + 4;
  const MmaMap<S, NT> mp;
  float z0[MAXA], z1[MAXA];
#pragma unroll
  for (int a = 0; a < MAXA; ++a) z0[a] = z1[a] = 0.f;
#pragma unroll 1
  for (int nt = 0; nt < 4; ++nt) {
    const int m = mp.m0 + 8 * nt + 2 * mp.t;
    const int base = m * SP + mp.s0 + mp.g;
    float* hp = H + base;
    // elements (m, g) (m+1, g) (m, g+8) (m+1, g+8); the odd row m+1 is stored with its column ^ 8
    const float p0 = hp[0], p1 = hp[SP + 8], p2 = hp[8], p3 = hp[SP];
    float h0, h1, h2, h3;
    if constexpr (FULL) {
      float d0, d1, d2, d3;
      act_fwd_grad_t<ACT>(p0, h0, d0); act_fwd_grad_t<ACT>(p1, h1, d1);
      act_fwd_grad_t<ACT>(p2, h2, d2); act_fwd_grad_t<ACT>(p3, h3, d3);
      float* dp = D + base;
      dp[0] = d0; dp[SP + 8] = d1; dp[8] = d2; dp[SP] = d3;
    } else {
      h0 = act_fwd_t<ACT>(p0); h1 = act_fwd_t<ACT>(p1); h2 = act_fwd_t<ACT>(p2); h3 = act_fwd_t<ACT>(p3);
    }
    hp[0] = h0; hp[SP + 8] = h1; hp[8] = h2; hp[SP] = h3;
    if (W3 != nullptr) {
#pragma unroll
      for (int a = 0; a < MAXA; ++a)
        if (a < out) {
          const float w0 = W3[a * 64 + m], w1 = W3[a * 64 + m + 1];
          z0[a] = fmaf(w1, h1, fmaf(w0, h0, z0[a]));     // sample s0 + g
          z1[a] = fmaf(w1, h3, fmaf(w0, h2, z1[a]));     // sample s0 + g + 8
        }
    }
  }
  if (W3 != nullptr) {
    const int half = mp.m0 >> 5;
#pragma unroll
    for (int a = 0; a < MAXA; ++a)
      if (a < out) {
        float u = z0[a], v = z1[a];
        u += __shfl_xor_sync(0xffffffffu, u, 1); v += __shfl_xor_sync(0xffffffffu, v, 1);
        u += __shfl_xor_sync(0xffffffffu, u, 2); v += __shfl_xor_sync(0xffffffffu, v, 2);
        if (mp.t == 0) {
          const float bb = half == 0 ? b3[a] : 0.f;
          Zout[(4 * half + a) * ldz + mp.s0 + mp.g] = u + bb;
          Zout[(4 * half + a) * ldz + mp.s0 + mp.g + 8] = v + bb;
        }
      }
  }
}

template <int S, int NT>
__device__ __forceinline__ void act_pass_frag(float* __restrict__ H, float* __restrict__ D, int act,
                                              const float* __restrict__ W3, const float* __restrict__ b3, int out,
                                              float* __restrict__ Zout, int ldz) {
#define GOPS_APF(A)                                                                  \
  do {                                                                               \
    if (D != nullptr) act_pass_frag_t<S, NT, A, true>(H, D, W3, b3, out, Zout, ldz); \
    else act_pass_frag_t<S, NT, A, false>(H, D, W3, b3, out, Zout, ldz);             \
  } while (0)
  GOPS_ACT_SWITCH(act, GOPS_APF)
#undef GOPS_APF
}

// D[m][s] <- D[m][s] * sum_a W3[a][m] * Zb[a][s] on the fragment-owned elements (stripe-local delta2)
template <int S, int NT>
__device__ __noinline__ void delta_from_out_frag(const float* __restrict__ W3, const float* __restrict__ Zb, int ldz,
                                                 int out, float* __restrict__ D) {
  constexpr int SP = S + 4;
  const MmaMap<S, NT> mp;
  float za[MAXA], zb[MAXA];
#pragma unroll
  for (int a = 0; a < MAXA; ++a) {
    za[a] = a < out ? Zb[a * ldz + mp.s0 + mp.g] : 0.f;
    zb[a] = a < out ? Zb[a * ldz + mp.s0 + mp.g + 8] : 0.f;
  }
#pragma unroll 1
  for (int nt = 0; nt < 4; ++nt) {
    const int m = mp.m0 + 8 * nt + 2 * mp.t;
    float* p = D + m * SP + mp.s0 + mp.g;
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
    for (int a = 0; a < MAXA; ++a)
      if (a < out) {
        const float w0 = W3[a * 64 + m], w1 = W3[a * 64 + m + 1];
        c0 = fmaf(w0, za[a], c0); c1 = fmaf(w1, za[a], c1);
        c2 = fmaf(w0, zb[a], c2); c3 = fmaf(w1, zb[a], c3);
      }
    p[0] *= c0; p[SP + 8] *= c1; p[8] *= c2; p[SP] *= c3;
  }
}

// Xb[i][s] = sum_o W1[i][o] * Dl[o][s] for i < M (stripe-local input gradient); n-tiles alternate between the
// two warps of the pair.  W1 planes: [round8(in)][HP] k-major, read transposed like gemm_bwd_mma.
template <int S, int NT, int HP>
__device__ __noinline__ void gemm_dx_mma(const float* __restrict__ Whi, const float* __restrict__ Wlo,
                                         const float* __restrict__ Dl, int M, float* __restrict__ Xb, int ldx) {
  constexpr int SP = S + 4;
  const MmaMap<S, NT> mp;
  const int half = mp.m0 >> 5, ntiles = (M + 7) >> 3;
  const int sw = (mp.t & 1) << 3;
  const float* ap = Dl + mp.t * SP + mp.s0 + (mp.g ^ sw);
  const float* ap8 = Dl + mp.t * SP + mp.s0 + ((mp.g + 8) ^ sw);
  for (int nt = half; nt < ntiles; nt += 2) {
    float c[4] = {0.f, 0.f, 0.f, 0.f};
    const int swz = mp.g & 4;
    const float* wh = Whi + (8 * nt + mp.g) * HP + (mp.t ^ swz);
    const float* wl = Wlo + (8 * nt + mp.g) * HP + (mp.t ^ swz);
    const float* wh4 = Whi + (8 * nt + mp.g) * HP + ((mp.t + 4) ^ swz);
    const float* wl4 = Wlo + (8 * nt + mp.g) * HP + ((mp.t + 4) ^ swz);
#pragma unroll 2
    for (int k0 = 0; k0 < 64; k0 += 8) {
      uint32_t ah[4], al[4], bh[2], bl[2];
      split_tf32(ap[k0 * SP], ah[0], al[0]);
      split_tf32(ap8[k0 * SP], ah[1], al[1]);
      split_tf32(ap[(k0 + 4) * SP], ah[2], al[2]);
      split_tf32(ap8[(k0 + 4) * SP], ah[3], al[3]);
      bh[0] = __float_as_uint(wh[k0]); bh[1] = __float_as_uint(wh4[k0]);
      bl[0] = __float_as_uint(wl[k0]); bl[1] = __float_as_uint(wl4[k0]);
      mma_3xtf32(c, ah, al, bh, bl);
    }
    const int i = 8 * nt + 2 * mp.t;
    float* p = Xb + i * ldx + mp.s0 + mp.g;
    if (i < M) { p[0] = c[0]; p[8] = c[2]; }
    if (i + 1 < M) { p[ldx] = c[1]; p[ldx + 8] = c[3]; }
  }
}

// ---------------------------------------------------------------------------------------------
// D[i][s] <- D[i][s] * sum_o W[i][o] * Dl[o][s]     (delta of a hidden layer, in place over D)
// The k-major weight planes [64][HP] are read transposed as the B operand: B[k = o][n = i] = W[i][o].
// ---------------------------------------------------------------------------------------------
template <int S, int NT, int HP>
__device__ __noinline__ void gemm_bwd_mma(const float* __restrict__ Whi, const float* __restrict__ Wlo,
                                          const float* __restrict__ Dl, float* __restrict__ D) {
  constexpr int SP = S + 4;
  const MmaMap<S, NT> mp;
  float c[4][4];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) c[nt][0] = c[nt][1] = c[nt][2] = c[nt][3] = 0.f;
  const int sw = (mp.t & 1) << 3;       // activation-tile swizzle of the delta rows k0+t / k0+4+t
  const float* ap = Dl + mp.t * SP + mp.s0 + (mp.g ^ sw);
  const float* ap8 = Dl + mp.t * SP + mp.s0 + ((mp.g + 8) ^ sw);
  const int swz = mp.g & 4;             // row (m0 + 8 nt + g) has bit 2 == bit 2 of g: its columns are stored ^ 4
  const float* wh = Whi + (mp.m0 + mp.g) * HP + (mp.t ^ swz);
  const float* wl = Wlo + (mp.m0 + mp.g) * HP + (mp.t ^ swz);
  const float* wh4 = Whi + (mp.m0 + mp.g) * HP + ((mp.t + 4) ^ swz);
  const float* wl4 = Wlo + (mp.m0 + mp.g) * HP + ((mp.t + 4) ^ swz);
#pragma unroll 2
  for (int k0 = 0; k0 < 64; k0 += 8) {
    uint32_t ah[4], al[4];
    split_tf32(ap[k0 * SP], ah[0], al[0]);
    split_tf32(ap8[k0 * SP], ah[1], al[1]);
    split_tf32(ap[(k0 + 4) * SP], ah[2], al[2]);
    split_tf32(ap8[(k0 + 4) * SP], ah[3], al[3]);
    uint32_t bh[4][2], bl[4][2];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      bh[nt][0] = __float_as_uint(wh[8 * nt * HP + k0]);
      bh[nt][1] = __float_as_uint(wh4[8 * nt * HP + k0]);
      bl[nt][0] = __float_as_uint(wl[8 * nt * HP + k0]);
      bl[nt][1] = __float_as_uint(wl4[8 * nt * HP + k0]);
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) mma_tf32(c[nt], al, bh[nt]);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) mma_tf32(c[nt], ah, bl[nt]);
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) mma_tf32(c[nt], ah, bh[nt]);
  }
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    float* p = D + (mp.m0 + 8 * nt + 2 * mp.t) * SP + mp.s0 + mp.g;
    p[0] *= c[nt][0]; p[SP + 8] *= c[nt][1]; p[8] *= c[nt][2]; p[SP] *= c[nt][3];
  }
}

// ---------------------------------------------------------------------------------------------
// dst[o][i] += sum_s Dl[o][s] * Xl[i][s]   for o < 64, i < RI   (weight gradient, k = sample)
// Work unit = 16 (o) x 16 (i) block (two n-tiles), units are dealt round-robin to the warps; both operands
// are activations and are split on the fly.  Rows RI .. round8(RI)-1 of Xl must be finite (they are zero).
// ---------------------------------------------------------------------------------------------
template <int S, int NT>
__device__ __noinline__ void dw_accum_mma(const float* __restrict__ Dl, int ldd, const float* __restrict__ Xl, int ldx,
                                          int RI, float* __restrict__ dst, int ld, int woff, bool swz_x) {
  constexpr int NW = NT / 32;
  const int w = ((threadIdx.x >> 5) + NW - (woff % NW)) % NW, l = threadIdx.x & 31, g = l >> 2, t = l & 3;
  const int ntiles = (RI + 7) >> 3, npairs = (ntiles + 1) >> 1;
  for (int unit = w; unit < 4 * npairs; unit += NW) {
    const int o0 = (unit & 3) * 16, i0 = (unit >> 2) * 16;
    const bool two = (i0 + 8) < 8 * ntiles;
    float c[2][4];
#pragma unroll
    for (int q = 0; q < 2; ++q) c[q][0] = c[q][1] = c[q][2] = c[q][3] = 0.f;
    // both delta rows (o0+g, o0+g+8) and X rows (i0+g, i0+8+g) have parity g & 1: activation-tile column swizzle
    const int swa = (g & 1) << 3, swb = swz_x ? swa : 0;
    const float* ap = Dl + (o0 + g) * ldd + t;
    const float* bp = Xl + (i0 + g) * ldx + t;
#pragma unroll 2
    for (int s = 0; s < S; s += 8) {
      uint32_t ah[4], al[4], bh[2], bl[2];
      const int sa = s ^ swa, sb = s ^ swb;
      split_tf32(ap[sa], ah[0], al[0]);
      split_tf32(ap[8 * ldd + sa], ah[1], al[1]);
      split_tf32(ap[sa + 4], ah[2], al[2]);
      split_tf32(ap[8 * ldd + sa + 4], ah[3], al[3]);
      uint32_t ch[2], cl[2];
      split_tf32(bp[sb], bh[0], bl[0]);
      split_tf32(bp[sb + 4], bh[1], bl[1]);
      if (two) {
        split_tf32(bp[8 * ldx + sb], ch[0], cl[0]);
        split_tf32(bp[8 * ldx + sb + 4], ch[1], cl[1]);
        mma_tf32(c[0], al, bh); mma_tf32(c[1], al, ch);
        mma_tf32(c[0], ah, bl); mma_tf32(c[1], ah, cl);
        mma_tf32(c[0], ah, bh); mma_tf32(c[1], ah, ch);
      } else {
        mma_3xtf32(c[0], ah, al, bh, bl);
      }
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = i0 + 8 * q + 2 * t;
      if (q == 1 && !two) break;
      if (i < RI) { dst[(o0 + g) * ld + i] += c[q][0]; dst[(o0 + g + 8) * ld + i] += c[q][2]; }
      if (i + 1 < RI) { dst[(o0 + g) * ld + i + 1] += c[q][1]; dst[(o0 + g + 8) * ld + i + 1] += c[q][3]; }
    }
  }
}

}  // namespace gops
