// Fused wgmma rollout kernel (64-wide nets, <= 16 inputs, state == obs models): one 256-thread group per CTA owning one
// 128-sample sub-tile at a time.
//
//   row = sample.  Each sample row is served by a thread PAIR (h = 0 owner in warpgroup 0, h = 1 helper in warpgroup 1,
//   both with r = thread index in the warpgroup).  The owner keeps the sample's model state and adjoint in registers
//   for the whole horizon, runs the dynamics / adjoint and writes the observation row straight into the bf16x3 operand
//   planes; owner and helper each read their 32 accumulator columns of the row back, apply bias / activation / output
//   layer and multiply their deltas.  The only other exchange is the helper's half of the output dot product and the
//   owner's output adjoint (4 KB).
//
//   Every dense product is a warpgroup MMA (wgmma, M = 64): warpgroup h computes rows [64 h, 64 h + 64) of the 128-row
//   layer / delta / input-gradient products and stores its register fragments into a row-major fp32 accumulator tile in
//   shared memory, from which the row owners read.  The reductions over samples run on the tensor core as well
//   (MN-major view of the same operand planes): warpgroup 0 forms dW2 / dW1, warpgroup 1 db2 / db1 (against a column
//   of ones), and each adds its fragment straight into the group's FP32 global partial after every horizon step.
//   dW3 / db3 are warp shuffles.
//
// Arithmetic (bars: loss 1e-4, gradient 2e-4 against the CPU oracle):
//   layer products        x . W^T      BF16x3 x BF16x3, six terms (FP32-accurate; the loss depends on these)
//   delta / input grad    delta . W    delta in TWO bf16 planes (2^-17 relative: the gradient bar is 2e-4), W in three
//   weight gradients      delta^T . h  (delta_b0 + delta_b1) . (h_b0 + h_b1): four terms, FP32 accumulation
//
// Shared memory (~206 KB of 227): weights 31.5 KB (TMA-staged) + H1 planes 48 KB, delta planes 32 KB (delta2, then delta1
// in the same buffer), observation planes 12 KB, exchange 4 KB, accumulator tiles: products 34 KB, act'(layer 1) 34 KB,
// input gradient 10 KB.
#pragma once
#include "models.cuh"
#include "mlp_tc_full.cuh"

namespace gops {
namespace tc2 {

constexpr int GT = 128;                 // rows (= samples) per sub-tile = two wgmma M = 64 halves
constexpr int GTH = 256;                // threads per group: owner warpgroup (h = 0) + helper warpgroup (h = 1)
constexpr int NG = 1;                   // groups per CTA
constexpr int NT2 = GTH * NG;
constexpr int AS = 68, XS = 20;         // row strides (floats) of the accumulator tiles (padded: conflict-free row reads)
constexpr int HPL = tcf::HPLANE, XPL = tcf::XPLANE;
constexpr int P_BYTES = 3 * HPL, Q_BYTES = 2 * HPL, XP_BYTES = 3 * XPL;
constexpr int XCH_BYTES = 2 * GT * MAXA * 4;   // helper -> owner output partials | owner -> helper output adjoints
constexpr int ACC_BYTES = GT * AS * 4, DX_BYTES = GT * XS * 4;
constexpr int GROUP_BYTES = P_BYTES + Q_BYTES + XP_BYTES + XCH_BYTES + 2 * ACC_BYTES + DX_BYTES;
constexpr int HDR_BYTES = 256;

__host__ __device__ inline size_t smem_bytes(int w_floats) {
  return HDR_BYTES + (size_t)w_floats * 4 + tcf::ONES_B + (size_t)NG * GROUP_BYTES;
}

__device__ __forceinline__ void group_sync(int g) { asm volatile("bar.sync %0, 256;" ::"r"(1 + g) : "memory"); }

// (x0, x1) -> packed bf16x2 words of two planes (low half = x0)
__device__ __forceinline__ void split2(f32x2::u64 X, uint32_t& p0, uint32_t& p1) {
  float r0, r1;
  f32x2::upk(X, r0, r1);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p0) : "f"(r1), "f"(r0));
  f32x2::upk(f32x2::fma(tcf::bf16x2_as_f32x2(p0), f32x2::rep(-1.f), X), r0, r1);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p1) : "f"(r1), "f"(r0));
}

// Per-thread view of its group's resources.  g, h, wg are warp-uniform (derived from a __shfl_sync'ed warp id).
struct Grp {
  unsigned char *P, *Q, *Xp;        // H1 planes (3), delta planes (2), observation planes (3)
  float *zp, *zb;                   // exchange: helper -> owner output partials [128][MAXA]; owner -> helper adjoints
  float *A, *D1, *DX;               // accumulator tiles: products [128][AS], act'(layer 1) [128][AS], input gradient [128][XS]
  const unsigned char* ones;
  int g, h, wg, r;                  // group, half (0 owner / 1 helper), warp in group, row (= sample of the sub-tile)
  // staged weights of the network in use
  const unsigned char *W1, *W2;
  const float *W3, *b1, *b2, *b3;
};

__device__ __forceinline__ void bind(Grp& G, const float* Wsm, const NetL& L) {
  G.W1 = reinterpret_cast<const unsigned char*>(Wsm + L.o_w1);
  G.W2 = reinterpret_cast<const unsigned char*>(Wsm + L.o_w2);
  G.W3 = Wsm + L.o_w3; G.b1 = Wsm + L.o_b1; G.b2 = Wsm + L.o_b2; G.b3 = Wsm + L.o_b3;
}
// make this thread's shared-memory writes visible to the tensor core, then meet the group
__device__ __forceinline__ void publish(const Grp& G) {
  fence_proxy_async();
  group_sync(G.g);
}

// A . B^T with the six BF16x3 terms (small ones first), KS steps of K = 16; A K-major (this warpgroup's 64 rows)
template <int N, int TB, int KS>
__device__ __forceinline__ void mma6(float* d, const tcf::Op& A, const tcf::Op& B) {
  using namespace tcf;
  const uint64_t a0 = dsc(A, 0), a1 = dsc(A, 1), a2 = dsc(A, 2), b0 = dsc(B, 0), b1 = dsc(B, 1), b2 = dsc(B, 2);
  const uint64_t ka = A.kadv >> 4, kb = B.kadv >> 4;
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16<N, 0, TB>(d, a2 + ks * ka, b0 + ks * kb, ks > 0 ? 1u : 0u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16<N, 0, TB>(d, a0 + ks * ka, b2 + ks * kb, 1u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16<N, 0, TB>(d, a1 + ks * ka, b1 + ks * kb, 1u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16<N, 0, TB>(d, a1 + ks * ka, b0 + ks * kb, 1u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16<N, 0, TB>(d, a0 + ks * ka, b1 + ks * kb, 1u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16<N, 0, TB>(d, a0 + ks * ka, b0 + ks * kb, 1u);
}
// delta (2 planes, K-major A) x W (MN-major B): a1b0, a0b1, a0b0 -- small terms first.  The dropped terms (a1b1, a0b2)
// are 2^-17 relative, the size of delta's own two-plane truncation.
template <int N, int KS>
__device__ __forceinline__ void mma_dw(float* d, const tcf::Op& A, const tcf::Op& B) {
  using namespace tcf;
  const uint64_t a0 = dsc(A, 0), a1 = dsc(A, 1), b0 = dsc(B, 0), b1 = dsc(B, 1);
  const uint64_t ka = A.kadv >> 4, kb = B.kadv >> 4;
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16<N, 0, 1>(d, a1 + ks * ka, b0 + ks * kb, ks > 0 ? 1u : 0u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16<N, 0, 1>(d, a0 + ks * ka, b1 + ks * kb, 1u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16<N, 0, 1>(d, a0 + ks * ka, b0 + ks * kb, 1u);
}
// weight gradient over the sub-tile's 128 samples: D = (A_b0 + A_b1)^T . (B_b0 + .. + B_b{BP-1}), both MN-major
template <int N, int BP>
__device__ __forceinline__ void mma_wgrad(float* d, const tcf::Op& A, const tcf::Op& B) {
  using namespace tcf;
  const uint64_t ka = A.kadv >> 4, kb = B.kadv >> 4;
  uint32_t acc = 0u;
#pragma unroll
  for (int p = BP - 1; p >= 0; --p)
#pragma unroll
    for (int q = 1; q >= 0; --q) {
      const uint64_t a = dsc(A, q), b = dsc(B, p);
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) { wg::mma_bf16<N, 1, 1>(d, a + ks * ka, b + ks * kb, acc); acc = 1u; }
    }
}
// this warpgroup's fragment of a 128-row product -> rows [64 h, 64 h + 64) of a row-major tile
template <int N>
__device__ __forceinline__ void store_frag(const Grp& G, float* dst, int ld, const float* d) {
#pragma unroll
  for (int i = 0; i < N / 2; i += 2)
    *reinterpret_cast<float2*>(dst + (64 * G.h + wg::frag_row(G.r, i)) * ld + wg::frag_col(G.r, i)) = make_float2(d[i], d[i + 1]);
}
// this warpgroup's fragment of a [64 output rows][N] weight gradient added into the FP32 partial (row stride ld,
// columns < ncols)
template <int N>
__device__ __forceinline__ void add_frag(float* __restrict__ dst, int ld, int ncols, const float* d, int r) {
#pragma unroll
  for (int i = 0; i < N / 2; ++i) {
    const int row = wg::frag_row(r, i), col = wg::frag_col(r, i);
    if (col < ncols) dst[row * ld + col] += d[i];
  }
}
// the group's 128-row product A . B^T (A = k_act(...) planes, six terms) into the product tile; ends with the group
// barrier: the results are visible and every wgmma operand read has retired
template <int KS>
__device__ __forceinline__ void layer_product(const Grp& G, const tcf::Op& Ain, const tcf::Op& B) {
  tcf::Op A = Ain;
  A.base += 1024u * G.h;                          // + 8 row groups of 128 B
  float d[32];
  wg::fence();
  mma6<64, 0, KS>(d, A, B);
  wg::commit();
  wg::wait<0>();
  store_frag<64>(G, G.A, AS, d);
  group_sync(G.g);
}
__device__ __forceinline__ void read16(const float* src, float* v) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 x = reinterpret_cast<const float4*>(src)[q];
    v[4 * q] = x.x; v[4 * q + 1] = x.y; v[4 * q + 2] = x.z; v[4 * q + 3] = x.w;
  }
}

// owner: this row's input (K1 = 16 values, zero padded) -> the three observation planes.  nch = 1: the inputs fit the
// first 8-feature chunk (idpendulum: 6 + time), the second chunk was zeroed once at kernel start.
__device__ __forceinline__ void write_x_row(const Grp& G, const float* x, int nch) {
  using namespace tcf;
#pragma unroll
  for (int ch = 0; ch < 2; ++ch) {
    if (ch >= nch) break;
    uint32_t w[3][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) split3(x[8 * ch + 2 * i], x[8 * ch + 2 * i + 1], w[0][i], w[1][i], w[2][i]);
#pragma unroll
    for (int p = 0; p < 3; ++p)
      *reinterpret_cast<uint4*>(G.Xp + p * XPL + (ch * 128 + G.r) * 16) = make_uint4(w[p][0], w[p][1], w[p][2], w[p][3]);
  }
}

// layer 1, first half: observation planes . W1^T into the product tile
template <int NS>
__device__ __forceinline__ void layer1_issue(Grp& G, const NetL& L, const float* st, float vt) {
  using namespace tcf;
  if (G.h == 0) {
    float x[16];
#pragma unroll
    for (int f = 0; f < 16; ++f) x[f] = (f < NS && f < L.obs) ? st[f < NS ? f : 0] : 0.f;
    if (L.time_input) {
#pragma unroll
      for (int f = 0; f < 16; ++f)
        if (f == L.in - 1) x[f] = vt;
    }
    write_x_row(G, x, L.in <= 8 ? 1 : 2);
  }
  publish(G);
  layer_product<1>(G, k_act(G.Xp, XPL), k_w(G.W1, W1PLANE));
}
// AF: hidden activation fixed at compile time (>= 0), or -1 = dispatch on the runtime id.  With the activation fixed (the
// headline configurations use GELU) the other six epilogue variants are not compiled in.
#define GOPS_TC2_ACT_SWITCH(AF, act, M)     \
  if constexpr ((AF) >= 0) { M(AF); }       \
  else { GOPS_ACT_SWITCH(act, M) }

// layer 1, second half: + b1, activation -> this thread's columns of the H1 planes (FULL: act' into the D1 tile).
// [lo, hi): the 16-column blocks of the row this thread converts (forward sweep: owner 0-1, helper 2-3; reverse sweep:
// the helper takes all four while the owner runs the adjoint of the dynamics).
template <bool FULL, int AF>
__device__ __forceinline__ void layer1_finish(Grp& G, const NetL& L, int lo, int hi) {
  using namespace tcf;
#pragma unroll 1
  for (int c16 = lo; c16 < hi; ++c16) {
    float v[16], d[16];
    read16(G.A + G.r * AS + 16 * c16, v);
    const float* bias = G.b1 + 16 * c16;
#define GOPS_TC2_A1(A)                                                      \
  _Pragma("unroll") for (int e = 0; e < 16; e += 2) {                                         \
    const f32x2::u64 pre = f32x2::add(f32x2::pk(v[e], v[e + 1]), f32x2::ld(bias + e));       \
    if constexpr (FULL) act_fwd_grad_pair_t<A>(pre, v[e], v[e + 1], d[e], d[e + 1]);          \
    else act_fwd_pair_t<A>(pre, v[e], v[e + 1]);                                              \
  }
    GOPS_TC2_ACT_SWITCH(AF, L.hact, GOPS_TC2_A1)
#undef GOPS_TC2_A1
    store16(G.P, HPL, c16, G.r, v);
    if constexpr (FULL) {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        reinterpret_cast<float4*>(G.D1 + G.r * AS + 16 * c16)[q] = make_float4(d[4 * q], d[4 * q + 1], d[4 * q + 2], d[4 * q + 3]);
    }
  }
}

// layer 2 + output layer, forward only: the owner gets z[a] = b3[a] + W3[a] . act(H1 . W2^T + b2)
template <int AF>
__device__ __forceinline__ void layer2_out(Grp& G, const NetL& L, float* z) {
  using namespace tcf;
  publish(G);
  layer_product<4>(G, k_act(G.P, HPL), k_w(G.W2, W2PLANE));
  float zp[MAXA];
#pragma unroll
  for (int a = 0; a < MAXA; ++a) zp[a] = 0.f;
#pragma unroll 1
  for (int cb = 0; cb < 2; ++cb) {
    const int c16 = 2 * G.h + cb;
    float v[16];
    read16(G.A + G.r * AS + 16 * c16, v);
    const float* bias = G.b2 + 16 * c16;
#define GOPS_TC2_A2(A)                               \
  _Pragma("unroll") for (int e = 0; e < 16; e += 2)  \
      act_fwd_pair_t<A>(f32x2::add(f32x2::pk(v[e], v[e + 1]), f32x2::ld(bias + e)), v[e], v[e + 1]);
    GOPS_TC2_ACT_SWITCH(AF, L.hact, GOPS_TC2_A2)
#undef GOPS_TC2_A2
#pragma unroll
    for (int a = 0; a < MAXA; ++a)
      if (a < L.out) {
        const float* w = G.W3 + a * 64 + 16 * c16;
        f32x2::u64 S = f32x2::rep(0.f);           // (even, odd) column partial sums
#pragma unroll
        for (int e = 0; e < 16; e += 2) S = f32x2::fma(f32x2::ld(w + e), f32x2::pk(v[e], v[e + 1]), S);
        float s0, s1;
        f32x2::upk(S, s0, s1);
        zp[a] += s0 + s1;
      }
  }
  if (G.h == 1) {
#pragma unroll
    for (int a = 0; a < MAXA; ++a)
      if (a < L.out) G.zp[G.r * MAXA + a] = zp[a];
  }
  group_sync(G.g);
  if (G.h == 0) {
#pragma unroll
    for (int a = 0; a < MAXA; ++a) z[a] = a < L.out ? G.b3[a] + (zp[a] + G.zp[G.r * MAXA + a]) : 0.f;
  }
}

// Per-thread accumulators of the output-layer gradients: after the transposing warp reduction lane l holds the warp's
// column sum of column 32 h + 16 q + col16(l) in slot q; they are combined across warps once, at the end of the kernel.
struct Acc3 {
  float w0[MAXA], w1[MAXA];
  float b[MAXA];
};

// layer 2 recompute fused with the start of the backward pass: z for the owner (WANT_Z), dW3 / db3 partial sums, and
// delta2 = (W3^T zbar) * act'(pre2) -> this thread's 32 columns of the two delta planes.
// zbar: the owner's output adjoint of its row (the helper receives it through shared memory).
template <bool WANT_DW, bool WANT_Z, int AF>
__device__ __forceinline__ void layer2_back(Grp& G, const NetL& L, const float* zbar, float* z, Acc3& acc3) {
  using namespace tcf;
  if (G.h == 0) {
#pragma unroll
    for (int a = 0; a < MAXA; ++a)
      if (a < L.out) G.zb[G.r * MAXA + a] = zbar[a];
  }
  publish(G);
  layer_product<4>(G, k_act(G.P, HPL), k_w(G.W2, W2PLANE));
  float zb[MAXA];
#pragma unroll
  for (int a = 0; a < MAXA; ++a) zb[a] = a < L.out ? G.zb[G.r * MAXA + a] : 0.f;
  const int lane = G.r & 31;
  float zp[MAXA];
#pragma unroll
  for (int a = 0; a < MAXA; ++a) zp[a] = 0.f;
#pragma unroll 1
  for (int cb = 0; cb < 2; ++cb) {
    const int c16 = 2 * G.h + cb;
    float v[16], d[16];
    read16(G.A + G.r * AS + 16 * c16, v);
    const float* bias = G.b2 + 16 * c16;
#define GOPS_TC2_A3(A)                               \
  _Pragma("unroll") for (int e = 0; e < 16; e += 2)  \
      act_fwd_grad_pair_t<A>(f32x2::add(f32x2::pk(v[e], v[e + 1]), f32x2::ld(bias + e)), v[e], v[e + 1], d[e], d[e + 1]);
    GOPS_TC2_ACT_SWITCH(AF, L.hact, GOPS_TC2_A3)
#undef GOPS_TC2_A3
    const float* w3 = G.W3 + 16 * c16;
    if constexpr (WANT_Z) {
#pragma unroll
      for (int a = 0; a < MAXA; ++a)
        if (a < L.out) {
          f32x2::u64 S = f32x2::rep(0.f);
#pragma unroll
          for (int e = 0; e < 16; e += 2) S = f32x2::fma(f32x2::ld(w3 + a * 64 + e), f32x2::pk(v[e], v[e + 1]), S);
          float s0, s1;
          f32x2::upk(S, s0, s1);
          zp[a] += s0 + s1;
        }
    }
    if constexpr (WANT_DW) {
#pragma unroll
      for (int a = 0; a < MAXA; ++a)
        if (a < L.out) {
          float t[16];
#pragma unroll
          for (int e = 0; e < 16; e += 2) f32x2::upk(f32x2::mul(f32x2::rep(zb[a]), f32x2::pk(v[e], v[e + 1])), t[e], t[e + 1]);
          warp_reduce16(t, lane);
          acc3.w0[a] += cb == 0 ? t[0] : 0.f;
          acc3.w1[a] += cb == 0 ? 0.f : t[0];
        }
    }
    f32x2::u64 D2[8];                              // delta2 pairs = act'(pre2) * (W3^T zbar)
#pragma unroll
    for (int e = 0; e < 16; e += 2) {
      f32x2::u64 gs = f32x2::rep(0.f);
#pragma unroll
      for (int a = 0; a < MAXA; ++a)
        if (a < L.out) gs = f32x2::fma(f32x2::ld(w3 + a * 64 + e), f32x2::rep(zb[a]), gs);
      D2[e / 2] = f32x2::mul(f32x2::pk(d[e], d[e + 1]), gs);
    }
    // two delta planes: chunks 2 c16, 2 c16 + 1 of row r
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      uint32_t w0[4], w1[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) split2(D2[4 * c + i], w0[i], w1[i]);
      *reinterpret_cast<uint4*>(G.Q + ((2 * c16 + c) * 128 + G.r) * 16) = make_uint4(w0[0], w0[1], w0[2], w0[3]);
      *reinterpret_cast<uint4*>(G.Q + HPL + ((2 * c16 + c) * 128 + G.r) * 16) = make_uint4(w1[0], w1[1], w1[2], w1[3]);
    }
  }
  if constexpr (WANT_DW) {
    if (G.h == 0) {
#pragma unroll
      for (int a = 0; a < MAXA; ++a)
        if (a < L.out) {
          float sz = zb[a];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) sz += __shfl_xor_sync(0xffffffffu, sz, o);
          acc3.b[a] += sz;
        }
    }
  }
  if constexpr (WANT_Z) {
    if (G.h == 1) {
#pragma unroll
      for (int a = 0; a < MAXA; ++a)
        if (a < L.out) G.zp[G.r * MAXA + a] = zp[a];
    }
    group_sync(G.g);
    if (G.h == 0) {
#pragma unroll
      for (int a = 0; a < MAXA; ++a) z[a] = a < L.out ? G.b3[a] + (zp[a] + G.zp[G.r * MAXA + a]) : 0.f;
    }
  }
}

// delta2 planes -> delta1 = (delta2 . W2) * act'(pre1) (same planes, once the readers of delta2 retired) -> input
// gradient rows in the DX tile (want_dx; the owner reads them with collect_dx) and, WANT_DW, the weight gradients of both
// layers added into the group's partial `part`: warpgroup 0 forms dW2 / dW1, warpgroup 1 db2 / db1.
template <bool WANT_DW>
__device__ __forceinline__ void backprop(Grp& G, const NetL& L, bool want_dx, float* __restrict__ part) {
  using namespace tcf;
  publish(G);
  {
    Op A = k_act(G.Q, HPL);
    A.base += 1024u * G.h;
    float d[32];
    wg::fence();
    mma_dw<64, 4>(d, A, mn_w(G.W2, W2PLANE));
    wg::commit();
    if constexpr (WANT_DW) {
      const Op Ad = mn_act(G.Q, HPL);
      if (G.h == 0) {
        float w[32];
        wg::fence();
        mma_wgrad<64, 2>(w, Ad, mn_act(G.P, HPL));
        wg::commit();
        wg::wait<0>();
        wg::reg_fence<32>(w);
        add_frag<64>(part + L.g_w2, 64, 64, w, G.r);
      } else {
        float w[8];
        wg::fence();
        mma_wgrad<16, 1>(w, Ad, Op{smem_u32(G.ones), 0u, 128u, 256u, 0u});
        wg::commit();
        wg::wait<0>();
        wg::reg_fence<8>(w);
        add_frag<16>(part + L.g_b2, 1, 1, w, G.r);
      }
    }
    wg::wait<0>();
    wg::reg_fence<32>(d);
    store_frag<64>(G, G.A, AS, d);
  }
  group_sync(G.g);                               // delta2 . W2 visible; every reader of delta2 / H1 has retired
  if (!WANT_DW && !want_dx) return;
  {
    float ra[32], rb[32];
    read16(G.A + G.r * AS + 32 * G.h, ra);
    read16(G.A + G.r * AS + 32 * G.h + 16, ra + 16);
    read16(G.D1 + G.r * AS + 32 * G.h, rb);
    read16(G.D1 + G.r * AS + 32 * G.h + 16, rb + 16);
    uint32_t w0[16], w1[16];                     // delta1 planes of this thread's 32 columns
#pragma unroll
    for (int i = 0; i < 16; ++i)
      split2(f32x2::mul(f32x2::pk(ra[2 * i], ra[2 * i + 1]), f32x2::pk(rb[2 * i], rb[2 * i + 1])), w0[i], w1[i]);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      *reinterpret_cast<uint4*>(G.Q + ((4 * G.h + c) * 128 + G.r) * 16) = make_uint4(w0[4 * c], w0[4 * c + 1], w0[4 * c + 2], w0[4 * c + 3]);
      *reinterpret_cast<uint4*>(G.Q + HPL + ((4 * G.h + c) * 128 + G.r) * 16) = make_uint4(w1[4 * c], w1[4 * c + 1], w1[4 * c + 2], w1[4 * c + 3]);
    }
  }
  publish(G);
  if (want_dx) {
    Op A = k_act(G.Q, HPL);
    A.base += 1024u * G.h;
    float d[8];
    wg::fence();
    mma_dw<16, 4>(d, A, mn_w(G.W1, W1PLANE));
    wg::commit();
    wg::wait<0>();
    wg::reg_fence<8>(d);
    store_frag<16>(G, G.DX, XS, d);
  }
  if constexpr (WANT_DW) {
    const Op Ad = mn_act(G.Q, HPL);
    float w[8];
    wg::fence();
    if (G.h == 0) mma_wgrad<16, 2>(w, Ad, mn_act(G.Xp, XPL));
    else mma_wgrad<16, 1>(w, Ad, Op{smem_u32(G.ones), 0u, 128u, 256u, 0u});
    wg::commit();
    wg::wait<0>();
    wg::reg_fence<8>(w);
    if (G.h == 0) add_frag<16>(part + L.g_w1, L.in, L.in, w, G.r);
    else add_frag<16>(part + L.g_b1, 1, 1, w, G.r);
  }
  group_sync(G.g);                               // input gradient visible; delta1 / X planes free
}

// owner half: the input gradient of the last backprop(..., want_dx = true)
__device__ __forceinline__ void collect_dx(const Grp& G, float* dx) {
  float v[16];
  read16(G.DX + G.r * XS, v);
#pragma unroll
  for (int f = 0; f < 16; ++f) dx[f] = v[f];
}

}  // namespace tc2

// ---------------------------------------------------------------------------------------------------------------
// The kernel.  grid = min(#SM, #sub-tiles) CTAs of 256 threads, one CTA per SM (shared memory).
// Slot s = NG * blockIdx.x + group owns the contiguous sub-tile range [NSUB s / slots, NSUB (s + 1) / slots).
// INFADP swaps weight blobs (policy <-> v_target <-> v) through the one staging buffer: those swap points are CTA-wide
// barriers, so with NG > 1 all groups run the same number of (possibly empty) sub-tile iterations.
// ---------------------------------------------------------------------------------------------------------------
template <class M, int ALG, int AF = -1>
__global__ void __launch_bounds__(tc2::NT2, 1) rollout_tc2_kernel(const __grid_constant__ KParams p) {
  using namespace tc2;
  static_assert(M::KIND == 0, "wgmma rollout kernel: state == obs models");
  constexpr int NS = M::NS, alg = ALG;
  extern __shared__ __align__(16) float smem[];
  unsigned char* sm = reinterpret_cast<unsigned char*>(smem);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm);           // [0] weights landed
  float* Wsm = reinterpret_cast<float*>(sm + HDR_BYTES);
  unsigned char* ones = sm + HDR_BYTES + (size_t)p.w_floats * 4;
  unsigned char* gbase = ones + tcf::ONES_B;

  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);      // warp-uniform by construction
  Grp G;
  G.g = warp >> 3;
  G.wg = warp & 7;
  G.h = G.wg >> 2;
  G.r = 32 * (G.wg & 3) + (tid & 31);
  G.P = gbase + G.g * GROUP_BYTES;
  G.Q = G.P + P_BYTES;
  G.Xp = G.Q + Q_BYTES;
  G.zp = reinterpret_cast<float*>(G.Xp + XP_BYTES);
  G.zb = G.zp + GT * MAXA;
  G.A = reinterpret_cast<float*>(G.Xp + XP_BYTES + XCH_BYTES);
  G.D1 = G.A + GT * AS;
  G.DX = G.D1 + GT * AS;
  G.ones = ones;
  const bool own = G.h == 0;

  if (tid == 0) {
    mbar_init(bars, 1);
    fence_mbar_init();
  }
  if (tid < 256) {  // `ones`: [2 mn-groups][16 rows][8 bf16], feature 0 = 1.0
    uint16_t* o16 = reinterpret_cast<uint16_t*>(ones);
    o16[tid] = (tid < 128 && (tid & 7) == 0) ? (uint16_t)0x3f80 : (uint16_t)0;
  }
  uint32_t wphase = 0;
  auto stage = [&](const float* gsrc, int floats) {      // CTA-wide: both groups call it at the same program points
    __syncthreads();
    if (tid == 0) {
      fence_proxy_async();
      const uint32_t bytes = (uint32_t)floats * 4u;
      mbar_expect_tx(bars, bytes);
      for (uint32_t off = 0; off < bytes; off += 32768u) {
        const uint32_t n = bytes - off < 32768u ? bytes - off : 32768u;
        tma_bulk_g2s(reinterpret_cast<char*>(Wsm) + off, reinterpret_cast<const char*>(gsrc) + off, n, bars);
      }
    }
    mbar_wait(bars, wphase);
    wphase ^= 1u;
  };

  const NetL& P = p.pol;
  const NetL& V = p.val;
  const int H = p.horizon, obs_dim = P.obs, TCH = p.tape_ch;
  const long long B = p.batch;
  const int slot = blockIdx.x * NG + G.g, slots = gridDim.x * NG;
  float* part = p.partial + (size_t)slot * p.part_stride;
  for (int i = G.h * GT + G.r; i < p.part_stride; i += GTH) part[i] = 0.f;
  float* tape = p.tape + (size_t)slot * (size_t)H * TCH * GT;
  Acc3 acc3;
#pragma unroll
  for (int a = 0; a < MAXA; ++a) acc3.w0[a] = acc3.w1[a] = acc3.b[a] = 0.f;
  float loss_acc = 0.f, vmean_acc = 0.f, done_acc = 0.f;

  for (int i = G.h * GT + G.r; i < XP_BYTES / 16; i += GTH) reinterpret_cast<uint4*>(G.Xp)[i] = make_uint4(0u, 0u, 0u, 0u);
  stage(p.blob_pol, P.blob);      // (its leading CTA barrier also publishes the zeroed planes)
  bind(G, Wsm, P);

  const long long nsub = (B + GT - 1) / GT;
  const long long s0 = nsub * slot / slots, s1 = nsub * (slot + 1) / slots;
  // INFADP: equal iteration counts for both groups of the CTA (stage() is a CTA-wide barrier)
  long long iters = s1 - s0;
  if (NG > 1 && (alg == ALG_PIM || alg == ALG_PEV)) {
    const long long o0 = nsub * (slot ^ 1) / slots, o1 = nsub * ((slot ^ 1) + 1) / slots;
    iters = (o1 - o0) > iters ? (o1 - o0) : iters;
  }

  for (long long it = 0; it < iters; ++it) {
    const long long sub = s0 + it;
    const bool have = sub < s1;                   // false: idle iteration that only takes part in the blob swaps
    const long long gs = sub * GT + G.r;
    const bool valid = have && gs < B;
    float st[NS];
#pragma unroll
    for (int f = 0; f < NS; ++f) st[f] = (own && valid && f < obs_dim) ? p.obs[gs * obs_dim + f] : 0.f;
    bool dn = (own && valid) ? (p.done[gs] != 0.f) : true;
    float vacc = 0.f;

    // ================================ forward sweep ================================
    if (have) {
      for (int k = 0; k < H; ++k) {
        if (own) {
          if (alg == ALG_FHADP || alg == ALG_PIM) {
#pragma unroll
            for (int f = 0; f < NS; ++f) tape[(k * TCH + f) * GT + G.r] = st[f];
            tape[(k * TCH + NS) * GT + G.r] = dn ? 1.f : 0.f;
          }
        }
        float z[MAXA];
        layer1_issue<NS>(G, P, st, (float)(k + 1));
        layer1_finish<false, AF>(G, P, 2 * G.h, 2 * G.h + 2);
        layer2_out<AF>(G, P, z);
        if (own) {
          float a[MAXA], g[MAXA], apol[MAXA];
          if (alg == ALG_FHADP || alg == ALG_PIM) {
#pragma unroll
            for (int j = 0; j < MAXA; ++j)
              if (j < P.out) tape[(k * TCH + NS + 1 + j) * GT + G.r] = z[j];
          }
          process_action(p, P.out, z, a, g, apol);
          const bool active = valid && (p.mask_at_done ? !dn : true);
          float r = 0.f;
          if (valid) {
            float in[NS];
#pragma unroll
            for (int f = 0; f < NS; ++f) in[f] = (p.obs_scaling && f < obs_dim) ? st[f] / p.osc[f] - p.osh[f] : st[f];
            if (active) {
              bool md = false;
              const int reps = p.repeat_num > 0 ? p.repeat_num : 1;
              float rsum = 0.f, rj = 0.f;
              for (int j = 0; j < reps; ++j) {
                M::step(p, in, a, rj, md);
                rsum += rj;
              }
              r = (p.repeat_num > 0 && p.sum_reward) ? rsum : rj;
              dn = md;
            }
#pragma unroll
            for (int f = 0; f < NS; ++f) {
              float o = (p.obs_scaling && f < obs_dim) ? (in[f] + p.osh[f]) * p.osc[f] : in[f];
              if (p.clip_obs) o = fminf(fmaxf(o, p.obs_low[f]), p.obs_high[f]);
              st[f] = o;
            }
            if (p.reward_shaping) r = (r + p.reward_shift) * p.reward_scale;
            vacc += r * p.gpow[k];
          }
          if (alg == ALG_TRACE && valid) {
            const size_t row = (size_t)k * B + gs;
            if (p.tr_obs)
              for (int f = 0; f < obs_dim; ++f) p.tr_obs[row * obs_dim + f] = st[f];
            if (p.tr_act)
              for (int j = 0; j < P.out; ++j) p.tr_act[row * P.out + j] = apol[j];
            if (p.tr_rew) p.tr_rew[row] = r;
            if (p.tr_done) p.tr_done[row] = dn ? 1.f : 0.f;
          }
        }
      }
      if (own && valid && dn) done_acc += 1.f;
    }
    if (alg == ALG_TRACE) continue;

    // ============================ terminal value (INFADP) ============================
    float lam[NS];
#pragma unroll
    for (int f = 0; f < NS; ++f) lam[f] = 0.f;
    if (alg != ALG_FHADP) {
      stage(p.blob_vtg, V.blob);
      bind(G, Wsm, V);
      if (have) {
        const float gn = p.gpow[H];
        const bool term = own && valid && !dn;
        float zv[MAXA], zb[MAXA], dx[16];
#pragma unroll
        for (int j = 0; j < MAXA; ++j) zb[j] = zv[j] = 0.f;
        if (alg == ALG_PIM) {
          zb[0] = term ? -gn * p.inv_B : 0.f;
          layer1_issue<NS>(G, V, st, 0.f);
          layer1_finish<true, AF>(G, V, 2 * G.h, 2 * G.h + 2);
          layer2_back<false, true, AF>(G, V, zb, zv, acc3);
          backprop<false>(G, V, true, part);
          collect_dx(G, dx);
          if (term) {
#pragma unroll
            for (int f = 0; f < NS; ++f)
              if (f < obs_dim) lam[f] = dx[f];
          }
        } else {
          layer1_issue<NS>(G, V, st, 0.f);
          layer1_finish<false, AF>(G, V, 2 * G.h, 2 * G.h + 2);
          layer2_out<AF>(G, V, zv);
        }
        if (term) vacc += gn * zv[0];
      }
    }

    if (alg == ALG_PEV) {
      // loss_v = mean((v(o_0) - backup)^2), gradient w.r.t. the value net only
      stage(p.blob_val, V.blob);
      bind(G, Wsm, V);
      if (have) {
        float o0[NS];
#pragma unroll
        for (int f = 0; f < NS; ++f) o0[f] = (own && valid && f < obs_dim) ? p.obs[gs * obs_dim + f] : 0.f;
        float zv[MAXA], zb[MAXA];
#pragma unroll
        for (int j = 0; j < MAXA; ++j) zb[j] = zv[j] = 0.f;
        // the output adjoint needs v(o_0) first: forward to the output, then recompute layer 2 fused with the backward
        layer1_issue<NS>(G, V, o0, 0.f);
        layer1_finish<true, AF>(G, V, 2 * G.h, 2 * G.h + 2);
        layer2_out<AF>(G, V, zv);
        if (own && valid) {
          const float diff = zv[0] - vacc;
          loss_acc += diff * diff * p.inv_B;
          vmean_acc += zv[0] * p.inv_B;
          zb[0] = 2.f * diff * p.inv_B;
        }
        layer2_back<true, false, AF>(G, V, zb, nullptr, acc3);
        backprop<true>(G, V, false, part);
      }
      stage(p.blob_pol, P.blob);
      bind(G, Wsm, P);
      continue;
    }

    if (own && valid) loss_acc += -vacc * p.inv_B;
    if (alg == ALG_PIM) {
      stage(p.blob_pol, P.blob);
      bind(G, Wsm, P);
    }
    if (!have) continue;

    // ================================ reverse sweep ================================
    // the owner prefetches step k - 1's state while step k's adjoint and MMAs run
    float nst[NS];
    bool ndn = false;
    if (own) {
#pragma unroll
      for (int f = 0; f < NS; ++f) nst[f] = tape[((H - 1) * TCH + f) * GT + G.r];
      ndn = tape[((H - 1) * TCH + NS) * GT + G.r] != 0.f;
    }
    bool dx_pending = false, dx_add = false;
    for (int k = H - 1; k >= 0; --k) {
      float zt[MAXA];
      const bool dnk = ndn;
#pragma unroll
      for (int f = 0; f < NS; ++f) st[f] = nst[f];
#pragma unroll
      for (int j = 0; j < MAXA; ++j) zt[j] = 0.f;
      if (own) {
#pragma unroll
        for (int j = 0; j < MAXA; ++j)
          if (j < P.out) zt[j] = tape[(k * TCH + NS + 1 + j) * GT + G.r];
      }
      layer1_issue<NS>(G, P, st, (float)(k + 1));     // recompute of step k's layer 1
      if (own && dx_pending) {                        // input gradient of step k + 1
        float dxn[16];
        collect_dx(G, dxn);
        if (dx_add) {
#pragma unroll
          for (int f = 0; f < NS; ++f)
            if (f < obs_dim) lam[f] += dxn[f];
        }
      }
      float zb[MAXA];
#pragma unroll
      for (int j = 0; j < MAXA; ++j) zb[j] = 0.f;
      const bool active = own && valid && (p.mask_at_done ? !dnk : true);
      if (own) {
        if (k > 0) {
#pragma unroll
          for (int f = 0; f < NS; ++f) nst[f] = tape[((k - 1) * TCH + f) * GT + G.r];
          ndn = tape[((k - 1) * TCH + NS) * GT + G.r] != 0.f;
        }
        if (active) {
          float a[MAXA], g[MAXA], abar[MAXA];
          process_action(p, P.out, zt, a, g, nullptr);
          const float rho = -p.gpow[k] * p.inv_B * (p.reward_shaping ? p.reward_scale : 1.f);
#pragma unroll
          for (int j = 0; j < MAXA; ++j) abar[j] = 0.f;
          // lam = adjoint of the OUTER observation obs_{k+1}.  Chain of step k:
          //   obs_k -(1/scale, -shift)-> inner_0 -[model step x reps, same action]-> inner_reps
          //         -(+shift, *scale)-> clip -> obs_{k+1}
          const int reps = p.repeat_num > 0 ? p.repeat_num : 1;
          float in0[NS], cur[NS];
#pragma unroll
          for (int f = 0; f < NS; ++f) in0[f] = (p.obs_scaling && f < obs_dim) ? st[f] / p.osc[f] - p.osh[f] : st[f];
          if (p.clip_obs) {            // clip passes gradient only where the raw next observation is inside
            float rr;
            bool md;
#pragma unroll
            for (int f = 0; f < NS; ++f) cur[f] = in0[f];
            for (int j = 0; j < reps; ++j) M::step(p, cur, a, rr, md);
#pragma unroll
            for (int f = 0; f < NS; ++f) {
              const float o = (p.obs_scaling && f < obs_dim) ? (cur[f] + p.osh[f]) * p.osc[f] : cur[f];
              if (o < p.obs_low[f] || o > p.obs_high[f]) lam[f] = 0.f;
            }
          }
          if (p.obs_scaling) {
#pragma unroll
            for (int f = 0; f < NS; ++f)
              if (f < obs_dim) lam[f] *= p.osc[f];
          }
          for (int j = reps - 1; j >= 0; --j) {
            float rr, aj[MAXA];
            bool md;
#pragma unroll
            for (int f = 0; f < NS; ++f) cur[f] = in0[f];
            for (int q = 0; q < j; ++q) M::step(p, cur, a, rr, md);      // state before repeat j
            const float rho_j = (p.repeat_num == 0 || p.sum_reward || j == reps - 1) ? rho : 0.f;
#pragma unroll
            for (int q = 0; q < MAXA; ++q) aj[q] = 0.f;
            M::step_bwd(p, cur, a, rho_j, lam, aj);
#pragma unroll
            for (int q = 0; q < MAXA; ++q) abar[q] += aj[q];
          }
          if (p.obs_scaling) {
#pragma unroll
            for (int f = 0; f < NS; ++f)
              if (f < obs_dim) lam[f] /= p.osc[f];
          }
#pragma unroll
          for (int j = 0; j < MAXA; ++j) zb[j] = abar[j] * g[j];
        }
      }
      layer1_finish<true, AF>(G, P, 0, G.h == 0 ? 0 : 4);      // the helper converts the whole row meanwhile
      layer2_back<true, false, AF>(G, P, zb, nullptr, acc3);
      backprop<true>(G, P, k > 0, part);
      dx_pending = k > 0;
      dx_add = active && k > 0;
    }
  }

  // ============================ per-group partials ============================
  group_sync(G.g);
  if (alg != ALG_TRACE) {
    const NetL& U = (alg == ALG_PEV) ? V : P;
    const int lane = G.r & 31, wq = G.wg & 3;
    constexpr int stride = MAXA * 64 + MAXA;
    float* rg = reinterpret_cast<float*>(G.P);                         // [4 quarters][stride]: the planes are dead
    if ((lane & 1) == 0) {
#pragma unroll
      for (int a = 0; a < MAXA; ++a)
        if (a < U.out) {
          rg[wq * stride + a * 64 + 32 * G.h + tcf::col16(lane)] = acc3.w0[a];
          rg[wq * stride + a * 64 + 32 * G.h + 16 + tcf::col16(lane)] = acc3.w1[a];
        }
    }
    if (own && lane == 0) {
#pragma unroll
      for (int a = 0; a < MAXA; ++a)
        if (a < U.out) rg[wq * stride + MAXA * 64 + a] = acc3.b[a];
    }
    group_sync(G.g);
    const int t = G.h * GT + G.r;
    for (int i = t; i < U.out * 64; i += GTH) {
      const int a = i >> 6, j = i & 63;
      part[U.g_w3 + i] = (rg[a * 64 + j] + rg[stride + a * 64 + j]) + (rg[2 * stride + a * 64 + j] + rg[3 * stride + a * 64 + j]);
    }
    if (t < U.out)
      part[U.g_b3 + t] = (rg[MAXA * 64 + t] + rg[stride + MAXA * 64 + t]) +
                         (rg[2 * stride + MAXA * 64 + t] + rg[3 * stride + MAXA * 64 + t]);
    group_sync(G.g);
  }
  {  // the three scalars of the group (fixed order; only owner threads carry values)
    float* sc = reinterpret_cast<float*>(G.P);
    if (own) { sc[G.r] = loss_acc; sc[GT + G.r] = vmean_acc; sc[2 * GT + G.r] = done_acc; }
    group_sync(G.g);
    if (own && G.r < 3) {
      const int nparam = (alg == ALG_PEV) ? V.nparam : P.nparam;
      float s = 0.f;
      for (int i = 0; i < GT; ++i) s += sc[G.r * GT + i];
      part[nparam + G.r] = s;
    }
  }
}

}  // namespace gops
