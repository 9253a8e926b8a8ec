// Fused wgmma rollout kernel (64-wide nets, <= 16 inputs, state == obs models): every warpgroup of the CTA owns one
// 64-sample sub-tile at a time and walks it through the whole horizon on its own.
//
//   row = sample.  Every dense product is one warpgroup MMA (wgmma, M = 64 = the sub-tile) whose FP32 fragment stays in
//   registers: thread t (warp w = t / 32, lane l) holds rows 16 w + l / 4 and 16 w + l / 4 + 8, columns 8 j + 2 (l % 4)
//   + {0, 1} (wgmma.cuh).  Bias, activation, act', the split into bf16 planes, the output layer (summed over the four
//   lanes of a quad by shuffles), delta2 = act'(pre2) * (W3^T zbar) and delta1 = (delta2 . W2) * act'(pre1) are all
//   computed on that fragment; act'(layer 1) stays in registers from the recompute until delta1 is formed.  The m64n64
//   accumulator fragment is the register-A fragment of the next m64nNk16 product (k-step ks = registers 8 ks .. 8 ks + 7),
//   so a forward-only layer 2 takes its three bf16 A planes straight from the layer-1 fragment, without shared memory.
//   Lanes 4q and 4q + 1 of warp w own rows 16 w + q and 16 w + q + 8: they keep the sample's model state and adjoint for
//   the whole horizon, run the dynamics / adjoint and write the observation row into the operand planes.  z, zbar and
//   the input gradient move within the quad by shuffles.  In the fixed-chain FHADP kernel (NA = 1) the forward sweep's
//   layer 1 takes A from registers too (layer1_issue_ra): each lane of the quad gets the owners' inputs by shuffles
//   and forms the bf16 words of its own feature pairs, so a forward step writes no observation planes and meets no
//   barrier.  The reverse sweep still writes them: dW1 contracts over their MN-major view.  That kernel's reverse step
//   feeds layer 2 from registers as well, and stores the same A words to the H1 planes for dW2 while the product runs,
//   so no fence and barrier stand between the layer-1 epilogue and the layer-2 wgmma.
//
//   Tape (FHADP / PIM; the owner's row of its slot's columns): per step the state, the done flag, and per policy output
//   the action a handed to the model and d a / d z, so that the reverse step neither re-reads z nor repeats the squash.
//
//   The reductions over samples run on the tensor core as well (MN-major view of the same operand planes, K = 64):
//   dW2 / db2 / dW1 / db1 (db against a column of ones).  dW2 is added into the warpgroup's FP32 sum in shared memory
//   (add.rn.ftz: the rounding of red.global.add.f32) and written to its global partial once, at the end; dW1, db2 and
//   db1 are added into the partial with red.global.add.  Every address has one writing thread, which adds in program
//   order, so the gradient is bit-reproducible.  dW3 / db3 are shuffle / register sums, written once at the end.
//
// Synchronisation: a warpgroup meets only itself (128-thread named barrier, fence.proxy.async before a wgmma reads
// planes the threads just wrote).  FHADP has no CTA-wide barrier after the initial weight stage; INFADP swaps weight
// blobs (policy <-> v_target <-> v) through the one staging buffer, CTA-wide, so there all warpgroups of a CTA run the
// same number of (possibly empty) sub-tile iterations.  Each warp waits only for its own share of a wgmma, so a plane
// is rewritten only after a barrier that follows every warp's wait for the last product that read it.  The fixed-chain
// kernel's reverse step meets five barriers, three of them after a proxy fence: put_x's, the layer-1 publish, the
// delta2 publish, the barrier before delta1 is written and the delta1 publish.  Its H1 stores (during the layer-2
// wgmma) follow the previous step's barrier before delta1, which follows that step's dW2 wait; the delta2 publish makes
// them visible to this step's dW2.
//
// Arithmetic (bars: loss 1e-4, gradient 2e-4 against the CPU oracle):
//   layer products        x . W^T      BF16x3 x BF16x3, six terms (FP32-accurate; the loss depends on these)
//   delta / input grad    delta . W    delta in TWO bf16 planes (2^-17 relative: the gradient bar is 2e-4), W in three
//   weight gradients      delta^T . h  (delta_b0 + delta_b1) . (h_b0 + h_b1): four terms, FP32 accumulation
//
// Shared memory (~218 KB of 227 with three warpgroups): weights 31.5 KB (TMA-staged), ones 0.5 KB, and per warpgroup
// H1 planes 24 KB, delta planes 16 KB (delta2, then delta1 in the same buffer), observation planes 6 KB (one buffer:
// put_x meets the warpgroup before it overwrites rows the last wgmma may still read; the fixed-chain kernel's forward
// sweep does not use them) and the FP32 sum of dW2 16 KB.
#pragma once
#include "models.cuh"
#include "mlp_tc_full.cuh"
#include "tc2_probe.cuh"

namespace gops {
namespace tc2 {

constexpr int WGS = 3;                  // warpgroups (= independent sub-tiles) per CTA
constexpr int GT = 64;                  // rows (= samples) per sub-tile = wgmma M
constexpr int NT2 = 128 * WGS;          // threads per CTA
constexpr int HPL = tcf::HPLANE, XPL = tcf::XPLANE;
constexpr int P_BYTES = 3 * HPL, Q_BYTES = 2 * HPL, XP_BYTES = 3 * XPL;
constexpr int ACC_BYTES = 64 * 64 * 4;  // FP32 dW2 sum, in fragment order (acc_frag)
constexpr int GROUP_BYTES = P_BYTES + Q_BYTES + XP_BYTES + ACC_BYTES;
constexpr int HDR_BYTES = 256;

__host__ __device__ inline size_t smem_bytes(int w_floats) {
  return HDR_BYTES + (size_t)w_floats * 4 + tcf::ONES_B + (size_t)WGS * GROUP_BYTES;
}

// (x0, x1) -> packed bf16x2 words of two planes (low half = x0)
__device__ __forceinline__ void split2(f32x2::u64 X, uint32_t& p0, uint32_t& p1) {
  float r0, r1;
  f32x2::upk(X, r0, r1);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p0) : "f"(r1), "f"(r0));
  f32x2::upk(f32x2::fma(tcf::bf16x2_as_f32x2(p0), f32x2::rep(-1.f), X), r0, r1);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p1) : "f"(r1), "f"(r0));
}

// FP32 add into global memory whose result is not used (no load on the issuing thread's path)
__device__ __forceinline__ void red_add(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
// a + b rounded as red.global.add.f32 rounds: to nearest even, subnormal inputs and result flushed to signed zero
__device__ __forceinline__ float add_ftz(float a, float b) {
  float r;
  asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// Per-thread view of its warpgroup's resources (kept small: everything else is an offset from P / Wsm).
struct Grp {
  unsigned char* P;                 // this warpgroup's planes: H1 (3) | delta (2) | observation (3) | dW2 sum
  const float* Wsm;                 // staged weight blob of the network in use (NetL offsets); `ones` precedes it
  int g, t, c;                      // warpgroup, thread in the warpgroup, t % 4 (column pair of the fragment)
  int row;                          // owned row of the sub-tile (lanes 4q, 4q + 1 of a quad; see own)
  bool own;
  __device__ __forceinline__ unsigned char* Q() const { return P + P_BYTES; }
  __device__ __forceinline__ unsigned char* X() const { return P + P_BYTES + Q_BYTES; }
  __device__ __forceinline__ float* acc() const { return reinterpret_cast<float*>(P + P_BYTES + Q_BYTES + XP_BYTES); }
  __device__ __forceinline__ const unsigned char* ones() const {
    return reinterpret_cast<const unsigned char*>(Wsm) - tcf::ONES_B;
  }
  __device__ __forceinline__ const unsigned char* W1(const NetL& L) const { return reinterpret_cast<const unsigned char*>(Wsm + L.o_w1); }
  __device__ __forceinline__ const unsigned char* W2(const NetL& L) const { return reinterpret_cast<const unsigned char*>(Wsm + L.o_w2); }
  __device__ __forceinline__ const float* W3(const NetL& L) const { return Wsm + L.o_w3; }
  __device__ __forceinline__ const float* b1(const NetL& L) const { return Wsm + L.o_b1; }
  __device__ __forceinline__ const float* b2(const NetL& L) const { return Wsm + L.o_b2; }
  __device__ __forceinline__ const float* b3(const NetL& L) const { return Wsm + L.o_b3; }
};

// make this thread's shared-memory writes visible to the tensor core, then meet the warpgroup
__device__ __forceinline__ void publish(const Grp& G) {
  fence_proxy_async();
  wg::wg_sync(G.g);
}

// A . B^T with the six BF16x3 terms (small ones first), KS steps of K = 16; A K-major (the sub-tile's 64 rows)
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
// the same product with A from registers: a[p][4 ks .. 4 ks + 3] = plane p's words of k-step ks (wgmma.cuh), same six
// terms in the same order as mma6; B K-major
template <int KS>
__device__ __forceinline__ void mma6_ra(float* d, const uint32_t (*a)[4 * KS], const tcf::Op& B) {
  using namespace tcf;
  const uint64_t b0 = dsc(B, 0), b1 = dsc(B, 1), b2 = dsc(B, 2);
  const uint64_t kb = B.kadv >> 4;
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16_n64_ra<0>(d, a[2] + 4 * ks, b0 + ks * kb, ks > 0 ? 1u : 0u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16_n64_ra<0>(d, a[0] + 4 * ks, b2 + ks * kb, 1u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16_n64_ra<0>(d, a[1] + 4 * ks, b1 + ks * kb, 1u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16_n64_ra<0>(d, a[1] + 4 * ks, b0 + ks * kb, 1u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16_n64_ra<0>(d, a[0] + 4 * ks, b1 + ks * kb, 1u);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wg::mma_bf16_n64_ra<0>(d, a[0] + 4 * ks, b0 + ks * kb, 1u);
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
// weight gradient over the sub-tile's 64 samples: D = (A_b0 + A_b1)^T . (B_b0 + .. + B_b{BP-1}), both MN-major
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
      for (int ks = 0; ks < GT / 16; ++ks) { wg::mma_bf16<N, 1, 1>(d, a + ks * ka, b + ks * kb, acc); acc = 1u; }
    }
}
__device__ __forceinline__ tcf::Op ones_op(const Grp& G) { return tcf::Op{smem_u32(G.ones()), 0u, 128u, 256u, 0u}; }

// this thread's m64n64 fragment (column pairs) -> NP bf16 planes of `buf` (BF16x3 for NP = 3, two planes for NP = 2)
template <int NP>
__device__ __forceinline__ void frag_to_planes(unsigned char* buf, const Grp& G, const float* v) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int off = (i >> 2) * (GT * 16) + wg::frag_row(G.t, i) * 16 + 4 * G.c;
    uint32_t w0, w1, w2;
    if constexpr (NP == 3) tcf::split3(v[i], v[i + 1], w0, w1, w2);
    else split2(f32x2::pk(v[i], v[i + 1]), w0, w1);
    *reinterpret_cast<uint32_t*>(buf + off) = w0;
    *reinterpret_cast<uint32_t*>(buf + HPL + off) = w1;
    if constexpr (NP == 3) *reinterpret_cast<uint32_t*>(buf + 2 * HPL + off) = w2;
  }
}
// a [64 output rows][N] weight-gradient fragment added into the FP32 partial (row stride ld, columns < ncols)
template <int N>
__device__ __forceinline__ void red_frag(float* __restrict__ dst, int ld, int ncols, const float* d, int t) {
#pragma unroll
  for (int i = 0; i < N / 2; i += 2) {
    const int row = wg::frag_row(t, i), col = wg::frag_col(t, i);
    if (col < ncols) red_add(dst + row * ld + col, d[i]);
    if (col + 1 < ncols) red_add(dst + row * ld + col + 1, d[i + 1]);
  }
}
// the m64n64 dW2 fragment added into this thread's own slots of the warpgroup's sum, kept in fragment order
// ([16 register pairs][128 threads] of float2: a warp's lanes touch 256 contiguous bytes, no bank conflict)
__device__ __forceinline__ void acc_frag(const Grp& G, const float* d) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    float2* s = reinterpret_cast<float2*>(G.acc()) + (i >> 1) * 128 + G.t;
    float2 v = *s;
    v.x = add_ftz(v.x, d[i]);
    v.y = add_ftz(v.y, d[i + 1]);
    *s = v;
  }
}
// column 0 of an m64n16 fragment (a product against the ones column) -> the bias gradient.  (Summed in shared memory
// like dW2, db2 / db1 made ptxas spill more in the fixed-chain kernel: 110 B / 84 B of spill stores instead of 60 B.)
__device__ __forceinline__ void red_bias(const Grp& G, float* part, int off, const float* d) {
  if (G.c == 0) {
    red_add(part + off + wg::frag_row(G.t, 0), d[0]);
    red_add(part + off + wg::frag_row(G.t, 2), d[2]);
  }
}

// owner: this row's input (K1 = 16 values, zero padded) -> the three observation planes.  nch = 1: the inputs fit the
// first 8-feature chunk (idpendulum: 6 + time), the second chunk was zeroed once at kernel start.  Called by every
// thread of the warpgroup: the planes have one buffer, and each warp waited on its own for the last wgmma that read
// them (layer 1 of the forward step, dW1 of the reverse step), so the warpgroup meets before an owner overwrites its
// row.
template <int NS>
__device__ __forceinline__ void put_x(const Grp& G, const NetL& L, const float* st, float vt) {
  using namespace tcf;
  wg::wg_sync(G.g);
  if (!G.own) return;
  unsigned char* x = G.X();
  float v[16];
#pragma unroll
  for (int f = 0; f < 16; ++f) v[f] = (f < NS && f < L.obs) ? st[f < NS ? f : 0] : 0.f;
  if (L.time_input) {
#pragma unroll
    for (int f = 0; f < 16; ++f)
      if (f == L.in - 1) v[f] = vt;
  }
  const int nch = L.in <= 8 ? 1 : 2;
#pragma unroll
  for (int ch = 0; ch < 2; ++ch) {
    if (ch >= nch) break;
    uint32_t w[3][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) split3(v[8 * ch + 2 * i], v[8 * ch + 2 * i + 1], w[0][i], w[1][i], w[2][i]);
#pragma unroll
    for (int p = 0; p < 3; ++p)
      *reinterpret_cast<uint4*>(x + p * XPL + (ch * GT + G.row) * 16) = make_uint4(w[p][0], w[p][1], w[p][2], w[p][3]);
  }
}

// AF: hidden activation fixed at compile time (>= 0), or -1 = dispatch on the runtime id.  With the activation fixed (the
// headline configurations use GELU) the other six epilogue variants are not compiled in.
#define GOPS_TC2_ACT_SWITCH(AF, act, M)     \
  if constexpr ((AF) >= 0) { M(AF); }       \
  else { GOPS_ACT_SWITCH(act, M) }

// layer 1, issue: observation planes . W1^T -> d (asynchronous; layer1_finish waits)
__device__ __forceinline__ void layer1_issue(const Grp& G, const NetL& L, float* d) {
  using namespace tcf;
  publish(G);                                     // observation rows visible
  wg::fence();
  mma6<64, 0, 1>(d, k_act(G.X(), XPL), k_w(G.W1(L), W1PLANE));
  wg::commit();
}
// the same product with A from registers (K = 16: one k-step), for a forward step that needs no observation planes.
// Lane c of each quad takes the owners' inputs of both quad rows by shuffles and forms the split3 words of feature pairs
// c and 4 + c (wgmma.cuh, mma_bf16_n64_ra) -- the words put_x stores for them -- then issues mma6's six terms in
// mma6's order, so the result is bit-identical.  No shared memory, no barrier.  a: the A words, which the caller keeps
// live (reg_fence_u32) until layer1_finish has waited.
template <int NS>
__device__ __forceinline__ void layer1_issue_ra(const Grp& G, const NetL& L, const float* st, float vt, float* d,
                                                uint32_t (*a)[4]) {
  using namespace tcf;
  const int qb = (G.t & 31) & ~3;
  float x[2][NS];                                 // the owners' state: row 16 w + q (lane 4q), row + 8 (lane 4q + 1)
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int f = 0; f < NS; ++f) x[r][f] = __shfl_sync(0xffffffffu, st[f], qb + r);
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int h = 0; h < 2; ++h) {                 // word 2 h + r: row r, features 8 h + 2 c + {0, 1}
      float v[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int f = 8 * h + 2 * G.c + e;        // as put_x: the state (f < obs), the time input, else 0
        float s = 0.f;
#pragma unroll
        for (int g = 0; g < NS; ++g)
          if (g == f && g < L.obs) s = x[r][g];
        if (L.time_input && f == L.in - 1) s = vt;
        v[e] = s;
      }
      split3(v[0], v[1], a[0][2 * h + r], a[1][2 * h + r], a[2][2 * h + r]);
    }
  wg::fence();
  mma6_ra<1>(d, a, k_w(G.W1(L), W1PLANE));
  wg::commit();
}
// layer 1, epilogue: + b1, activation -> d; FULL (a backward pass follows): act'(pre1) into a1p and, H1P, d -> the H1
// planes
template <bool FULL, int AF, bool H1P = FULL>
__device__ __forceinline__ void layer1_finish(const Grp& G, const NetL& L, float* d, float* a1p) {
  wg::wait<0>();
  wg::reg_fence<32>(d);
#define GOPS_TC2_A1(A)                                                                             \
  _Pragma("unroll") for (int i = 0; i < 32; i += 2) {                                              \
    const f32x2::u64 pre = f32x2::add(f32x2::pk(d[i], d[i + 1]), f32x2::ld(G.b1(L) + wg::frag_col(G.t, i))); \
    if constexpr (FULL) act_fwd_grad_pair_t<A>(pre, d[i], d[i + 1], a1p[i], a1p[i + 1]);           \
    else act_fwd_pair_t<A>(pre, d[i], d[i + 1]);                                                   \
  }
  GOPS_TC2_ACT_SWITCH(AF, L.hact, GOPS_TC2_A1)
#undef GOPS_TC2_A1
  if constexpr (H1P) frag_to_planes<3>(G.P, G, d);
}

// layer 2 product H1 . W2^T -> d (waited)
__device__ __forceinline__ void layer2_product(const Grp& G, const NetL& L, float* d) {
  using namespace tcf;
  publish(G);                                     // H1 planes visible
  wg::fence();
  mma6<64, 0, 4>(d, k_act(G.P, HPL), k_w(G.W2(L), W2PLANE));
  wg::commit();
  wg::wait<0>();
  wg::reg_fence<32>(d);
}
// the same product with A from registers: h = this thread's H1 fragment, split into three bf16 planes of A words.
// H1P (a backward pass follows): the same words also go to the H1 planes for dW2, stored while the product runs (the
// caller has met the warpgroup since the last wgmma that read them retired; the delta2 publish makes them visible)
template <bool H1P = false>
__device__ __forceinline__ void layer2_product_ra(const Grp& G, const NetL& L, const float* h, float* d) {
  using namespace tcf;
  uint32_t a[3][16];
#pragma unroll
  for (int i = 0; i < 32; i += 2) split3(h[i], h[i + 1], a[0][i >> 1], a[1][i >> 1], a[2][i >> 1]);
  wg::fence();
  mma6_ra<4>(d, a, k_w(G.W2(L), W2PLANE));
  wg::commit();
  if constexpr (H1P) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {              // frag_to_planes<3>'s layout
      const int off = (i >> 2) * (GT * 16) + wg::frag_row(G.t, i) * 16 + 4 * G.c;
#pragma unroll
      for (int p = 0; p < 3; ++p) *reinterpret_cast<uint32_t*>(G.P + p * HPL + off) = a[p][i >> 1];
    }
  }
  wg::wait<0>();
  wg::reg_fence<32>(d);
#pragma unroll
  for (int p = 0; p < 3; ++p) wg::reg_fence_u32<16>(a[p]);
}
// NA: the kernel's action count = length of the per-output arrays (z, zbar, S, Acc3).  Every net has at least one
// output; with NA = 1 that is all of them (the host selects such a kernel only for nets with one output), so output a
// is live without a test.
template <int NA>
__device__ __forceinline__ bool live(int a, const NetL& L) { return NA == 1 || a < L.out; }

// output layer: S[q][a] = this thread's (even, odd) column sums of W3[a] . h for fragment row q; reduced over the four
// lanes of the quad, the owner of each row takes z[a] = b3[a] + W3[a] . h
template <int NA>
__device__ __forceinline__ void output_sum(const Grp& G, const NetL& L, f32x2::u64 (*S)[NA], float* z) {
#pragma unroll
  for (int a = 0; a < NA; ++a) {
    z[a] = 0.f;
    if (live<NA>(a, L)) {
      float s[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        float s0, s1;
        f32x2::upk(S[q][a], s0, s1);
        s[q] = s0 + s1;
        s[q] += __shfl_xor_sync(0xffffffffu, s[q], 1);
        s[q] += __shfl_xor_sync(0xffffffffu, s[q], 2);
      }
      z[a] = G.b3(L)[a] + (G.c == 0 ? s[0] : s[1]);
    }
  }
}
template <int NA>
__device__ __forceinline__ void output_layer(const Grp& G, const NetL& L, const float* h, float* z) {
  f32x2::u64 S[2][NA];
#pragma unroll
  for (int a = 0; a < NA; ++a) S[0][a] = S[1][a] = f32x2::rep(0.f);
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int col = wg::frag_col(G.t, i), q = (i >> 1) & 1;
#pragma unroll
    for (int a = 0; a < NA; ++a)
      if (live<NA>(a, L)) S[q][a] = f32x2::fma(f32x2::ld(G.W3(L) + a * 64 + col), f32x2::pk(h[i], h[i + 1]), S[q][a]);
  }
  output_sum<NA>(G, L, S, z);
}

// layer 2 + output layer, forward only: the owner gets z[a] = b3[a] + W3[a] . act(H1 . W2^T + b2).  REGA: H1 from
// this thread's fragment h (layer2_product_ra), else from the H1 planes
template <int AF, int NA, bool REGA>
__device__ __forceinline__ void layer2_out(const Grp& G, const NetL& L, const float* h, float* z) {
  float d[32];
  if constexpr (REGA) layer2_product_ra(G, L, h, d);
  else layer2_product(G, L, d);
#define GOPS_TC2_A2(A)                                \
  _Pragma("unroll") for (int i = 0; i < 32; i += 2)   \
      act_fwd_pair_t<A>(f32x2::add(f32x2::pk(d[i], d[i + 1]), f32x2::ld(G.b2(L) + wg::frag_col(G.t, i))), d[i], d[i + 1]);
  GOPS_TC2_ACT_SWITCH(AF, L.hact, GOPS_TC2_A2)
#undef GOPS_TC2_A2
  output_layer<NA>(G, L, d, z);
}

// Per-thread accumulators of the output-layer gradients: lane l of warp w holds dW3[a] of columns 8 (l / 4) + 2 (l % 4)
// + {0, 1}, summed over the warp's 16 rows; the owners hold their rows' db3.  Combined across the warps once, at the end
// of the kernel.
template <int NA>
struct Acc3 {
  float w[NA][2];
  float b[NA];
};

// layer 2 epilogue of the backward pass, one column pair of both fragment rows at a time: h = act(pre2), then
// delta2 = act'(pre2) * (W3^T zbar) straight into the two delta planes, WANT_DW: the dW3 sums (over the warp's rows by
// an xor butterfly over the quads), WANT_Z: the output-layer partial sums S (output_layer).  zr: zbar of the two rows.
template <int A, bool WANT_DW, bool WANT_Z, int NA>
__device__ __forceinline__ void delta2_epilogue(const Grp& G, const NetL& L, float* d, const float (*zr)[NA],
                                                Acc3<NA>& acc3, f32x2::u64 (*S)[NA]) {
  const int q4 = (G.t & 31) >> 2;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = 8 * j + 2 * G.c;
    float h[2][2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int i = 4 * j + 2 * q;
      float g0, g1;
      act_fwd_grad_pair_t<A>(f32x2::add(f32x2::pk(d[i], d[i + 1]), f32x2::ld(G.b2(L) + col)), h[q][0], h[q][1], g0, g1);
      f32x2::u64 gs = f32x2::rep(0.f);
#pragma unroll
      for (int a = 0; a < NA; ++a)
        if (live<NA>(a, L)) gs = f32x2::fma(f32x2::ld(G.W3(L) + a * 64 + col), f32x2::rep(zr[q][a]), gs);
      uint32_t w0, w1;
      split2(f32x2::mul(f32x2::pk(g0, g1), gs), w0, w1);
      const int off = j * (GT * 16) + wg::frag_row(G.t, i) * 16 + 4 * G.c;
      *reinterpret_cast<uint32_t*>(G.Q() + off) = w0;
      *reinterpret_cast<uint32_t*>(G.Q() + HPL + off) = w1;
      if constexpr (WANT_Z) {
#pragma unroll
        for (int a = 0; a < NA; ++a)
          if (live<NA>(a, L)) S[q][a] = f32x2::fma(f32x2::ld(G.W3(L) + a * 64 + col), f32x2::pk(h[q][0], h[q][1]), S[q][a]);
      }
    }
    if constexpr (WANT_DW) {
#pragma unroll
      for (int a = 0; a < NA; ++a)
        if (live<NA>(a, L)) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float v = fmaf(zr[1][a], h[1][e], zr[0][a] * h[0][e]);
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 8);
            v += __shfl_xor_sync(0xffffffffu, v, 16);
            if (q4 == j) acc3.w[a][e] += v;
          }
        }
    }
  }
}

// layer 2 recompute fused with the start of the backward pass: z for the owner (WANT_Z), dW3 / db3 sums, and
// delta2 -> the two delta planes.  zbar: the owner's output adjoint of its row.  REGA: H1 from this thread's fragment h
// (layer2_product_ra, which also stores the H1 planes), else from the H1 planes
template <bool WANT_DW, bool WANT_Z, int AF, int NA, bool REGA = false>
__device__ __forceinline__ void layer2_back(const Grp& G, const NetL& L, const float* h, const float* zbar, float* z,
                                            Acc3<NA>& acc3) {
  float d[32];
  if constexpr (REGA) layer2_product_ra<true>(G, L, h, d);
  else layer2_product(G, L, d);
  const int qb = (G.t & 31) & ~3;
  float zr[2][NA];                                // zbar of the fragment's two rows
#pragma unroll
  for (int a = 0; a < NA; ++a) {
    zr[0][a] = __shfl_sync(0xffffffffu, zbar[a], qb);
    zr[1][a] = __shfl_sync(0xffffffffu, zbar[a], qb + 1);
  }
  f32x2::u64 S[2][NA];
#pragma unroll
  for (int a = 0; a < NA; ++a) S[0][a] = S[1][a] = f32x2::rep(0.f);
#define GOPS_TC2_A3(A) delta2_epilogue<A, WANT_DW, WANT_Z, NA>(G, L, d, zr, acc3, S);
  GOPS_TC2_ACT_SWITCH(AF, L.hact, GOPS_TC2_A3)
#undef GOPS_TC2_A3
  if constexpr (WANT_Z) output_sum<NA>(G, L, S, z);
  if constexpr (WANT_DW) {
#pragma unroll
    for (int a = 0; a < NA; ++a)
      if (live<NA>(a, L) && G.own) acc3.b[a] += zbar[a];
  }
}

// delta2 planes -> delta1 = (delta2 . W2) * act'(pre1) (same planes, once the readers of delta2 retired) -> the owner's
// input gradient dx (want_dx) and, WANT_DW, the weight gradients of both layers: dW2 into the warpgroup's shared-memory
// sum, the others added into the partial `part`.  pr: phase probe (tc2_probe.cuh), stamps the delta2 / dW2 part.
// OVERLAP (WANT_DW): delta2 . W2 and the layer-2 weight gradients go out as two commit groups of one issue, and delta1
// is formed while the second runs.  Its 40 accumulators are live across delta1, so only the NA = 1 kernels take it (with
// MAXA outputs ptxas spills more).
template <bool WANT_DW, int NS, bool OVERLAP>
__device__ __forceinline__ void backprop(const Grp& G, const NetL& L, bool want_dx, float* __restrict__ part,
                                         const float* a1p, float* dx, Probe& pr) {
  using namespace tcf;
  publish(G);                                     // delta2 planes visible
  // delta2 . W2 and the layer-2 weight gradients read only the delta2 and H1 planes
  constexpr bool overlap = WANT_DW && OVERLAP;
  float g1[32], w[32], wb[8];
  wg::fence();
  mma_dw<64, 4>(g1, k_act(G.Q(), HPL), mn_w(G.W2(L), W2PLANE));
  wg::commit();
  if constexpr (overlap) {
    mma_wgrad<64, 2>(w, mn_act(G.Q(), HPL), mn_act(G.P, HPL));
    mma_wgrad<16, 1>(wb, mn_act(G.Q(), HPL), ones_op(G));
    wg::commit();
    wg::wait<1>();
  } else {
    wg::wait<0>();
  }
  wg::reg_fence<32>(g1);
  if (!WANT_DW && !want_dx) return;
#pragma unroll
  for (int i = 0; i < 32; ++i) g1[i] *= a1p[i];   // delta1, written once the wgmma reads of delta2 have retired
  if constexpr (WANT_DW) {
    if constexpr (!overlap) {
      wg::fence();
      mma_wgrad<64, 2>(w, mn_act(G.Q(), HPL), mn_act(G.P, HPL));
      mma_wgrad<16, 1>(wb, mn_act(G.Q(), HPL), ones_op(G));
      wg::commit();
    }
    wg::wait<0>();
    wg::reg_fence<32>(w);
    wg::reg_fence<8>(wb);
    acc_frag(G, w);
    red_bias(G, part, L.g_b2, wb);
  }
  pr.stamp(kRevD2);
  wg::wg_sync(G.g);                               // every wgmma read of delta2 retired
  frag_to_planes<2>(G.Q(), G, g1);
  publish(G);                                     // delta1 planes visible
  float d[8], w1[8], wb1[8];
  if (want_dx) {
    wg::fence();
    mma_dw<16, 4>(d, k_act(G.Q(), HPL), mn_w(G.W1(L), W1PLANE));
    wg::commit();
  }
  if constexpr (WANT_DW) {
    wg::fence();
    mma_wgrad<16, 2>(w1, mn_act(G.Q(), HPL), mn_act(G.X(), XPL));
    mma_wgrad<16, 1>(wb1, mn_act(G.Q(), HPL), ones_op(G));
    wg::commit();
  }
  wg::wait<0>();
  if constexpr (WANT_DW) {
    wg::reg_fence<8>(w1);
    wg::reg_fence<8>(wb1);
    red_frag<16>(part + L.g_w1, L.in, L.in, w1, G.t);
    red_bias(G, part, L.g_b1, wb1);
  }
  if (want_dx) {
    wg::reg_fence<8>(d);
    // register i = 4 j + 2 h + e of lane 4q + c' holds row 16 w + q + 8 h, column 8 j + 2 c' + e; owner h = c
    const int qb = (G.t & 31) & ~3;
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int cc = 0; cc < 4; ++cc)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int f = 8 * j + 2 * cc + e;
          if (f < NS) {
            const float v0 = __shfl_sync(0xffffffffu, d[4 * j + e], qb + cc);
            const float v1 = __shfl_sync(0xffffffffu, d[4 * j + 2 + e], qb + cc);
            dx[f] = G.c == 0 ? v0 : v1;
          }
        }
  }
}

}  // namespace tc2

// ---------------------------------------------------------------------------------------------------------------
// The kernel.  grid = min(#SM, #sub-tiles) CTAs of WGS warpgroups, one CTA per SM (shared memory).
// Slot s = WGS * blockIdx.x + warpgroup owns the contiguous sub-tile range [NSUB s / slots, NSUB (s + 1) / slots), its
// tape columns and its row of the gradient partials.
// AF: hidden activation (GOPS_TC2_ACT_SWITCH).  NA: action count, MAXA (policy outputs read from the plan) or 1 (nets
// with one output: the per-output arrays and tests drop out).  W: wrapper flags (models.cuh, WrapRt / WrapFixed).
// ---------------------------------------------------------------------------------------------------------------
template <class M, int ALG, int AF, int NA, class W>
__global__ void __launch_bounds__(tc2::NT2, 1) rollout_tc2_kernel(const __grid_constant__ KParams p) {
  using namespace tc2;
  static_assert(M::KIND == 0, "wgmma rollout kernel: state == obs models");
  static_assert(NA == 1 || NA == MAXA, "wgmma rollout kernel: NA is MAXA or 1");
  constexpr int NS = M::NS, alg = ALG;
  // the fixed-chain FHADP kernel (NA = 1) feeds the forward sweep's layer 1 (layer1_issue_ra) and the reverse sweep's
  // layer 2 (layer2_product_ra<true>) from registers
  constexpr bool kRegA = alg == ALG_FHADP && NA == 1;
  extern __shared__ __align__(16) float smem[];
  unsigned char* sm = reinterpret_cast<unsigned char*>(smem);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm);           // [0] weights landed
  unsigned char* ones = sm + HDR_BYTES;
  float* Wsm = reinterpret_cast<float*>(ones + tcf::ONES_B);
  unsigned char* gbase = reinterpret_cast<unsigned char*>(Wsm + p.w_floats);

  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);      // warp-uniform by construction
  Grp G;
  G.g = warp >> 2;
  G.t = tid & 127;
  G.c = tid & 3;
  G.row = wg::frag_row(G.t, 2 * (G.c & 1));                   // lanes 4q, 4q + 1: rows 16 w + q, 16 w + q + 8
  G.own = G.c < 2;
  G.P = gbase + G.g * GROUP_BYTES;
  G.Wsm = Wsm;
  const bool own = G.own;

  if (tid == 0) {
    mbar_init(bars, 1);
    fence_mbar_init();
  }
  if (tid < 256) {  // `ones`: [2 mn-groups][16 rows][8 bf16], feature 0 = 1.0
    uint16_t* o16 = reinterpret_cast<uint16_t*>(ones);
    o16[tid] = (tid < 128 && (tid & 7) == 0) ? (uint16_t)0x3f80 : (uint16_t)0;
  }
  uint32_t wphase = 0;
  auto stage = [&](const float* gsrc, int floats) {      // CTA-wide: every warpgroup calls it at the same program points
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
  const int pout = NA == 1 ? 1 : P.out;                        // policy outputs
  const long long B = p.batch;
  const int slot = blockIdx.x * WGS + G.g, slots = gridDim.x * WGS;
  // zeroed before the first red.global.add into it: stage() below is a CTA barrier
  float* part = p.partial + (size_t)slot * p.part_stride;
  for (int i = G.t; i < p.part_stride; i += 128) part[i] = 0.f;
  float* tape = p.tape + (size_t)slot * (size_t)H * TCH * GT;
  Acc3<NA> acc3;
#pragma unroll
  for (int a = 0; a < NA; ++a) acc3.w[a][0] = acc3.w[a][1] = acc3.b[a] = 0.f;
  float loss_acc = 0.f, vmean_acc = 0.f, done_acc = 0.f;
  Probe pr;
  pr.init(G.t);

  // the observation planes and the dW2 sum that follows them
  for (int i = G.t; i < (XP_BYTES + ACC_BYTES) / 16; i += 128) reinterpret_cast<uint4*>(G.X())[i] = make_uint4(0u, 0u, 0u, 0u);
  stage(p.blob_pol, P.blob);      // (its leading CTA barrier also publishes the zeroed planes)

  const long long nsub = (B + GT - 1) / GT;
  const long long s0 = nsub * slot / slots, s1 = nsub * (slot + 1) / slots;
  // INFADP: equal iteration counts for all warpgroups of the CTA (stage() is a CTA-wide barrier)
  long long iters = s1 - s0;
  if (WGS > 1 && (alg == ALG_PIM || alg == ALG_PEV)) {
    for (int o = 0; o < WGS; ++o) {
      const long long os = (long long)blockIdx.x * WGS + o;
      const long long n = nsub * (os + 1) / slots - nsub * os / slots;
      iters = n > iters ? n : iters;
    }
  }

  for (long long it = 0; it < iters; ++it) {
    const long long sub = s0 + it;
    const bool have = sub < s1;                   // false: idle iteration that only takes part in the blob swaps
    const long long gs = sub * GT + G.row;
    const bool valid = own && have && gs < B;
    float st[NS];
#pragma unroll
    for (int f = 0; f < NS; ++f) st[f] = (valid && f < obs_dim) ? p.obs[gs * obs_dim + f] : 0.f;
    bool dn = valid ? (p.done[gs] != 0.f) : true;
    float vacc = 0.f;

    // ================================ forward sweep ================================
    if (have) {
      for (int k = 0; k < H; ++k) {
        pr.mark();
        if (own) {
          if (alg == ALG_FHADP || alg == ALG_PIM) {
#pragma unroll
            for (int f = 0; f < NS; ++f) tape[(k * TCH + f) * GT + G.row] = st[f];
            tape[(k * TCH + NS) * GT + G.row] = dn ? 1.f : 0.f;
          }
        }
        float z[NA], d1[32];
        if constexpr (kRegA) {
          uint32_t x1[3][4];
          layer1_issue_ra<NS>(G, P, st, (float)(k + 1), d1, x1);
          layer1_finish<false, AF>(G, P, d1, nullptr);
#pragma unroll
          for (int q = 0; q < 3; ++q) wg::reg_fence_u32<4>(x1[q]);
        } else {
          put_x<NS>(G, P, st, (float)(k + 1));
          layer1_issue(G, P, d1);
          layer1_finish<false, AF>(G, P, d1, nullptr);
        }
        pr.stamp(kFwdL1);
        layer2_out<AF, NA, true>(G, P, d1, z);
        pr.stamp(kFwdL2);
        if (own) {
          float a[NA], g[NA], apol[NA];
          process_action<NA, W>(p, pout, z, a, g, apol);
          if (alg == ALG_FHADP || alg == ALG_PIM) {
#pragma unroll
            for (int j = 0; j < NA; ++j)
              if (j < pout) {
                tape[(k * TCH + NS + 1 + j) * GT + G.row] = a[j];
                tape[(k * TCH + NS + 1 + pout + j) * GT + G.row] = g[j];
              }
          }
          const bool active = valid && (p.mask_at_done ? !dn : true);
          float r = 0.f;
          if (valid) {
            wrapped_step<M, W>(p, obs_dim, st, a, active, r, dn);
            r = shape_reward(p, r);
            vacc += r * p.gpow[k];
          }
          if (alg == ALG_TRACE && valid) {
            const size_t row = (size_t)k * B + gs;
            if (p.tr_obs)
              for (int f = 0; f < obs_dim; ++f) p.tr_obs[row * obs_dim + f] = st[f];
            if (p.tr_act)
              for (int j = 0; j < pout; ++j) p.tr_act[row * pout + j] = apol[j];
            if (p.tr_rew) p.tr_rew[row] = r;
            if (p.tr_done) p.tr_done[row] = dn ? 1.f : 0.f;
          }
        }
        pr.stamp(kFwdDyn);
        pr.step(true);
      }
      if (valid && dn) done_acc += 1.f;
    }
    if (alg == ALG_TRACE) continue;

    // ============================ terminal value (INFADP) ============================
    float lam[NS];
#pragma unroll
    for (int f = 0; f < NS; ++f) lam[f] = 0.f;
    if (alg != ALG_FHADP) {
      stage(p.blob_vtg, V.blob);
      if (have) {
        const float gn = p.gpow[H];
        const bool term = valid && !dn;
        float zv[NA], zb[NA], d1[32], a1p[32];
#pragma unroll
        for (int j = 0; j < NA; ++j) zb[j] = zv[j] = 0.f;
        put_x<NS>(G, V, st, 0.f);
        layer1_issue(G, V, d1);
        if (alg == ALG_PIM) {
          float dx[NS];
          zb[0] = term ? -gn * p.inv_B : 0.f;
          layer1_finish<true, AF>(G, V, d1, a1p);
          layer2_back<false, true, AF, NA>(G, V, nullptr, zb, zv, acc3);
          backprop<false, NS, NA == 1>(G, V, true, part, a1p, dx, pr);
          if (term) {
#pragma unroll
            for (int f = 0; f < NS; ++f)
              if (f < obs_dim) lam[f] = dx[f];
          }
        } else {
          layer1_finish<false, AF>(G, V, d1, nullptr);
          layer2_out<AF, NA, true>(G, V, d1, zv);
        }
        if (term) vacc += gn * zv[0];
      }
    }

    if (alg == ALG_PEV) {
      // loss_v = mean((v(o_0) - backup)^2), gradient w.r.t. the value net only
      stage(p.blob_val, V.blob);
      if (have) {
        float o0[NS];
#pragma unroll
        for (int f = 0; f < NS; ++f) o0[f] = (valid && f < obs_dim) ? p.obs[gs * obs_dim + f] : 0.f;
        float zv[NA], zb[NA], d1[32], a1p[32];
#pragma unroll
        for (int j = 0; j < NA; ++j) zb[j] = zv[j] = 0.f;
        // the output adjoint needs v(o_0) first: forward to the output, then recompute layer 2 fused with the backward
        put_x<NS>(G, V, o0, 0.f);
        layer1_issue(G, V, d1);
        layer1_finish<true, AF>(G, V, d1, a1p);
        layer2_out<AF, NA, false>(G, V, d1, zv);        // from the H1 planes, which layer2_back reads again
        if (valid) {
          const float diff = zv[0] - vacc;
          loss_acc += diff * diff * p.inv_B;
          vmean_acc += zv[0] * p.inv_B;
          zb[0] = 2.f * diff * p.inv_B;
        }
        layer2_back<true, false, AF, NA>(G, V, nullptr, zb, nullptr, acc3);
        backprop<true, NS, NA == 1>(G, V, false, part, a1p, nullptr, pr);
      }
      stage(p.blob_pol, P.blob);
      continue;
    }

    if (valid) loss_acc += -vacc * p.inv_B;
    if (alg == ALG_PIM) {
      stage(p.blob_pol, P.blob);
    }
    if (!have) continue;

    // ================================ reverse sweep ================================
    // the owner prefetches step k - 1's state while step k's adjoint and MMAs run
    float nst[NS];
    bool ndn = false;
    if (own) {
#pragma unroll
      for (int f = 0; f < NS; ++f) nst[f] = tape[((H - 1) * TCH + f) * GT + G.row];
      ndn = tape[((H - 1) * TCH + NS) * GT + G.row] != 0.f;
    }
    for (int k = H - 1; k >= 0; --k) {
      pr.mark();
      float a[NA], g[NA];                            // step k's action and d a / d z, from the forward sweep
      const bool dnk = ndn;
#pragma unroll
      for (int f = 0; f < NS; ++f) st[f] = nst[f];
#pragma unroll
      for (int j = 0; j < NA; ++j) a[j] = g[j] = 0.f;
      if (own) {
#pragma unroll
        for (int j = 0; j < NA; ++j)
          if (j < pout) {
            a[j] = tape[(k * TCH + NS + 1 + j) * GT + G.row];
            g[j] = tape[(k * TCH + NS + 1 + pout + j) * GT + G.row];
          }
      }
      float d1[32], a1p[32];
      put_x<NS>(G, P, st, (float)(k + 1));
      layer1_issue(G, P, d1);                        // recompute of step k's layer 1, overlapped with the adjoint
      pr.stamp(kRevL1);
      float zb[NA];
#pragma unroll
      for (int j = 0; j < NA; ++j) zb[j] = 0.f;
      const bool active = valid && (p.mask_at_done ? !dnk : true);
      if (own) {
        if (k > 0) {
#pragma unroll
          for (int f = 0; f < NS; ++f) nst[f] = tape[((k - 1) * TCH + f) * GT + G.row];
          ndn = tape[((k - 1) * TCH + NS) * GT + G.row] != 0.f;
        }
        if (active) {
          float abar[NA];
#pragma unroll
          for (int j = 0; j < NA; ++j) abar[j] = 0.f;
          // lam: adjoint of obs_{k+1}.  The NA = 1 kernel has the registers for an unrolled model adjoint; with MAXA
          // outputs ptxas spills more
          wrapped_step_bwd<M, NA, W, NA == 1>(p, obs_dim, st, a, reward_adjoint(p, k), lam, abar);
#pragma unroll
          for (int j = 0; j < NA; ++j) zb[j] = abar[j] * g[j];
        }
      }
      pr.stamp(kRevAdj);
      // kRegA: layer 2 from this thread's layer-1 fragment, which goes to the H1 planes (for dW2) while it runs
      layer1_finish<true, AF, !kRegA>(G, P, d1, a1p);
      pr.stamp(kRevL1);
      layer2_back<true, false, AF, NA, kRegA>(G, P, d1, zb, nullptr, acc3);
      pr.stamp(kRevL2);
      float dx[NS];
      backprop<true, NS, NA == 1>(G, P, k > 0, part, a1p, dx, pr);
      if (active && k > 0) {                          // + the policy's input gradient of step k
#pragma unroll
        for (int f = 0; f < NS; ++f)
          if (f < obs_dim) lam[f] += dx[f];
      }
      pr.stamp(kRevD1);
      pr.step(false);
    }
  }

  // ============================ per-warpgroup partials ============================
  wg::wg_sync(G.g);
  const int lane = G.t & 31, w4 = G.t >> 5;
  if (alg != ALG_TRACE) {
    const NetL& U = (alg == ALG_PEV) ? V : P;
    // the dW2 sum: each thread its own fragment
#pragma unroll
    for (int i = 0; i < 32; i += 2)
      *reinterpret_cast<float2*>(part + U.g_w2 + wg::frag_row(G.t, i) * 64 + wg::frag_col(G.t, i)) =
          reinterpret_cast<const float2*>(G.acc())[(i >> 1) * 128 + G.t];
    constexpr int stride = NA * 64 + NA;
    float* rg = reinterpret_cast<float*>(G.P);                         // [4 warps][stride]: the planes are dead
#pragma unroll
    for (int a = 0; a < NA; ++a)
      if (live<NA>(a, U)) {
        const int col = 8 * (lane >> 2) + 2 * G.c;
        rg[w4 * stride + a * 64 + col] = acc3.w[a][0];
        rg[w4 * stride + a * 64 + col + 1] = acc3.w[a][1];
        float sb = acc3.b[a];                                          // owners' rows; 0 elsewhere
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sb += __shfl_xor_sync(0xffffffffu, sb, o);
        if (lane == 0) rg[w4 * stride + NA * 64 + a] = sb;
      }
    wg::wg_sync(G.g);
    for (int i = G.t; i < U.out * 64; i += 128) {
      const int a = i >> 6, j = i & 63;
      part[U.g_w3 + i] = (rg[a * 64 + j] + rg[stride + a * 64 + j]) + (rg[2 * stride + a * 64 + j] + rg[3 * stride + a * 64 + j]);
    }
    if (G.t < U.out)
      part[U.g_b3 + G.t] = (rg[NA * 64 + G.t] + rg[stride + NA * 64 + G.t]) +
                           (rg[2 * stride + NA * 64 + G.t] + rg[3 * stride + NA * 64 + G.t]);
    wg::wg_sync(G.g);
  }
  {  // the three scalars of the sub-tile slot (fixed order over its 64 rows; only owner threads carry values)
    float* sc = reinterpret_cast<float*>(G.P);
    if (own) { sc[G.row] = loss_acc; sc[GT + G.row] = vmean_acc; sc[2 * GT + G.row] = done_acc; }
    wg::wg_sync(G.g);
    if (G.t < 3) {
      const int nparam = (alg == ALG_PEV) ? V.nparam : P.nparam;
      float s = 0.f;
      for (int i = 0; i < GT; ++i) s += sc[G.t * GT + i];
      part[nparam + G.t] = s;
    }
  }
  pr.finish(alg, WGS);
}

}  // namespace gops
