// BF16x3 operand primitives of the warpgroup tensor-core kernels (rollout_tc2.cuh, dense_tc.cuh): operand descriptors
// of the canonical plane layout and the fp32 -> three-plane split.
//
// Arithmetic: BF16x3.  x = b0 + b1 + b2 (three bf16 planes, residual <= 2^-27 |x|), a product keeps the six terms of
// order <= 2 (b0b0, b0b1, b1b0, b1b1, b0b2, b2b0; neglected <= 2^-26), FP32 accumulation: at least as accurate as the
// 3xTF32 split of the other paths (parity tests hold it to the same bars).  Why bf16 and not tf32: wgmma reads a 16-bit
// operand transposed (MN-major) from the plain no-swizzle layout, so ONE shared-memory buffer [sample][feature] serves
// the layer products (K-major: contraction over features) and the weight-gradient products (MN-major: contraction over
// samples); 32-bit operands are K-major only.
//
// Operand layout: plane[p][k/8][row][8] bf16 (p = 0..2), i.e. the no-swizzle canonical layout with chunk stride
// rows*16 B and 8-row group stride 128 B.  K-major view: rows = M/N, K along k.  MN-major view (same bytes): M/N along
// k, K = rows (wgmma.cuh).
#pragma once
#include "rollout.cuh"
#include "wgmma.cuh"

namespace gops {

namespace tcf {
constexpr int K1 = 16;                           // layer-1 K extent (inputs padded to 16)
constexpr int HPLANE = 8 * 64 * 16;              // bytes of one hidden-activation plane ([8 chunks][64 rows][16 B])
constexpr int XPLANE = 2 * 64 * 16;              // bytes of one observation plane
constexpr int W2PLANE = 8 * 64 * 16, W1PLANE = 2 * 64 * 16;
constexpr int ONES_B = 2 * 16 * 16;              // bytes: [2 mn-groups][16 rows][16 B]

struct Op {            // one operand: smem address of plane 0, plane stride, descriptor strides, advance per K = 16 step
  uint32_t base, pstride, lbo, sbo, kadv;
};
__device__ __forceinline__ Op k_act(const unsigned char* b, int plane_bytes) {     // activations K-major, 64 rows
  return Op{smem_u32(b), (uint32_t)plane_bytes, 1024u, 128u, 2048u};
}
__device__ __forceinline__ Op k_w(const unsigned char* b, int plane_bytes) {       // weights K-major, 64 rows
  return Op{smem_u32(b), (uint32_t)plane_bytes, 1024u, 128u, 2048u};
}
__device__ __forceinline__ Op mn_act(const unsigned char* b, int plane_bytes) {    // activations transposed: K = 64 samples
  return Op{smem_u32(b), (uint32_t)plane_bytes, 128u, 1024u, 256u};
}
__device__ __forceinline__ Op mn_w(const unsigned char* b, int plane_bytes) {      // weights transposed: K = output rows
  return Op{smem_u32(b), (uint32_t)plane_bytes, 128u, 1024u, 256u};
}
__device__ __forceinline__ uint64_t dsc(const Op& o, int plane) {
  return wg::smem_desc(o.base + plane * o.pstride, o.lbo, o.sbo);
}

// (x0, x1) -> packed bf16x2 words of the three planes (low half = x0); the residuals x - hi are formed by one pair
// FMA (hi * -1 + x: the same rounding as the subtraction)
__device__ __forceinline__ f32x2::u64 bf16x2_as_f32x2(uint32_t p) {
  return f32x2::pk(__uint_as_float(p << 16), __uint_as_float(p & 0xffff0000u));
}
__device__ __forceinline__ void split3(f32x2::u64 X, uint32_t& p0, uint32_t& p1, uint32_t& p2) {
  float r0, r1;
  f32x2::upk(X, r0, r1);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p0) : "f"(r1), "f"(r0));
  f32x2::u64 R = f32x2::fma(bf16x2_as_f32x2(p0), f32x2::rep(-1.f), X);
  f32x2::upk(R, r0, r1);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p1) : "f"(r1), "f"(r0));
  R = f32x2::fma(bf16x2_as_f32x2(p1), f32x2::rep(-1.f), R);
  f32x2::upk(R, r0, r1);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p2) : "f"(r1), "f"(r0));
}
__device__ __forceinline__ void split3(float x0, float x1, uint32_t& p0, uint32_t& p1, uint32_t& p2) {
  split3(f32x2::pk(x0, x1), p0, p1, p2);
}

}  // namespace tcf

}  // namespace gops
