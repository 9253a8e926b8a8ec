// Generic dense layers on the Hopper warpgroup tensor cores (wgmma) in FP32-accurate BF16x3 arithmetic: the building block of the layer-wise paths
// (wide nets: FHADP veh3dof_tracking [256,256]; DSAC [256,256,256]; FHADP2's open-loop policy) where a whole-horizon
// fusion does not fit one SM's shared memory.
//
//   forward   Y[r][n] = act(sum_k X[r][k] W[n][k] + b[n])           (optionally also D = act'(pre))
//   dgrad     dX[r][k] = (sum_n dY[r][n] W[n][k]) * M[r][k]          (M: saved act' of the layer below, optional)
//   wgrad     dW[n][k] = sum_r dY[r][n] X[r][k]                       (row-split partials, fixed-order reduction)
//
// All three are C = A . B^T GEMMs with M = 128 rows per CTA (two warpgroups of 64 rows), operands as bf16 planes in the
// no-swizzle canonical layout plane[chunk = col/8][row][8] (wgmma.cuh):
//   * activations (fp32, row-major in HBM) are converted by the CTA while it stages them: thread = (8-column chunk, row),
//     one 32-byte global read, one 16-byte shared store per plane (conflict-free: consecutive lanes = consecutive rows);
//   * weights are pre-split once per update by pack_dense_kernel into exactly the shared-memory image of each
//     (column split, K slice) and fetched with one TMA bulk copy per slice;
//   * K is consumed in slices of 64 (four K = 16 MMA steps), accumulators live in registers (<= 128 columns per CTA:
//     64 fp32 registers per thread);
//   * forward products keep six BF16x3 terms (FP32-accurate), gradient products three (2-plane delta, 2^-16).
// wgrad contracts over ROWS: the same planes, MN-major view (A = dY^T, B = X^T), 8 K-steps per 128-row tile.
#pragma once
#include "mlp_tc_full.cuh"

namespace gops {
namespace dense {

constexpr int TM = 128;          // rows per CTA tile (two wgmma M = 64 halves)
constexpr int KS = 64;           // K slice
constexpr int NCMAX = 128;       // output columns per CTA
constexpr int NTH = 256;         // threads per CTA

__host__ __device__ inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
// columns per CTA (a wgmma tile width: 16, 32, 64 or 128) / number of column splits for an output width n
__host__ __device__ inline int nc_of(int n) { return n <= 16 ? 16 : n <= 32 ? 32 : n <= 64 ? 64 : NCMAX; }
__host__ __device__ inline int splits_of(int n) { return (round_up(n, 16) + NCMAX - 1) / NCMAX; }
__host__ __device__ inline int slices_of(int k) { return (k + KS - 1) / KS; }
// bytes of one packed (split, slice) image: 3 planes x 8 chunks x NC rows x 16 B
__host__ __device__ inline size_t slice_bytes(int nc) { return (size_t)3 * 8 * nc * 16; }
__host__ __device__ inline size_t packed_bytes(int n_out, int k_in) {
  return (size_t)splits_of(n_out) * slices_of(k_in) * slice_bytes(nc_of(n_out));
}

// W [n_out][k_in] (torch Linear, row-major) -> images for  Y = X . W^T  (B rows = n, contraction over k)
//                                       and  -> images for dX = dY . W   (B rows = k, contraction over n)
__global__ void pack_dense_kernel(const float* __restrict__ W, int n_out, int k_in, unsigned char* __restrict__ fwd,
                                  unsigned char* __restrict__ bwd) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthreads = gridDim.x * blockDim.x;
  auto put3 = [](float w, __nv_bfloat16* dst, size_t pstride) {
    const __nv_bfloat16 b0 = __float2bfloat16_rn(w);
    const float r1 = w - __bfloat162float(b0);
    const __nv_bfloat16 b1 = __float2bfloat16_rn(r1);
    dst[0] = b0; dst[pstride] = b1; dst[2 * pstride] = __float2bfloat16_rn(r1 - __bfloat162float(b1));
  };
  {
    const int nc = nc_of(n_out), ns = splits_of(n_out), nsl = slices_of(k_in);
    const size_t plane = (size_t)8 * nc * 8;                  // bf16 elements per plane
    const long long total = (long long)ns * nsl * plane;
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(fwd);
    for (long long i = tid; i < total; i += nthreads) {
      const long long img = i / plane;
      const int rem = (int)(i - img * plane), kc = rem / (nc * 8), r = (rem / 8) % nc, e = rem & 7;
      const int s = (int)(img / nsl), t = (int)(img % nsl);
      const int n = s * nc + r, k = t * KS + kc * 8 + e;
      put3((n < n_out && k < k_in) ? W[(size_t)n * k_in + k] : 0.f, out + img * 3 * plane + rem, plane);
    }
  }
  if (bwd != nullptr) {
    const int nc = nc_of(k_in), ns = splits_of(k_in), nsl = slices_of(n_out);
    const size_t plane = (size_t)8 * nc * 8;
    const long long total = (long long)ns * nsl * plane;
    __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(bwd);
    for (long long i = tid; i < total; i += nthreads) {
      const long long img = i / plane;
      const int rem = (int)(i - img * plane), kc = rem / (nc * 8), r = (rem / 8) % nc, e = rem & 7;
      const int s = (int)(img / nsl), t = (int)(img % nsl);
      const int k = s * nc + r, n = t * KS + kc * 8 + e;       // row = input feature k, contraction index = n
      put3((n < n_out && k < k_in) ? W[(size_t)n * k_in + k] : 0.f, out + img * 3 * plane + rem, plane);
    }
  }
}

enum Epi { EPI_ACT = 0, EPI_LINEAR = 1, EPI_MUL = 2, EPI_PLAIN = 3 };

struct GemmArgs {
  const float* A; int lda; long long rows; int k;            // activations [rows][k] (row stride lda)
  const unsigned char* Bimg; int n;                           // packed weights (fwd or bwd images), output width
  const float* bias;                                          // [n] (EPI_ACT / EPI_LINEAR)
  const float* mul; int ldm;                                  // [rows][n] factor (EPI_MUL)
  float* Y; int ldy;                                          // [rows][n]
  float* D; int ldd;                                          // [rows][n] act'(pre) (EPI_ACT, optional)
  int act;
};

// rows [r0, r0 + 128) x columns [k0, k0 + 64) of a row-major fp32 matrix -> NPL bf16 planes [8 chunks][128 rows][8]
// (`PL`: byte stride between planes; the 8 chunks land at planes + chunk * 2048).  Split into a LOAD half (global ->
// registers; all 32-byte reads of a tile are issued back to back, so their HBM / L2 latencies overlap -- and callers
// prefetch the next tile while the tensor core works on the current one) and a STORE half (split + shared stores).
struct TileRegs {
  float v[(8 * TM) / NTH][8];
};
__device__ __forceinline__ void load_tile(const float* __restrict__ src, int ld, long long r0, long long rows, int k0,
                                          int kcols, TileRegs& t) {
#pragma unroll
  for (int i = 0; i < (8 * TM) / NTH; ++i) {
    const int idx = threadIdx.x + NTH * i, kc = idx >> 7, r = idx & 127;
    const long long row = r0 + r;
    const int k = k0 + 8 * kc;
    if (row < rows && k + 8 <= kcols && ((ld & 3) == 0)) {
      const float4 a = *reinterpret_cast<const float4*>(src + row * ld + k);
      const float4 b = *reinterpret_cast<const float4*>(src + row * ld + k + 4);
      t.v[i][0] = a.x; t.v[i][1] = a.y; t.v[i][2] = a.z; t.v[i][3] = a.w;
      t.v[i][4] = b.x; t.v[i][5] = b.y; t.v[i][6] = b.z; t.v[i][7] = b.w;
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) t.v[i][e] = (row < rows && k + e < kcols) ? src[row * ld + k + e] : 0.f;
    }
  }
}
template <int NPL>
__device__ __forceinline__ void store_tile(const TileRegs& t, unsigned char* planes, int PL = 8 * TM * 16) {
#pragma unroll
  for (int i = 0; i < (8 * TM) / NTH; ++i) {
    const int idx = threadIdx.x + NTH * i, kc = idx >> 7, r = idx & 127;
    const float* v = t.v[i];
    uint32_t w[3][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if constexpr (NPL == 3) tcf::split3(v[2 * j], v[2 * j + 1], w[0][j], w[1][j], w[2][j]);
      else {
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(w[0][j]) : "f"(v[2 * j + 1]), "f"(v[2 * j]));
        float q0, q1;
        f32x2::upk(f32x2::fma(tcf::bf16x2_as_f32x2(w[0][j]), f32x2::rep(-1.f), f32x2::pk(v[2 * j], v[2 * j + 1])), q0, q1);
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(w[1][j]) : "f"(q1), "f"(q0));
      }
    }
#pragma unroll
    for (int p = 0; p < NPL; ++p)
      *reinterpret_cast<uint4*>(planes + p * PL + (kc * TM + r) * 16) = make_uint4(w[p][0], w[p][1], w[p][2], w[p][3]);
  }
}

// One 128-row x NC-column output tile.  grid = (row tiles, column splits), 256 threads = two warpgroups, warpgroup w
// owns rows [64 w, 64 w + 64) of the tile and their NC accumulator columns in registers.
// GRAD: gradient product (A in two planes, three terms); else forward product (three planes, six terms).
// K slices are double buffered: while the tensor core works on slice t the CTA converts slice t + 1 into the other
// operand buffer and its weight image arrives by TMA; a warpgroup keeps at most one slice's wgmma group in flight.
template <int EPI, int NC, int ACT>
__device__ __forceinline__ void gemm_epilogue(const GemmArgs& g, const float* acc, long long r0, int split) {
  const int wgi = threadIdx.x >> 7, t = threadIdx.x & 127;
#pragma unroll
  for (int i = 0; i < NC / 2; i += 2) {
    const long long row = r0 + 64 * wgi + wg::frag_row(t, i);
    const int n = split * NC + wg::frag_col(t, i);
    if (row >= g.rows) continue;
    float v0 = acc[i], v1 = acc[i + 1], d0 = 0.f, d1 = 0.f;
    if constexpr (EPI == EPI_ACT) {
      const float b0 = n < g.n ? g.bias[n] : 0.f, b1 = n + 1 < g.n ? g.bias[n + 1] : 0.f;
      act_fwd_grad_pair_t<ACT>(f32x2::add(f32x2::pk(v0, v1), f32x2::pk(b0, b1)), v0, v1, d0, d1);
    } else if constexpr (EPI == EPI_LINEAR) {
      v0 += n < g.n ? g.bias[n] : 0.f;
      v1 += n + 1 < g.n ? g.bias[n + 1] : 0.f;
    } else if constexpr (EPI == EPI_MUL) {
      v0 *= n < g.n ? g.mul[row * g.ldm + n] : 0.f;
      v1 *= n + 1 < g.n ? g.mul[row * g.ldm + n + 1] : 0.f;
    }
    if (n < g.n) g.Y[row * g.ldy + n] = v0;
    if (n + 1 < g.n) g.Y[row * g.ldy + n + 1] = v1;
    if constexpr (EPI == EPI_ACT) {
      if (g.D != nullptr) {
        if (n < g.n) g.D[row * g.ldd + n] = d0;
        if (n + 1 < g.n) g.D[row * g.ldd + n + 1] = d1;
      }
    }
  }
}

template <int EPI, bool GRAD, int NC>
__device__ __forceinline__ void dense_gemm_body(const GemmArgs& g, unsigned char* dsm) {
  uint64_t* bars = reinterpret_cast<uint64_t*>(dsm);           // [0..1] weights landed (per buffer)
  constexpr int APL = 8 * TM * 16, NPA = GRAD ? 2 : 3;
  const int tid = threadIdx.x, wgi = tid >> 7;
  const int nsl = slices_of(g.k);
  const size_t img = slice_bytes(NC);
  unsigned char* Abuf = dsm + 128;
  unsigned char* Bbuf = Abuf + 2 * NPA * APL;
  const int split = blockIdx.y;
  const long long r0 = (long long)blockIdx.x * TM;
  if (tid == 0) {
    mbar_init(bars, 1);
    mbar_init(bars + 1, 1);
    fence_mbar_init();
  }
  const unsigned char* Bsrc = g.Bimg + (size_t)split * nsl * img;
  float acc[NC / 2];
#pragma unroll
  for (int i = 0; i < NC / 2; ++i) acc[i] = 0.f;
  TileRegs regs;
  load_tile(g.A, g.lda, r0, g.rows, 0, g.k, regs);
  for (int t = 0; t < nsl; ++t) {
    const int bf = t & 1;
    const uint32_t ph = (uint32_t)(t >> 1) & 1u;
    unsigned char* Ap = Abuf + bf * NPA * APL;
    unsigned char* Bp = Bbuf + (size_t)bf * img;
    __syncthreads();                                // both warpgroups retired slice t - 2, the reader of this buffer pair
    if (tid == 0) {
      fence_proxy_async();
      mbar_expect_tx(bars + bf, (uint32_t)img);
      for (size_t off = 0; off < img; off += 32768)
        tma_bulk_g2s(Bp + off, Bsrc + (size_t)t * img + off, (uint32_t)(img - off < 32768 ? img - off : 32768), bars + bf);
    }
    store_tile<NPA>(regs, Ap);
    if (t + 1 < nsl) load_tile(g.A, g.lda, r0, g.rows, (t + 1) * KS, g.k, regs);   // next slice's reads are in flight
    fence_proxy_async();
    mbar_wait(bars + bf, ph);
    __syncthreads();
    {
      using namespace tcf;
      const Op A{smem_u32(Ap) + 1024u * wgi, (uint32_t)APL, 2048u, 128u, 4096u};     // this warpgroup's 64 rows
      const Op B{smem_u32(Bp), (uint32_t)(8 * NC * 16), (uint32_t)(NC * 16), 128u, (uint32_t)(2 * NC * 16)};
      const uint64_t ka = A.kadv >> 4, kb = B.kadv >> 4;
      const uint64_t a0 = dsc(A, 0), a1 = dsc(A, 1), b0 = dsc(B, 0), b1 = dsc(B, 1), b2 = dsc(B, 2);
      uint32_t first = t == 0 ? 0u : 1u;
      wg::fence();
      if constexpr (!GRAD) {
        const uint64_t a2 = dsc(A, 2);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) { wg::mma_bf16<NC, 0, 0>(acc, a2 + ks * ka, b0 + ks * kb, first); first = 1u; }
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) wg::mma_bf16<NC, 0, 0>(acc, a0 + ks * ka, b2 + ks * kb, 1u);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) wg::mma_bf16<NC, 0, 0>(acc, a1 + ks * ka, b1 + ks * kb, 1u);
      }
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) { wg::mma_bf16<NC, 0, 0>(acc, a1 + ks * ka, b0 + ks * kb, first); first = 1u; }
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) wg::mma_bf16<NC, 0, 0>(acc, a0 + ks * ka, b1 + ks * kb, 1u);
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) wg::mma_bf16<NC, 0, 0>(acc, a0 + ks * ka, b0 + ks * kb, 1u);
      wg::commit();
    }
    wg::wait<1>();
  }
  wg::wait<0>();
  wg::reg_fence<NC / 2>(acc);
  if constexpr (EPI == EPI_ACT) {
#define GOPS_DENSE_EPI(A) gemm_epilogue<EPI, NC, A>(g, acc, r0, split)
    GOPS_ACT_SWITCH(g.act, GOPS_DENSE_EPI)
#undef GOPS_DENSE_EPI
  } else {
    gemm_epilogue<EPI, NC, GOPS_ACT_LINEAR>(g, acc, r0, split);
  }
}

template <int EPI, bool GRAD>
__device__ __forceinline__ void dense_gemm_tile(const GemmArgs& g, unsigned char* dsm) {
  switch (nc_of(g.n)) {
    case 16: dense_gemm_body<EPI, GRAD, 16>(g, dsm); break;
    case 32: dense_gemm_body<EPI, GRAD, 32>(g, dsm); break;
    case 64: dense_gemm_body<EPI, GRAD, 64>(g, dsm); break;
    default: dense_gemm_body<EPI, GRAD, 128>(g, dsm); break;
  }
}

template <int EPI, bool GRAD>
__global__ void __launch_bounds__(NTH, 1) dense_gemm_kernel(const __grid_constant__ GemmArgs g) {
  extern __shared__ __align__(128) unsigned char dsm[];
  dense_gemm_tile<EPI, GRAD>(g, dsm);
}

// Two networks of identical shape in one launch (twin critics): blockIdx.z selects the network, every CTA of network z
// computes exactly the tile the single-network kernel computes for it.
struct GemmPair {
  GemmArgs g[2];
};
template <int EPI, bool GRAD>
__global__ void __launch_bounds__(NTH, 1) dense_gemm_pair_kernel(const __grid_constant__ GemmPair p) {
  extern __shared__ __align__(128) unsigned char dsm[];
  dense_gemm_tile<EPI, GRAD>(p.g[blockIdx.z], dsm);
}

inline size_t gemm_smem(int n, bool grad) { return 128 + 2 * ((size_t)(grad ? 2 : 3) * 8 * TM * 16 + slice_bytes(nc_of(n))); }

// dW partial of one (128 output features, <= 128 input features) block over a chunk of the rows:
// grid = (n blocks * k blocks, row chunks).  A = dY^T (2 planes), B = X^T (2 planes), contraction over rows: the planes are
// the K-major images of the [row][feature] tiles, read MN-major (wgmma.cuh), three terms a1b0 + a0b1 + a0b0.
// The rows may be spread over `nslots` equally shaped slabs (the per-step slots of a rollout): slab s of dY starts at
// dY + s * sy * ldy, of X at X + s * sx * ldx, each with `rows` valid rows -> ONE contraction over all steps and samples.
struct WgradArgs {
  const float* dY; int ldy; const float* X; int ldx; long long rows; int n, k;
  float* partial;            // [row chunks][n][k]
  int tiles_per_chunk;
  int nslots; long long sy, sx;
};
template <int KW>
__device__ __forceinline__ void dense_wgrad_body(const WgradArgs& g, unsigned char* dsm, int n0, int k0) {
  constexpr int PL = 16 * TM * 16;                            // one plane: 128 features = 16 chunks x 128 rows x 16 B
  unsigned char* Yp = dsm + 128;
  unsigned char* Xp = Yp + 2 * PL;
  const int tid = threadIdx.x, wgi = tid >> 7, tw = tid & 127;
  const long long t0 = (long long)blockIdx.y * g.tiles_per_chunk;
  const long long tps = (g.rows + TM - 1) / TM, ttot = tps * g.nslots;      // tiles per slab, tiles in total
  uint32_t first = 0u;
  float acc[KW / 2];
#pragma unroll
  for (int i = 0; i < KW / 2; ++i) acc[i] = 0.f;
  // tile q of row tile tt: q = 0 / 1 the dY columns [n0, n0 + 64) / [n0 + 64, n0 + 128), q = 2 / 3 the X columns
  auto load_q = [&](long long tt, int q, TileRegs& r) {
    const long long slab = tt / tps, r0 = (tt - slab * tps) * TM;
    if (q < 2) load_tile(g.dY + slab * g.sy * g.ldy, g.ldy, r0, g.rows, n0 + 64 * q, g.n, r);
    else load_tile(g.X + slab * g.sx * g.ldx, g.ldx, r0, g.rows, k0 + 64 * (q - 2), g.k, r);
  };
  auto store_q = [&](int q, const TileRegs& r) { store_tile<2>(r, (q < 2 ? Yp : Xp) + (q & 1) * 8 * TM * 16, PL); };
  constexpr int NQ = KW > 64 ? 4 : 3;
  // each tile is loaded and stored in turn (no prefetch across the MMAs: three or four tiles held in registers next to
  // up to 64 accumulator registers per thread spill)
  TileRegs rt;
  for (int t = 0; t < g.tiles_per_chunk; ++t) {
    const long long tt = t0 + t;
    if (tt >= ttot) break;
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
      load_q(tt, q, rt);
      store_q(q, rt);
    }
    fence_proxy_async();
    __syncthreads();
    {
      using namespace tcf;
      // M = this warpgroup's 64 output features (chunks 8 wgi ..), N = input features, K = the tile's 128 rows
      const Op A{smem_u32(Yp) + (uint32_t)(8 * TM * 16) * wgi, (uint32_t)PL, 128u, 2048u, 256u};
      const Op B{smem_u32(Xp), (uint32_t)PL, 128u, 2048u, 256u};
      const uint64_t ka = A.kadv >> 4, kbv = B.kadv >> 4;
      const uint64_t a0 = dsc(A, 0), a1 = dsc(A, 1), b0 = dsc(B, 0), b1 = dsc(B, 1);
      wg::fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) { wg::mma_bf16<KW, 1, 1>(acc, a1 + ks * ka, b0 + ks * kbv, first); first = 1u; }
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) wg::mma_bf16<KW, 1, 1>(acc, a0 + ks * ka, b1 + ks * kbv, 1u);
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) wg::mma_bf16<KW, 1, 1>(acc, a0 + ks * ka, b0 + ks * kbv, 1u);
      wg::commit();
    }
    wg::wait<0>();
    __syncthreads();                                                     // both warpgroups are done with the planes
  }
  wg::reg_fence<KW / 2>(acc);
  // epilogue: fragment row = output feature, column = input feature
  float* out = g.partial + (size_t)blockIdx.y * g.n * g.k;
#pragma unroll
  for (int i = 0; i < KW / 2; ++i) {
    const int n = n0 + 64 * wgi + wg::frag_row(tw, i), k = k0 + wg::frag_col(tw, i);
    if (n < g.n && k < g.k) out[(size_t)n * g.k + k] = first ? acc[i] : 0.f;     // a chunk past the last row writes zeros
  }
}

// dW partial of one (128 output features, <= 128 input features) block over a chunk of the rows
__device__ __forceinline__ void dense_wgrad_block(const WgradArgs& g, unsigned char* dsm) {
  const int kb = (g.k + 127) / 128, nb_i = blockIdx.x / kb, kb_i = blockIdx.x % kb;
  const int n0 = nb_i * 128, k0 = kb_i * 128;
  const int kw = (g.k - k0) < 128 ? (g.k - k0) : 128;                   // input features of this block
  if (kw <= 16) dense_wgrad_body<16>(g, dsm, n0, k0);
  else if (kw <= 32) dense_wgrad_body<32>(g, dsm, n0, k0);
  else if (kw <= 64) dense_wgrad_body<64>(g, dsm, n0, k0);
  else dense_wgrad_body<128>(g, dsm, n0, k0);
}
__global__ void __launch_bounds__(NTH, 1) dense_wgrad_kernel(const __grid_constant__ WgradArgs g) {
  extern __shared__ __align__(128) unsigned char dsm[];
  dense_wgrad_block(g, dsm);
}
struct WgradPair {
  WgradArgs g[2];
};
__global__ void __launch_bounds__(NTH, 1) dense_wgrad_pair_kernel(const __grid_constant__ WgradPair p) {
  extern __shared__ __align__(128) unsigned char dsm[];
  dense_wgrad_block(p.g[blockIdx.z], dsm);
}
inline size_t wgrad_smem() { return 128 + (size_t)4 * 16 * TM * 16; }

// grad[i] (+)= sum_c partial[c][i] in fixed chunk order
__device__ __forceinline__ void dense_reduce_elem(const float* __restrict__ partial, int chunks, long long n,
                                                  float* __restrict__ grad, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int c = 0; c < chunks; ++c) s += partial[(size_t)c * n + i];
  grad[i] = accumulate ? grad[i] + s : s;
}
__global__ void dense_reduce_kernel(const float* __restrict__ partial, int chunks, long long n, float* __restrict__ grad,
                                    int accumulate) {
  dense_reduce_elem(partial, chunks, n, grad, accumulate);
}
// the same for two networks (blockIdx.z)
__global__ void dense_reduce_pair_kernel(const float* __restrict__ partial0, const float* __restrict__ partial1, int chunks,
                                         long long n, float* __restrict__ grad0, float* __restrict__ grad1, int accumulate) {
  dense_reduce_elem(blockIdx.z ? partial1 : partial0, chunks, n, blockIdx.z ? grad1 : grad0, accumulate);
}
// db[n] (+)= sum_r dY[r][n]: one warp per (column, row chunk) pair would be the fast way; the layer widths here are
// <= 256 and this is 0.1 % of the update, so: block = 32 columns x 8 row-lanes, fixed-order tree, partials per block row
__device__ __forceinline__ void dense_colsum_block(const float* __restrict__ dY, int ld, long long rows, int n,
                                                   float* __restrict__ partial, long long rows_per_block, int nslots,
                                                   long long sy, float (*sm)[33]) {
  const int c = blockIdx.x * 32 + threadIdx.x, ry = threadIdx.y;
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
  float s = 0.f;
  if (c < n)
    for (int sl = 0; sl < nslots; ++sl) {
      const float* base = dY + (size_t)sl * sy * ld;
      for (long long r = r0 + ry; r < r1; r += 8) s += base[r * ld + c];
    }
  sm[ry][threadIdx.x] = s;
  __syncthreads();
  if (ry == 0 && c < n) {
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += sm[j][threadIdx.x];
    partial[(size_t)blockIdx.y * n + c] = t;
  }
}
__global__ void dense_colsum_kernel(const float* __restrict__ dY, int ld, long long rows, int n, float* __restrict__ partial,
                                    long long rows_per_block, int nslots, long long sy) {
  __shared__ float sm[8][33];
  dense_colsum_block(dY, ld, rows, n, partial, rows_per_block, nslots, sy, sm);
}
// the same for two networks (blockIdx.z); both read `ld` floats per row of their dY
__global__ void dense_colsum_pair_kernel(const float* __restrict__ dY0, const float* __restrict__ dY1, int ld, long long rows,
                                         int n, float* __restrict__ partial0, float* __restrict__ partial1,
                                         long long rows_per_block) {
  __shared__ float sm[8][33];
  dense_colsum_block(blockIdx.z ? dY1 : dY0, ld, rows, n, blockIdx.z ? partial1 : partial0, rows_per_block, 1, 0, sm);
}

}  // namespace dense
}  // namespace gops
