// MinAtar CNN conv device code shared by the conv kernels of pqn_net.cu and the conv-fused dense forward GEMM of
// pqn_tc.cu: the packed-observation patch words, the fp16 mma.sync conv chain, its quad LayerNorm and the fp16 split
// of the activation.  One copy, so that every kernel that computes h1 lands on the same bits.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pqn_b200.h"
#include "tc_common.cuh"

namespace pqn {

constexpr float LN_EPS = 1e-6f;
constexpr int CONV_O = 16;   // conv output channels
constexpr int CONV_PIX = 64; // 8x8 output pixels
constexpr int HID_CNN = 128;
constexpr int FLAT_CNN = CONV_PIX * CONV_O;  // 1024

template <int C>
struct ConvCfg {
  static constexpr int TAPS = 9 * C;
  static constexpr int OBS_BITS = 100 * C;
  static constexpr int OBS_WORDS = (OBS_BITS + 31) / 32;
  static constexpr int PW = (OBS_WORDS + 3) / 4 * 4;       // packed row words (matches env OBS_WORDS_PAD)
  static constexpr int SW = PW + 1;                        // smem row (+1 so the funnel shift may read past the end)
};

// im2col "patch" of one output pixel as bits: bit k = tap k = (di*3+dj)*C + c, i.e. obs bit
// ((y+di)*10 + x+dj)*C + c.  9C <= 90 bits -> PatchCfg::WORDS words; bits beyond 9C are zero.  Built once per
// sample into shared memory (patch[pixel][word]); the MMA fragment builders then test bits with a shift instead of
// re-deriving the observation bit address for every (pixel, tap) pair.
template <int C>
struct PatchCfg {
  static constexpr int WORDS = (9 * C + 31) / 32;
};

// The 9C patch bits of output pixel `pix` as PatchCfg::WORDS words.  The packed observation is pixel-major /
// channel-minor, so the three taps (dj = 0..2) x C channels of one patch row are 3C CONSECUTIVE bits of the input row:
// three funnel-shift extracts instead of nine per-pixel ones.
template <int C>
__device__ __forceinline__ void patch_bits(const uint32_t* __restrict__ so, int pix, uint32_t (&w)[PatchCfg<C>::WORDS]) {
  constexpr int W = PatchCfg<C>::WORDS;
#pragma unroll
  for (int k = 0; k < W; ++k) w[k] = 0u;
  const int y = pix >> 3, x = pix & 7;
#pragma unroll
  for (int di = 0; di < 3; ++di) {
    const int f0 = ((y + di) * 10 + x) * C;
    const uint32_t r = __funnelshift_r(so[f0 >> 5], so[(f0 >> 5) + 1], f0 & 31) & ((1u << (3 * C)) - 1u);
    const int o = 3 * C * di;  // compile-time after unrolling
    w[o >> 5] |= r << (o & 31);
    if ((o & 31) + 3 * C > 32) w[min((o >> 5) + 1, W - 1)] |= r >> (32 - (o & 31));
  }
}

// LayerNorm statistics over the 16 channels of pixel rows g (z[.][0..1]) and g+8 (z[.][2..3]); quad reduction.
// Every rounding is spelled out (no FMA contraction left to the compiler): the fp16 conv backward rebuilds rstd and
// xhat with this function and must land on the training forward's bits.
__device__ __forceinline__ void ln16_quad(const float (&z)[2][4], float& mean0, float& rstd0, float& mean1,
                                          float& rstd1) {
  float s0 = z[0][0] + z[0][1] + z[1][0] + z[1][1];
  float q0 = fmaf(z[1][1], z[1][1], fmaf(z[1][0], z[1][0], fmaf(z[0][0], z[0][0], __fmul_rn(z[0][1], z[0][1]))));
  float s1 = z[0][2] + z[0][3] + z[1][2] + z[1][3];
  float q1 = fmaf(z[1][3], z[1][3], fmaf(z[1][2], z[1][2], fmaf(z[0][2], z[0][2], __fmul_rn(z[0][3], z[0][3]))));
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o); q0 += __shfl_xor_sync(0xffffffffu, q0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o); q1 += __shfl_xor_sync(0xffffffffu, q1, o);
  }
  mean0 = __fmul_rn(s0, 1.0f / CONV_O); mean1 = __fmul_rn(s1, 1.0f / CONV_O);
  // MUFU.RSQ (2 ulp) instead of the IEEE 1/sqrt sequence, whose slow-path branches cost more than the conv MMAs
  rstd0 = rsqrtf(fmaxf(fmaf(q0, 1.0f / CONV_O, -__fmul_rn(mean0, mean0)), 0.f) + LN_EPS);
  rstd1 = rsqrtf(fmaxf(fmaf(q1, 1.0f / CONV_O, -__fmul_rn(mean1, mean1)), 0.f) + LN_EPS);
}

// ---------------------------------------------------------------------------------------------------------------
// conv forward on fp16 warp-level MMA (mma.sync.m16n8k16, fp32 accumulate) -- the default conv path of round 2.
// Same structure as conv_fwd_mma_kernel (one sample per warp, quad-level LayerNorm), but
//   * the {0,1} im2col operand is fp16 and "exponent coded": per output pixel and k-step of 16 taps two words hold the
//     tap bits at the exponent bits 10..13 of the low half and 26..29 of the high half; lane t of the fragment masks
//     bit (10 + t) / (26 + t), which turns a set bit into the fp16 power of two 2^(2^t - 15) (one LOP3 per register
//     that carries TWO k values) and row k of B is pre-multiplied by the inverse power of two (exact), so every product
//     equals the plain 0/1 product;
//   * weights/255 are split into fp16 hi + lo (22 significant bits, like the tf32 hi/lo pair);
//   * K = 9C taps padded to 16 needs ceil(9C/16) k-steps (3 for C = 4) instead of ceil(9C/8) = 5 tf32 ones: 48 MMAs
//     and 48 fragment LOP3s per sample instead of 80 / 80 (the tf32 kernel's top stall was the mma.sync pipe).
// k order inside a k-step (free to choose, B is laid out to match): fragment column 2t <-> tap 16s + t,
// 2t+1 <-> 16s + 4 + t, 2t+8 <-> 16s + 8 + t, 2t+9 <-> 16s + 12 + t.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_f16_16n8k16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int C>
struct Conv16 {
  static constexpr int TAPS = 9 * C;
  static constexpr int KS = (TAPS + 15) / 16;          // k-steps of 16 taps
  static constexpr int ROW = 2 * KS < 8 ? 8 : 2 * KS;  // padded row: 8 or 12 words keep the 4-row LDS.64 groups apart
};

// Output channel of column n (0..7) of n-tile h.  NOT the natural 8h + n: with 4 (n / 2) + 2h + (n % 2) the accumulator
// columns (2t, 2t+1) of the two n-tiles are the four CONSECUTIVE channels 4t .. 4t+3 of a pixel, so a thread stores 16
// bytes of fp32 h1 / 8 bytes of each fp16 plane per pixel with one instruction and no lane exchange (the kernel's time
// follows its store instructions).
__host__ __device__ constexpr int conv16_channel(int h, int n) { return 4 * (n >> 1) + 2 * h + (n & 1); }

// tap of fragment column kk (0..15) of k-step s, see the k order above
__host__ __device__ constexpr int conv16_tap(int s, int kk) {
  return 16 * s + (kk < 8 ? 0 : 8) + ((kk & 1) ? 4 : 0) + ((kk & 7) >> 1);
}

// B fragments of weights/255 as fp16 (hi, lo), pre-scaled by the inverse of the A coding: wb[s][h][lane] = uint4
// {b0_hi, b1_hi, b0_lo, b1_lo} (b0 = columns k = 2t, 2t+1; b1 = k = 2t+8, 2t+9; n = 8h + g)
// Threads tid = 0 .. nt - 1 of the block take part (the conv kernels: all of them; the fused GEMM: its consumers).
template <int C>
__device__ __forceinline__ void conv16_load_weights(const float* __restrict__ prm, const pqn_net_layout_t& L, uint4* wb,
                                                    float* cb, float* sc, float* bi, int tid, int nt) {
  using M = Conv16<C>;
  const float inv255 = 1.0f / 255.0f;
  for (int i = tid; i < M::KS * 2 * 32; i += nt) {
    const int ln = i & 31, h = (i >> 5) & 1, s = i >> 6;
    const int gg = ln >> 2, tt = ln & 3;
    const int o = conv16_channel(h, gg);
    const float scale = __uint_as_float((uint32_t)(127 + 15 - (1 << tt)) << 23);   // 2^(15 - 2^t), exact
    float v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {   // q: 0 -> k=2t, 1 -> 2t+1, 2 -> 2t+8, 3 -> 2t+9
      const int tap = conv16_tap(s, 2 * tt + (q & 1) + (q >> 1) * 8);
      v[q] = tap < M::TAPS ? __ldg(prm + L.conv_w + tap * CONV_O + o) * inv255 * scale : 0.f;
      v[q] = fminf(fmaxf(v[q], -65000.f), 65000.f);
    }
    const __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
    const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
    const __half2 l0 = __floats2half2_rn(v[0] - f0.x, v[1] - f0.y), l1 = __floats2half2_rn(v[2] - f1.x, v[3] - f1.y);
    wb[i] = make_uint4(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1),
                       *reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
  }
  if (tid < CONV_O) {
    cb[tid] = __ldg(prm + L.conv_b + tid);
    sc[tid] = __ldg(prm + L.ln0_scale + tid);
    bi[tid] = __ldg(prm + L.ln0_bias + tid);
  }
}

// exponent-coded fp16 patch words of one output pixel: out[2s], out[2s+1] for k-step s (taps 16s..16s+7, 16s+8..16s+15).
// Only bits 10..13 and 26..29 are meaningful (the fragment mask picks one of them per half); tap 16s+j, j<4 sits at bit
// 10+j and tap 16s+4+j at bit 26+j.
template <int C>
__device__ __forceinline__ void build_patch16(const uint32_t* __restrict__ so, int pix, uint32_t* __restrict__ out) {
  constexpr int W = PatchCfg<C>::WORDS;
  uint32_t w[W];
  patch_bits<C>(so, pix, w);
#pragma unroll
  for (int b = 0; b < 2 * Conv16<C>::KS; ++b) {
    const int o = 8 * b;                                   // bit offset of this byte in the patch string
    uint32_t v = (o >> 5) < W ? w[(o >> 5) < W ? (o >> 5) : 0] : 0u;
    const int sh = o & 31;
    const uint32_t lo = sh >= 10 ? v >> (sh - 10) : v << (10 - sh);          // bits sh..sh+3   -> 10..13
    const uint32_t hi = sh + 4 <= 26 ? v << (26 - sh - 4) : v >> (sh + 4 - 26);  // bits sh+4..sh+7 -> 26..29
    out[b] = __byte_perm(lo, hi, 0x7610);                  // low half from lo, high half from hi
  }
}

// patch row of one pixel -> shared memory with 128-bit stores (ROW is 8 or 12 words; pad words are never read)
template <int C>
__device__ __forceinline__ void store_patch16(const uint32_t* __restrict__ so, int pix, uint32_t* __restrict__ row) {
  using M = Conv16<C>;
  uint32_t w[M::ROW];
#pragma unroll
  for (int k = 0; k < M::ROW; ++k) w[k] = 0u;
  build_patch16<C>(so, pix, w);
#pragma unroll
  for (int q = 0; q < M::ROW / 4; ++q)
    *reinterpret_cast<uint4*>(row + 4 * q) = make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
}

// conv output z of NB blocks of 16 pixels from patch rows ra (fragment row g of block 0), rb (row g + 8 of block 0) and
// ra / rb + i * BSTRIDE words for block i; cb4 = conv bias of the thread's channels 4t .. 4t+3.  PAIRED: the two rows
// are interleaved per k-step at ra (words 4s, 4s+1 of row g, 4s+2, 4s+3 of row g + 8: one 16-byte load; rb unused).
// Which pixel feeds which fragment row does not change any accumulator's MMA sequence, so every caller gets the same
// bits per pixel.
template <int C, int NB, int BSTRIDE, bool PAIRED = false>
__device__ __forceinline__ void conv16_blocks_rows(const uint32_t* __restrict__ ra, const uint32_t* __restrict__ rb,
                                                   const uint4* __restrict__ wb, const float (&cb4)[4], int lane,
                                                   float (&z)[NB][2][4]) {
  using M = Conv16<C>;
  const int t = lane & 3;
  const uint32_t mask = (1u << (10 + t)) | (1u << (26 + t));
#pragma unroll
  for (int i = 0; i < NB; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      z[i][h][0] = z[i][h][2] = cb4[2 * h];       // conv16_channel(h, 2t), (h, 2t + 1)
      z[i][h][1] = z[i][h][3] = cb4[2 * h + 1];
    }
#pragma unroll
  for (int s = 0; s < M::KS; ++s) {
    uint32_t a[NB][4];
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      uint2 w0, w1;   // fragment rows g and g + 8
      if (PAIRED) {
        const uint4 v = *reinterpret_cast<const uint4*>(ra + i * BSTRIDE + 4 * s);
        w0 = make_uint2(v.x, v.y); w1 = make_uint2(v.z, v.w);
      } else {
        w0 = *reinterpret_cast<const uint2*>(ra + i * BSTRIDE + 2 * s);
        w1 = *reinterpret_cast<const uint2*>(rb + i * BSTRIDE + 2 * s);
      }
      a[i][0] = w0.x & mask; a[i][1] = w1.x & mask; a[i][2] = w0.y & mask; a[i][3] = w1.y & mask;
    }
    uint4 b[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) b[h] = wb[(s * 2 + h) * 32 + lane];
    // lo pass of all accumulators, then the hi pass: no back-to-back dependent MMAs
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NB; ++i) mma_f16_16n8k16(z[i][h], a[i], b[h].z, b[h].w);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NB; ++i) mma_f16_16n8k16(z[i][h], a[i], b[h].x, b[h].y);
  }
}

// conv output z of the NB m-blocks mb0 .. mb0 + NB - 1 (m-block mb = pixels 16 mb .. 16 mb + 15): z[i] holds pixel
// rows 16 (mb0 + i) + g and + 8.  The training forward runs two m-blocks at a time; every accumulator sees the same MMA
// sequence however many blocks share a call, so the backward's rebuild (conv16_blocks_rows) gets the same bits.
template <int C, int NB>
__device__ __forceinline__ void conv16_blocks(const uint32_t* __restrict__ xp, const uint4* __restrict__ wb,
                                              const float* __restrict__ cb, int mb0, int lane, float (&z)[NB][2][4]) {
  using M = Conv16<C>;
  const int g = lane >> 2, t = lane & 3;
  const float cb4[4] = {cb[4 * t], cb[4 * t + 1], cb[4 * t + 2], cb[4 * t + 3]};
  const uint32_t* r00 = xp + (16 * mb0 + g) * M::ROW;
  conv16_blocks_rows<C, NB, 16 * M::ROW>(r00, r00 + 8 * M::ROW, wb, cb4, lane, z);
}

// LayerNorm of one m-block of conv16_blocks: xhat of pixel rows 16 mb + g (x0) and + 8 (x1) in the thread's channels
// 4t .. 4t+3, and the rows' rstd.  xhat = z * rstd - mean * rstd: one FFMA per element.
__device__ __forceinline__ void conv16_xhat(const float (&z)[2][4], float (&x0)[4], float (&x1)[4], float& rstd0,
                                            float& rstd1) {
  float mean0, mean1;
  ln16_quad(z, mean0, rstd0, mean1, rstd1);
  const float nm0 = -__fmul_rn(mean0, rstd0), nm1 = -__fmul_rn(mean1, rstd1);
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      x0[2 * h + c] = fmaf(z[h][c], rstd0, nm0);
      x1[2 * h + c] = fmaf(z[h][2 + c], rstd1, nm1);
    }
}

__device__ __forceinline__ uint32_t cvt_f16x2_satfinite(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// h1 of pixel rows 16 mb + g (v0) and + 8 (v1) from conv16_blocks' z: LayerNorm, scale / bias, ReLU in the thread's
// channels 4t .. 4t+3, whose LayerNorm scale and bias are sc4 / bi4.
__device__ __forceinline__ void conv16_act(const float (&z)[2][4], const float (&sc4)[4], const float (&bi4)[4],
                                           float (&v0)[4], float (&v1)[4]) {
  float x0[4], x1[4], rstd0, rstd1;
  conv16_xhat(z, x0, x1, rstd0, rstd1);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    v0[c] = fmaxf(fmaf(x0[c], sc4[c], bi4[c]), 0.f);
    v1[c] = fmaxf(fmaf(x1[c], sc4[c], bi4[c]), 0.f);
  }
}

// fp16 split planes of four consecutive channels of h1 (>= 0): hi = fp16(v) (saturating: no inf),
// lo' = fp16((v - hi) * 2^11); hw[h] / lw[h] = channels 2h, 2h + 1 as one f16x2 word each
__device__ __forceinline__ void conv16_split(const float (&v)[4], uint32_t (&hw)[2], uint32_t (&lw)[2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    hw[h] = cvt_f16x2_satfinite(v[2 * h], v[2 * h + 1]);
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hw[h]));
    const __half2 l = __floats2half2_rn((v[2 * h] - f.x) * tc::TC_LO_SCALE, (v[2 * h + 1] - f.y) * tc::TC_LO_SCALE);
    lw[h] = *reinterpret_cast<const uint32_t*>(&l);
  }
}

namespace tc {
// conv input of the conv-fused dense forward GEMM (pqn_tc.cu): packed observation rows [S][rows_per_seed][PW] read
// through the optional minibatch index gather[S][M], and the network layout for the conv parameters
struct ConvIn {
  const uint32_t* obs;
  int64_t obs_rows_per_seed;
  const int32_t* gather;
  pqn_net_layout_t L;
};
// Z = conv(obs) . W1 with the LayerNorm epilogue EPI (EPI_LN_HEAD; the kernel takes EPI_LN_TRAIN as well, but the
// training forward does not use it and it is not instantiated): tb = {W1 hi, W1 lo'} fp16 maps
// ([S][1024][128], boxes of 64 rows), gs.M rows per seed, gs.S seeds; C in {4, 6, 7, 10}
int launch_conv_gemm16(int C, int epi, const CUtensorMap* tb, const GemmShape& gs, const EpiParams& ep, const ConvIn& ci,
                       cudaStream_t st, int kernel_id);
}  // namespace tc


}  // namespace pqn
