// wgmma / TMA path for the dense contractions of the Q-network (sm_90a): one
// warp-specialised, persistent GEMM kernel used for
//   forward   Z  = H1 [rows,1024] . W1 [1024,128]        (A K-major,  B MN-major)
//   wgrad     dW = H1^T [1024,rows] . dZ [rows,128]      (A MN-major, B MN-major)
//   dgrad     dX = dZ [rows,128] . W1^T [128,1024]       (A K-major,  B K-major)
// with fp32 accuracy from fp16-split operands: every operand x is fed as the
// planes hi = fp16(x), lo' = fp16((x - hi) * 2^11) (pqn_tc_split16), and
// D = A_hi.B_hi + (A_lo'.B_hi + A_hi.B_lo') * 2^-11 accumulates in fp32.
//
// Reference arithmetic: nn.Dense(128) of CNN (purejaxql/pqn_minatar.py:48) and
// its autodiff; XLA itself runs these as TF32 tensor-core GEMMs on GPU.
//
// Pipeline (per CTA, 288 threads, one CTA per SM, 128 x 128 output tiles):
//   warp 8      TMA producer   cp.async.bulk.tensor (SWIZZLE_128B boxes) -> 2-stage smem ring
//   warps 0-7   consumers      two warpgroups, rows 0-63 / 64-127 of the tile: wgmma m64n128k16 into register
//                              accumulators, promotion into an fp32 tile in shared memory, then the epilogue
// Barriers: full[stage] (TMA -> consumers, tx bytes), empty[stage] (8 consumer warps -> TMA).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pqn_b200.h"
#include "api_common.h"
#include "tc_common.cuh"
#include "conv16.cuh"

namespace pqn {
namespace tc {

// ---------------------------------------------------------------------------
// LayerNorm epilogues: each of the 128 threads of warps 0-3 owns one row of the 128x128 tile, read from the fp32
// tile into registers (acc[128], fully unrolled static indexing)
// ---------------------------------------------------------------------------
// Coalesced tile-row-block store: the warp's 32 rows x 32 columns chunk goes through a padded shared-memory
// stage so that 8 lanes write one 128-byte row segment (4 rows per store instruction) instead of 32 lanes
// writing 32 different rows.  `vals` = this lane's row, columns [0,32) of the chunk.
constexpr int STG_LD = 36;  // floats per staged row (16-byte aligned, conflict-free for 128-bit accesses)

__device__ __forceinline__ void store_chunk_coalesced(float* stage, const float (&vals)[32], int lane, float* dst,
                                                      int64_t ld, int m_base, int M) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
    *reinterpret_cast<float4*>(stage + lane * STG_LD + 4 * j) =
        make_float4(vals[4 * j], vals[4 * j + 1], vals[4 * j + 2], vals[4 * j + 3]);
  __syncwarp();
  const int r_in = lane >> 3, c4 = lane & 7;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int r = it * 4 + r_in;
    if (m_base + r < M)
      *reinterpret_cast<float4*>(dst + (int64_t)r * ld + 4 * c4) = *reinterpret_cast<const float4*>(stage + r * STG_LD + 4 * c4);
  }
  __syncwarp();
}

// Shared-memory copy of the per-seed epilogue parameters (LN epilogues), staged once per tile by the 128 epilogue
// threads: every thread needs all of them, and 128-bit broadcast reads cost a quarter of the per-element loads.
constexpr int SP_B = 0, SP_SC = 128, SP_BI = 256, SP_HW = 384 /* [PQN_TC_MAX_A][128] */,
              SP_HB = SP_HW + PQN_TC_MAX_A * 128, SP_FLOATS = SP_HB + PQN_TC_MAX_A;
static_assert(SP_FLOATS == TC_SP_FLOATS, "matches the TC_SMEM_BYTES budget in tc_common.cuh");

__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
__device__ __forceinline__ void consumer_bar_sync() { asm volatile("bar.sync 2, 256;" ::: "memory"); }

template <int EPI>
__device__ __forceinline__ void stage_epi_params(const EpiParams& ep, float* sp, int seed, int et /*0..127*/) {
  const float* __restrict__ prm = ep.params + (int64_t)seed * ep.P;
  epi_bar_sync();  // everyone is done with the previous tile's parameters
  sp[SP_B + et] = __ldg(prm + ep.off_b + et);
  sp[SP_SC + et] = __ldg(prm + ep.off_scale + et);
  sp[SP_BI + et] = __ldg(prm + ep.off_bias + et);
  if constexpr (EPI == EPI_LN_HEAD) {
    for (int a = 0; a < ep.A; ++a) sp[SP_HW + a * 128 + et] = __ldg(prm + ep.off_hw + (int64_t)et * ep.A + a);
    if (et < ep.A) sp[SP_HB + et] = __ldg(prm + ep.off_hb + et);
  }
  epi_bar_sync();
}

// bias + LayerNorm(128) + ReLU, then either (h, xhat, rstd) or the fused Q-head.  `m_base` = first row of this warp's
// 32-row block; the lane's own row is m_base + lane.
template <int EPI>
__device__ __forceinline__ void epilogue_ln_row(const EpiParams& ep, float (&acc)[128], float* stage, const float* sp,
                                                int lane, int seed, int m_base, int M) {
  const int m = m_base + lane;
  const bool row_ok = m < M;
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int j4 = 0; j4 < 32; ++j4) {
    const float4 b = *reinterpret_cast<const float4*>(sp + SP_B + 4 * j4);
    const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = 4 * j4 + e;
      acc[j] += bb[e];
      s1 += acc[j];
      s2 = fmaf(acc[j], acc[j], s2);
    }
  }
  const float mean = s1 * (1.0f / 128.f);
  const float var = fmaxf(s2 * (1.0f / 128.f) - mean * mean, 0.f);
  const float rstd = 1.0f / sqrtf(var + 1e-6f);
  const int64_t grow = (int64_t)seed * ep.rows + m;
  if constexpr (EPI == EPI_LN_TRAIN) {
    float* hbase = ep.H + ((int64_t)seed * ep.rows + m_base) * 128;
    float* xbase = ep.XHAT + ((int64_t)seed * ep.rows + m_base) * 128;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float xh[32], h[32];
#pragma unroll
      for (int j4 = 0; j4 < 8; ++j4) {
        const float4 s4 = *reinterpret_cast<const float4*>(sp + SP_SC + c * 32 + 4 * j4);
        const float4 b4 = *reinterpret_cast<const float4*>(sp + SP_BI + c * 32 + 4 * j4);
        const float ss[4] = {s4.x, s4.y, s4.z, s4.w}, bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int j = 4 * j4 + e;
          xh[j] = (acc[c * 32 + j] - mean) * rstd;
          h[j] = fmaxf(xh[j] * ss[e] + bb[e], 0.f);
        }
      }
      store_chunk_coalesced(stage, h, lane, hbase + c * 32, 128, m_base, M);
      store_chunk_coalesced(stage, xh, lane, xbase + c * 32, 128, m_base, M);
    }
    if (row_ok) ep.RSTD[grow] = rstd;
  } else {  // EPI_LN_HEAD
    float q[PQN_TC_MAX_A];
#pragma unroll
    for (int a = 0; a < PQN_TC_MAX_A; ++a) q[a] = 0.f;
#pragma unroll
    for (int j4 = 0; j4 < 32; ++j4) {
      const float4 s4 = *reinterpret_cast<const float4*>(sp + SP_SC + 4 * j4);
      const float4 b4 = *reinterpret_cast<const float4*>(sp + SP_BI + 4 * j4);
      float h[4];
      h[0] = fmaxf((acc[4 * j4 + 0] - mean) * rstd * s4.x + b4.x, 0.f);
      h[1] = fmaxf((acc[4 * j4 + 1] - mean) * rstd * s4.y + b4.y, 0.f);
      h[2] = fmaxf((acc[4 * j4 + 2] - mean) * rstd * s4.z + b4.z, 0.f);
      h[3] = fmaxf((acc[4 * j4 + 3] - mean) * rstd * s4.w + b4.w, 0.f);
#pragma unroll
      for (int a = 0; a < PQN_TC_MAX_A; ++a)
        if (a < ep.A) {
          const float4 w4 = *reinterpret_cast<const float4*>(sp + SP_HW + a * 128 + 4 * j4);
          q[a] = fmaf(h[0], w4.x, q[a]); q[a] = fmaf(h[1], w4.y, q[a]);
          q[a] = fmaf(h[2], w4.z, q[a]); q[a] = fmaf(h[3], w4.w, q[a]);
        }
    }
    if (row_ok) {
#pragma unroll
      for (int a = 0; a < PQN_TC_MAX_A; ++a)
        if (a < ep.A) ep.Q[grow * ep.A + a] = q[a] + sp[SP_HB + a];
    }
  }
}

// ---------------------------------------------------------------------------
// TF32 consumers (3xTF32 / single-pass).  Hopper's wgmma reads 32-bit operands only K-major, and the forward and
// weight-gradient products have MN-major operands, so this variant runs warp-level mma.sync.m16n8k8.tf32 on fragments
// read from the same TMA ring (SWIZZLE_128B tiles of 128 rows x 32 fp32).  Warp w owns tile rows 32 (w % 4) .. +31 and
// columns 64 (w / 4) .. +63: 2 x 8 MMAs per k-step and product.
// ---------------------------------------------------------------------------
// fp32 element (r = M or N index, k) of a 128 x 32 operand tile as TMA writes it with SWIZZLE_128B:
//   K-major : 128-byte rows r, 16-byte chunk (k / 4) ^ (r % 8)
//   MN-major: 4 boxes of [32 k rows][32 mn] at 4096 B, 128-byte rows k, chunk ((r % 32) / 4) ^ (k % 8)
template <int MN>
__device__ __forceinline__ float lds_tf32(const uint8_t* tile, int r, int k) {
  const int off = MN ? ((r >> 5) * 4096 + k * 128 + ((((r & 31) >> 2) ^ (k & 7)) << 4) + ((r & 3) << 2))
                     : (r * 128 + (((k >> 2) ^ (r & 7)) << 4) + ((k & 3) << 2));
  return *reinterpret_cast<const float*>(tile + off);
}
__device__ __forceinline__ uint32_t tf32_trunc_bits(float x) { return __float_as_uint(x) & 0xFFFFE000u; }
__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// One output tile into tile_s (promotion as in the fp16 path; the cross products are in the units of the result).
// split3: 0 single TF32 pass; 1 3xTF32 with A_lo from memory; 2 3xTF32 with A_lo = A - trunc_tf32(A) in registers.
template <int A_MN, int B_MN>
__device__ __forceinline__ void tf32_tile(const uint8_t* smem_al, float* tile_s, uint64_t* full, uint64_t* empty,
                                          int& stage, uint32_t& phase, int kbn, int split3, float osc, int warp,
                                          int lane) {
  const int g = lane >> 2, tq = lane & 3;
  const int wr = (warp & 3) * 32, wc = (warp >> 2) * 64;
  float mainacc[2][8][4], corr[2][8][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 8; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) { mainacc[mi][ni][e] = 0.f; corr[mi][ni][e] = 0.f; }
  for (int kb = 0; kb < kbn; ++kb) {
    mbar_wait(&full[stage], phase);
    const uint8_t* sb = smem_al + stage * TC_STAGE_BYTES;
    if (kb % TC_PROMOTE == 0) {
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 8; ++ni)
#pragma unroll
          for (int e = 0; e < 4; ++e) mainacc[mi][ni][e] = 0.f;
    }
#pragma unroll
    for (int ks = 0; ks < TC_BK / 8; ++ks) {
      const int k = ks * 8 + tq;
      uint32_t ahi[2][4], alo[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const int r0 = wr + mi * 16 + g;
        const int rr[4] = {r0, r0 + 8, r0, r0 + 8}, kk[4] = {k, k, k + 4, k + 4};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float x = lds_tf32<A_MN>(sb + TC_A_HI, rr[e], kk[e]);
          ahi[mi][e] = tf32_trunc_bits(x);
          const float lo = split3 == 1 ? lds_tf32<A_MN>(sb + TC_A_LO, rr[e], kk[e]) : x - __uint_as_float(ahi[mi][e]);
          alo[mi][e] = tf32_trunc_bits(lo);
        }
      }
#pragma unroll
      for (int ni = 0; ni < 8; ++ni) {
        const int n = wc + ni * 8 + g;
        const uint32_t bh0 = tf32_trunc_bits(lds_tf32<B_MN>(sb + TC_B_HI, n, k));
        const uint32_t bh1 = tf32_trunc_bits(lds_tf32<B_MN>(sb + TC_B_HI, n, k + 4));
        if (split3) {
          const uint32_t bl0 = tf32_trunc_bits(lds_tf32<B_MN>(sb + TC_B_LO, n, k));
          const uint32_t bl1 = tf32_trunc_bits(lds_tf32<B_MN>(sb + TC_B_LO, n, k + 4));
#pragma unroll
          for (int mi = 0; mi < 2; ++mi) {
            mma_tf32_16x8x8(corr[mi][ni], alo[mi], bh0, bh1);
            mma_tf32_16x8x8(corr[mi][ni], ahi[mi], bl0, bl1);
          }
        }
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) mma_tf32_16x8x8(mainacc[mi][ni], ahi[mi], bh0, bh1);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);   // this warp's fragment reads of the slot are done
    if (++stage == TC_STAGES) { stage = 0; phase ^= 1u; }
    if ((kb + 1) % TC_PROMOTE == 0 || kb == kbn - 1) {
      const bool first = kb < TC_PROMOTE;
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 8; ++ni)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float2* p = reinterpret_cast<float2*>(tile_s + (wr + mi * 16 + g + 8 * h) * TC_ACC_LD + wc + ni * 8 + 2 * tq);
            const float2 v = make_float2(mainacc[mi][ni][2 * h], mainacc[mi][ni][2 * h + 1]);
            if (first) *p = v;
            else { const float2 o = *p; *p = make_float2(o.x + v.x, o.y + v.y); }
          }
    }
  }
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 8; ++ni)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2* p = reinterpret_cast<float2*>(tile_s + (wr + mi * 16 + g + 8 * h) * TC_ACC_LD + wc + ni * 8 + 2 * tq);
        float2 o = kbn > 0 ? *p : make_float2(0.f, 0.f);
        o.x += corr[mi][ni][2 * h];
        o.y += corr[mi][ni][2 * h + 1];
        *p = make_float2(o.x * osc, o.y * osc);
      }
}

// ---------------------------------------------------------------------------
// the kernel
//
// Accuracy: the tensor core's fp32 accumulation is not round-to-nearest, so a long chain of MMAs into one
// accumulator drifts.  Two-level accumulation keeps fp32 accuracy:
//   * the correction terms A_lo'.B_hi + A_hi.B_lo' (2^-11 of the result) get their own register accumulator for the
//     whole K -- their accumulation error is negligible at that magnitude;
//   * the main A_hi.B_hi chain is cut every TC_PROMOTE k-blocks (16 k-steps): the partial is added to the fp32 tile in
//     shared memory (round-to-nearest FADD) and the chain restarts with scale-d = 0.
//
// ReLU-mask epilogues of the fp16 kernel (the input gradients) finish the tile in registers and store it through TMA
// (tm_out): the mask words are loaded before the tile's MMAs, each warpgroup writes its 64 rows into a swizzled
// staging area and one thread issues the bulk store, which runs while the warpgroup goes on to the next tile's MMAs.
// The two warpgroups do not synchronise with each other.  Rows >= gs.M are clipped by the tensor map.
// ---------------------------------------------------------------------------
// Tile steps of the conv-fused kernel below, written as the fp16 path of tc_gemm_kernel writes them inline (kept
// inline there so that its code does not change); the two must stay the same arithmetic.
// main partial of the fp16 wgmma chain -> fp32 tile (first: store, else add); rows fr, fr + 8, columns 8 j + fc, + 1
__device__ __forceinline__ void promote_main(float* tile_s, const float (&mainacc)[64], int fr, int fc, bool first) {
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float2* p = reinterpret_cast<float2*>(tile_s + (fr + 8 * h) * TC_ACC_LD + 8 * j + fc);
      const float2 v = make_float2(mainacc[4 * j + 2 * h], mainacc[4 * j + 2 * h + 1]);
      if (first) *p = v;
      else { const float2 o = *p; *p = make_float2(o.x + v.x, o.y + v.y); }
    }
}

// the correction accumulator (units of 2^-11), then the power-of-two output scale (exact)
__device__ __forceinline__ void finish_corr(float* tile_s, const float (&corr)[64], int fr, int fc, int kbn, float osc) {
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float2* p = reinterpret_cast<float2*>(tile_s + (fr + 8 * h) * TC_ACC_LD + 8 * j + fc);
      float2 o = kbn > 0 ? *p : make_float2(0.f, 0.f);
      if (kbn > 0) {
        o.x = fmaf(corr[4 * j + 2 * h], TC_LO_INV, o.x);
        o.y = fmaf(corr[4 * j + 2 * h + 1], TC_LO_INV, o.y);
      }
      *p = make_float2(o.x * osc, o.y * osc);
    }
}

// LayerNorm epilogues of a finished fp32 tile: thread t < 128 takes tile row t
template <int EPI>
__device__ __forceinline__ void ln_epilogue_tile(const EpiParams& ep, float* tile_s, float* sp_all, int t, int warp,
                                                 int lane, int seed, int m0, int M) {
  stage_epi_params<EPI>(ep, sp_all, seed, t);
  float acc[128];
  const float* row = tile_s + t * TC_ACC_LD;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float4 v = *reinterpret_cast<const float4*>(row + 4 * j);
    acc[4 * j] = v.x; acc[4 * j + 1] = v.y; acc[4 * j + 2] = v.z; acc[4 * j + 3] = v.w;
  }
  __syncwarp();   // the warp's own 32 rows of tile_s become its store staging area
  epilogue_ln_row<EPI>(ep, acc, tile_s + warp * 32 * TC_ACC_LD, sp_all, lane, seed, m0 + warp * 32, M);
}

template <int EPI, bool F16>
__host__ __device__ constexpr bool tma_store_epilogue() { return F16 && (EPI == EPI_RELU_MASK || EPI == EPI_RELU_BITS); }

__device__ __forceinline__ void wg_bar_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(3 + wg) : "memory"); }

template <int A_MN, int B_MN, int EPI, bool F16 = true>
__global__ void __launch_bounds__(TC_THREADS, 1)
    tc_gemm_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                   const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                   const __grid_constant__ CUtensorMap tm_out, const GemmShape gs, const EpiParams ep) {
  constexpr bool TMA_EPI = tma_store_epilogue<EPI, F16>();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte aligned operand ring (swizzle atoms), then the fp32 tile, the epilogue parameters and the barriers
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_al = smem_raw + (smem_base - smem_u32(smem_raw));
  float* tile_s = reinterpret_cast<float*>(smem_al + TC_STAGES * TC_STAGE_BYTES);   // [128][TC_ACC_LD]
  float* sp_all = tile_s + 128 * TC_ACC_LD;                                            // [SP_FLOATS]
  uint64_t* full = reinterpret_cast<uint64_t*>(sp_all + TC_SP_FLOATS);                // [TC_STAGES]  TMA -> MMA
  uint64_t* empty = full + TC_STAGES;                                                 // [TC_STAGES]  MMA -> TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo);
    if (TMA_EPI) prefetch_tmap(&tm_out);
    for (int i = 0; i < TC_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TC_CONSUMERS / 32); }
    fence_barrier_init();
  }
  __syncthreads();

  // split-K: tile index -> (seed, m/n tile, k range).  k_split == 1 is the plain case.
  const int ksplit = gs.k_split > 1 ? gs.k_split : 1;
  const int kb_per = (gs.k_blocks + ksplit - 1) / ksplit;
  const int tiles_per_seed = gs.m_tiles * gs.n_tiles * ksplit;
  const int num_tiles = tiles_per_seed * gs.S;
  auto decode = [&](int tile, int& seed, int& m0, int& n0, int& kb0, int& kbn) {
    seed = tile / tiles_per_seed;
    const int rem = tile - seed * tiles_per_seed;
    const int ks = rem % ksplit, mn = rem / ksplit;
    m0 = (mn / gs.n_tiles) * 128; n0 = (mn % gs.n_tiles) * 128;
    kb0 = ks * kb_per;
    kbn = min(kb_per, gs.k_blocks - kb0);
    if (kbn < 0) kbn = 0;
    return ks;
  };

  // F16: 64-element k-blocks, 2 MN-major boxes of 64; TF32: 32-element k-blocks, 4 MN-major boxes of 32
  constexpr int BKE = F16 ? TC_BK16 : TC_BK;
  constexpr int MNB = F16 ? 2 : 4;                        // MN-major TMA boxes per 128-wide tile
  constexpr int MNB_ELEMS = F16 ? 64 : 32, MNB_BYTES = F16 ? 8192 : 4096;
  const bool a_lo_tma = F16 || gs.split3 == 1, b_lo_tma = F16 || gs.split3 != 0;
  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int seed, m0, n0, kb0, kbn;
        decode(tile, seed, m0, n0, kb0, kbn);
        for (int kb = kb0; kb < kb0 + kbn; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1u);
          const uint32_t sb = smem_base + stage * TC_STAGE_BYTES;
          mbar_expect_tx(&full[stage], (2 + (a_lo_tma ? 1 : 0) + (b_lo_tma ? 1 : 0)) * TC_TILE_BYTES);
          const int k0 = kb * BKE;
          if (A_MN) {
#pragma unroll
            for (int j = 0; j < MNB; ++j) {
              tma_load_3d(sb + TC_A_HI + j * MNB_BYTES, &tm_a_hi, &full[stage], m0 + MNB_ELEMS * j, k0, seed);
              if (a_lo_tma) tma_load_3d(sb + TC_A_LO + j * MNB_BYTES, &tm_a_lo, &full[stage], m0 + MNB_ELEMS * j, k0, seed);
            }
          } else {
            tma_load_3d(sb + TC_A_HI, &tm_a_hi, &full[stage], k0, m0, seed);
            if (a_lo_tma) tma_load_3d(sb + TC_A_LO, &tm_a_lo, &full[stage], k0, m0, seed);
          }
          if (B_MN) {
#pragma unroll
            for (int j = 0; j < MNB; ++j) {
              tma_load_3d(sb + TC_B_HI + j * MNB_BYTES, &tm_b_hi, &full[stage], n0 + MNB_ELEMS * j, k0, seed);
              if (b_lo_tma) tma_load_3d(sb + TC_B_LO + j * MNB_BYTES, &tm_b_lo, &full[stage], n0 + MNB_ELEMS * j, k0, seed);
            }
          } else {
            tma_load_3d(sb + TC_B_HI, &tm_b_hi, &full[stage], k0, n0, seed);
            if (b_lo_tma) tma_load_3d(sb + TC_B_LO, &tm_b_lo, &full[stage], k0, n0, seed);
          }
          if (++stage == TC_STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // ===================== consumers (warps 0-7) =====================
  const int t = threadIdx.x;                 // 0..255
  const int wg = t >> 7;                     // warpgroup: tile rows 64 * wg ..
  // A operand of this warpgroup: rows 64 * wg.. of a K-major tile (64 rows x 128 B) or the second 64-wide MN box
  const uint32_t a_off = wg * 8192;
  // fragment coordinates (see wgmma_f16_m64n128): rows fr, fr + 8; columns 8 j + fc, 8 j + fc + 1
  const int fr = 64 * wg + 16 * ((t & 127) >> 5) + (lane >> 2), fc = 2 * (lane & 3);
  const int et = t & 127;                    // thread in the warpgroup; et == 0 issues the warpgroup's bulk stores
  uint8_t* out_stage = reinterpret_cast<uint8_t*>(tile_s) + wg * TC_OUT_STAGE_WG;   // TMA_EPI only
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int seed, m0, n0, kb0, kbn;
    const int ks_idx = decode(tile, seed, m0, n0, kb0, kbn);
    uint32_t rbits[2][4];   // EPI_RELU_BITS: the mask words of rows fr, fr + 8 (bit c of word w = column 32 w + c)
    if constexpr (TMA_EPI) {
      // fetch the tile's ReLU mask now, so that its latency hides behind the MMAs
      if constexpr (EPI == EPI_RELU_BITS) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = m0 + fr + 8 * h;
          const uint4 w = m < gs.M ? __ldg(reinterpret_cast<const uint4*>(
                                         ep.relu_bits + ((int64_t)seed * ep.rows + m) * (ep.ld_out >> 5) + (n0 >> 5)))
                                   : make_uint4(0u, 0u, 0u, 0u);
          rbits[h][0] = w.x; rbits[h][1] = w.y; rbits[h][2] = w.z; rbits[h][3] = w.w;
        }
      } else {   // fp32 mask: 64 KB per tile is too much to hold, so it is pulled into L2 for the epilogue's loads
        const int m = m0 + 64 * wg + (et >> 1);
        const float* p = ep.mask + (int64_t)seed * ep.out_seed_stride + (int64_t)m * ep.ld_out + n0 + 64 * (et & 1);
        if (m < gs.M) {
          asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
          asm volatile("prefetch.global.L2 [%0];" ::"l"(p + 32));
        }
      }
      if (kbn > TC_PROMOTE) {   // the promotions below write tile rows that hold the previous tile's output staging
        if (et == 0) bulk_wait_read_all();
        wg_bar_sync(wg);
      }
    } else {
      consumer_bar_sync();   // the previous tile's epilogue is done with tile_s
    }
    if constexpr (!F16) {
      tf32_tile<A_MN, B_MN>(smem_al, tile_s, full, empty, stage, phase, kbn, gs.split3,
                            ep.out_scale != 0.f ? ep.out_scale : 1.0f, warp, lane);
    } else {
    float mainacc[64], corr[64];   // scoped to the k loop: dead (no registers) during the epilogue
#pragma unroll
    for (int i = 0; i < 64; ++i) { mainacc[i] = 0.f; corr[i] = 0.f; }
    for (int kb = 0; kb < kbn; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sb = smem_base + stage * TC_STAGE_BYTES;
      const uint32_t first_corr = kb == 0 ? 0u : 1u, first_main = kb % TC_PROMOTE == 0 ? 0u : 1u;
      fence_operands(mainacc); fence_operands(corr);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t a_hi = make_gdesc16<A_MN>(sb + TC_A_HI + a_off, ks), a_lo = make_gdesc16<A_MN>(sb + TC_A_LO + a_off, ks);
        const uint64_t b_hi = make_gdesc16<B_MN>(sb + TC_B_HI, ks), b_lo = make_gdesc16<B_MN>(sb + TC_B_LO, ks);
        wgmma_f16_m64n128<A_MN, B_MN>(corr, a_lo, b_hi, ks == 0 ? first_corr : 1u);
        wgmma_f16_m64n128<A_MN, B_MN>(corr, a_hi, b_lo, 1u);
        wgmma_f16_m64n128<A_MN, B_MN>(mainacc, a_hi, b_hi, ks == 0 ? first_main : 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_operands(mainacc); fence_operands(corr);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);   // smem slot free: this warp's MMAs have retired
      if (++stage == TC_STAGES) { stage = 0; phase ^= 1u; }
      // promote the main partial into the fp32 tile (TMA_EPI adds the last partial in registers instead)
      const bool promote = TMA_EPI ? (kb + 1) % TC_PROMOTE == 0 && kb != kbn - 1
                                   : (kb + 1) % TC_PROMOTE == 0 || kb == kbn - 1;
      if (promote) {
        const bool first = kb < TC_PROMOTE;
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float2* p = reinterpret_cast<float2*>(tile_s + (fr + 8 * h) * TC_ACC_LD + 8 * j + fc);
            const float2 v = make_float2(mainacc[4 * j + 2 * h], mainacc[4 * j + 2 * h + 1]);
            if (first) *p = v;
            else { const float2 o = *p; *p = make_float2(o.x + v.x, o.y + v.y); }
          }
      }
    }
    if constexpr (TMA_EPI) {
      // the same operations as the fp32-tile path below: main (+ promoted partials), + corr * 2^-11, * out_scale;
      // then the ReLU mask
      const float osc = ep.out_scale != 0.f ? ep.out_scale : 1.0f;
      const float* mrow = ep.mask + (int64_t)seed * ep.out_seed_stride + n0;   // EPI_RELU_MASK
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = 4 * j + 2 * h;
          float2 o = make_float2(mainacc[i], mainacc[i + 1]);
          if (kbn > TC_PROMOTE) {
            const float2 p = *reinterpret_cast<const float2*>(tile_s + (fr + 8 * h) * TC_ACC_LD + 8 * j + fc);
            o = make_float2(p.x + o.x, p.y + o.y);
          }
          mainacc[i] = fmaf(corr[i], TC_LO_INV, o.x) * osc;
          mainacc[i + 1] = fmaf(corr[i + 1], TC_LO_INV, o.y) * osc;
        }
#pragma unroll
      for (int j = 0; j < 16; ++j)   // a second pass: the fp32 mask's loads do not compete with corr for registers
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float& x = mainacc[4 * j + 2 * h];
          float& y = mainacc[4 * j + 2 * h + 1];
          if constexpr (EPI == EPI_RELU_BITS) {
            const uint32_t b = rbits[h][j >> 2] >> (8 * (j & 3) + fc);
            x = (b & 1u) ? x : 0.f; y = (b & 2u) ? y : 0.f;
          } else {
            const int m = m0 + fr + 8 * h;
            if (m < gs.M) {   // rows >= gs.M are not stored
              const float2 mk = *reinterpret_cast<const float2*>(mrow + (int64_t)m * ep.ld_out + 8 * j + fc);
              x = mk.x > 0.f ? x : 0.f; y = mk.y > 0.f ? y : 0.f;
            }
          }
        }
      if (et == 0) bulk_wait_read_all();   // the previous tile's store has read the staging area
      wg_bar_sync(wg);
      // staging: box j / 4 holds columns 32 (j / 4) ..; 128-byte rows, 16-byte chunk c of row r at c ^ (r % 8)
      const int rl = fr - 64 * wg;   // rl % 8 == lane / 4, rows rl and rl + 8
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int chunk = 2 * (j & 3) + (fc >> 2);
          const int off = (j >> 2) * TC_OUT_BOX_BYTES + (rl + 8 * h) * 128 + ((chunk ^ (lane >> 2)) << 4) + (fc & 3) * 4;
          *reinterpret_cast<float2*>(out_stage + off) = make_float2(mainacc[4 * j + 2 * h], mainacc[4 * j + 2 * h + 1]);
        }
      fence_proxy_async_smem();
      wg_bar_sync(wg);
      if (et == 0) {
#pragma unroll
        for (int b = 0; b < 4; ++b)
          tma_store_3d(&tm_out, smem_u32(out_stage + b * TC_OUT_BOX_BYTES), n0 + 32 * b, m0 + 64 * wg, seed);
        bulk_commit();
      }
      continue;
    }
    {   // the correction accumulator (units of 2^-11), then the power-of-two output scale (exact)
      const float osc = ep.out_scale != 0.f ? ep.out_scale : 1.0f;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float2* p = reinterpret_cast<float2*>(tile_s + (fr + 8 * h) * TC_ACC_LD + 8 * j + fc);
          float2 o = kbn > 0 ? *p : make_float2(0.f, 0.f);
          if (kbn > 0) {
            o.x = fmaf(corr[4 * j + 2 * h], TC_LO_INV, o.x);
            o.y = fmaf(corr[4 * j + 2 * h + 1], TC_LO_INV, o.y);
          }
          *p = make_float2(o.x * osc, o.y * osc);
        }
    }
    }
    consumer_bar_sync();   // tile_s complete

    if constexpr (EPI == EPI_LN_TRAIN || EPI == EPI_LN_HEAD) {
      if (t < 128) {
        stage_epi_params<EPI>(ep, sp_all, seed, t);
        float acc[128];
        const float* row = tile_s + t * TC_ACC_LD;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const float4 v = *reinterpret_cast<const float4*>(row + 4 * j);
          acc[4 * j] = v.x; acc[4 * j + 1] = v.y; acc[4 * j + 2] = v.z; acc[4 * j + 3] = v.w;
        }
        __syncwarp();   // the warp's own 32 rows of tile_s become its store staging area
        epilogue_ln_row<EPI>(ep, acc, tile_s + warp * 32 * TC_ACC_LD, sp_all, lane, seed, m0 + warp * 32, gs.M);
      }
    } else {
      // EPI_STORE / EPI_RELU_MASK / EPI_RELU_BITS: the 256 consumers copy tile rows out, 512 B per row and warp
      // instruction; the ReLU masks are read with the same addressing (dgrad runs in place: out may equal mask)
      const int64_t base = (int64_t)seed * ep.out_seed_stride + n0;
      float* out = ep.out + (EPI == EPI_STORE ? (int64_t)ks_idx * ep.split_stride : 0) + base;
      for (int i = t; i < 128 * 32; i += TC_CONSUMERS) {
        const int r = i >> 5, c4 = i & 31, m = m0 + r;
        if (m >= gs.M) break;   // rows ascend with i
        float4 v = *reinterpret_cast<const float4*>(tile_s + r * TC_ACC_LD + 4 * c4);
        if constexpr (EPI == EPI_RELU_MASK) {
          const float4 mk = *reinterpret_cast<const float4*>(ep.mask + base + (int64_t)m * ep.ld_out + 4 * c4);
          v.x = mk.x > 0.f ? v.x : 0.f; v.y = mk.y > 0.f ? v.y : 0.f;
          v.z = mk.z > 0.f ? v.z : 0.f; v.w = mk.w > 0.f ? v.w : 0.f;
        }
        if constexpr (EPI == EPI_RELU_BITS) {
          // packed ReLU mask written by the conv forward: one word per (row, 32 columns)
          const uint32_t wd = __ldg(ep.relu_bits + ((int64_t)seed * ep.rows + m) * (ep.ld_out >> 5) + ((n0 >> 5) + (c4 >> 3)));
          const uint32_t b = wd >> (4 * (c4 & 7));
          v.x = (b & 1u) ? v.x : 0.f; v.y = (b & 2u) ? v.y : 0.f;
          v.z = (b & 4u) ? v.z : 0.f; v.w = (b & 8u) ? v.w : 0.f;
        }
        *reinterpret_cast<float4*>(out + (int64_t)m * ep.ld_out + 4 * c4) = v;
      }
    }
  }
  if constexpr (TMA_EPI) {
    if (et == 0) bulk_wait_all();   // the staging area must outlive the last bulk store's reads
  }
}

// ---------------------------------------------------------------------------
// Conv-fused dense forward: Z = H1 . W1 with H1 built in registers from the packed observations, so that h1 never goes
// through HBM or shared memory.  The LayerNorm of the conv covers the 16 channels of one pixel, so the A operand of one
// k-step of 16 (k = pixel * 16 + channel) is the conv output of one pixel for the warp's 16 rows (samples):
//   * per k-block (4 pixels) lane (g, t) writes the exponent-coded patch words of pixel 4 kb + t for its warp's rows g
//     and g + 8 (store_patch16) into the warp's patch buffer;
//   * per pair of pixels the warp runs the conv chain of the conv kernels with samples as the MMA rows
//     (conv16_blocks<C, 2>: bias, k-steps in order, lo pass then hi pass), the quad LayerNorm, scale / bias / ReLU and
//     the fp16 split (conv16_act, conv16_split) -- the same instructions on the same operands as conv_fwd_mma16_kernel,
//     so the same bits;
//   * eight shuffles inside the quad turn lane t's channels 4t .. 4t+3 into the wgmma A layout (2t, 2t+1, 2t+8, 2t+9),
//     and the three wgmmas of each pixel (lo.hi, hi.lo into corr; hi.hi into main) go out with A from registers, in the
//     order and with the promotion of tc_gemm_kernel.
// The A fragments are double-buffered: pixels p + 2, p + 3 are built while the wgmmas of p, p + 1 run
// (wgmma.wait_group 1 before their registers are rewritten).  The producer loads only the W1 planes (32 KB per
// k-block).  Observation rows of the next tile are copied (cp.async) into a second buffer during the current tile.
// Rows >= gs.M read row gs.M - 1 and are never stored.
// ---------------------------------------------------------------------------
constexpr int CV_STAGE_BYTES = 2 * TC_TILE_BYTES;   // W1 hi, lo' of one k-block: MN-major boxes [64 k][64 n] x 2 each
constexpr int CV_B_HI = 0, CV_B_LO = TC_TILE_BYTES;
constexpr int CV_WARPS = TC_CONSUMERS / 32;
// a whole producer warpgroup (warps 8-11, one thread of which issues the TMA loads), so that setmaxnreg can move its
// registers to the consumers: 128 x 40 + 256 x 232 <= 64 K.  The consumers hold 128 accumulators, two A fragment
// buffers and the conv chain at once.
constexpr int CV_THREADS = TC_CONSUMERS + 128;
constexpr int CV_PRODUCER_REGS = 40, CV_CONSUMER_REGS = 232;
constexpr int CV_KB = FLAT_CNN / TC_BK16;           // 16 k-blocks of 4 pixels

template <int C>
struct ConvGemm {
  static constexpr int PW = ConvCfg<C>::PW;
  static constexpr int OLD = PW + 4;                          // words per observation row: 16-byte rows + zero pad words
  static constexpr int PB_PIX = 16 * Conv16<C>::ROW;          // patch words of one pixel for a warp's 16 rows
  // byte offsets from the 1024-aligned base
  static constexpr int TILE = TC_STAGES * CV_STAGE_BYTES;
  static constexpr int SP = TILE + 128 * TC_ACC_LD * 4;
  static constexpr int WB = SP + TC_SP_FLOATS * 4;
  static constexpr int CB = WB + Conv16<C>::KS * 2 * 32 * 16;
  static constexpr int OBS = CB + 3 * CONV_O * 4;             // [2 buffers][warp][16 rows][OLD]
  static constexpr int PB = OBS + 2 * CV_WARPS * 16 * OLD * 4;  // [warp][4 pixels][16 rows][ROW]
  static constexpr int BAR = PB + CV_WARPS * 4 * PB_PIX * 4;
  static constexpr int SMEM = BAR + 2 * TC_STAGES * 8 + 1024 /*align slack*/;
  static_assert(WB % 16 == 0 && OBS % 16 == 0 && PB % 16 == 0 && BAR % 8 == 0, "aligned regions");
  static_assert(SMEM <= 227 * 1024, "dynamic shared memory of the conv-fused GEMM exceeds the per-CTA limit");
};

__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
// keeps the registers of an A fragment alive (in the compiler's view) until here: an in-flight wgmma reads them
__device__ __forceinline__ void fence_frag(uint32_t (&a)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(a[i])::"memory");
}

// x[0], x[1] = channel pairs 2t', 2t'+1 (channels 4t' .. 4t'+3) of lane t' of the quad -> pair t (lo) and pair t + 4
// (hi) of lane t: two shuffles, each source lane sending the word its reader needs
__device__ __forceinline__ void quad_pairs(const uint32_t (&x)[2], int lane, uint32_t& lo, uint32_t& hi) {
  const int t = lane & 3, base = lane & ~3;
  const uint32_t sa = (t >> 1) ? x[1] : x[0], sb = (t >> 1) ? x[0] : x[1];
  const uint32_t ra = __shfl_sync(0xffffffffu, sa, base | ((t & 1) << 1) | (t >> 1));
  const uint32_t rb = __shfl_sync(0xffffffffu, sb, base | (((t & 1) ^ 1) << 1) | (t >> 1));
  lo = (t & 1) ? rb : ra;
  hi = (t & 1) ? ra : rb;
}

template <int C, int EPI>
__global__ void __launch_bounds__(CV_THREADS, 1)
    tc_conv_gemm_kernel(const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                        const GemmShape gs, const EpiParams ep, const ConvIn ci) {
  using G = ConvGemm<C>;
  using M = Conv16<C>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_al = smem_raw + (smem_base - smem_u32(smem_raw));
  float* tile_s = reinterpret_cast<float*>(smem_al + G::TILE);    // [128][TC_ACC_LD]
  float* sp_all = reinterpret_cast<float*>(smem_al + G::SP);      // [TC_SP_FLOATS]
  uint4* wb = reinterpret_cast<uint4*>(smem_al + G::WB);          // conv B fragments (conv16_load_weights)
  float* cb = reinterpret_cast<float*>(smem_al + G::CB);
  float* sc = cb + CONV_O;
  float* bi = sc + CONV_O;
  uint32_t* obs_s = reinterpret_cast<uint32_t*>(smem_al + G::OBS);
  uint32_t* pb_s = reinterpret_cast<uint32_t*>(smem_al + G::PB);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_al + G::BAR);
  uint64_t* empty = full + TC_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo);
    for (int i = 0; i < TC_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TC_CONSUMERS / 32); }
    fence_barrier_init();
  }
  __syncthreads();
  const int tiles_per_seed = gs.m_tiles;   // one 128-wide n-tile, no split-K
  const int num_tiles = tiles_per_seed * gs.S;

  if (warp >= 8) {
    // ===================== TMA producer: W1 planes only =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(CV_PRODUCER_REGS));
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int seed = tile / tiles_per_seed;
        for (int kb = 0; kb < CV_KB; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1u);
          const uint32_t sb = smem_base + stage * CV_STAGE_BYTES;
          mbar_expect_tx(&full[stage], 2 * TC_TILE_BYTES);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            tma_load_3d(sb + CV_B_HI + j * 8192, &tm_b_hi, &full[stage], 64 * j, kb * TC_BK16, seed);
            tma_load_3d(sb + CV_B_LO + j * 8192, &tm_b_lo, &full[stage], 64 * j, kb * TC_BK16, seed);
          }
          if (++stage == TC_STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // ===================== consumers (warps 0-7): conv + wgmma =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CV_CONSUMER_REGS));
  const int t = threadIdx.x;                   // 0..255
  const int g = lane >> 2, tq = lane & 3;
  const int fr = 16 * warp + g, fc = 2 * tq;   // accumulator rows fr, fr + 8 of the tile (warpgroup warp / 4)
  uint32_t* my_pb = pb_s + warp * 4 * G::PB_PIX;
  for (int i = t; i < 2 * CV_WARPS * 16; i += TC_CONSUMERS)
    for (int w = G::PW; w < G::OLD; ++w) obs_s[i * G::OLD + w] = 0u;   // pad words read by the funnel shifts
  // observation rows of this warp's 16 tile rows: lane l copies row l % 16, 16-byte chunks l / 16, + 2, ..
  auto obs_src = [&](int tile) -> const uint32_t* {
    const int seed = tile / tiles_per_seed;
    int m = (tile - seed * tiles_per_seed) * 128 + 16 * warp + (lane & 15);
    m = m < gs.M ? m : gs.M - 1;
    const int64_t src = ci.gather ? __ldg(ci.gather + (int64_t)seed * gs.M + m) : m;
    return ci.obs + ((int64_t)seed * ci.obs_rows_per_seed + src) * G::PW;
  };
  auto obs_copy = [&](const uint32_t* src, int buf) {
    const uint32_t dst = smem_u32(obs_s + ((buf * CV_WARPS + warp) * 16 + (lane & 15)) * G::OLD);
    for (int j = lane >> 4; j < G::PW / 4; j += 2) cp_async16(dst + 16 * j, src + 4 * j);
    cp_async_commit();
  };
  if ((int)blockIdx.x < num_tiles) obs_copy(obs_src(blockIdx.x), 0);

  int cur_seed = -1, buf = 0;
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int seed = tile / tiles_per_seed, m0 = (tile - seed * tiles_per_seed) * 128;
    const int next = tile + gridDim.x;
    const uint32_t* next_src = next < num_tiles ? obs_src(next) : nullptr;   // copied after the first k-block
    consumer_bar_sync();   // the previous epilogue is done with tile_s, every warp with the previous conv weights
    if (seed != cur_seed) {
      conv16_load_weights<C>(ep.params + (int64_t)seed * ep.P, ci.L, wb, cb, sc, bi, t, TC_CONSUMERS);
      consumer_bar_sync();
      cur_seed = seed;
    }
    cp_async_wait_all();
    __syncwarp();
    const uint32_t* my_obs = obs_s + (buf * CV_WARPS + warp) * 16 * G::OLD;

    // A fragments (hi, lo') of pixels 4 kb + 2 half and + 1 for rows fr, fr + 8: the two pixels' conv chains run
    // interleaved (conv16_blocks with two m-blocks, as in the conv kernel), which halves the latency per pixel
    auto build_pair = [&](int kb, int half, uint32_t (&ah)[2][4], uint32_t (&al)[2][4]) {
      if (half == 0) {
        __syncwarp();   // the previous k-block's patch rows have been read
        store_patch16<C>(my_obs + g * G::OLD, 4 * kb + tq, my_pb + tq * G::PB_PIX + g * M::ROW);
        store_patch16<C>(my_obs + (g + 8) * G::OLD, 4 * kb + tq, my_pb + tq * G::PB_PIX + (g + 8) * M::ROW);
        __syncwarp();
      }
      float z2[2][2][4];
      conv16_blocks<C, 2>(my_pb, wb, cb, 2 * half, lane, z2);   // m-block i = pixel 2 half + i of the k-block
      const float4 s4 = *reinterpret_cast<const float4*>(sc + 4 * tq), b4 = *reinterpret_cast<const float4*>(bi + 4 * tq);
      const float sc4[4] = {s4.x, s4.y, s4.z, s4.w}, bi4[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float v0[4], v1[4];
        conv16_act(z2[i], sc4, bi4, v0, v1);
        uint32_t hw0[2], lw0[2], hw1[2], lw1[2];
        conv16_split(v0, hw0, lw0);
        conv16_split(v1, hw1, lw1);
        quad_pairs(hw0, lane, ah[i][0], ah[i][2]);
        quad_pairs(hw1, lane, ah[i][1], ah[i][3]);
        quad_pairs(lw0, lane, al[i][0], al[i][2]);
        quad_pairs(lw1, lane, al[i][1], al[i][3]);
      }
    };

    float mainacc[64], corr[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { mainacc[i] = 0.f; corr[i] = 0.f; }
    uint32_t ahi[2][2][4], alo[2][2][4];   // [pixel pair of the k-block][pixel][register]
    build_pair(0, 0, ahi[0], alo[0]);
    int prev_stage = 0;
    for (int kb = 0; kb < CV_KB; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sb = smem_base + stage * CV_STAGE_BYTES;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int nxt = half ^ 1;
        wgmma_fence();
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int ks = 2 * half + i;
          const uint64_t b_hi = make_gdesc16<1>(sb + CV_B_HI, ks), b_lo = make_gdesc16<1>(sb + CV_B_LO, ks);
          wgmma_f16_m64n128_ra<1>(corr, alo[half][i], b_hi, (ks == 0 && kb == 0) ? 0u : 1u);
          wgmma_f16_m64n128_ra<1>(corr, ahi[half][i], b_lo, 1u);
          wgmma_f16_m64n128_ra<1>(mainacc, ahi[half][i], b_hi, (ks == 0 && kb % TC_PROMOTE == 0) ? 0u : 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous pixel pair's wgmmas have retired
#pragma unroll
        for (int i = 0; i < 2; ++i) { fence_frag(ahi[nxt][i]); fence_frag(alo[nxt][i]); }
        if (half == 0 && kb > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[prev_stage]);   // the previous k-block's W1 slot is free
        }
        if (half == 0 && kb == 0 && next_src) obs_copy(next_src, buf ^ 1);
        if (half == 0) build_pair(kb, 1, ahi[1], alo[1]);
        else if (kb + 1 < CV_KB) build_pair(kb + 1, 0, ahi[0], alo[0]);
      }
      prev_stage = stage;
      if (++stage == TC_STAGES) { stage = 0; phase ^= 1u; }
      if ((kb + 1) % TC_PROMOTE == 0) {
        wgmma_wait<0>();
        fence_operands(mainacc); fence_operands(corr);
#pragma unroll
        for (int i = 0; i < 2; ++i) { fence_frag(ahi[0][i]); fence_frag(alo[0][i]); }
        promote_main(tile_s, mainacc, fr, fc, kb < TC_PROMOTE);
      }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) { fence_frag(ahi[1][i]); fence_frag(alo[1][i]); }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev_stage]);
    finish_corr(tile_s, corr, fr, fc, CV_KB, ep.out_scale != 0.f ? ep.out_scale : 1.0f);
    consumer_bar_sync();   // tile_s complete
    if (t < 128) ln_epilogue_tile<EPI>(ep, tile_s, sp_all, t, warp, lane, seed, m0, gs.M);
    buf ^= 1;
  }
  cp_async_wait_all();
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static int num_sms() { return device_sm_count(); }

// 3-D fp32 tensor [seeds][mid][inner] with a {32, box_mid, 1} box (128 bytes x box_mid), SWIZZLE_128B for both majors
int make_tmap(CUtensorMap* tm, const float* base, uint64_t inner, uint64_t mid, uint64_t seeds, uint64_t mid_stride_elems,
              uint64_t seed_stride_elems, uint32_t box_mid) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error(PQN_E_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t dims[3] = {inner, mid, seeds};
  cuuint64_t strides[2] = {mid_stride_elems * 4, seed_stride_elems * 4};
  cuuint32_t box[3] = {32, box_mid, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(PQN_E_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return PQN_OK;
}

template <int A_MN, int B_MN, int EPI, bool F16>
static int launch_t(const CUtensorMap* t, const GemmShape& gs, const EpiParams& ep, cudaStream_t st, int kid) {
  auto kfn = tc_gemm_kernel<A_MN, B_MN, EPI, F16>;
  static_assert(TC_SMEM_BYTES <= 227 * 1024, "dynamic shared memory of the GEMM kernel exceeds the per-CTA limit");
  if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES) != cudaSuccess)
    return check_launch("tc_gemm(cudaFuncSetAttribute)");
  CUtensorMap tm_out = t[0];   // not read unless the epilogue stores through TMA
  if (tma_store_epilogue<EPI, F16>()) {
    // out[S][M][ld_out] in boxes of 64 rows x 32 floats; the row bound clips a ragged last m-tile
    if (ep.ld_out != (int64_t)gs.n_tiles * 128 || gs.k_split > 1)
      return set_error(PQN_E_INVALID, "tc_gemm16: ReLU-mask epilogues need ld_out == N and no split-K");
    int rc = make_tmap(&tm_out, ep.out, (uint64_t)ep.ld_out, (uint64_t)gs.M, (uint64_t)gs.S, (uint64_t)ep.ld_out,
                       (uint64_t)ep.out_seed_stride, 64);
    if (rc) return rc;
  }
  const int tiles = gs.m_tiles * gs.n_tiles * gs.S * (gs.k_split > 1 ? gs.k_split : 1);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  {
    LaunchScope _ls(kid < 0 ? (int)K_TC_GEMM : kid, st);
    kfn<<<grid, TC_THREADS, TC_SMEM_BYTES, st>>>(t[0], t[1], t[2], t[3], tm_out, gs, ep);
  }
  return check_launch("tc_gemm");
}

template <int C, int EPI>
static int launch_conv_t(const CUtensorMap* tb, const GemmShape& gs, const EpiParams& ep, const ConvIn& ci,
                         cudaStream_t st, int kid) {
  auto kfn = tc_conv_gemm_kernel<C, EPI>;
  constexpr int smem = ConvGemm<C>::SMEM;
  if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
    return check_launch("tc_conv_gemm(cudaFuncSetAttribute)");
  const int tiles = gs.m_tiles * gs.S;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  {
    LaunchScope _ls(kid, st);
    kfn<<<grid, CV_THREADS, smem, st>>>(tb[0], tb[1], gs, ep, ci);
  }
  return check_launch("tc_conv_gemm");
}

int launch_conv_gemm16(int C, int epi, const CUtensorMap* tb, const GemmShape& gs, const EpiParams& ep, const ConvIn& ci,
                       cudaStream_t st, int kernel_id) {
  if (gs.n_tiles != 1 || gs.k_split > 1 || gs.k_blocks != CV_KB)
    return set_error(PQN_E_INVALID, "tc_conv_gemm16: N = 128, K = 1024 and no split-K");
#define PQN_CONV_CASE(CC) \
  if (C == CC && epi == EPI_LN_HEAD) return launch_conv_t<CC, EPI_LN_HEAD>(tb, gs, ep, ci, st, kernel_id);
  PQN_CONV_CASE(4)
  PQN_CONV_CASE(6)
  PQN_CONV_CASE(7)
  PQN_CONV_CASE(10)
#undef PQN_CONV_CASE
  return set_error(PQN_E_UNSUPPORTED, "tc_conv_gemm16: combination C=%d epi=%d not instantiated", C, epi);
}

int launch_gemm(int a_mn, int b_mn, int epi, const CUtensorMap* t, const GemmShape& gs, const EpiParams& ep,
                cudaStream_t st, int kernel_id) {
#define PQN_TC_CASE(A, B, E) \
  if (a_mn == A && b_mn == B && epi == E) return launch_t<A, B, E, false>(t, gs, ep, st, kernel_id);
  PQN_TC_CASE(0, 1, EPI_STORE)
  PQN_TC_CASE(0, 1, EPI_LN_TRAIN)
  PQN_TC_CASE(0, 1, EPI_LN_HEAD)
  PQN_TC_CASE(1, 1, EPI_STORE)
  PQN_TC_CASE(0, 0, EPI_STORE)
  PQN_TC_CASE(0, 0, EPI_RELU_MASK)
  PQN_TC_CASE(0, 0, EPI_RELU_BITS)
#undef PQN_TC_CASE
  return set_error(PQN_E_UNSUPPORTED, "tc_gemm: combination a_mn=%d b_mn=%d epi=%d not instantiated", a_mn, b_mn, epi);
}

int launch_gemm16(int a_mn, int b_mn, int epi, const CUtensorMap* t, const GemmShape& gs, const EpiParams& ep,
                  cudaStream_t st, int kernel_id) {
#define PQN_TC_CASE(A, B, E) \
  if (a_mn == A && b_mn == B && epi == E) return launch_t<A, B, E, true>(t, gs, ep, st, kernel_id);
  PQN_TC_CASE(0, 1, EPI_STORE)
  PQN_TC_CASE(0, 1, EPI_LN_TRAIN)
  PQN_TC_CASE(0, 1, EPI_LN_HEAD)
  PQN_TC_CASE(1, 1, EPI_STORE)
  PQN_TC_CASE(0, 0, EPI_STORE)
  PQN_TC_CASE(0, 0, EPI_RELU_MASK)
  PQN_TC_CASE(0, 0, EPI_RELU_BITS)
#undef PQN_TC_CASE
  return set_error(PQN_E_UNSUPPORTED, "tc_gemm16: combination a_mn=%d b_mn=%d epi=%d not instantiated", a_mn, b_mn, epi);
}

int make_tmap16(CUtensorMap* tm, const void* base, uint64_t inner, uint64_t mid, uint64_t seeds, uint64_t mid_stride_elems,
                uint64_t seed_stride_elems, uint32_t box_mid) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error(PQN_E_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t dims[3] = {inner, mid, seeds};
  cuuint64_t strides[2] = {mid_stride_elems * 2, seed_stride_elems * 2};
  cuuint32_t box[3] = {64, box_mid, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(PQN_E_CUDA, "cuTensorMapEncodeTiled(fp16) failed (%d)", (int)r);
  return PQN_OK;
}

__global__ void split_lo_kernel(const float* __restrict__ x, float* __restrict__ lo, int64_t n4) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
  float4 o;
  o.x = tf32_lo(v.x); o.y = tf32_lo(v.y); o.z = tf32_lo(v.z); o.w = tf32_lo(v.w);
  reinterpret_cast<float4*>(lo)[i] = o;
}

// fp16 split planes of an fp32 tensor (optionally pre-scaled by a power of two): hi = fp16(x*scale),
// lo = fp16((x*scale - hi) * 2^11)
__global__ void split16_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo, int64_t n4,
                               float scale) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
  __half2 h0, h1, l0, l1;
  split16x2(v.x * scale, v.y * scale, h0, l0);
  split16x2(v.z * scale, v.w * scale, h1, l1);
  reinterpret_cast<uint2*>(hi)[i] = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
  reinterpret_cast<uint2*>(lo)[i] = make_uint2(*reinterpret_cast<uint32_t*>(&l0), *reinterpret_cast<uint32_t*>(&l1));
}

}  // namespace tc
}  // namespace pqn

using namespace pqn;
using namespace pqn::tc;

extern "C" {

int pqn_tc_split_lo(const float* x, float* lo, int64_t n, void* stream) {
  if (!x || !lo || n < 0 || (n & 3)) return set_error(PQN_E_INVALID, "pqn_tc_split_lo: bad argument (n %% 4 == 0)");
  if (n == 0) return PQN_OK;
  {
    LaunchScope _ls(K_TC_SPLIT, (cudaStream_t)stream);
    split_lo_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, lo, n / 4);
  }
  return check_launch("pqn_tc_split_lo");
}

int pqn_tc_split16(const float* x, void* hi, void* lo, int64_t n, float scale, void* stream) {
  if (!x || !hi || !lo || n < 0 || (n & 3)) return set_error(PQN_E_INVALID, "pqn_tc_split16: bad argument (n %% 4 == 0)");
  if (n == 0) return PQN_OK;
  {
    LaunchScope _ls(K_TC_SPLIT, (cudaStream_t)stream);
    split16_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, (__half*)hi, (__half*)lo, n / 4,
                                                                                       scale);
  }
  return check_launch("pqn_tc_split16");
}

// Test hook: D[s] = A[s] . B[s] * out_scale on the fp16-split wgmma path; operands are the (hi, lo') planes written
// by pqn_tc_split16.
//   a_mn = 0: A is [S][M][K] (K contiguous)   a_mn = 1: A is [S][K][M] (M contiguous)
//   b_mn = 0: B is [S][N][K] (K contiguous)   b_mn = 1: B is [S][K][N] (N contiguous)
// N % 128 == 0; rows of a ragged M are guarded, a ragged K is zero-filled by TMA.
int pqn_tc_gemm16_test(const void* a_hi, const void* a_lo, const void* b_hi, const void* b_lo, float* d, int32_t S,
                       int32_t M, int32_t N, int32_t K, int a_mn, int b_mn, float out_scale, void* stream) {
  if (!a_hi || !a_lo || !b_hi || !b_lo || !d || S <= 0 || M <= 0 || N <= 0 || K <= 0 || (N % 128) || (K % 8) || (M % 8))
    return set_error(PQN_E_INVALID, "pqn_tc_gemm16_test: bad argument");
  CUtensorMap t[4];
  int rc;
  const void* ap[2] = {a_hi, a_lo};
  const void* bp[2] = {b_hi, b_lo};
  for (int i = 0; i < 2; ++i) {
    if (a_mn) { if ((rc = make_tmap16(&t[i], ap[i], M, K, S, M, (uint64_t)M * K, 64))) return rc; }
    else { if ((rc = make_tmap16(&t[i], ap[i], K, M, S, K, (uint64_t)M * K, 128))) return rc; }
    if (b_mn) { if ((rc = make_tmap16(&t[2 + i], bp[i], N, K, S, N, (uint64_t)N * K, 64))) return rc; }
    else { if ((rc = make_tmap16(&t[2 + i], bp[i], K, N, S, K, (uint64_t)N * K, 128))) return rc; }
  }
  GemmShape gs = {};
  gs.S = S; gs.M = M; gs.m_tiles = (M + 127) / 128; gs.n_tiles = N / 128; gs.k_blocks = (K + TC_BK16 - 1) / TC_BK16;
  EpiParams ep = {};
  ep.out = d; ep.ld_out = N; ep.out_seed_stride = (int64_t)M * N; ep.out_scale = out_scale;
  return launch_gemm16(a_mn, b_mn, EPI_STORE, t, gs, ep, (cudaStream_t)stream);
}

// Test hook for the input-gradient epilogues: D[s] = mask[s] * (A[s] . B[s]^T) * out_scale on the fp16-split wgmma
// path, A [S][M][K] and B [S][N][K] as planes (both K-major, the dgrad layout).
//   epi = 0 (EPI_STORE): no mask;  3 (EPI_RELU_MASK): mask[s][m][n] > 0, mask may equal d (in place);
//   4 (EPI_RELU_BITS): bit n % 32 of relu_bits[s][m][n / 32].
// N % 128 == 0; rows of a ragged M are not written.
int pqn_tc_dgrad16_test(const void* a_hi, const void* a_lo, const void* b_hi, const void* b_lo, const float* mask,
                        const uint32_t* relu_bits, float* d, int32_t S, int32_t M, int32_t N, int32_t K, int epi,
                        float out_scale, void* stream) {
  if (!a_hi || !a_lo || !b_hi || !b_lo || !d || S <= 0 || M <= 0 || N <= 0 || K <= 0 || (N % 128) || (K % 8) ||
      (M % 8) || !(epi == EPI_STORE || epi == EPI_RELU_MASK || epi == EPI_RELU_BITS) ||
      (epi == EPI_RELU_MASK && !mask) || (epi == EPI_RELU_BITS && !relu_bits))
    return set_error(PQN_E_INVALID, "pqn_tc_dgrad16_test: bad argument");
  CUtensorMap t[4];
  int rc;
  const void* p[4] = {a_hi, a_lo, b_hi, b_lo};
  for (int i = 0; i < 2; ++i) {
    if ((rc = make_tmap16(&t[i], p[i], K, M, S, K, (uint64_t)M * K, 128))) return rc;
    if ((rc = make_tmap16(&t[2 + i], p[2 + i], K, N, S, K, (uint64_t)N * K, 128))) return rc;
  }
  GemmShape gs = {};
  gs.S = S; gs.M = M; gs.m_tiles = (M + 127) / 128; gs.n_tiles = N / 128; gs.k_blocks = (K + TC_BK16 - 1) / TC_BK16;
  EpiParams ep = {};
  ep.out = d; ep.mask = mask; ep.relu_bits = relu_bits; ep.rows = M;
  ep.ld_out = N; ep.out_seed_stride = (int64_t)M * N; ep.out_scale = out_scale;
  return launch_gemm16(0, 0, epi, t, gs, ep, (cudaStream_t)stream);
}

// Test hook: D[s] = A[s] . B[s] on the TF32 path (fp32 in, fp32 out).  Layout flags as in pqn_tc_gemm16_test.
//   split3 = 1: 3xTF32 (a_lo / b_lo must hold x - trunc_tf32(x)); 2: same, but A_lo is derived in the kernel
//   (a_lo unused); 0: single-pass TF32.  N % 128 == 0; rows of a ragged M are guarded, a ragged K is zero-filled.
int pqn_tc_gemm_test(const float* a, const float* a_lo, const float* b, const float* b_lo, float* d, int32_t S,
                     int32_t M, int32_t N, int32_t K, int a_mn, int b_mn, int split3, void* stream) {
  if (!a || !b || !d || S <= 0 || M <= 0 || N <= 0 || K <= 0 || (N % 128) || split3 < 0 || split3 > 2 ||
      (split3 && !b_lo) || (split3 == 1 && !a_lo))
    return set_error(PQN_E_INVALID, "pqn_tc_gemm_test: bad argument");
  CUtensorMap t[4];
  int rc;
  const float* al = split3 == 1 ? a_lo : a;
  const float* bl = split3 ? b_lo : b;
  const float* ap[2] = {a, al};
  const float* bp[2] = {b, bl};
  for (int i = 0; i < 2; ++i) {
    if (a_mn) { if ((rc = make_tmap(&t[i], ap[i], M, K, S, M, (uint64_t)M * K, 32))) return rc; }
    else { if ((rc = make_tmap(&t[i], ap[i], K, M, S, K, (uint64_t)M * K, 128))) return rc; }
    if (b_mn) { if ((rc = make_tmap(&t[2 + i], bp[i], N, K, S, N, (uint64_t)N * K, 32))) return rc; }
    else { if ((rc = make_tmap(&t[2 + i], bp[i], K, N, S, K, (uint64_t)N * K, 128))) return rc; }
  }
  GemmShape gs = {};
  gs.S = S; gs.M = M; gs.m_tiles = (M + 127) / 128; gs.n_tiles = N / 128; gs.k_blocks = (K + TC_BK - 1) / TC_BK;
  gs.split3 = split3;
  EpiParams ep = {};
  ep.out = d; ep.ld_out = N; ep.out_seed_stride = (int64_t)M * N;
  return launch_gemm(a_mn, b_mn, EPI_STORE, t, gs, ep, (cudaStream_t)stream);
}

}  // extern "C"
