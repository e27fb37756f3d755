// Dense_0 of the MLP Q-network on packed MinAtar observation bits (PQN_NET_MLP_BITS): pqn_gymnax.py's QNetwork on a
// MinAtar env behind FlattenObservationWrapper, whose D = 100 * C inputs are {0,1}.
//
// Forward   Z[s][r][n] = sum_f bit[r][f] * W0'[f][n] + b0'[n]        (fwd_kernel)
// Gradient  G[s][f][n] = sum_r bit[r][f] * dz0[r][n]                  (wgrad_kernel)
// both on fp16 mma.sync.m16n8k16 with fp32 accumulation, read straight from the packed rows (no fp32 or fp16 copy of
// the observations is written).  The {0,1} operand is exact in fp16; the other one is the fp16-split pair
// (hi, lo' = (x - hi) * 2^11).  A set bit becomes the fp16 value 2^-11 with ONE shift + AND of a "spread" word (the
// bit sits on fp16 exponent bit 12), and 1.0 for the hi product with one more shift + IMUL (2^-11 << 11): both planes
// accumulate into the same fp32 accumulator (1.0 * hi + 2^-11 * lo' = x).  Tensor-core accumulation does not round
// to nearest, so the MMA chains are cut every few k-steps and added to fp32 registers with FADD.
//
// k order inside a k-step of 16 (free to choose, the other operand is laid out to match; as in conv16_tap):
// fragment column 2t <-> element t, 2t+1 <-> 4+t, 2t+8 <-> 8+t, 2t+9 <-> 12+t of the 16.  So a 16-bit chunk c of
// bits spreads into two words (spread16): bits 0..3 of c at bits 12..15, 4..7 at 28..31 (word x), 8..11 at 12..15,
// 12..15 at 28..31 (word y), and lane t's A register is (x >> t) & 0x10001000.
//
// The padding bits of a packed row past D never reach a result: the forward's B rows past D are zero and the weight
// gradient stores only rows f < D.  The BatchNorm_0 statistics are per-feature popcounts (count_kernel).
//
// Included inside namespace pqn of pqn_net.cu (uses its mma / split helpers and launch_split_reduce).
#pragma once

namespace bits {

constexpr int KC = 8;                            // k-steps per MMA accumulation chain (forward)
constexpr int FWD_WARPS = 4, FWD_ROWS = 32 * FWD_WARPS;   // forward CTA tile: 128 rows x 8 * NT columns
constexpr int WG_ROWS = 64;                      // rows (4 k-steps) per staged chunk of the weight gradient
constexpr int WG_FEAT = 128;                     // features per weight-gradient CTA
constexpr int CNT_BLOCKS = 64;                   // row chunks per seed of the two-stage popcount
constexpr uint32_t AMASK = 0x10001000u;          // fp16 2^-11 in both halves

__host__ __device__ inline int packed_words(int D) { return ((D + 31) / 32 + 3) / 4 * 4; }
__host__ __device__ inline int ksteps(int D) { return (D + 15) / 16; }

__device__ __forceinline__ uint2 spread16(uint32_t c) {
  return make_uint2(((c & 0xFu) << 12) | ((c & 0xF0u) << 24), ((c & 0xF00u) << 4) | ((c & 0xF000u) << 16));
}
// A registers of lane t from the spread words of its two rows (xa: row g, xb: row g + 8): lo = 2^-11 coded, hi = 1.0
__device__ __forceinline__ void a_frag(uint2 xa, uint2 xb, int t, uint32_t (&lo)[4], uint32_t (&hi)[4]) {
  lo[0] = (xa.x >> t) & AMASK; lo[1] = (xb.x >> t) & AMASK; lo[2] = (xa.y >> t) & AMASK; lo[3] = (xb.y >> t) & AMASK;
#pragma unroll
  for (int q = 0; q < 4; ++q) hi[q] = (lo[q] >> 2) * 15u;   // bit 12 -> bits 10..13: fp16 1.0
}
__device__ __forceinline__ uint32_t h2u(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }

// Dense_0 kernel, optionally row-scaled by dvec[f] and negated where flip[s] has bit f (NORM_INPUT), as B fragments
// of fp16 (hi, lo') planes:
// wf[s][ks][n / 8][lane] = {b0_hi, b1_hi, b0_lo, b1_lo}; lane = 4g + t holds column 8 (n / 8) + g and the features
// 16 ks + t, +4 (b0) and +8, +12 (b1); rows past D are zero.  grid = (ceil(KS * H * 4 / 256), S)
__global__ void wfrag_kernel(const float* __restrict__ params, int64_t P, int64_t off_w, const float* __restrict__ dvec,
                             const uint32_t* __restrict__ flip, int D, int H, int KS, uint4* __restrict__ wf) {
  const int seed = blockIdx.y;
  const int64_t n_per = (int64_t)KS * (H / 8) * 32;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_per) return;
  const int lane = (int)(i & 31), nt = (int)((i >> 5) % (H / 8)), ks = (int)(i / (32 * (H / 8)));
  const int n = nt * 8 + (lane >> 2), t = lane & 3;
  const float* __restrict__ W = params + (int64_t)seed * P + off_w;
  const float* __restrict__ dv = dvec ? dvec + (int64_t)seed * 2 * D : nullptr;
  float v[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int f = 16 * ks + 4 * q + t;
    v[q] = f < D ? W[(int64_t)f * H + n] * (dv ? dv[f] : 1.f) : 0.f;
    if (flip && ((flip[(int64_t)seed * packed_words(D) + (f >> 5)] >> (f & 31)) & 1u)) v[q] = -v[q];
  }
  __half2 h0, l0, h1, l1;
  tc::split16x2(v[0], v[1], h0, l0);
  tc::split16x2(v[2], v[3], h1, l1);
  wf[(int64_t)seed * n_per + i] = make_uint4(h2u(h0), h2u(h1), h2u(l0), h2u(l1));
}

// Z[s][r][n0 .. n0+8NT-1] = bits(row r) . W0' + bias.  CTA = 4 warps; its 8NT-column slice of the B fragments (all
// k-steps) stays in shared memory while the CTA walks row tiles of 128 (grid-stride); warp = 32 rows x 8NT columns.
// NT = 8 (64 columns) up to 44 k-steps (D = 700); NT = 4 (32 columns) at D = 1000, whose 63 k-steps of 64-column B
// fragments (252 KB) would not fit in shared memory.  Same MMA chains and fp32 adds per column either way.
// grid = (row-tile CTAs, H / (8NT), S), dynamic shared memory fwd_smem(KS, NT)
template <int NT>
__global__ void __launch_bounds__(FWD_WARPS * 32, 1)
    fwd_kernel(const uint32_t* __restrict__ obs, int64_t orps, const int32_t* __restrict__ gather, int rows, int D,
               int KS, const uint4* __restrict__ wf, int H, const float* __restrict__ bias, int64_t bias_stride,
               const uint32_t* __restrict__ flip, float* __restrict__ Z) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint4* sB = reinterpret_cast<uint4*>(smem_raw);                      // [KS][8 n-tiles][32 lanes]
  uint2* sA = reinterpret_cast<uint2*>(sB + (int64_t)KS * NT * 32);    // [128 rows][LDA] spread k-chunks
  const int LDA = KS | 1;                                              // odd: conflict-free fragment loads
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int seed = blockIdx.z, nt0 = blockIdx.y * NT;
  const int PW = packed_words(D);
  const uint4* __restrict__ wsrc = wf + (int64_t)seed * KS * (H / 8) * 32;
  for (int i = tid; i < KS * NT * 32; i += blockDim.x)
    sB[i] = __ldg(wsrc + ((int64_t)(i / (NT * 32)) * (H / 8) + nt0 + ((i >> 5) % NT)) * 32 + (i & 31));
  const float* __restrict__ bv = bias + (int64_t)seed * bias_stride + nt0 * 8;
  float2 bcol[NT];
#pragma unroll
  for (int j = 0; j < NT; ++j) bcol[j] = make_float2(bv[8 * j + 2 * t], bv[8 * j + 2 * t + 1]);

  for (int r0 = blockIdx.x * FWD_ROWS; r0 < rows; r0 += gridDim.x * FWD_ROWS) {
    __syncthreads();   // sB is loaded / the previous tile's sA is consumed
    {
      const int row = r0 + tid;   // one row per thread: packed words -> spread k-chunks
      uint2* __restrict__ dst = sA + tid * LDA;
      if (row < rows) {
        const int64_t src = gather ? gather[(int64_t)seed * rows + row] : row;
        const uint4* __restrict__ p = reinterpret_cast<const uint4*>(obs + ((int64_t)seed * orps + src) * PW);
        for (int q = 0; q < PW / 4; ++q) {
          uint4 v = __ldg(p + q);
          if (flip) {
            const uint4 fl = reinterpret_cast<const uint4*>(flip + (int64_t)seed * PW)[q];
            v.x ^= fl.x; v.y ^= fl.y; v.z ^= fl.z; v.w ^= fl.w;
          }
          const uint32_t wv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int ks = 8 * q + 2 * e;   // word 4q + e holds k-steps 2(4q + e) and 2(4q + e) + 1
            if (ks < KS) dst[ks] = spread16(wv[e] & 0xFFFFu);
            if (ks + 1 < KS) dst[ks + 1] = spread16(wv[e] >> 16);
          }
        }
      } else {
        for (int ks = 0; ks < KS; ++ks) dst[ks] = make_uint2(0u, 0u);
      }
    }
    __syncthreads();
    float tot[2][NT][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) tot[m][j][q] = 0.f;
    const uint2* __restrict__ arow = sA + (warp * 32 + g) * LDA;
    for (int c0 = 0; c0 < KS; c0 += KC) {
      float acc[2][NT][4];
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[m][j][q] = 0.f;
      const int c1 = min(KS, c0 + KC);
      for (int ks = c0; ks < c1; ++ks) {
        uint32_t alo[2][4], ahi[2][4];
#pragma unroll
        for (int m = 0; m < 2; ++m) a_frag(arow[(16 * m) * LDA + ks], arow[(16 * m + 8) * LDA + ks], t, alo[m], ahi[m]);
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const uint4 b = sB[(ks * NT + j) * 32 + lane];
#pragma unroll
          for (int m = 0; m < 2; ++m) {
            mma_f16_16n8k16(acc[m][j], ahi[m], b.x, b.y);
            mma_f16_16n8k16(acc[m][j], alo[m], b.z, b.w);
          }
        }
      }
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
          for (int q = 0; q < 4; ++q) tot[m][j][q] += acc[m][j][q];
    }
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const int row = r0 + warp * 32 + 16 * m + g;
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const int col = (nt0 + j) * 8 + 2 * t;
        if (row < rows)
          *reinterpret_cast<float2*>(Z + ((int64_t)seed * rows + row) * H + col) =
              make_float2(tot[m][j][0] + bcol[j].x, tot[m][j][1] + bcol[j].y);
        if (row + 8 < rows)
          *reinterpret_cast<float2*>(Z + ((int64_t)seed * rows + row + 8) * H + col) =
              make_float2(tot[m][j][2] + bcol[j].x, tot[m][j][3] + bcol[j].y);
      }
    }
  }
}
static size_t fwd_smem(int KS, int NT) {
  return (size_t)KS * NT * 32 * sizeof(uint4) + (size_t)FWD_ROWS * (KS | 1) * sizeof(uint2);
}
static int fwd_ntiles(int KS) { return fwd_smem(KS, 8) <= 227u * 1024u ? 8 : 4; }

// G[f][n] = sum_r bit[r][f] * dz[r][n] over this CTA's row split, for 128 features x BNC columns: the bits of a 64-row
// chunk are transposed to feature-major spread words with warp ballots, dz * gscale is split into fp16 (hi, lo') B
// fragments while it is staged; warp = 32 features x 64 columns; one accumulation chain per chunk (4 k-steps).
// out + split * split_stride + seed * out_seed_stride receives rows f < D of the (unscaled) result.
// grid = (ceil(D / 128), H / BNC, splits * S)
template <int BNC>
__global__ void __launch_bounds__(BNC / 16 * 32, 1)
    wgrad_kernel(const uint32_t* __restrict__ obs, int64_t orps, const int32_t* __restrict__ gather, int rows, int D,
                 const float* __restrict__ DZ, int H, float gscale, int S, int rows_per_split,
                 const uint32_t* __restrict__ flip, float* __restrict__ out, int64_t out_seed_stride, int64_t split_stride) {
  constexpr int NWARP = BNC / 16, NT = BNC / 8, LDX = 5;
  __shared__ uint32_t sRows[WG_ROWS][4];
  __shared__ uint2 sX[WG_FEAT * LDX];        // [feature][k-step] spread bits over the chunk's rows
  __shared__ uint4 sZ[4 * NT * 32];          // [k-step][n-tile][lane] dz fragments
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int seed = blockIdx.z % S, split = blockIdx.z / S;
  const int f0 = blockIdx.x * WG_FEAT, n0 = blockIdx.y * BNC, fg = warp & 3, cg = warp >> 2;
  const int PW = packed_words(D), w0 = f0 / 32;
  const int r_begin = split * rows_per_split, r_end = min(rows, r_begin + rows_per_split);
  float tot[2][8][4];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) tot[m][j][q] = 0.f;
  for (int r0 = r_begin; r0 < r_end; r0 += WG_ROWS) {
    __syncthreads();
    for (int i = tid; i < WG_ROWS * 4; i += NWARP * 32) {
      const int r = i >> 2, wd = i & 3, row = r0 + r;
      uint32_t v = 0u;
      if (row < r_end && w0 + wd < PW) {
        const int64_t src = gather ? gather[(int64_t)seed * rows + row] : row;
        v = __ldg(obs + ((int64_t)seed * orps + src) * PW + w0 + wd);
        if (flip) v ^= flip[(int64_t)seed * PW + w0 + wd];
      }
      sRows[r][wd] = v;
    }
    for (int i = tid; i < 4 * NT * 32; i += NWARP * 32) {
      const int ln = i & 31, nt = (i >> 5) % NT, ks = i / (32 * NT);
      const int n = n0 + 8 * nt + (ln >> 2), tt = ln & 3;
      float v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int row = r0 + 16 * ks + 4 * q + tt;
        v[q] = row < r_end ? __ldg(DZ + ((int64_t)seed * rows + row) * H + n) * gscale : 0.f;
      }
      __half2 h0, l0, h1, l1;
      tc::split16x2(v[0], v[1], h0, l0);
      tc::split16x2(v[2], v[3], h1, l1);
      sZ[i] = make_uint4(h2u(h0), h2u(h1), h2u(l0), h2u(l1));
    }
    __syncthreads();
    // transpose: warp takes (word wd, 32-row half rh); lane j keeps feature 32 wd + j's bits over those 32 rows
    for (int combo = warp; combo < 8; combo += NWARP) {
      const int wd = combo & 3, rh = combo >> 2;
      const uint32_t v = sRows[rh * 32 + lane][wd];
      uint32_t mine = 0u;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const uint32_t m = __ballot_sync(0xffffffffu, (v >> j) & 1u);
        if (lane == j) mine = m;
      }
      const int f = wd * 32 + lane;
      sX[f * LDX + 2 * rh] = spread16(mine & 0xFFFFu);
      sX[f * LDX + 2 * rh + 1] = spread16(mine >> 16);
    }
    __syncthreads();
    float acc[2][8][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[m][j][q] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t alo[2][4], ahi[2][4];
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        const int fa = fg * 32 + 16 * m + g;
        a_frag(sX[fa * LDX + ks], sX[(fa + 8) * LDX + ks], t, alo[m], ahi[m]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint4 b = sZ[(ks * NT + cg * 8 + j) * 32 + lane];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          mma_f16_16n8k16(acc[m][j], ahi[m], b.x, b.y);
          mma_f16_16n8k16(acc[m][j], alo[m], b.z, b.w);
        }
      }
    }
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) tot[m][j][q] += acc[m][j][q];
  }
  const float inv = 1.0f / gscale;
  float* __restrict__ o = out + (int64_t)split * split_stride + (int64_t)seed * out_seed_stride;
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    const int f = f0 + fg * 32 + 16 * m + g;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + (cg * 8 + j) * 8 + 2 * t;
      if (f < D) *reinterpret_cast<float2*>(o + (int64_t)f * H + n) = make_float2(tot[m][j][0] * inv, tot[m][j][1] * inv);
      if (f + 8 < D)
        *reinterpret_cast<float2*>(o + (int64_t)(f + 8) * H + n) = make_float2(tot[m][j][2] * inv, tot[m][j][3] * inv);
    }
  }
}

// per-feature set-bit counts of the (gathered) rows over each block's row chunk: part[S][nb][D], exact integers
// (shared-memory integer atomics: the result does not depend on their order).  One row per warp, one word per lane.
// grid = (CNT_BLOCKS, S), block = 256
__global__ void __launch_bounds__(256) count_kernel(const uint32_t* __restrict__ obs, int64_t orps,
                                                    const int32_t* __restrict__ gather, int rows, int D,
                                                    int* __restrict__ part) {
  __shared__ int cnt[1024];
  const int seed = blockIdx.y, b = blockIdx.x, nb = gridDim.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int PW = packed_words(D);
  for (int i = tid; i < D; i += 256) cnt[i] = 0;
  __syncthreads();
  const int chunk = (rows + nb - 1) / nb, r0 = b * chunk, r1 = min(rows, r0 + chunk);
  // bits of word `lane` that are features (< D)
  const uint32_t keep = lane * 32 + 32 <= D ? 0xffffffffu : (lane * 32 < D ? (1u << (D - lane * 32)) - 1u : 0u);
  for (int row = r0 + warp; row < r1; row += 8) {
    const int64_t src = gather ? gather[(int64_t)seed * rows + row] : row;
    uint32_t w = lane < PW ? __ldg(obs + ((int64_t)seed * orps + src) * PW + lane) & keep : 0u;
    while (w) {
      const int bit = __ffs(w) - 1;
      w &= w - 1u;
      atomicAdd(&cnt[lane * 32 + bit], 1);
    }
  }
  __syncthreads();
  for (int i = tid; i < D; i += 256) part[((int64_t)seed * nb + b) * D + i] = cnt[i];
}

// second stage, blocks in index order: sums[S][2][D] = (count, count) (x in {0,1}: sum x = sum x^2); bn_sums, when
// given, receives the same (BatchNorm_0 statistics of the minibatch for pqn_bn_stats_update)
__global__ void count_final_kernel(const int* __restrict__ part, int nb, int D, float* __restrict__ sums,
                                   float* __restrict__ bn_sums) {
  const int seed = blockIdx.y, f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= D) return;
  int c = 0;
  for (int b = 0; b < nb; ++b) c += part[((int64_t)seed * nb + b) * D + f];
  const float v = (float)c;
  if (sums) { sums[(int64_t)seed * 2 * D + f] = v; sums[(int64_t)seed * 2 * D + D + f] = v; }
  if (bn_sums) { bn_sums[(int64_t)seed * 2 * D + f] = v; bn_sums[(int64_t)seed * 2 * D + D + f] = v; }
}

// NORM_INPUT: the input BatchNorm of a {0,1} feature is BN(x_f) = a0_f + bit * d_f with d_f = rstd_f * scale_f and
// a0_f = bias_f - mean_f * d_f, mr[S][2][D] = (mean, rstd) (batch or running statistics).  Writes aff[S][2][D] =
// (d, a0).  A feature that is mostly 1 (mean > 1/2) is folded around 1 instead: BN(x_f) = a1_f - (1 - bit) * d_f with
// a1_f = bias_f + (1 - mean_f) * d_f, its bit flipped (flip[S][packed words], read by the product kernels) and its
// Dense_0 row negated -- otherwise a constant-1 column (rstd = 1/sqrt(eps)) would add two large cancelling terms.
// Effective Dense_0 bias beff[S][H] = b0 + sum_f a_f W0[f] (a = a0 or a1).  grid = (ceil(H / 128), S), block = 128
__global__ void eff_kernel(const float* __restrict__ params, int64_t P, int64_t off_bs, int64_t off_bb, int64_t off_w,
                           int64_t off_b, const float* __restrict__ mr, int D, int H, float* __restrict__ aff,
                           uint32_t* __restrict__ flip, float* __restrict__ beff) {
  __shared__ float a0s[1024];
  const int seed = blockIdx.y;
  const float* __restrict__ prm = params + (int64_t)seed * P;
  for (int f = threadIdx.x; f < D; f += blockDim.x) {
    const float mean = mr[(int64_t)seed * 2 * D + f], rstd = mr[(int64_t)seed * 2 * D + D + f];
    const float dd = rstd * prm[off_bs + f], aa = prm[off_bb + f] - mean * dd;
    a0s[f] = mean > 0.5f ? prm[off_bb + f] + (1.0f - mean) * dd : aa;
    if (blockIdx.x == 0) { aff[(int64_t)seed * 2 * D + f] = dd; aff[(int64_t)seed * 2 * D + D + f] = aa; }
  }
  const int PW = packed_words(D);
  if (blockIdx.x == 0 && (int)threadIdx.x < PW) {
    uint32_t m = 0u;
    for (int b = 0; b < 32; ++b) {
      const int f = threadIdx.x * 32 + b;
      if (f < D && mr[(int64_t)seed * 2 * D + f] > 0.5f) m |= 1u << b;
    }
    flip[(int64_t)seed * PW + threadIdx.x] = m;
  }
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= H) return;
  float s = prm[off_b + n];
  for (int f = 0; f < D; ++f) s = fmaf(prm[off_w + (int64_t)f * H + n], a0s[f], s);
  beff[(int64_t)seed * H + n] = s;
}

// NORM_INPUT gradients from G = bits^T dz0 ([S][D][H]; rows of flipped features hold (1 - bit)^T dz0 = sdz - G) and
// sdz = sum_r dz0 (sdz + seed * sdz_stride, [H]), no dgrad:
//   dW0[f] = d_f G[f] + a0_f sdz     d bias_f = W0[f] . sdz     d scale_f = rstd_f (W0[f] . G[f] - mean_f W0[f] . sdz)
// one warp per feature.  grid = (ceil(D / 8), S), block = 256
__global__ void grad_finish_kernel(const float* __restrict__ G, const float* __restrict__ sdz, int64_t sdz_stride,
                                   const float* __restrict__ aff, const uint32_t* __restrict__ flip, const float* __restrict__ mr,
                                   const float* __restrict__ params, int64_t P, int64_t off_w, int64_t off_bs,
                                   int64_t off_bb, int D, int H, float* __restrict__ grads) {
  const int seed = blockIdx.y, lane = threadIdx.x & 31, f = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (f >= D) return;
  const float dd = aff[(int64_t)seed * 2 * D + f], aa = aff[(int64_t)seed * 2 * D + D + f];
  const float mean = mr[(int64_t)seed * 2 * D + f], rstd = mr[(int64_t)seed * 2 * D + D + f];
  const float* __restrict__ W = params + (int64_t)seed * P + off_w + (int64_t)f * H;
  const float* __restrict__ Gf = G + ((int64_t)seed * D + f) * H;
  const float* __restrict__ sz = sdz + (int64_t)seed * sdz_stride;
  float* __restrict__ gw = grads + (int64_t)seed * P + off_w + (int64_t)f * H;
  const bool flipped = (flip[(int64_t)seed * packed_words(D) + (f >> 5)] >> (f & 31)) & 1u;
  float s1 = 0.f, s2 = 0.f;
  for (int n = lane; n < H; n += 32) {
    const float w = W[n], z = sz[n], gv = flipped ? z - Gf[n] : Gf[n];
    gw[n] = fmaf(dd, gv, aa * z);
    s1 = fmaf(w, gv, s1);
    s2 = fmaf(w, z, s2);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if (lane == 0) {
    grads[(int64_t)seed * P + off_bb + f] = s2;
    grads[(int64_t)seed * P + off_bs + f] = rstd * (s1 - mean * s2);
  }
}

// tensor-core path off: the gathered bits as fp32 rows X[S][rows][D] for the PQN_NET_MLP kernels
__global__ void expand_kernel(const uint32_t* __restrict__ obs, int64_t orps, const int32_t* __restrict__ gather,
                              int rows, int D, float* __restrict__ X) {
  const int seed = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)rows * D) return;
  const int r = (int)(i / D), f = (int)(i - (int64_t)r * D);
  const int64_t src = gather ? gather[(int64_t)seed * rows + r] : r;
  const uint32_t w = __ldg(obs + ((int64_t)seed * orps + src) * packed_words(D) + (f >> 5));
  X[((int64_t)seed * rows + r) * D + f] = ((w >> (f & 31)) & 1u) ? 1.f : 0.f;
}

// ---- host side ------------------------------------------------------------------------------------------------------
// Scratch of this kind, placed after the PQN_NET_MLP workspace of the same shape.
struct BitsWs {
  float* x;          // path 0: expanded fp32 rows [S][rows][D]
  uint4* wf;         // B fragments of Dense_0 [S][KS][H/8][32]
  int* cntp;         // popcount partials [S][CNT_BLOCKS][D]
  float *aff, *beff; // NORM_INPUT: (d, a0) [S][2][D], effective bias [S][H]
  uint32_t* flip;    // NORM_INPUT: features folded around 1 [S][packed words]
  float* G;          // NORM_INPUT: bits^T dz0 [S][D][H]
  float* part;       // split partials of the weight gradient [splits][S][D][H]
};

// row splits of the weight gradient: about two CTAs per SM over all seeds, >= 256 rows each, at most 64
static int wgrad_splits(int S, int rows, int D, int H) {
  const int bnc = H >= 128 ? 128 : 64;
  const int ctas = (D + WG_FEAT - 1) / WG_FEAT * (H / bnc) * S;
  int s = (2 * device_sm_count() + ctas - 1) / ctas;
  const int maxs = (rows + 255) / 256;
  if (s > maxs) s = maxs;
  if (s > 64) s = 64;
  if (s < 1) s = 1;
  return s;
}
static int split_rows(int rows, int splits) {
  const int per = (rows + splits - 1) / splits;
  return (per + WG_ROWS - 1) / WG_ROWS * WG_ROWS;
}

static int64_t carve_bits(const pqn_net_desc_t* d, int32_t S, int64_t rows, char* base, BitsWs* w) {
  int64_t off = 0;
  auto take = [&](int64_t nfloats) -> float* {
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += (nfloats * 4 + 255) / 256 * 256;
    return p;
  };
  BitsWs tmp;
  BitsWs* ww = w ? w : &tmp;
  const int D = d->in_c, H = d->hidden, KS = ksteps(D);
  const int64_t R = (int64_t)S * rows;
  const int sp = wgrad_splits(S, (int)rows, D, H);
  const int splits = (int)((rows + split_rows((int)rows, sp) - 1) / split_rows((int)rows, sp));
  ww->x = take(R * D);
  ww->wf = reinterpret_cast<uint4*>(take((int64_t)S * KS * H * 16));
  ww->cntp = reinterpret_cast<int*>(take((int64_t)S * CNT_BLOCKS * D));
  ww->aff = take((int64_t)S * 2 * D);
  ww->beff = take((int64_t)S * H);
  ww->flip = reinterpret_cast<uint32_t*>(take((int64_t)S * packed_words(D)));
  ww->G = take((int64_t)S * D * H);
  ww->part = take((int64_t)(splits > 1 ? splits : 0) * S * D * H);
  return off;
}

// Dense_0' = diag(dvec) . W0 (dvec NULL: W0) -> wf
static void launch_wfrag(const float* params, int64_t P, int64_t off_w, const float* dvec, const uint32_t* flip, int D,
                         int H, int S, uint4* wf, cudaStream_t st) {
  const int64_t n = (int64_t)ksteps(D) * H * 4;
  LaunchScope _ls(K_TC_SPLIT, st);
  wfrag_kernel<<<dim3(cdiv(n, 256), S), 256, 0, st>>>(params, P, off_w, dvec, flip, D, H, ksteps(D), wf);
}

// Z[S][rows][H] = bits . Dense_0' + bias (bias + seed * bias_stride, [H])
static int launch_fwd(const uint32_t* obs, int64_t orps, const int32_t* gather, int rows, int D, int H, const uint4* wf,
                      const float* bias, int64_t bias_stride, const uint32_t* flip, float* Z, int S, cudaStream_t st) {
  const int KS = ksteps(D), NT = fwd_ntiles(KS);
  const size_t sm = fwd_smem(KS, NT);
  auto kfn = NT == 8 ? fwd_kernel<8> : fwd_kernel<4>;
  if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm) != cudaSuccess)
    return check_launch("bits fwd(cudaFuncSetAttribute)");
  const int tiles = (rows + FWD_ROWS - 1) / FWD_ROWS, slices = H / (8 * NT);
  int per = (device_sm_count() + slices * S - 1) / (slices * S);   // one CTA per SM over all seeds and slices
  if (per > tiles) per = tiles;
  if (per < 1) per = 1;
  LaunchScope _ls(K_BITS_FWD, st);
  kfn<<<dim3(per, slices, S), FWD_WARPS * 32, sm, st>>>(obs, orps, gather, rows, D, KS, wf, H, bias, bias_stride, flip, Z);
  return 0;
}

// dW0 (or G) = bits^T . dz; out + seed * out_seed_stride, [D][H].  The row splits' partials are added in split order.
static void launch_wgrad(const uint32_t* obs, int64_t orps, const int32_t* gather, int rows, int D, int H, const float* dz,
                         float gscale, const uint32_t* flip, float* out, int64_t out_seed_stride, const BitsWs& w, int S,
                         cudaStream_t st) {
  const int rps = split_rows(rows, wgrad_splits(S, rows, D, H));
  const int splits = (rows + rps - 1) / rps;
  const int64_t n = (int64_t)D * H;
  float* dst = splits > 1 ? w.part : out;
  const int64_t dss = splits > 1 ? n : out_seed_stride;
  const unsigned fx = (unsigned)((D + WG_FEAT - 1) / WG_FEAT);
  { LaunchScope _ls(K_BITS_WGRAD, st);
    if (H >= 128)
      wgrad_kernel<128><<<dim3(fx, H / 128, splits * S), 256, 0, st>>>(obs, orps, gather, rows, D, dz, H, gscale, S, rps, flip, dst,
                                                                       dss, (int64_t)S * n);
    else
      wgrad_kernel<64><<<dim3(fx, H / 64, splits * S), 128, 0, st>>>(obs, orps, gather, rows, D, dz, H, gscale, S, rps, flip, dst,
                                                                     dss, (int64_t)S * n); }
  if (splits > 1) launch_split_reduce(w.part, splits, (int64_t)S * n, n, S, out, out_seed_stride, st);
}

// per-feature popcounts of the gathered minibatch -> sums and / or bn_sums ([S][2][D] each, may be NULL)
static void launch_counts(const uint32_t* obs, int64_t orps, const int32_t* gather, int rows, int D, const BitsWs& w,
                          float* sums, float* bn_sums, int S, cudaStream_t st) {
  { LaunchScope _ls(K_NORM_REDUCE, st); count_kernel<<<dim3(CNT_BLOCKS, S), 256, 0, st>>>(obs, orps, gather, rows, D, w.cntp); }
  { LaunchScope _ls(K_GRAD_FINAL, st); count_final_kernel<<<dim3(cdiv(D, 256), S), 256, 0, st>>>(w.cntp, CNT_BLOCKS, D, sums, bn_sums); }
}

static void launch_expand(const uint32_t* obs, int64_t orps, const int32_t* gather, int rows, int D, float* X, int S,
                          cudaStream_t st) {
  LaunchScope _ls(K_GATHER_ROWS, st);
  expand_kernel<<<dim3(cdiv((int64_t)rows * D, 256), S), 256, 0, st>>>(obs, orps, gather, rows, D, X);
}

// the PQN_NET_MLP descriptor of the same network (what the layout and the fp32 kernels see)
static inline pqn_net_desc_t as_mlp(const pqn_net_desc_t* d) {
  pqn_net_desc_t m = *d;
  m.kind = PQN_NET_MLP;
  return m;
}

}  // namespace bits
