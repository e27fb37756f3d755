// Q-network forward / loss-gradient kernels for sm_90a, batched over S
// independent seeds (blockIdx.y or .z = seed; every seed has its own weights).
//
// Reference: QNetwork/CNN  purejaxql/pqn_minatar.py:24-69,
//            MLP QNetwork  purejaxql/pqn_gymnax.py:29-58,
//            _loss_fn      purejaxql/pqn_minatar.py:271-291.
// fp32 throughout (the north star asks for 1e-5 agreement with an fp32 oracle):
// the dense contractions are register-tiled FFMA GEMMs (128x128x16 CTA tiles,
// 8x8 per thread, double-buffered shared memory, 128-bit LDS) with the
// bias + LayerNorm + ReLU (+ Q-head) epilogue fused in registers; the 3x3 conv
// consumes the bit-packed observations directly (its input is {0,1}/255, so a
// tap contributes either w/255 or nothing) and skips taps no lane of the warp
// has set.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pqn_b200.h"
#include "api_common.h"
#include "tc_common.cuh"
#include "conv16.cuh"

namespace pqn {

constexpr int GT = 256;   // threads per GEMM CTA (16 x 16)
constexpr int BK = 16;    // reduce-dim tile

// wgmma path for the CNN dense layer (pqn_set_tensor_core_path); default on
static int g_use_tc = 2;  // 0 FFMA, 1 3xTF32 on mma.sync (A_lo derived in the kernel), 2 wgmma on fp16-split planes (default)
// warp-level tensor-core (mma.sync tf32) conv kernels (pqn_set_conv_mma_path); default on
static int g_conv_mma = 1;   // 0: fp32 CUDA cores, 1: fp16 mma.sync forward (default), 3: tf32 mma.sync forward
                             // (1, 3: mma.sync backward)
// the Q-value forward (rollout, bootstrap, evaluation) computes the conv inside the dense forward GEMM
// (pqn_set_conv_fusion), with tensor-core path 2 and conv path 1; default on
static int g_conv_fuse = 1;

__host__ __device__ static inline int64_t align4(int64_t x) { return (x + 3) & ~(int64_t)3; }

static int make_layout(const pqn_net_desc_t* d, pqn_net_layout_t* L) {
  int64_t off = 0;
  auto take = [&](int64_t n) { int64_t o = off; off += align4(n); return o; };
  L->d1_w = L->d1_b = L->ln1_scale = L->ln1_bias = L->conv_w = L->conv_b = -1;
  L->gru_ir_w = L->gru_ir_b = L->gru_iz_w = L->gru_iz_b = L->gru_in_w = L->gru_in_b = -1;
  L->gru_hr_w = L->gru_hz_w = L->gru_hn_w = L->gru_hn_b = -1;
  const int A = d->num_actions;
  const bool has_norm = d->norm_type != PQN_NORM_NONE;   // layer_norm and batch_norm have (scale, bias) of the same shape
  if (d->kind == PQN_NET_MINATAR_CNN) {
    const int C = d->in_c;
    L->bn_scale = take(C); L->bn_bias = take(C);
    L->conv_w = take(9 * C * CONV_O); L->conv_b = take(CONV_O);
    L->ln0_scale = L->ln0_bias = -1;   // norm_type none: the network has no normalisation parameters
    if (has_norm) { L->ln0_scale = take(CONV_O); L->ln0_bias = take(CONV_O); }
    L->d0_w = take((int64_t)FLAT_CNN * HID_CNN); L->d0_b = take(HID_CNN);
    if (has_norm) { L->ln1_scale = take(HID_CNN); L->ln1_bias = take(HID_CNN); }
    L->head_w = take((int64_t)HID_CNN * A); L->head_b = take(A);
  } else if (d->kind == PQN_NET_MLP || d->kind == PQN_NET_RNN || d->kind == PQN_NET_MLP_BITS) {
    const int D = d->in_c, H = d->hidden;
    L->bn_scale = take(D); L->bn_bias = take(D);
    L->d0_w = take((int64_t)D * H); L->d0_b = take(H);
    L->ln0_scale = L->ln0_bias = -1;
    if (has_norm) { L->ln0_scale = take(H); L->ln0_bias = take(H); }
    // layers >= 2 follow layer 1 in the same pattern; dense_off restates this order for any layer (keep the two in step)
    for (int l = 1; l < d->layers; ++l) {
      const int64_t w = take((int64_t)H * H), b = take(H);
      const int64_t sc = has_norm ? take(H) : -1, bi = has_norm ? take(H) : -1;
      if (l == 1) { L->d1_w = w; L->d1_b = b; L->ln1_scale = sc; L->ln1_bias = bi; }
    }
    if (d->kind == PQN_NET_RNN) {   // flax GRUCell: input denses with bias, recurrent ones without (except hn)
      L->gru_ir_w = take((int64_t)(H + A) * H); L->gru_ir_b = take(H);
      L->gru_iz_w = take((int64_t)(H + A) * H); L->gru_iz_b = take(H);
      L->gru_in_w = take((int64_t)(H + A) * H); L->gru_in_b = take(H);
      L->gru_hr_w = take((int64_t)H * H); L->gru_hz_w = take((int64_t)H * H);
      L->gru_hn_w = take((int64_t)H * H); L->gru_hn_b = take(H);
    }
    L->head_w = take((int64_t)H * A); L->head_b = take(A);
  } else {
    return -1;
  }
  L->total = off;
  return 0;
}

// Offsets of hidden layer l (Dense_l kernel / bias, its norm's scale / bias; -1 where there is none) of an MLP / GRU
// layout: layers 0 and 1 are the d0/ln0 and d1/ln1 fields, layers >= 2 follow layer 1's norm with the same stride.
struct DenseOff { int64_t w, b, g, bi; };
__host__ __device__ inline DenseOff dense_off(const pqn_net_layout_t& L, int H, int l) {
  if (l == 0) return DenseOff{L.d0_w, L.d0_b, L.ln0_scale, L.ln0_bias};
  if (l == 1) return DenseOff{L.d1_w, L.d1_b, L.ln1_scale, L.ln1_bias};
  const bool norm = L.ln1_scale >= 0;
  const int64_t stride = align4((int64_t)H * H) + (norm ? 3 : 1) * align4(H);
  const int64_t w = (norm ? L.ln1_bias : L.d1_b) + align4(H) + (l - 2) * stride;
  const int64_t b = w + align4((int64_t)H * H);
  return DenseOff{w, b, norm ? b + align4(H) : -1, norm ? b + 2 * align4(H) : -1};
}

static int check_desc(const pqn_net_desc_t* d, const char* who) {
  if (!d) return set_error(PQN_E_INVALID, "%s: desc is NULL", who);
  if (d->num_actions < 1 || d->num_actions > 32) return set_error(PQN_E_INVALID, "%s: num_actions=%d out of [1,32]", who, d->num_actions);
  if (d->norm_type < 0 || d->norm_type > 2 || d->norm_input < 0 || d->norm_input > 1)
    return set_error(PQN_E_INVALID, "%s: norm_type=%d norm_input=%d", who, d->norm_type, d->norm_input);
  if (d->kind == PQN_NET_MLP || d->kind == PQN_NET_RNN || d->kind == PQN_NET_MLP_BITS) {
    const int H = d->hidden;
    if (H != 64 && H != 128 && H != 256 && H != 512)
      return set_error(PQN_E_UNSUPPORTED, "%s: hidden=%d (64, 128, 256 or 512 built)", who, H);
    if (d->layers < 1 || d->layers > PQN_MAX_LAYERS)
      return set_error(PQN_E_UNSUPPORTED, "%s: layers=%d (1 to %d built)", who, d->layers, PQN_MAX_LAYERS);
  }
  {
    // row_bwd_kernel keeps [A][N] head weights + eight warp-private [A][N] gradient slices in shared memory
    const int Nh = d->kind == PQN_NET_MINATAR_CNN ? 128 : d->hidden;
    const size_t need = (size_t)(24 * Nh + 9 * d->num_actions * Nh + 8 * d->num_actions + 16) * sizeof(float);
    if (need > 227u * 1024u)
      return set_error(PQN_E_UNSUPPORTED, "%s: hidden=%d with num_actions=%d needs %zu B of shared memory for the head "
                       "backward (limit 227 KB)", who, Nh, d->num_actions, need);
  }
  if (d->kind == PQN_NET_MINATAR_CNN) {
    if (d->in_c != 4 && d->in_c != 6 && d->in_c != 7 && d->in_c != 10)
      return set_error(PQN_E_UNSUPPORTED, "%s: CNN in_c=%d (MinAtar uses 4/6/7/10)", who, d->in_c);
    return PQN_OK;
  }
  if (d->kind == PQN_NET_MLP_BITS) {
    if (d->in_c != 400 && d->in_c != 600 && d->in_c != 700 && d->in_c != 1000)
      return set_error(PQN_E_UNSUPPORTED, "%s: MLP on packed MinAtar observations with in_c=%d (100 * C: 400, 600 or 700 "
                       "built, and 1000 for Seaquest)", who, d->in_c);
    return PQN_OK;
  }
  if (d->kind == PQN_NET_MLP || d->kind == PQN_NET_RNN) {
    if (d->in_c < 1 || d->in_c > 4096) return set_error(PQN_E_INVALID, "%s: MLP in dim %d", who, d->in_c);
    return PQN_OK;
  }
  return set_error(PQN_E_INVALID, "%s: unknown net kind %d", who, d->kind);
}

// ---------------------------------------------------------------------------
// GEMM tile core: acc[TM][TN] += As[k][rows of thread] * Bs[k][cols of thread]
// thread (tx, ty) owns rows  {c*64 + ty*4 + i}  and cols {c*64 + tx*4 + j}.
// ---------------------------------------------------------------------------
template <int BM, int BN, int TM, int TN>
__device__ __forceinline__ void tile_mma(const float* __restrict__ As, const float* __restrict__ Bs, int tx, int ty,
                                         float (&acc)[TM][TN]) {
#pragma unroll
  for (int kk = 0; kk < BK; ++kk) {
    float a[TM], b[TN];
#pragma unroll
    for (int c = 0; c < TM / 4; ++c) {
      const float4 v = *reinterpret_cast<const float4*>(As + kk * BM + c * 64 + ty * 4);
      a[4 * c] = v.x; a[4 * c + 1] = v.y; a[4 * c + 2] = v.z; a[4 * c + 3] = v.w;
    }
#pragma unroll
    for (int c = 0; c < TN / 4; ++c) {
      const float4 v = *reinterpret_cast<const float4*>(Bs + kk * BN + c * 64 + tx * 4);
      b[4 * c] = v.x; b[4 * c + 1] = v.y; b[4 * c + 2] = v.z; b[4 * c + 3] = v.w;
    }
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
  }
}

// Load 4 consecutive reduce-dim elements src[0..3] (bounds: r0+j < R), vector if allowed.
__device__ __forceinline__ float4 load4_guard(const float* __restrict__ src, int r0, int R, bool vec_ok, bool row_ok) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!row_ok) return v;
  if (vec_ok && r0 + 3 < R) return __ldg(reinterpret_cast<const float4*>(src));
  if (r0 < R) v.x = __ldg(src);
  if (r0 + 1 < R) v.y = __ldg(src + 1);
  if (r0 + 2 < R) v.z = __ldg(src + 2);
  if (r0 + 3 < R) v.w = __ldg(src + 3);
  return v;
}

// ---------------------------------------------------------------------------
// dense_fwd: Y = LayerNorm(X @ W + b) -> ReLU  [-> head]
//   MODE 0: write H          (inference hidden layer)
//   MODE 1: write H, XHAT, RSTD  (training forward: what the backward needs)
//   MODE 2: write Q = H @ Wh + bh only (inference last layer, Q-head fused)
//   MODE 3: write the raw pre-activation X @ W + b to H (no LayerNorm; modular NORM_TYPE path)
// grid = (ceil(rows/BM), S, column tiles); more than one column tile (rows of gridDim.z * BN outputs) for MODE 3 only
// ---------------------------------------------------------------------------
template <int BN, int MODE>
__global__ void __launch_bounds__(GT) dense_fwd_kernel(
    const float* __restrict__ X, int64_t x_seed_stride, int ldx, const float* __restrict__ params, int64_t P,
    int64_t off_w, int64_t off_b, int64_t off_scale, int64_t off_bias, int64_t off_hw, int64_t off_hb, int A,
    float* __restrict__ H, float* __restrict__ XHAT, float* __restrict__ RSTD, float* __restrict__ Q, int rows,
    int K) {
  constexpr int BM = (BN == 128) ? 128 : 64;
  constexpr int TM = BM / 16, TN = BN / 16;
  constexpr int A_LD = BM / 64, B_LD = BN / 64;
  __shared__ __align__(16) float As[2][BK * BM];
  __shared__ __align__(16) float Bs[2][BK * BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int seed = blockIdx.y;
  const int m0 = blockIdx.x * BM;
  const int n0 = blockIdx.z * BN, ldn = gridDim.z * BN;   // this CTA's output columns, row stride of W and H
  const float* __restrict__ Xs = X + (int64_t)seed * x_seed_stride;
  const float* __restrict__ prm = params + (int64_t)seed * P;
  const float* __restrict__ W = prm + off_w + n0;
  const bool vecA = (ldx % 4 == 0) && ((reinterpret_cast<uintptr_t>(Xs) & 15) == 0);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nk = (K + BK - 1) / BK;
  float4 ra[A_LD], rb[B_LD];
  auto gload = [&](int kt) {
#pragma unroll
    for (int i = 0; i < A_LD; ++i) {
      const int f = tid + i * GT;
      const int m = f >> 2, r4 = f & 3;
      const int row = m0 + m;
      const int k = kt * BK + r4 * 4;
      ra[i] = load4_guard(Xs + (int64_t)row * ldx + k, k, K, vecA, row < rows);
    }
#pragma unroll
    for (int i = 0; i < B_LD; ++i) {
      const int f = tid + i * GT;
      const int r = f / (BN / 4), n4 = f % (BN / 4);
      const int k = kt * BK + r;
      rb[i] = (k < K) ? __ldg(reinterpret_cast<const float4*>(W + (int64_t)k * ldn + n4 * 4))
                      : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_LD; ++i) {
      const int f = tid + i * GT;
      const int m = f >> 2, r4 = f & 3;
      float* dst = &As[buf][(r4 * 4) * BM + m];
      dst[0] = ra[i].x; dst[BM] = ra[i].y; dst[2 * BM] = ra[i].z; dst[3 * BM] = ra[i].w;
    }
#pragma unroll
    for (int i = 0; i < B_LD; ++i) {
      const int f = tid + i * GT;
      const int r = f / (BN / 4), n4 = f % (BN / 4);
      *reinterpret_cast<float4*>(&Bs[buf][r * BN + n4 * 4]) = rb[i];
    }
  };

  gload(0);
  sstore(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    if (kt + 1 < nk) gload(kt + 1);
    tile_mma<BM, BN, TM, TN>(As[kt & 1], Bs[kt & 1], tx, ty, acc);
    if (kt + 1 < nk) sstore((kt + 1) & 1);
    __syncthreads();
  }

  // ---- epilogue: bias, LayerNorm over the BN columns of each row, ReLU
  const float* __restrict__ bvec = prm + (off_b >= 0 ? off_b + n0 : 0);
  const float* __restrict__ sc = prm + off_scale;
  const float* __restrict__ bi = prm + off_bias;
  float colb[TN], cols_[TN], colbi[TN];
#pragma unroll
  for (int j = 0; j < TN; ++j) {
    const int col = (j >> 2) * 64 + tx * 4 + (j & 3);
    colb[j] = off_b >= 0 ? __ldg(bvec + col) : 0.f; cols_[j] = __ldg(sc + col); colbi[j] = __ldg(bi + col);
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int row = m0 + (i >> 2) * 64 + ty * 4 + (i & 3);
    if (MODE == 3) {  // raw pre-activation (bias only): the modular NORM_TYPE path normalises in its own kernels
      if (row < rows) {
        const int64_t grow3 = (int64_t)seed * rows + row;
#pragma unroll
        for (int c = 0; c < TN / 4; ++c)
          *reinterpret_cast<float4*>(H + grow3 * ldn + n0 + c * 64 + tx * 4) =
              make_float4(acc[i][4 * c] + colb[4 * c], acc[i][4 * c + 1] + colb[4 * c + 1], acc[i][4 * c + 2] + colb[4 * c + 2],
                          acc[i][4 * c + 3] + colb[4 * c + 3]);
      }
      continue;
    }
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      acc[i][j] += colb[j];
      s1 += acc[i][j];
      s2 += acc[i][j] * acc[i][j];
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const float mean = s1 * (1.0f / BN);
    const float var = fmaxf(s2 * (1.0f / BN) - mean * mean, 0.f);
    const float rstd = 1.0f / sqrtf(var + LN_EPS);
    float xh[TN], h[TN];
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      xh[j] = (acc[i][j] - mean) * rstd;
      h[j] = fmaxf(xh[j] * cols_[j] + colbi[j], 0.f);
    }
    const bool row_ok = row < rows;
    const int64_t grow = (int64_t)seed * rows + row;
    if (MODE == 0 || MODE == 1) {
      if (row_ok) {
#pragma unroll
        for (int c = 0; c < TN / 4; ++c) {
          const int col = c * 64 + tx * 4;
          *reinterpret_cast<float4*>(H + grow * BN + col) = make_float4(h[4 * c], h[4 * c + 1], h[4 * c + 2], h[4 * c + 3]);
          if (MODE == 1)
            *reinterpret_cast<float4*>(XHAT + grow * BN + col) =
                make_float4(xh[4 * c], xh[4 * c + 1], xh[4 * c + 2], xh[4 * c + 3]);
        }
        if (MODE == 1 && tx == 0) RSTD[grow] = rstd;
      }
    } else {
      const float* __restrict__ HW = prm + off_hw;
      const float* __restrict__ HB = prm + off_hb;
      for (int a = 0; a < A; ++a) {
        float pq = 0.f;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
          const int col = (j >> 2) * 64 + tx * 4 + (j & 3);
          pq = fmaf(h[j], __ldg(HW + (int64_t)col * A + a), pq);
        }
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) pq += __shfl_xor_sync(0xffffffffu, pq, o);
        if (tx == 0 && row_ok) Q[grow * A + a] = pq + __ldg(HB + a);
      }
    }
  }
}

// ---------------------------------------------------------------------------
// wgrad: dW[kin][n] (+)= sum_rows X[row][kin] * dZ[row][n]
// grid = (ceil(Kin/128), N/BN, S*splits); splits > 1 writes per-split partials (launch through run_wgrad_ffma).
// BN = 128, or 64 for a 64-wide layer (HIDDEN_SIZE 64)
// ---------------------------------------------------------------------------
template <int BN>
__global__ void __launch_bounds__(GT) wgrad_kernel(const float* __restrict__ X, int64_t x_seed_stride, int ldx,
                                                   const float* __restrict__ DZ, int64_t dz_seed_stride, int N,
                                                   float* __restrict__ grads, int64_t P, int64_t off_w, int rows,
                                                   int Kin, int splits, float* __restrict__ part) {
  constexpr int BM = 128, TM = 8, TN = BN / 16, B_LD = BN / 64;
  __shared__ __align__(16) float As[2][BK * BM];
  __shared__ __align__(16) float Bs[2][BK * BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int seed = blockIdx.z / splits, split = blockIdx.z % splits;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const float* __restrict__ Xs = X + (int64_t)seed * x_seed_stride;
  const float* __restrict__ Zs = DZ + (int64_t)seed * dz_seed_stride;
  int chunk = (rows + splits - 1) / splits;
  chunk = (chunk + BK - 1) / BK * BK;
  const int r_begin = split * chunk;
  const int r_end = min(rows, r_begin + chunk);
  const bool vecA = (ldx % 4 == 0) && ((reinterpret_cast<uintptr_t>(Xs) & 15) == 0);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nk = (r_end > r_begin) ? (r_end - r_begin + BK - 1) / BK : 0;
  float4 ra[2], rb[B_LD];
  auto gload = [&](int kt) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int f = tid + i * GT;
      const int r = f >> 5, m4 = f & 31;
      const int row = r_begin + kt * BK + r;
      const int kin = m0 + m4 * 4;
      ra[i] = load4_guard(Xs + (int64_t)row * ldx + kin, kin, Kin, vecA, row < r_end);
    }
#pragma unroll
    for (int i = 0; i < B_LD; ++i) {
      const int f = tid + i * GT;
      const int r = f / (BN / 4), n4 = f % (BN / 4);
      const int row = r_begin + kt * BK + r;
      rb[i] = (row < r_end) ? __ldg(reinterpret_cast<const float4*>(Zs + (int64_t)row * N + n0 + n4 * 4))
                            : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int f = tid + i * GT;
      const int r = f >> 5, m4 = f & 31;
      *reinterpret_cast<float4*>(&As[buf][r * BM + m4 * 4]) = ra[i];
    }
#pragma unroll
    for (int i = 0; i < B_LD; ++i) {
      const int f = tid + i * GT;
      const int r = f / (BN / 4), n4 = f % (BN / 4);
      *reinterpret_cast<float4*>(&Bs[buf][r * BN + n4 * 4]) = rb[i];
    }
  };
  if (nk > 0) {
    gload(0);
    sstore(0);
  }
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    if (kt + 1 < nk) gload(kt + 1);
    tile_mma<BM, BN, TM, TN>(As[kt & 1], Bs[kt & 1], tx, ty, acc);
    if (kt + 1 < nk) sstore((kt + 1) & 1);
    __syncthreads();
  }
  // splits == 1: the gradient itself; otherwise this row range's partial [split][seed][Kin][N], added in split order by
  // wgrad_split_reduce_kernel (no float atomics)
  float* __restrict__ dW = splits == 1 ? grads + (int64_t)seed * P + off_w
                                       : part + ((int64_t)split * (gridDim.z / splits) + seed) * Kin * N;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int kin = m0 + (i >> 2) * 64 + ty * 4 + (i & 3);
    if (kin >= Kin) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + (j >> 2) * 64 + tx * 4 + (j & 3);
      dW[(int64_t)kin * N + n] = acc[i][j];
    }
  }
}

// ---------------------------------------------------------------------------
// dgrad: OUT[row][c] = (HPREV[row][c] > 0) * sum_n dZ[row][n] * W[c][n]
// (ReLU mask of the previous layer fused; OUT may alias HPREV)
// grid = (ceil(rows/128), Kprev/BN, S); BN = 128, or 64 for a 64-wide layer (launch through launch_dgrad)
// ---------------------------------------------------------------------------
template <int BN>
__global__ void __launch_bounds__(GT) dgrad_kernel(const float* __restrict__ DZ, int64_t dz_seed_stride, int N,
                                                   const float* __restrict__ params, int64_t P, int64_t off_w,
                                                   const float* HPREV, float* OUT, int64_t h_seed_stride, int rows,
                                                   int Kprev, int accumulate) {
  constexpr int BM = 128, TM = 8, TN = BN / 16, B_LD = BN / 64;
  __shared__ __align__(16) float As[2][BK * BM];
  __shared__ __align__(16) float Bs[2][BK * BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int seed = blockIdx.z;
  const int m0 = blockIdx.x * BM, c0 = blockIdx.y * BN;
  const float* __restrict__ Zs = DZ + (int64_t)seed * dz_seed_stride;
  const float* __restrict__ W = params + (int64_t)seed * P + off_w;  // [Kprev][N]

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  const int nk = N / BK;
  float4 ra[2], rb[B_LD];
  auto gload = [&](int kt) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int f = tid + i * GT;
      const int m = f >> 2, r4 = f & 3;
      const int n = kt * BK + r4 * 4;
      const int row = m0 + m;
      ra[i] = (row < rows) ? __ldg(reinterpret_cast<const float4*>(Zs + (int64_t)row * N + n))
                           : make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < B_LD) rb[i] = __ldg(reinterpret_cast<const float4*>(W + (int64_t)(c0 + m) * N + n));
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int f = tid + i * GT;
      const int m = f >> 2, r4 = f & 3;
      float* da = &As[buf][(r4 * 4) * BM + m];
      da[0] = ra[i].x; da[BM] = ra[i].y; da[2 * BM] = ra[i].z; da[3 * BM] = ra[i].w;
      if (i < B_LD) {
        float* db = &Bs[buf][(r4 * 4) * BN + m];
        db[0] = rb[i].x; db[BN] = rb[i].y; db[2 * BN] = rb[i].z; db[3 * BN] = rb[i].w;
      }
    }
  };
  gload(0);
  sstore(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    if (kt + 1 < nk) gload(kt + 1);
    tile_mma<BM, BN, TM, TN>(As[kt & 1], Bs[kt & 1], tx, ty, acc);
    if (kt + 1 < nk) sstore((kt + 1) & 1);
    __syncthreads();
  }
  const float* Hs = HPREV + (int64_t)seed * h_seed_stride;   // ReLU mask source (the layer output: h > 0)
  float* Os = OUT + (int64_t)seed * h_seed_stride;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int row = m0 + (i >> 2) * 64 + ty * 4 + (i & 3);
    if (row >= rows) continue;
#pragma unroll
    for (int c = 0; c < TN / 4; ++c) {
      const int col = c0 + c * 64 + tx * 4;
      const float4 hv = *reinterpret_cast<const float4*>(Hs + (int64_t)row * Kprev + col);
      float4 o;
      o.x = hv.x > 0.f ? acc[i][4 * c] : 0.f;
      o.y = hv.y > 0.f ? acc[i][4 * c + 1] : 0.f;
      o.z = hv.z > 0.f ? acc[i][4 * c + 2] : 0.f;
      o.w = hv.w > 0.f ? acc[i][4 * c + 3] : 0.f;
      if (accumulate) {   // OUT += ... (sum of several products, e.g. the three GRU gates; OUT must not alias HPREV)
        const float4 prev = *reinterpret_cast<const float4*>(Os + (int64_t)row * Kprev + col);
        o.x += prev.x; o.y += prev.y; o.z += prev.z; o.w += prev.w;
      }
      *reinterpret_cast<float4*>(Os + (int64_t)row * Kprev + col) = o;
    }
  }
}

// ---------------------------------------------------------------------------
// row backward: one warp per sample.
//   HEAD=1: q = h @ Wh + bh, loss/qsa accumulation, dq, dWh, dbh, dh = dq*Wh[:,a],
//           ReLU mask from h.      HEAD=0: dy read from DH (already ReLU-masked).
//   then LayerNorm backward -> DZ, accumulating dscale, dbias and db (= sum dz).
// grid = (ceil(rows/ROWS_PER_CTA), S)
// ---------------------------------------------------------------------------

// V consecutive features of a lane (V = 4: float4, V = 2: float2)
template <int V>
__device__ __forceinline__ void ld_feat(const float* p, float* o) {
  if constexpr (V == 4) {
    const float4 v = *reinterpret_cast<const float4*>(p);
    o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
  } else {
    const float2 v = *reinterpret_cast<const float2*>(p);
    o[0] = v.x; o[1] = v.y;
  }
}
template <int V>
__device__ __forceinline__ void st_feat(float* p, const float* o) {
  if constexpr (V == 4) *reinterpret_cast<float4*>(p) = make_float4(o[0], o[1], o[2], o[3]);
  else *reinterpret_cast<float2*>(p) = make_float2(o[0], o[1]);
}

template <int N, bool HEAD>
__global__ void __launch_bounds__(256) row_bwd_kernel(
    const float* __restrict__ Hh, const float* __restrict__ XHAT, const float* __restrict__ RSTD,
    const float* DH, float* DZ, float* DZLO, __half* DZ16H, __half* DZ16L, float gscale,
    const float* __restrict__ params, float* __restrict__ grads, int64_t P,
    int64_t off_scale, int64_t off_dscale, int64_t off_dbias, int64_t off_db, int64_t off_hw, int64_t off_hb, int A,
    const int32_t* __restrict__ gather, const int32_t* __restrict__ action, const float* __restrict__ target,
    int64_t tr_rows_per_seed, float* __restrict__ part, int rows) {
  // Reductions over rows are deterministic: lane-private registers -> warp-private shared-memory slices -> a fixed-order
  // sum over the 8 warps -> this CTA's partial vector part[seed][cta][3N (+ A*N + A + 2)], which row_bwd_final_kernel
  // adds over the CTAs in index order (no float atomics anywhere).
  constexpr int F = N / 32;  // features per lane, in chunks of V at lane*V + c*32*V
  constexpr int V = N >= 128 ? 4 : 2, CW = 32 * V;
  extern __shared__ float smem[];
  float* s_red3 = smem;           // [8 warps][3N]  d scale, d bias, d dense-bias slices
  float* s_hw = smem + 24 * N;    // [A][N]  head weights, transposed copy (HEAD)
  float* s_dhw = s_hw + (HEAD ? A * N : 0);   // [8 warps][A][N]  warp-private head-weight gradient slices (HEAD);
                                              // 16-byte aligned for the float4 accesses, scalars go last
  float* s_dhb = s_dhw + (HEAD ? 8 * A * N : 0);  // [8 warps][A]
  float* s_ls = s_dhb + (HEAD ? 8 * A : 0);       // [8 warps][2] loss, qsa
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int seed = blockIdx.y;
  const float* __restrict__ prm = params + (int64_t)seed * P;
  const int nsm = 24 * N + (HEAD ? A * N + 8 * A + 16 + 8 * A * N : 0);
  for (int i = tid; i < nsm; i += 256) smem[i] = 0.f;
  __syncthreads();
  if (HEAD)
    for (int i = tid; i < A * N; i += 256) s_hw[(i % A) * N + i / A] = __ldg(prm + off_hw + i);
  __syncthreads();
  float scale[F];
#pragma unroll
  for (int j = 0; j < F; ++j) scale[j] = __ldg(prm + off_scale + (j / V) * CW + lane * V + (j % V));
  float a_dsc[F], a_dbi[F], a_db[F];
#pragma unroll
  for (int j = 0; j < F; ++j) a_dsc[j] = a_dbi[j] = a_db[j] = 0.f;
  float a_loss = 0.f, a_qsa = 0.f;
  const float invB = 1.0f / (float)rows;
  float* my_dhw = s_dhw + warp * A * N;

  // grid-stride over the seed's rows, one row per warp (grid.x is sized in whole waves, see conv_mma_ctas)
  for (int row = blockIdx.x * 8 + warp; row < rows; row += gridDim.x * 8) {
    const int64_t grow = (int64_t)seed * rows + row;
    float h[F], xh[F], dy[F];
#pragma unroll
    for (int c = 0; c < F / V; ++c) ld_feat<V>(XHAT + grow * N + c * CW + lane * V, xh + V * c);
    const float rstd = RSTD[grow];
    if (HEAD) {
#pragma unroll
      for (int c = 0; c < F / V; ++c) ld_feat<V>(Hh + grow * N + c * CW + lane * V, h + V * c);
      const int src = gather ? gather[(int64_t)seed * rows + row] : row;
      const int act = action[(int64_t)seed * tr_rows_per_seed + src];
      const float tgt = target[(int64_t)seed * tr_rows_per_seed + src];
      // q_sa only needs column `act` of the head
      float pq = 0.f;
      float wcol[F];
#pragma unroll
      for (int c = 0; c < F / V; ++c) ld_feat<V>(s_hw + act * N + c * CW + lane * V, wcol + V * c);
#pragma unroll
      for (int j = 0; j < F; ++j) pq = fmaf(h[j], wcol[j], pq);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) pq += __shfl_xor_sync(0xffffffffu, pq, o);
      const float q_sa = pq + __ldg(prm + off_hb + act);
      const float diff = q_sa - tgt;
      const float dq = diff * invB;
      if (lane == 0) {
        a_loss += 0.5f * diff * diff * invB;
        a_qsa += q_sa * invB;
        s_dhb[warp * A + act] += dq;   // warp-private slot, one writer
      }
#pragma unroll
      for (int c = 0; c < F / V; ++c) {  // warp-private slice: plain read-modify-write, no atomics
        float* dst = my_dhw + act * N + c * CW + lane * V;
        float v[V];
        ld_feat<V>(dst, v);
#pragma unroll
        for (int k = 0; k < V; ++k) v[k] = fmaf(h[V * c + k], dq, v[k]);
        st_feat<V>(dst, v);
      }
#pragma unroll
      for (int j = 0; j < F; ++j) dy[j] = h[j] > 0.f ? dq * wcol[j] : 0.f;
    } else {
#pragma unroll
      for (int c = 0; c < F / V; ++c) ld_feat<V>(DH + grow * N + c * CW + lane * V, dy + V * c);
    }
    float m1 = 0.f, m2 = 0.f;
    float dxh[F];
#pragma unroll
    for (int j = 0; j < F; ++j) {
      a_dsc[j] = fmaf(dy[j], xh[j], a_dsc[j]);
      a_dbi[j] += dy[j];
      dxh[j] = dy[j] * scale[j];
      m1 += dxh[j];
      m2 = fmaf(dxh[j], xh[j], m2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      m1 += __shfl_xor_sync(0xffffffffu, m1, o);
      m2 += __shfl_xor_sync(0xffffffffu, m2, o);
    }
    m1 *= (1.0f / N);
    m2 *= (1.0f / N);
    float dz[F];
#pragma unroll
    for (int j = 0; j < F; ++j) {
      dz[j] = rstd * (dxh[j] - m1 - xh[j] * m2);
      a_db[j] += dz[j];
    }
#pragma unroll
    for (int c = 0; c < F / V; ++c)
    {
      const int64_t e = grow * N + c * CW + lane * V;
      if (DZ16H != nullptr) {  // fp16-split planes of dz * gscale for the tensor-core wgrad / dgrad (no fp32 copy)
        __half2 h0, h1, l0, l1;
        tc::split16x2(dz[V * c] * gscale, dz[V * c + 1] * gscale, h0, l0);
        if constexpr (V == 4) {
          tc::split16x2(dz[4 * c + 2] * gscale, dz[4 * c + 3] * gscale, h1, l1);
          *reinterpret_cast<uint2*>(DZ16H + e) =
              make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
          *reinterpret_cast<uint2*>(DZ16L + e) =
              make_uint2(*reinterpret_cast<uint32_t*>(&l0), *reinterpret_cast<uint32_t*>(&l1));
        } else {
          *reinterpret_cast<__half2*>(DZ16H + e) = h0;
          *reinterpret_cast<__half2*>(DZ16L + e) = l0;
        }
        continue;
      }
      st_feat<V>(DZ + e, dz + V * c);
      if (DZLO != nullptr) {
        float lo[V];
#pragma unroll
        for (int k = 0; k < V; ++k) lo[k] = tc::tf32_lo(dz[V * c + k]);
        st_feat<V>(DZLO + e, lo);
      }
    }
  }
  // warp-private slices (each lane owns its features: plain stores)
#pragma unroll
  for (int j = 0; j < F; ++j) {
    const int f = (j / V) * CW + lane * V + (j % V);
    s_red3[warp * 3 * N + f] = a_dsc[j];
    s_red3[warp * 3 * N + N + f] = a_dbi[j];
    s_red3[warp * 3 * N + 2 * N + f] = a_db[j];
  }
  if (HEAD && lane == 0) { s_ls[warp * 2] = a_loss; s_ls[warp * 2 + 1] = a_qsa; }
  __syncthreads();
  const int stride = 3 * N + (HEAD ? A * N + A + 2 : 0);
  float* __restrict__ o = part + ((int64_t)seed * gridDim.x + blockIdx.x) * stride;
  for (int i = tid; i < 3 * N; i += 256) {
    float v = 0.f;
#pragma unroll
    for (int wv = 0; wv < 8; ++wv) v += s_red3[wv * 3 * N + i];
    o[i] = v;
  }
  if (HEAD) {
    for (int i = tid; i < A * N; i += 256) {   // [A][N]
      float v = 0.f;
#pragma unroll
      for (int wv = 0; wv < 8; ++wv) v += s_dhw[wv * A * N + i];
      o[3 * N + i] = v;
    }
    if (tid < A + 2) {
      float v = 0.f;
      for (int wv = 0; wv < 8; ++wv) v += tid < A ? s_dhb[wv * A + tid] : s_ls[wv * 2 + (tid - A)];
      o[3 * N + A * N + tid] = v;
    }
  }
}

// Fixed-order column sum of `count` partial vectors (p[c * stride], c = 0..count-1) by a 256-thread block laid out as
// (256 / SL) columns x SL slices: slice s adds the partials c = s, s+SL, ... in order, the SL slice sums are then added
// in slice order.  Every thread of the block must call it; the result is valid in the threads of slice 0
// (threadIdx.x < 256 / SL).  SL = 8 for a few partials per seed (many seeds), 32 for hundreds (one seed): the chain of
// dependent-latency loads per thread stays short either way.
template <int SL>
__device__ __forceinline__ float ordered_partial_sum(const float* __restrict__ p, int count, int64_t stride, bool valid) {
  constexpr int COLS = 256 / SL;
  __shared__ float slice_sum[SL][COLS];
  const int col = threadIdx.x % COLS, sl = threadIdx.x / COLS;
  float v = 0.f;
  if (valid) {
#pragma unroll 4
    for (int c = sl; c < count; c += SL) v += p[(int64_t)c * stride];
  }
  slice_sum[sl][col] = v;
  __syncthreads();
  float r = 0.f;
  if (sl == 0) {
#pragma unroll
    for (int k = 0; k < SL; ++k) r += slice_sum[k][col];
  }
  return r;
}
// slices for `count` partials per output element
static inline int final_slices(int count) { return count > 48 ? 32 : 8; }

// Sums the per-CTA partial vectors of row_bwd_kernel in a fixed order and writes the gradients (and adds the
// minibatch's loss / mean q_sa to the running sums).  grid = (ceil(stride / (256 / SL)), S), block = 256
template <int SL>
__global__ void row_bwd_final_kernel(const float* __restrict__ part, int nctas, int N, int A, int head,
                                     float* __restrict__ grads, int64_t P, int64_t off_dscale, int64_t off_dbias,
                                     int64_t off_db, int64_t off_hw, int64_t off_hb, float* __restrict__ loss_sum,
                                     float* __restrict__ qsa_sum) {
  const int seed = blockIdx.y;
  const int stride = 3 * N + (head ? A * N + A + 2 : 0);
  const int i = blockIdx.x * (256 / SL) + threadIdx.x % (256 / SL);
  const float v = ordered_partial_sum<SL>(part + (int64_t)seed * nctas * stride + i, nctas, stride, i < stride);
  if (i >= stride || threadIdx.x >= 256 / SL) return;
  float* __restrict__ g = grads + (int64_t)seed * P;
  if (i < N) g[off_dscale + i] = v;
  else if (i < 2 * N) g[off_dbias + (i - N)] = v;
  else if (i < 3 * N) g[off_db + (i - 2 * N)] = v;
  else if (i < 3 * N + A * N) {
    const int j = i - 3 * N, a = j / N, f = j - a * N;   // partial layout [A][N]; the parameter is [N][A]
    g[off_hw + (int64_t)f * A + a] = v;
  } else if (i < 3 * N + A * N + A) g[off_hb + (i - 3 * N - A * N)] = v;
  else if (i == 3 * N + A * N + A) loss_sum[seed] += v;
  else qsa_sum[seed] += v;
}

// ---------------------------------------------------------------------------
// MinAtar conv 3x3 (C -> 16, VALID) + LayerNorm(16) + ReLU from bit-packed obs.
// thread = (sample, output pixel); block = 4 samples; grid = (ceil(rows/4), S)
// ---------------------------------------------------------------------------

// the C channel bits of input pixel p of a packed row held in shared memory
template <int C>
__device__ __forceinline__ uint32_t pixel_bits(const uint32_t* __restrict__ so, int p) {
  const int f0 = p * C;
  const uint32_t lo = so[f0 >> 5], hi = so[(f0 >> 5) + 1];
  return __funnelshift_r(lo, hi, f0 & 31) & ((1u << C) - 1u);
}

// conv pre-activation for one output pixel; ws = conv kernel * (1/255), [tap][16]
template <int C>
__device__ __forceinline__ void conv_pixel(const uint32_t* __restrict__ so, const float* __restrict__ ws,
                                           const float* __restrict__ cb, int y, int x, float (&acc)[CONV_O]) {
#pragma unroll
  for (int o = 0; o < CONV_O; ++o) acc[o] = cb[o];
#pragma unroll
  for (int di = 0; di < 3; ++di)
#pragma unroll
    for (int dj = 0; dj < 3; ++dj) {
      const uint32_t nib = pixel_bits<C>(so, (y + di) * 10 + (x + dj));
      if (__ballot_sync(0xffffffffu, nib != 0u) == 0u) continue;  // nobody in the warp has this patch cell set
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const bool bit = (nib >> c) & 1u;
        if (__ballot_sync(0xffffffffu, bit) == 0u) continue;
        const float* __restrict__ w = ws + ((di * 3 + dj) * C + c) * CONV_O;
#pragma unroll
        for (int o4 = 0; o4 < CONV_O / 4; ++o4) {
          const float4 wv = *reinterpret_cast<const float4*>(w + 4 * o4);
          if (bit) {
            acc[4 * o4] += wv.x; acc[4 * o4 + 1] += wv.y; acc[4 * o4 + 2] += wv.z; acc[4 * o4 + 3] += wv.w;
          }
        }
      }
    }
}

__device__ __forceinline__ void ln16(const float (&z)[CONV_O], float& mean, float& rstd) {
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int o = 0; o < CONV_O; ++o) { s1 += z[o]; s2 = fmaf(z[o], z[o], s2); }
  mean = s1 * (1.0f / CONV_O);
  const float var = fmaxf(s2 * (1.0f / CONV_O) - mean * mean, 0.f);
  rstd = 1.0f / sqrtf(var + LN_EPS);
}

template <int C>
__device__ __forceinline__ void conv_load_consts(const float* __restrict__ prm, const pqn_net_layout_t& L, float* ws,
                                                 float* cb, float* sc, float* bi) {
  const float inv255 = 1.0f / 255.0f;  // x/255 for x in {0,1}  (pqn_minatar.py:66)
  for (int i = threadIdx.x; i < ConvCfg<C>::TAPS * CONV_O; i += blockDim.x) ws[i] = __ldg(prm + L.conv_w + i) * inv255;
  if (threadIdx.x < CONV_O) {
    cb[threadIdx.x] = __ldg(prm + L.conv_b + threadIdx.x);
    sc[threadIdx.x] = __ldg(prm + L.ln0_scale + threadIdx.x);
    bi[threadIdx.x] = __ldg(prm + L.ln0_bias + threadIdx.x);
  }
}

template <int C, bool TRAIN>
__global__ void __launch_bounds__(256) conv_fwd_kernel(const uint32_t* __restrict__ obs, int64_t obs_rows_per_seed,
                                                       const int32_t* __restrict__ gather,
                                                       const float* __restrict__ params, int64_t P,
                                                       pqn_net_layout_t L, float* __restrict__ H1,
                                                       float* __restrict__ H1LO, float* __restrict__ bn_sums,
                                                       int rows) {
  using Cfg = ConvCfg<C>;
  __shared__ __align__(16) float ws[Cfg::TAPS * CONV_O];
  __shared__ float cb[CONV_O], sc[CONV_O], bi[CONV_O];
  __shared__ uint32_t so[4][Cfg::SW];
  __shared__ float s_cnt[C];
  const int tid = threadIdx.x, sl = tid >> 6, pix = tid & 63;
  const int seed = blockIdx.y;
  const int row = blockIdx.x * 4 + sl;
  const bool valid = row < rows;
  conv_load_consts<C>(params + (int64_t)seed * P, L, ws, cb, sc, bi);
  if (TRAIN && tid < C) s_cnt[tid] = 0.f;
  if (pix < Cfg::SW) {
    uint32_t w = 0u;
    if (valid && pix < Cfg::PW) {
      const int64_t src = gather ? gather[(int64_t)seed * rows + row] : row;
      w = __ldg(obs + ((int64_t)seed * obs_rows_per_seed + src) * Cfg::PW + pix);
    }
    so[sl][pix] = w;
  }
  __syncthreads();
  const int y = pix >> 3, x = pix & 7;
  float acc[CONV_O];
  conv_pixel<C>(so[sl], ws, cb, y, x, acc);
  float mean, rstd;
  ln16(acc, mean, rstd);
  if (valid) {
    float4* __restrict__ out = reinterpret_cast<float4*>(H1 + ((int64_t)seed * rows + row) * FLAT_CNN + pix * CONV_O);
#pragma unroll
    for (int o4 = 0; o4 < CONV_O / 4; ++o4) {
      float4 v;
      v.x = fmaxf((acc[4 * o4] - mean) * rstd * sc[4 * o4] + bi[4 * o4], 0.f);
      v.y = fmaxf((acc[4 * o4 + 1] - mean) * rstd * sc[4 * o4 + 1] + bi[4 * o4 + 1], 0.f);
      v.z = fmaxf((acc[4 * o4 + 2] - mean) * rstd * sc[4 * o4 + 2] + bi[4 * o4 + 2], 0.f);
      v.w = fmaxf((acc[4 * o4 + 3] - mean) * rstd * sc[4 * o4 + 3] + bi[4 * o4 + 3], 0.f);
      out[o4] = v;
      if (H1LO != nullptr) {  // 3xTF32 error-compensation operand
        float4* __restrict__ olo =
            reinterpret_cast<float4*>(H1LO + ((int64_t)seed * rows + row) * FLAT_CNN + pix * CONV_O);
        olo[o4] = make_float4(tc::tf32_lo(v.x), tc::tf32_lo(v.y), tc::tf32_lo(v.z), tc::tf32_lo(v.w));
      }
    }
  }
  if (TRAIN && bn_sums != nullptr) {
    // dummy input BatchNorm statistics: per-channel count of set bits (x in {0,1} => sum x == sum x^2)
    uint32_t b0 = pixel_bits<C>(so[sl], pix);
    uint32_t b1 = (pix + 64 < 100) ? pixel_bits<C>(so[sl], pix + 64) : 0u;
    if (!valid) { b0 = 0u; b1 = 0u; }
#pragma unroll
    for (int c = 0; c < C; ++c) {
      int cnt = (int)((b0 >> c) & 1u) + (int)((b1 >> c) & 1u);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      if ((tid & 31) == 0 && cnt) atomicAdd(&s_cnt[c], (float)cnt);
    }
    __syncthreads();
    if (tid < C && s_cnt[tid] != 0.f) {
      atomicAdd(bn_sums + (int64_t)seed * 2 * C + tid, s_cnt[tid]);
      atomicAdd(bn_sums + (int64_t)seed * 2 * C + C + tid, s_cnt[tid]);
    }
  }
}

// conv backward, one warp per sample (no block-level sync in the loop):
//   phase A  lane = output pixel (2 per lane): recompute conv + LN statistics, LN backward from DY1 (already
//            ReLU-masked by dgrad) -> dz staged in the warp's shared memory; d(ln0 scale/bias) in registers.
//   phase B  dW[tap][o] += x[pixel+tap] * dz[pixel][o] driven by the SET input bits only (MinAtar observations
//            are sparse): for each set bit (input pixel q, channel c) the 9 taps that see it add dz[q - tap][:]
//            into lane-private accumulators; lane = (tap parity, o), accumulators indexed [c][tap/2] statically.
//   d(conv bias)[o] = sum over pixels of dz, also taken from the staged dz.
// grid = (CONV_BWD_CTAS_X, S); each CTA strides over the seed's samples 8 at a time.
constexpr int CONV_BWD_WARPS = 8;
constexpr int SDZ_LD = 20;  // padded dz row (conflict-free 128-bit stores from 32 pixel-lanes)

template <int C>
__global__ void __launch_bounds__(CONV_BWD_WARPS * 32, 2)
    conv_bwd_kernel(const uint32_t* __restrict__ obs, int64_t obs_rows_per_seed, const int32_t* __restrict__ gather,
                    const float* __restrict__ params, int64_t P, pqn_net_layout_t L, const float* __restrict__ DY1,
                    float* __restrict__ grads, int rows) {
  using Cfg = ConvCfg<C>;
  constexpr int TAPS = Cfg::TAPS;
  __shared__ __align__(16) float ws[TAPS * CONV_O];
  __shared__ float cb[CONV_O], sc[CONV_O], bi[CONV_O];
  __shared__ uint32_t so[CONV_BWD_WARPS][Cfg::SW];
  __shared__ __align__(16) float sdz[CONV_BWD_WARPS][CONV_PIX * SDZ_LD];
  __shared__ float s_red[3 * CONV_O];
  float* s_w = &sdz[0][0];  // [TAPS*16], aliases the dz staging area once the sample loop is done
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int seed = blockIdx.y;
  const float* __restrict__ prm = params + (int64_t)seed * P;
  conv_load_consts<C>(prm, L, ws, cb, sc, bi);
  if (tid < 3 * CONV_O) s_red[tid] = 0.f;
  __syncthreads();

  float a_dsc[CONV_O], a_dbi[CONV_O];
#pragma unroll
  for (int o = 0; o < CONV_O; ++o) a_dsc[o] = a_dbi[o] = 0.f;
  // phase-B role: lane = (tap parity, output channel); 5 iterations cover the 9 taps
  const int o_b = lane & 15, tpar = lane >> 4;
  int t_di[5], t_dj[5];
#pragma unroll
  for (int it = 0; it < 5; ++it) {
    const int tap = it * 2 + tpar;
    t_di[it] = tap < 9 ? tap / 3 : 100;  // 100 => never valid
    t_dj[it] = tap < 9 ? tap % 3 : 0;
  }
  float wacc[C][5];
#pragma unroll
  for (int c = 0; c < C; ++c)
#pragma unroll
    for (int it = 0; it < 5; ++it) wacc[c][it] = 0.f;
  float a_dcb = 0.f;  // lane (tpar, o): sum of dz[pixel][o] over pixels of parity tpar

  uint32_t* __restrict__ my_so = so[warp];
  float* __restrict__ my_dz = sdz[warp];
  for (int row = blockIdx.x * CONV_BWD_WARPS + warp; row < rows; row += gridDim.x * CONV_BWD_WARPS) {
    __syncwarp();
    {
      const int64_t src = gather ? gather[(int64_t)seed * rows + row] : row;
      const uint32_t* __restrict__ orow = obs + ((int64_t)seed * obs_rows_per_seed + src) * Cfg::PW;
      for (int wi = lane; wi < Cfg::SW; wi += 32) my_so[wi] = wi < Cfg::PW ? __ldg(orow + wi) : 0u;
    }
    __syncwarp();
    // ---- phase A: two output pixels per lane
#pragma unroll 1
    for (int hh = 0; hh < 2; ++hh) {
      const int pix = lane + 32 * hh;
      float acc[CONV_O];
      conv_pixel<C>(my_so, ws, cb, pix >> 3, pix & 7, acc);
      float mean, rstd;
      ln16(acc, mean, rstd);
      const float4* __restrict__ dyp =
          reinterpret_cast<const float4*>(DY1 + ((int64_t)seed * rows + row) * FLAT_CNN + pix * CONV_O);
      float dy[CONV_O];
#pragma unroll
      for (int o4 = 0; o4 < CONV_O / 4; ++o4) {
        const float4 v = __ldg(dyp + o4);
        dy[4 * o4] = v.x; dy[4 * o4 + 1] = v.y; dy[4 * o4 + 2] = v.z; dy[4 * o4 + 3] = v.w;
      }
      float m1 = 0.f, m2 = 0.f;
#pragma unroll
      for (int o = 0; o < CONV_O; ++o) {
        acc[o] = (acc[o] - mean) * rstd;  // xhat
        a_dsc[o] = fmaf(dy[o], acc[o], a_dsc[o]);
        a_dbi[o] += dy[o];
        dy[o] *= sc[o];                   // dxhat
        m1 += dy[o];
        m2 = fmaf(dy[o], acc[o], m2);
      }
      m1 *= (1.0f / CONV_O);
      m2 *= (1.0f / CONV_O);
#pragma unroll
      for (int o4 = 0; o4 < CONV_O / 4; ++o4) {
        float4 dz;
        dz.x = rstd * (dy[4 * o4] - m1 - acc[4 * o4] * m2);
        dz.y = rstd * (dy[4 * o4 + 1] - m1 - acc[4 * o4 + 1] * m2);
        dz.z = rstd * (dy[4 * o4 + 2] - m1 - acc[4 * o4 + 2] * m2);
        dz.w = rstd * (dy[4 * o4 + 3] - m1 - acc[4 * o4 + 3] * m2);
        *reinterpret_cast<float4*>(&my_dz[pix * SDZ_LD + 4 * o4]) = dz;
      }
    }
    __syncwarp();
    // ---- d(conv bias): lane (tpar, o) sums dz over the pixels of its parity
#pragma unroll 8
    for (int p = tpar; p < CONV_PIX; p += 2) a_dcb += my_dz[p * SDZ_LD + o_b];
    // ---- phase B: sparse dW accumulation over the set input bits
#pragma unroll
    for (int c = 0; c < C; ++c) {
      for (int wi = 0; wi < Cfg::OBS_WORDS; ++wi) {
        // bits of word wi that belong to channel c: flat index f = wi*32 + b with f % C == c
        uint32_t bits = my_so[wi];
        if (C == 4) bits &= 0x11111111u << c;  // 32 % C == 0: channel c sits at a fixed bit phase in every word
        if (bits == 0u) continue;
        while (bits) {
          const int b = __ffs(bits) - 1;
          bits &= bits - 1u;
          const int f = wi * 32 + b;
          const int q = f / C;
          if (f - q * C != c) continue;
          const int qy = q / 10, qx = q - qy * 10;
#pragma unroll
          for (int it = 0; it < 5; ++it) {
            const int py = qy - t_di[it], px = qx - t_dj[it];
            if ((unsigned)py < 8u && (unsigned)px < 8u) wacc[c][it] += my_dz[(py * 8 + px) * SDZ_LD + o_b];
          }
        }
      }
    }
  }
  // ---- reduce and publish
  __syncthreads();
  for (int i = tid; i < TAPS * CONV_O; i += blockDim.x) s_w[i] = 0.f;
  __syncthreads();
  const float inv255 = 1.0f / 255.0f;
#pragma unroll
  for (int c = 0; c < C; ++c)
#pragma unroll
    for (int it = 0; it < 5; ++it) {
      const int tap = it * 2 + tpar;
      if (tap < 9) atomicAdd(&s_w[(tap * C + c) * CONV_O + o_b], wacc[c][it] * inv255);
    }
  atomicAdd(&s_red[2 * CONV_O + o_b], a_dcb);
#pragma unroll
  for (int o = 0; o < CONV_O; ++o) {
    float v0 = a_dsc[o], v1 = a_dbi[o];
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) {
      v0 += __shfl_xor_sync(0xffffffffu, v0, sft);
      v1 += __shfl_xor_sync(0xffffffffu, v1, sft);
    }
    if (lane == 0) {
      atomicAdd(&s_red[o], v0);
      atomicAdd(&s_red[CONV_O + o], v1);
    }
  }
  __syncthreads();
  float* __restrict__ g = grads + (int64_t)seed * P;
  for (int i = tid; i < TAPS * CONV_O; i += blockDim.x) atomicAdd(g + L.conv_w + i, s_w[i]);
  if (tid < CONV_O) {
    atomicAdd(g + L.ln0_scale + tid, s_red[tid]);
    atomicAdd(g + L.ln0_bias + tid, s_red[CONV_O + tid]);
    atomicAdd(g + L.conv_b + tid, s_red[2 * CONV_O + tid]);
  }
}

// ---------------------------------------------------------------------------
// conv on the warp-level tensor-core path (mma.sync.m16n8k8 tf32, fp32 accumulate).
// The 3x3 conv is a skinny GEMM  Z[64 pixels x 16] = Xcol[64 x 9C] . W[9C x 16]  per sample whose A operand is
// {0,1}: every lane builds its A-fragment elements straight from the packed observation bits (no im2col in
// memory), B fragments (weights/255 split into tf32 hi + lo: two passes keep fp32 accuracy, x is exact) come from
// shared memory, and the 16 channels of a pixel end up in the 4 lanes of a quad, so LayerNorm is two shuffles.
// The weight gradient is the transposed skinny GEMM dW[9C x 16] = Xcol^T[9C x 64] . dZ[64 x 16], accumulated per
// sample in fresh MMA accumulators (16-long chains) and added to fp32 registers (FADD) across samples.
// One warp per sample.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void mma_tf32_16n8k8(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int C>
struct ConvMma {
  static constexpr int TAPS = 9 * C;
  static constexpr int KS = (TAPS + 7) / 8;    // k-steps of the forward GEMM (taps)
  static constexpr int MT = (TAPS + 15) / 16;  // m-blocks of the weight-gradient GEMM (taps)
};


template <int C>
__device__ __forceinline__ void build_patch(const uint32_t* __restrict__ so, int pix, uint32_t* __restrict__ out) {
  constexpr int W = PatchCfg<C>::WORDS;
  uint32_t w[W];
  patch_bits<C>(so, pix, w);
#pragma unroll
  for (int k = 0; k < W; ++k) out[k] = w[k];
}

// both output pixels of a lane (pix = lane, lane + 32) -> patch[64][WORDS]
template <int C>
__device__ __forceinline__ void build_patches(const uint32_t* __restrict__ so, uint32_t* __restrict__ patch, int lane) {
  build_patch<C>(so, lane, patch + lane * PatchCfg<C>::WORDS);
  build_patch<C>(so, lane + 32, patch + (lane + 32) * PatchCfg<C>::WORDS);
}

__device__ __forceinline__ uint32_t bit_f32(uint32_t word, int shift) {
  return ((word >> shift) & 1u) ? 0x3F800000u : 0u;
}

// B fragments of the conv weights (scaled by 1/255), hi and lo, laid out [ks][half][lane] as float2 (b0, b1).
// EXPC: the A operand is "exponent coded" (see ExpPatch): the activation of tap k is the power of two
// 2^(2^(k%8) - 127) instead of 1, so row k of B carries the inverse factor 2^(127 - 2^(k%8)) (exact scaling).
template <int C, bool EXPC = false>
__device__ __forceinline__ void conv_mma_load_weights(const float* __restrict__ prm, const pqn_net_layout_t& L,
                                                      float2* wb_hi, float2* wb_lo, float* cb, float* sc, float* bi) {
  using M = ConvMma<C>;
  const float inv255 = 1.0f / 255.0f;
  for (int i = threadIdx.x; i < M::KS * 2 * 32; i += blockDim.x) {
    const int ln = i & 31, h = (i >> 5) & 1, ks = i >> 6;
    const int o = h * 8 + (ln >> 2);
    const int t0 = ks * 8 + (ln & 3), t1 = t0 + 4;
    float w0 = t0 < M::TAPS ? __ldg(prm + L.conv_w + t0 * CONV_O + o) * inv255 : 0.f;
    float w1 = t1 < M::TAPS ? __ldg(prm + L.conv_w + t1 * CONV_O + o) * inv255 : 0.f;
    if (EXPC) {
      w0 *= __uint_as_float((254u - (1u << (t0 & 7))) << 23);
      w1 *= __uint_as_float((254u - (1u << (t1 & 7))) << 23);
    }
    const float h0 = __uint_as_float(__float_as_uint(w0) & 0xFFFFE000u), h1 = __uint_as_float(__float_as_uint(w1) & 0xFFFFE000u);
    wb_hi[i] = make_float2(h0, h1);
    wb_lo[i] = make_float2(w0 - h0, w1 - h1);
  }
  if (threadIdx.x < CONV_O) {
    cb[threadIdx.x] = __ldg(prm + L.conv_b + threadIdx.x);
    sc[threadIdx.x] = __ldg(prm + L.ln0_scale + threadIdx.x);
    bi[threadIdx.x] = __ldg(prm + L.ln0_bias + threadIdx.x);
  }
}

// ---- exponent-coded im2col fragments (forward kernel) --------------------------------------------------------
// A tf32 MMA operand only has to be *some* exactly known value when the input bit is set, not 1.0: a word whose
// bits 23..30 (the fp32 exponent field) hold eight tap bits turns into an A element with ONE instruction,
//     a = word & (1 << (23 + j))      ->  0  or  2^(2^j - 127)        (a normal power of two, mantissa 0)
// and the matching row of B is pre-multiplied by 2^(127 - 2^j) (conv_mma_load_weights<C, true>), so every product
// is bit-for-bit the product of the plain 0/1 formulation.  Per output pixel the patch is stored as KS words,
// word ks = taps 8ks .. 8ks+7 at bits 23..30; lane (g, t) of the m16n8k8 fragment needs taps t and t+4.
template <int C>
struct ExpPatch {
  static constexpr int KS = ConvMma<C>::KS;
  static constexpr int LD = KS | 1;  // odd row stride: conflict-free for the 8 pixel rows a fragment load touches
};

template <int C>
__device__ __forceinline__ void build_exp_patch(const uint32_t* __restrict__ so, int pix, uint32_t* __restrict__ out) {
  constexpr int W = PatchCfg<C>::WORDS;
  uint32_t w[W];
  patch_bits<C>(so, pix, w);
#pragma unroll
  for (int ks = 0; ks < ExpPatch<C>::KS; ++ks)  // 8 | 32: a k-step never straddles two words; bits >= 9C are zero
    out[ks] = ((w[(8 * ks) >> 5] >> ((8 * ks) & 31)) & 0xFFu) << 23;
}

// conv pre-activation of the 32 pixels of m-blocks 2*mbp and 2*mbp+1 (two blocks share every B fragment load);
// z[i][h][0..3] is the C fragment of block mb = 2*mbp+i (pixel = 16*mb + g [+8]):
// z[i][h][0], z[i][h][1] -> pixel g, channels 8h+2t, 8h+2t+1 ; z[i][h][2], z[i][h][3] -> pixel g+8, same channels.
template <int C>
__device__ __forceinline__ void conv_mma_block2_exp(const uint32_t* __restrict__ xp, const float2* __restrict__ wb_hi,
                                                    const float2* __restrict__ wb_lo, const float* __restrict__ cb,
                                                    int mbp, int lane, float (&z)[2][2][4]) {
  using E = ExpPatch<C>;
  const int g = lane >> 2, t = lane & 3;
  const uint32_t m_lo = 1u << (23 + t), m_hi = 1u << (27 + t);
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      z[i][h][0] = z[i][h][2] = cb[8 * h + 2 * t];
      z[i][h][1] = z[i][h][3] = cb[8 * h + 2 * t + 1];
    }
  const uint32_t* r00 = xp + (32 * mbp + g) * E::LD;  // pixel rows g, g+8 of block 2mbp; +16, +24 of block 2mbp+1
#pragma unroll
  for (int ks = 0; ks < E::KS; ++ks) {
    uint32_t a[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t w0 = r00[(16 * i) * E::LD + ks], w1 = r00[(16 * i + 8) * E::LD + ks];
      a[i][0] = w0 & m_lo; a[i][1] = w1 & m_lo; a[i][2] = w0 & m_hi; a[i][3] = w1 & m_hi;
    }
    float2 bl[2], bh[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      bl[h] = wb_lo[(ks * 2 + h) * 32 + lane];
      bh[h] = wb_hi[(ks * 2 + h) * 32 + lane];
    }
    // four independent accumulators between the lo and the hi pass of the same one (no back-to-back dependency)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 2; ++i) mma_tf32_16n8k8(z[i][h], a[i], __float_as_uint(bl[h].x), __float_as_uint(bl[h].y));
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 2; ++i) mma_tf32_16n8k8(z[i][h], a[i], __float_as_uint(bh[h].x), __float_as_uint(bh[h].y));
  }
}


constexpr int CONV_MMA_WARPS = 8;

// H16: the activation goes out as the two fp16 planes of the fp16-split tensor-core path (H1 = hi plane, H1LO = lo'
// plane, both __half[rows][1024]) instead of fp32 h1 -- the same 4 bytes per element, so the dense GEMMs read
// (hi, lo') straight through TMA and no operand conversion happens in the GEMM kernel.
template <int C, bool TRAIN, bool H16 = false>
__global__ void __launch_bounds__(CONV_MMA_WARPS * 32, 3)
    conv_fwd_mma_kernel(const uint32_t* __restrict__ obs, int64_t obs_rows_per_seed, const int32_t* __restrict__ gather,
                        const float* __restrict__ params, int64_t P, pqn_net_layout_t L, float* __restrict__ H1,
                        float* __restrict__ H1LO, float* __restrict__ XH1, float* __restrict__ RS1,
                        uint32_t* __restrict__ RB, float* __restrict__ bn_sums, int rows) {
  using Cfg = ConvCfg<C>;
  using M = ConvMma<C>;
  __shared__ float2 wb_hi[M::KS * 2 * 32], wb_lo[M::KS * 2 * 32];
  __shared__ float cb[CONV_O], sc[CONV_O], bi[CONV_O];
  __shared__ uint32_t so[CONV_MMA_WARPS][Cfg::SW];
  __shared__ uint32_t sxp[CONV_MMA_WARPS][CONV_PIX * ExpPatch<C>::LD];
  __shared__ float s_cnt[C];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int seed = blockIdx.y;
  conv_mma_load_weights<C, true>(params + (int64_t)seed * P, L, wb_hi, wb_lo, cb, sc, bi);
  if (TRAIN && tid < C) s_cnt[tid] = 0.f;
  __syncthreads();
  int cnt[C];
  uint32_t cmask[C];  // bits of this lane's observation word (word index = lane) that belong to channel c
#pragma unroll
  for (int c = 0; c < C; ++c) {
    cnt[c] = 0;
    cmask[c] = 0u;
    if (TRAIN) {
      for (int b = 0; b < 32; ++b) {
        const int f = lane * 32 + b;
        if (f < Cfg::OBS_BITS && f % C == c) cmask[c] |= 1u << b;
      }
    }
  }
  uint32_t* __restrict__ my_so = so[warp];
  static_assert(Cfg::PW <= 32, "one packed observation word per lane");
  if (lane == 0) my_so[Cfg::PW] = 0u;  // pad word read by the funnel shift of the last pixel
  // software pipeline: the next sample's packed observation is fetched while the current one is processed
  const int row_stride = gridDim.x * CONV_MMA_WARPS;
  auto fetch = [&](int r) -> uint32_t {
    if (r >= rows || lane >= Cfg::PW) return 0u;
    const int64_t src = gather ? gather[(int64_t)seed * rows + r] : r;
    return __ldg(obs + ((int64_t)seed * obs_rows_per_seed + src) * Cfg::PW + lane);
  };
  uint32_t pre = fetch(blockIdx.x * CONV_MMA_WARPS + warp);
  for (int row = blockIdx.x * CONV_MMA_WARPS + warp; row < rows; row += row_stride) {
    __syncwarp();
    if (lane < Cfg::PW) my_so[lane] = pre;
    if (TRAIN && bn_sums != nullptr) {
      // dummy input BatchNorm statistics: per-channel popcount of the 100 input pixels (x in {0,1})
#pragma unroll
      for (int c = 0; c < C; ++c) cnt[c] += __popc(pre & cmask[c]);
    }
    __syncwarp();
    pre = fetch(row + row_stride);
    build_exp_patch<C>(my_so, lane, sxp[warp] + lane * ExpPatch<C>::LD);
    build_exp_patch<C>(my_so, lane + 32, sxp[warp] + (lane + 32) * ExpPatch<C>::LD);
    __syncwarp();
    float* __restrict__ hrow = H16 ? nullptr : H1 + ((int64_t)seed * rows + row) * FLAT_CNN;
    float* __restrict__ lrow = (!H16 && H1LO) ? H1LO + ((int64_t)seed * rows + row) * FLAT_CNN : nullptr;
    __half* __restrict__ hrow16 = H16 ? reinterpret_cast<__half*>(H1) + ((int64_t)seed * rows + row) * FLAT_CNN : nullptr;
    __half* __restrict__ lrow16 = H16 ? reinterpret_cast<__half*>(H1LO) + ((int64_t)seed * rows + row) * FLAT_CNN : nullptr;
    float* __restrict__ xrow = (TRAIN && XH1) ? XH1 + ((int64_t)seed * rows + row) * FLAT_CNN : nullptr;
    float* __restrict__ rrow = (TRAIN && RS1) ? RS1 + ((int64_t)seed * rows + row) * CONV_PIX : nullptr;
    // packed ReLU mask for the dense dgrad epilogue: bit (pixel * 16 + channel) = (h1 > 0), 16 bits per pixel
    uint16_t* __restrict__ brow =
        (TRAIN && RB) ? reinterpret_cast<uint16_t*>(RB + ((int64_t)seed * rows + row) * (FLAT_CNN / 32)) : nullptr;
#pragma unroll 1
    for (int mbp = 0; mbp < 2; ++mbp) {
     float z2[2][2][4];
     conv_mma_block2_exp<C>(sxp[warp], wb_hi, wb_lo, cb, mbp, lane, z2);
#pragma unroll
     for (int mi = 0; mi < 2; ++mi) {
      const int mb = 2 * mbp + mi;
      float (&z)[2][4] = z2[mi];
      float mean0, rstd0, mean1, rstd1;
      ln16_quad(z, mean0, rstd0, mean1, rstd1);
      uint32_t rb0 = 0u, rb1 = 0u;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o = 8 * h + 2 * t;
        float2 v0, v1;
        v0.x = fmaxf((z[h][0] - mean0) * rstd0 * sc[o] + bi[o], 0.f);
        v0.y = fmaxf((z[h][1] - mean0) * rstd0 * sc[o + 1] + bi[o + 1], 0.f);
        v1.x = fmaxf((z[h][2] - mean1) * rstd1 * sc[o] + bi[o], 0.f);
        v1.y = fmaxf((z[h][3] - mean1) * rstd1 * sc[o + 1] + bi[o + 1], 0.f);
        const int p0 = 16 * mb + g, p1 = p0 + 8;
        if (H16) {
          __half2 h0, l0, h1v, l1;
          // post-ReLU values are >= 0: one-sided saturation is enough
          tc::split16x2<false>(fminf(v0.x, 65000.f), fminf(v0.y, 65000.f), h0, l0);
          tc::split16x2<false>(fminf(v1.x, 65000.f), fminf(v1.y, 65000.f), h1v, l1);
          *reinterpret_cast<__half2*>(hrow16 + p0 * CONV_O + o) = h0;
          *reinterpret_cast<__half2*>(lrow16 + p0 * CONV_O + o) = l0;
          *reinterpret_cast<__half2*>(hrow16 + p1 * CONV_O + o) = h1v;
          *reinterpret_cast<__half2*>(lrow16 + p1 * CONV_O + o) = l1;
        } else {
          *reinterpret_cast<float2*>(hrow + p0 * CONV_O + o) = v0;
          *reinterpret_cast<float2*>(hrow + p1 * CONV_O + o) = v1;
        }
        if (TRAIN) {
          rb0 |= ((v0.x > 0.f ? 1u : 0u) | (v0.y > 0.f ? 2u : 0u)) << o;
          rb1 |= ((v1.x > 0.f ? 1u : 0u) | (v1.y > 0.f ? 2u : 0u)) << o;
        }
        if (xrow) {  // saved for the backward pass (no conv recompute there)
          *reinterpret_cast<float2*>(xrow + p0 * CONV_O + o) =
              make_float2((z[h][0] - mean0) * rstd0, (z[h][1] - mean0) * rstd0);
          *reinterpret_cast<float2*>(xrow + p1 * CONV_O + o) =
              make_float2((z[h][2] - mean1) * rstd1, (z[h][3] - mean1) * rstd1);
          if (h == 0 && t == 0) { rrow[p0] = rstd0; rrow[p1] = rstd1; }
        }
        if (lrow) {
          *reinterpret_cast<float2*>(lrow + p0 * CONV_O + o) = make_float2(tc::tf32_lo(v0.x), tc::tf32_lo(v0.y));
          *reinterpret_cast<float2*>(lrow + p1 * CONV_O + o) = make_float2(tc::tf32_lo(v1.x), tc::tf32_lo(v1.y));
        }
      }
      if (TRAIN && brow) {
        rb0 |= __shfl_xor_sync(0xffffffffu, rb0, 1); rb1 |= __shfl_xor_sync(0xffffffffu, rb1, 1);
        rb0 |= __shfl_xor_sync(0xffffffffu, rb0, 2); rb1 |= __shfl_xor_sync(0xffffffffu, rb1, 2);
        if (t == 0) { brow[16 * mb + g] = (uint16_t)rb0; brow[16 * mb + g + 8] = (uint16_t)rb1; }
      }
     }
    }
  }
  if (TRAIN && bn_sums != nullptr) {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      int v = cnt[c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0 && v) atomicAdd(&s_cnt[c], (float)v);
    }
    __syncthreads();
    if (tid < C && s_cnt[tid] != 0.f) {
      atomicAdd(bn_sums + (int64_t)seed * 2 * C + tid, s_cnt[tid]);
      atomicAdd(bn_sums + (int64_t)seed * 2 * C + C + tid, s_cnt[tid]);
    }
  }
}


// 4 warps per CTA, 5 CTAs per SM = 5 warps per scheduler: 96 registers per thread.  (With 8-warp CTAs x 3 the cap is 80
// registers and the epilogue spilled: ncu r2e, STL = 0.7 % of the instructions but 13 % of the stall samples; the
// kernel wants ~123 registers unconstrained.)
constexpr int CONV16_WARPS = 4;
constexpr int CONV16_CTAS_PER_SM = 5;

template <int C, bool TRAIN, bool H16>
__global__ void __launch_bounds__(CONV16_WARPS * 32, CONV16_CTAS_PER_SM)
    conv_fwd_mma16_kernel(const uint32_t* __restrict__ obs, int64_t obs_rows_per_seed, const int32_t* __restrict__ gather,
                          const float* __restrict__ params, int64_t P, pqn_net_layout_t L, float* __restrict__ H1,
                          float* __restrict__ H1LO, uint32_t* __restrict__ RB, float* __restrict__ bn_sums, int rows) {
  using Cfg = ConvCfg<C>;
  using M = Conv16<C>;
  __shared__ __align__(16) uint4 wb[M::KS * 2 * 32];
  __shared__ float cb[CONV_O], sc[CONV_O], bi[CONV_O];
  __shared__ uint32_t so[CONV16_WARPS][Cfg::SW];
  __shared__ __align__(16) uint32_t sxp[CONV16_WARPS][CONV_PIX * M::ROW];
  __shared__ float s_cnt[C];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int seed = blockIdx.y;
  conv16_load_weights<C>(params + (int64_t)seed * P, L, wb, cb, sc, bi, threadIdx.x, blockDim.x);
  if (TRAIN && tid < C) s_cnt[tid] = 0.f;
  __syncthreads();
  int cnt[C];
  uint32_t cmask[C];
#pragma unroll
  for (int c = 0; c < C; ++c) {
    cnt[c] = 0;
    cmask[c] = 0u;
    if (TRAIN) {
      for (int b = 0; b < 32; ++b) {
        const int f = lane * 32 + b;
        if (f < Cfg::OBS_BITS && f % C == c) cmask[c] |= 1u << b;
      }
    }
  }
  uint32_t* __restrict__ my_so = so[warp];
  static_assert(Cfg::PW <= 32, "one packed observation word per lane");
  if (lane == 0) my_so[Cfg::PW] = 0u;
  const int row_stride = gridDim.x * CONV16_WARPS;
  // two-deep prefetch: the gather index of row + 2 strides and the packed observation of row + 1 stride are in flight
  // while this row is computed, so the index -> observation load chain never stalls the in-order issue
  // unconditional loads from clamped addresses (rows past the end re-read the last row, lanes past the packed width
  // re-read word 0; neither is ever used): a predicated load with a default value made ptxas copy the result into the
  // loop-carried register ~125 instructions after the LDG, which stalled every warp on the load it had just issued
  // (13 % of all stall samples of the forward kernel, ncu r2m)
  auto fetch_index = [&](int r) -> int {
    const int rc = r < rows ? r : rows - 1;
    return gather ? __ldg(gather + (int64_t)seed * rows + rc) : rc;
  };
  auto fetch_obs = [&](int src) -> uint32_t {
    return __ldg(obs + ((int64_t)seed * obs_rows_per_seed + src) * Cfg::PW + (lane < Cfg::PW ? lane : 0));
  };
  const int row0 = blockIdx.x * CONV16_WARPS + warp;
  uint32_t pre = fetch_obs(fetch_index(row0));
  int src_next = fetch_index(row0 + row_stride);
  for (int row = row0; row < rows; row += row_stride) {
    __syncwarp();
    if (lane < Cfg::PW) my_so[lane] = pre;
    if (TRAIN && bn_sums != nullptr) {
#pragma unroll
      for (int c = 0; c < C; ++c) cnt[c] += __popc(pre & cmask[c]);
    }
    __syncwarp();
    pre = fetch_obs(src_next);
    src_next = fetch_index(row + 2 * row_stride);
    store_patch16<C>(my_so, lane, sxp[warp] + lane * M::ROW);
    store_patch16<C>(my_so, lane + 32, sxp[warp] + (lane + 32) * M::ROW);
    __syncwarp();
    const int64_t grow = (int64_t)seed * rows + row;
    float* __restrict__ hrow = H16 ? nullptr : H1 + grow * FLAT_CNN;
    __half* __restrict__ hrow16 = H16 ? reinterpret_cast<__half*>(H1) + grow * FLAT_CNN : nullptr;
    __half* __restrict__ lrow16 = H16 ? reinterpret_cast<__half*>(H1LO) + grow * FLAT_CNN : nullptr;
    uint16_t* __restrict__ brow = (TRAIN && RB) ? reinterpret_cast<uint16_t*>(RB + grow * (FLAT_CNN / 32)) : nullptr;
    // the ReLU masks of m-block t are kept by lane t of every quad and stored once per sample (2 store instructions
    // instead of 8 predicated ones)
    uint32_t keep_rb = 0u;
#pragma unroll 1
    for (int mbp = 0; mbp < 2; ++mbp) {
      float z2[2][2][4];
      conv16_blocks<C, 2>(sxp[warp], wb, cb, 2 * mbp, lane, z2);
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const int mb = 2 * mbp + mi;
        uint32_t rb0 = 0u, rb1 = 0u;
        // the thread's channels of pixel rows p0 = 16 mb + g and p1 = p0 + 8: 4t .. 4t+3 (n-tile h -> 4t + 2h, + 1)
        const int p0 = 16 * mb + g, p1 = p0 + 8, o4 = 4 * t;
        const float sc4[4] = {sc[o4], sc[o4 + 1], sc[o4 + 2], sc[o4 + 3]};
        const float bi4[4] = {bi[o4], bi[o4 + 1], bi[o4 + 2], bi[o4 + 3]};
        float v0[4], v1[4];
        conv16_act(z2[mi], sc4, bi4, v0, v1);
        if (H16) {
          // 8-byte stores of the (hi, lo') planes
          uint32_t hw0[2], hw1[2], lw0[2], lw1[2];
          conv16_split(v0, hw0, lw0);
          conv16_split(v1, hw1, lw1);
          *reinterpret_cast<uint2*>(hrow16 + p0 * CONV_O + o4) = make_uint2(hw0[0], hw0[1]);
          *reinterpret_cast<uint2*>(lrow16 + p0 * CONV_O + o4) = make_uint2(lw0[0], lw0[1]);
          *reinterpret_cast<uint2*>(hrow16 + p1 * CONV_O + o4) = make_uint2(hw1[0], hw1[1]);
          *reinterpret_cast<uint2*>(lrow16 + p1 * CONV_O + o4) = make_uint2(lw1[0], lw1[1]);
        } else {
          *reinterpret_cast<float4*>(hrow + p0 * CONV_O + o4) = make_float4(v0[0], v0[1], v0[2], v0[3]);
          *reinterpret_cast<float4*>(hrow + p1 * CONV_O + o4) = make_float4(v1[0], v1[1], v1[2], v1[3]);
        }
        if (TRAIN) {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            rb0 |= (v0[c] > 0.f ? 1u : 0u) << (o4 + c);
            rb1 |= (v1[c] > 0.f ? 1u : 0u) << (o4 + c);
          }
        }
        if (TRAIN && brow) {
          uint32_t rb = rb0 | (rb1 << 16);      // both pixel rows in one register: two shuffles instead of four
          rb |= __shfl_xor_sync(0xffffffffu, rb, 1);
          rb |= __shfl_xor_sync(0xffffffffu, rb, 2);
          if (t == mb) keep_rb = rb;
        }
      }
    }
    if (TRAIN && brow) { brow[16 * t + g] = (uint16_t)keep_rb; brow[16 * t + g + 8] = (uint16_t)(keep_rb >> 16); }
  }
  if (TRAIN && bn_sums != nullptr) {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      int v = cnt[c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0 && v) atomicAdd(&s_cnt[c], (float)v);
    }
    __syncthreads();
    if (tid < C && s_cnt[tid] != 0.f) {
      atomicAdd(bn_sums + (int64_t)seed * 2 * C + tid, s_cnt[tid]);
      atomicAdd(bn_sums + (int64_t)seed * 2 * C + C + tid, s_cnt[tid]);
    }
  }
}

constexpr int CDZ_LD = 16;  // staged dz / dy / xhat row stride (floats)
// Column swizzle of the [64 pixels][16 channels] shared-memory tiles of the conv backward: rows p and p+2 are 32 banks
// apart, so the column is XORed with 8 on every second row pair.  The float2 accesses of a fragment (8 pixel rows x
// 4 column pairs per half-warp pair) and the B-fragment reads (4 pixel rows x 8 columns) then touch every bank once.
__device__ __forceinline__ int cswz(int p, int col) { return col ^ (((p >> 1) & 1) << 3); }

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// per-warp shared-memory slice of the conv backward kernel (floats)
template <int C>
struct ConvBwdSmem {
  static constexpr int DY = 0;                                  // [64][16] upstream gradient of the sample
  static constexpr int XH = DY + FLAT_CNN;                      // [64][16] saved LayerNorm xhat
  static constexpr int RS = XH + FLAT_CNN;                      // [64]     saved rstd
  static constexpr int DZ = RS + CONV_PIX;                      // [64][CDZ_LD] dz stage (aliases the packed obs row)
  static constexpr int PATCH = DZ + CONV_PIX * CDZ_LD;          // [64][PatchCfg::WORDS] im2col bit patches
  static constexpr int WARP_FLOATS = (PATCH + CONV_PIX * PatchCfg<C>::WORDS + 3) / 4 * 4;
  static constexpr int WARPS = 8;
  static constexpr int BYTES = (WARPS * WARP_FLOATS + 4 * CONV_O) * 4;  // + sc[16] + s_red[48]
};

// Backward of conv3x3 + LayerNorm(16) + ReLU for one sample per warp, from the xhat / rstd the training forward
// saved (ReLU' is already folded into DY1 by the dense dgrad epilogue):
//   phase A  LayerNorm backward per pixel -> dz[pixel][16] (staged in shared memory), d(scale), d(bias), d(conv bias)
//   phase B  dW[tap][o] += sum_pixels x[pixel, tap] dz[pixel][o] on mma.sync (A = im2col bits, B = dz as hi + lo)
// The sample's DY1 / xhat / rstd rows (8.25 KB) are fetched with cp.async while phase B of the previous sample
// runs, so the HBM latency is off the dependent path (it was 42% of all stall samples before).
template <int C>
__global__ void __launch_bounds__(ConvBwdSmem<C>::WARPS * 32, 2)
    conv_bwd_mma_kernel(const uint32_t* __restrict__ obs, int64_t obs_rows_per_seed, const int32_t* __restrict__ gather,
                        const float* __restrict__ params, int64_t P, pqn_net_layout_t L, const float* __restrict__ DY1,
                        const float* __restrict__ XH1, const float* __restrict__ RS1, float* __restrict__ part,
                        int rows) {
  using Cfg = ConvCfg<C>;
  using M = ConvMma<C>;
  using SM = ConvBwdSmem<C>;
  constexpr int PWD = PatchCfg<C>::WORDS;
  extern __shared__ __align__(16) float smem_bwd[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int seed = blockIdx.y;
  float* my = smem_bwd + warp * SM::WARP_FLOATS;
  float* my_dy = my + SM::DY;
  float* my_xh = my + SM::XH;
  float* my_rs = my + SM::RS;
  float* my_dz = my + SM::DZ;
  uint32_t* my_so = reinterpret_cast<uint32_t*>(my + SM::DZ);  // only needed until the patches are built
  uint32_t* my_patch = reinterpret_cast<uint32_t*>(my + SM::PATCH);
  float* sc = smem_bwd + SM::WARPS * SM::WARP_FLOATS;
  float* s_red = sc + CONV_O;
  float* s_w = smem_bwd;  // block-level dW reduction buffer, aliases warp 0's slice; only used after the row loop
  static_assert(Cfg::SW <= CONV_PIX * CDZ_LD, "obs staging aliases the dz stage");
  static_assert(M::MT * 16 * CONV_O <= SM::WARP_FLOATS * SM::WARPS, "dW reduction buffer aliases the warp slices");
  static_assert(Cfg::PW <= 32, "one packed observation word per lane");
  if (tid < CONV_O) sc[tid] = __ldg(params + (int64_t)seed * P + L.ln0_scale + tid);
  if (tid < 3 * CONV_O) s_red[tid] = 0.f;
  __syncthreads();
  // lane-private accumulators: columns {2t, 2t+1, 8+2t, 8+2t+1}
  float a_dsc[4] = {0.f, 0.f, 0.f, 0.f}, a_dbi[4] = {0.f, 0.f, 0.f, 0.f}, a_dcb[4] = {0.f, 0.f, 0.f, 0.f};
  float wrun[M::MT][2][4];
#pragma unroll
  for (int mt = 0; mt < M::MT; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 4; ++j) wrun[mt][h][j] = 0.f;

  const int row_stride = gridDim.x * SM::WARPS;
  auto fetch_obs = [&](int r) -> uint32_t {
    if (r >= rows || lane >= Cfg::PW) return 0u;
    const int64_t src = gather ? gather[(int64_t)seed * rows + r] : r;
    return __ldg(obs + ((int64_t)seed * obs_rows_per_seed + src) * Cfg::PW + lane);
  };
  auto fetch_rows = [&](int r) {  // async copy of the sample's dy / xhat / rstd rows into this warp's slice
    if (r < rows) {
      const int64_t gr = (int64_t)seed * rows + r;
      const float* dsrc = DY1 + gr * FLAT_CNN;
      const float* xsrc = XH1 + gr * FLAT_CNN;
#pragma unroll
      for (int i = 0; i < FLAT_CNN / 4 / 32; ++i) {
        const int q = i * 32 + lane, prow = q >> 2;              // 16-byte chunk q = (pixel row, column quad)
        const int dst = prow * CONV_O + cswz(prow, (q & 3) * 4);  // the XOR moves whole chunks
        cp_async16(my_dy + dst, dsrc + q * 4);
        cp_async16(my_xh + dst, xsrc + q * 4);
      }
      if (lane < CONV_PIX / 4) cp_async16(my_rs + lane * 4, RS1 + gr * CONV_PIX + lane * 4);
    }
    cp_async_commit();
  };
  int row = blockIdx.x * SM::WARPS + warp;
  uint32_t pre = fetch_obs(row);
  fetch_rows(row);
  for (; row < rows; row += row_stride) {
    __syncwarp();
    if (lane < Cfg::PW) my_so[lane] = pre;
    if (lane == 0) my_so[Cfg::PW] = 0u;  // pad word read by the funnel shift of the last pixel
    __syncwarp();
    pre = fetch_obs(row + row_stride);
    build_patches<C>(my_so, my_patch, lane);
    cp_async_wait_all();
    __syncwarp();
    // ---- phase A: LayerNorm backward, stage dz
#pragma unroll 1
    for (int mb = 0; mb < 4; ++mb) {
      const int p0 = 16 * mb + g, p1 = p0 + 8;
      float z[2][4];  // xhat in C-fragment layout
      float2 dyv[2][2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        dyv[h][0] = *reinterpret_cast<const float2*>(my_dy + p0 * CONV_O + cswz(p0, 8 * h + 2 * t));
        dyv[h][1] = *reinterpret_cast<const float2*>(my_dy + p1 * CONV_O + cswz(p1, 8 * h + 2 * t));
        const float2 a0 = *reinterpret_cast<const float2*>(my_xh + p0 * CONV_O + cswz(p0, 8 * h + 2 * t));
        const float2 a1 = *reinterpret_cast<const float2*>(my_xh + p1 * CONV_O + cswz(p1, 8 * h + 2 * t));
        z[h][0] = a0.x; z[h][1] = a0.y; z[h][2] = a1.x; z[h][3] = a1.y;
      }
      const float rstd0 = my_rs[p0], rstd1 = my_rs[p1];
      float dxh[2][4];
      float m1a = 0.f, m2a = 0.f, m1b = 0.f, m2b = 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o = 8 * h + 2 * t;
        const float dy4[4] = {dyv[h][0].x, dyv[h][0].y, dyv[h][1].x, dyv[h][1].y};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = 2 * h + (j & 1);    // index into the lane's 4 columns; z[h][j] holds xhat
          a_dsc[col] = fmaf(dy4[j], z[h][j], a_dsc[col]);
          a_dbi[col] += dy4[j];
          dxh[h][j] = dy4[j] * sc[o + (j & 1)];
          if (j < 2) { m1a += dxh[h][j]; m2a = fmaf(dxh[h][j], z[h][j], m2a); }
          else { m1b += dxh[h][j]; m2b = fmaf(dxh[h][j], z[h][j], m2b); }
        }
      }
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        m1a += __shfl_xor_sync(0xffffffffu, m1a, o); m2a += __shfl_xor_sync(0xffffffffu, m2a, o);
        m1b += __shfl_xor_sync(0xffffffffu, m1b, o); m2b += __shfl_xor_sync(0xffffffffu, m2b, o);
      }
      m1a *= (1.0f / CONV_O); m2a *= (1.0f / CONV_O); m1b *= (1.0f / CONV_O); m2b *= (1.0f / CONV_O);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o = 8 * h + 2 * t;
        float dzv[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float rstd = j < 2 ? rstd0 : rstd1, m1 = j < 2 ? m1a : m1b, m2 = j < 2 ? m2a : m2b;
          dzv[j] = rstd * (dxh[h][j] - m1 - z[h][j] * m2);
          a_dcb[2 * h + (j & 1)] += dzv[j];
        }
        *reinterpret_cast<float2*>(my_dz + p0 * CDZ_LD + cswz(p0, o)) = make_float2(dzv[0], dzv[1]);
        *reinterpret_cast<float2*>(my_dz + p1 * CDZ_LD + cswz(p1, o)) = make_float2(dzv[2], dzv[3]);
      }
    }
    __syncwarp();
    fetch_rows(row + row_stride);  // overlaps phase B
    // ---- phase B: dW[tap][o] += sum_pixels x[pixel, tap] * dz[pixel][o]   (fresh accumulators per sample)
    float wacc[M::MT][2][4];
#pragma unroll
    for (int mt = 0; mt < M::MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 4; ++j) wacc[mt][h][j] = 0.f;
#pragma unroll 1
    for (int kk = 0; kk < 8; ++kk) {
      // B fragments: b0 = dz[pixel 8kk + t][o = 8h + g], b1 = dz[pixel 8kk + t + 4][o]
      uint32_t bh[2][2], bl[2][2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r0 = 8 * kk + t, r1 = r0 + 4;
        const float v0 = my_dz[r0 * CDZ_LD + cswz(r0, 8 * h + g)], v1 = my_dz[r1 * CDZ_LD + cswz(r1, 8 * h + g)];
        bh[h][0] = __float_as_uint(v0) & 0xFFFFE000u; bh[h][1] = __float_as_uint(v1) & 0xFFFFE000u;
        bl[h][0] = __float_as_uint(v0 - __uint_as_float(bh[h][0])); bl[h][1] = __float_as_uint(v1 - __uint_as_float(bh[h][1]));
      }
      // A fragments: x[tap, pixel]: a0 = (tap g, pixel 8kk+t), a1 = (tap g+8, same), a2 = (tap g, pixel+4), a3
      const int pa = 8 * kk + t, pb = pa + 4;
      uint32_t qa[PWD], qb[PWD];
#pragma unroll
      for (int k = 0; k < PWD; ++k) { qa[k] = my_patch[pa * PWD + k]; qb[k] = my_patch[pb * PWD + k]; }
#pragma unroll
      for (int mt = 0; mt < M::MT; ++mt) {
        // taps 16mt .. 16mt+15 live in one patch word (32 % 16 == 0, 16 mt < 9C <= 32 PWD); bits beyond 9C are zero
        const uint32_t wa = qa[(16 * mt) >> 5], wb = qb[(16 * mt) >> 5];
        const int sh = ((16 * mt) & 31) + g;
        uint32_t a[4];
        a[0] = bit_f32(wa, sh); a[1] = bit_f32(wa, sh + 8); a[2] = bit_f32(wb, sh); a[3] = bit_f32(wb, sh + 8);
        if (__ballot_sync(0xffffffffu, (a[0] | a[1] | a[2] | a[3]) != 0u) == 0u) continue;
        // lo pass of both column halves, then the hi pass: no back-to-back MMAs on one accumulator
        mma_tf32_16n8k8(wacc[mt][0], a, bl[0][0], bl[0][1]);
        mma_tf32_16n8k8(wacc[mt][1], a, bl[1][0], bl[1][1]);
        mma_tf32_16n8k8(wacc[mt][0], a, bh[0][0], bh[0][1]);
        mma_tf32_16n8k8(wacc[mt][1], a, bh[1][0], bh[1][1]);
      }
    }
#pragma unroll
    for (int mt = 0; mt < M::MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 4; ++j) wrun[mt][h][j] += wacc[mt][h][j];
  }
  cp_async_wait_all();
  // ---- reduce and publish (deterministic): wrun[mt][h][j] is dW[tap = 16mt + g (+8 for j>=2)][o = 8h + 2t + (j&1)].
  // The 8 warps add their registers to the block accumulator one after the other, lanes of a warp own distinct
  // elements; the CTA's partial vector goes to part[seed][cta][TAPS*16 + 48] and conv_bwd_final_kernel sums the CTAs
  // in index order.
  __syncthreads();  // all warps are done with their slices
  for (int w = 0; w < SM::WARPS; ++w) {
    if (warp == w) {
#pragma unroll
      for (int mt = 0; mt < M::MT; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int tap = 16 * mt + g + (j >= 2 ? 8 : 0);
            float* dst = &s_w[tap * CONV_O + 8 * h + 2 * t + (j & 1)];   // tap < 16 * MT: inside the buffer
            *dst = (w == 0 ? 0.f : *dst) + wrun[mt][h][j];
          }
    }
    __syncthreads();
  }
  // per-channel sums: lanes with the same t hold the same columns -> xor-shuffle tree (fixed), then warps in order
#pragma unroll
  for (int col = 0; col < 4; ++col) {
    float v0 = a_dsc[col], v1 = a_dbi[col], v2 = a_dcb[col];
#pragma unroll
    for (int sft = 4; sft <= 16; sft <<= 1) {
      v0 += __shfl_xor_sync(0xffffffffu, v0, sft);
      v1 += __shfl_xor_sync(0xffffffffu, v1, sft);
      v2 += __shfl_xor_sync(0xffffffffu, v2, sft);
    }
    a_dsc[col] = v0; a_dbi[col] = v1; a_dcb[col] = v2;
  }
  for (int w = 0; w < SM::WARPS; ++w) {
    if (warp == w && g == 0) {
#pragma unroll
      for (int col = 0; col < 4; ++col) {
        const int o = 8 * (col >> 1) + 2 * t + (col & 1);
        s_red[o] = (w == 0 ? 0.f : s_red[o]) + a_dsc[col];
        s_red[CONV_O + o] = (w == 0 ? 0.f : s_red[CONV_O + o]) + a_dbi[col];
        s_red[2 * CONV_O + o] = (w == 0 ? 0.f : s_red[2 * CONV_O + o]) + a_dcb[col];
      }
    }
    __syncthreads();
  }
  float* __restrict__ o = part + ((int64_t)seed * gridDim.x + blockIdx.x) * (M::TAPS * CONV_O + 3 * CONV_O);
  // x = bit / 255 (pqn_minatar.py:66): the A operand was the raw bit, so scale here
  for (int i = tid; i < M::TAPS * CONV_O; i += blockDim.x) o[i] = s_w[i] * (1.0f / 255.0f);
  if (tid < 3 * CONV_O) o[M::TAPS * CONV_O + tid] = s_red[tid];
}

// ---------------------------------------------------------------------------------------------------------------
// conv backward with the weight gradient on fp16 warp-level MMA (mma.sync.m16n8k16, fp32 accumulate) -- the default
// backward of the fp16 conv path.  Same phases as conv_bwd_mma_kernel; what changes is phase B,
// dW[tap][o] = sum_pixels x[pixel, tap] dz[pixel][o] with M = taps, N = 16 channels, K = 64 pixels in 4 k-steps of 16:
//   * A (the {0,1} im2col bits, tap-major) is "exponent coded" like the forward: for every PAIR of pixels (2j, 2j+1)
//     and group q of four taps one word holds the tap bits of pixel 2j at bits 10..13 and of pixel 2j+1 at bits 26..29;
//     a fragment register (row = tap, its two k values = the two pixels of a pair) is that word AND the lane's mask
//     (1 << (10 + g%4)) | (1 << (26 + g%4)): a set bit becomes the fp16 power of two 2^(2^(g%4) - 15).  The factor
//     depends only on the accumulator ROW, which is fixed per thread, so it is undone by one exact multiplication
//     when the accumulators are published -- 48 LOP3 per sample instead of 288 shift / and / select.
//   * B = dz * gs as fp16 hi + lo (lo = fp16(v - hi): 22 significant bits where it matters; gs is a power of two that
//     lifts the gradient-sized values out of the fp16 subnormals), written by phase A directly in fragment order:
//     dzT[plane][channel][pixel pair], the pairs (t, t + 4) of a k-step adjacent so that (b0, b1) is one LDS.64; the
//     k-step block of a channel row is XOR-swizzled so that the phase-A stores and the fragment loads are conflict free.
//   * 48 MMAs per sample (3 m-tiles x 2 n-tiles x 4 k-steps x {hi, lo}) instead of 96 tf32 ones.
// xhat and rstd are not read from memory: phase A reruns the training forward's conv MMAs and LayerNorm
// (conv16_blocks_rows, conv16_xhat) from the sample's packed observation with the same parameters, two m-blocks
// (pixels 16 mb .. 16 mb + 15) per call as the forward groups them (one at C = 10), so they are bit for bit what the
// forward computed.
// The rebuild's fragment row g is pixel 16 mb + 2g and row g + 8 is pixel 16 mb + 2g + 1, so thread (g, t) holds
// xhat and rstd of the pixel pair (16 mb + 2g, + 1) -- whose two dz values of a channel are exactly one B word -- in
// channels 4t .. 4t+3, and runs the LayerNorm backward there, in registers: only dy (one 16-byte load per pixel) and
// the dz planes go through shared memory.  The rebuild costs the forward's MMAs again (48 at C = 4, 96 at C = 10); it
// saves 4,352 bytes per sample of HBM writes in the forward and as many reads here.
// ---------------------------------------------------------------------------------------------------------------
template <int C>
struct ConvBwd16 {
  static constexpr int MT = ConvMma<C>::MT;
  static constexpr int NG = 4 * MT;                             // tap groups of 4 per pixel pair
  static constexpr int NGP = (NG % 8 == 4) ? NG : NG + 4;       // pair stride in words: the 4 t-lanes hit distinct banks
  static constexpr int DY = 0;                                  // [64][16] upstream gradient (rows swizzled, dy_off)
  static constexpr int DZT = DY + FLAT_CNN;                     // 2 planes x [16 ch][32 pair words]; aliases the obs row
  static constexpr int PW = DZT + 2 * CONV_O * 32;              // [32 pairs][NGP] exponent-coded pair words
  static constexpr int XP = PW + 32 * NGP;                      // [32 pairs][NGP] the forward's patch words, pair-interleaved
  static constexpr int WARP_FLOATS = XP + 32 * NGP;
  static constexpr int WARPS = (C == 4) ? 8 : 6;                // keeps two CTAs per SM for the wider observations
  static constexpr int WB = WARPS * WARP_FLOATS;                // the forward's weight fragments, Conv16::KS x 2 x 32 uint4
  static constexpr int BYTES = (WB + Conv16<C>::KS * 2 * 32 * 4 + 6 * CONV_O) * 4;  // + cb, sc, bi[16] + s_red[48]
  // m-blocks per conv rebuild: two (the training forward's grouping, more MMAs in flight) where the registers allow
  static constexpr int NBR = (C == 10) ? 1 : 2;
};

// float offset of the 16-byte chunk (pixel p, channels 4q .. 4q+3) in the [64][16] DY stage: rows 4i+2 and 4i+3 are
// swapped, so that the even pixels 2g (and the odd ones) that a quarter-warp reads cover the 32 banks once
__device__ __forceinline__ int dy_off(int p, int q) { return ((p ^ ((p >> 1) & 1)) << 4) + 4 * q; }
// word offset of (channel ch, k-step ks, position pos) in a dzT plane [16][32].  The k-step block of a channel row is
// swizzled by (ch / 4) ^ (ch % 4), which differs between the channels 4t + k of a phase-A store (t = 0..3) and between
// the channels 8h + g of a fragment load (g = 0..3 or 4..7); it sits in bits 3..4, so a thread reaches every block it
// stores or loads from one base word by XOR-ing a constant
__device__ __forceinline__ int dzt_word(int ch, int ks, int pos) {
  return (ch << 5) + ((ks ^ (ch >> 2) ^ (ch & 3)) << 3) + pos;
}

template <int C>
__global__ void __launch_bounds__(ConvBwd16<C>::WARPS * 32, 2)
    conv_bwd_mma16_kernel(const uint32_t* __restrict__ obs, int64_t obs_rows_per_seed, const int32_t* __restrict__ gather,
                          const float* __restrict__ params, int64_t P, pqn_net_layout_t L, const float* __restrict__ DY1,
                          float* __restrict__ part, int rows, float gs) {
  using Cfg = ConvCfg<C>;
  using M = ConvMma<C>;
  using SM = ConvBwd16<C>;
  constexpr int PWD = PatchCfg<C>::WORDS;
  extern __shared__ __align__(16) float smem_bwd[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int seed = blockIdx.y;
  float* my = smem_bwd + warp * SM::WARP_FLOATS;
  float* my_dy = my + SM::DY;
  uint32_t* my_dzt = reinterpret_cast<uint32_t*>(my + SM::DZT);   // plane 0 = hi, plane 1 = lo: 512 words each
  uint32_t* my_so = reinterpret_cast<uint32_t*>(my + SM::DZT);    // packed obs row: only needed until the patch words exist
  uint32_t* my_pw = reinterpret_cast<uint32_t*>(my + SM::PW);
  uint32_t* my_xp = reinterpret_cast<uint32_t*>(my + SM::XP);
  uint4* wb = reinterpret_cast<uint4*>(smem_bwd + SM::WB);
  float* cb = smem_bwd + SM::WB + Conv16<C>::KS * 2 * 32 * 4;
  float* sc = cb + CONV_O;
  float* bi = sc + CONV_O;   // loaded with the forward's weights, not used here
  float* s_red = bi + CONV_O;
  float* s_w = smem_bwd;  // block-level dW reduction buffer, aliases warp 0's slice; only used after the row loop
  static_assert(Cfg::SW <= 2 * CONV_O * 32, "obs staging aliases the dz planes");
  static_assert(M::MT * 16 * CONV_O <= SM::WARP_FLOATS * SM::WARPS, "dW reduction buffer aliases the warp slices");
  static_assert(Cfg::PW <= 32, "one packed observation word per lane");
  static_assert(SM::XP % 4 == 0 && SM::WB % 4 == 0, "16-byte aligned patch rows and weight fragments");
  static_assert(SM::NG == 4 * Conv16<C>::KS, "a pixel's patch words are exactly the pair words' tap groups");
  conv16_load_weights<C>(params + (int64_t)seed * P, L, wb, cb, sc, bi, threadIdx.x, blockDim.x);
  if (tid < 3 * CONV_O) s_red[tid] = 0.f;
  __syncthreads();
  float a_dsc[4] = {0.f, 0.f, 0.f, 0.f}, a_dbi[4] = {0.f, 0.f, 0.f, 0.f}, a_dcb[4] = {0.f, 0.f, 0.f, 0.f};
  float wrun[M::MT][2][4];
#pragma unroll
  for (int mt = 0; mt < M::MT; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 4; ++j) wrun[mt][h][j] = 0.f;
  const uint32_t amask = (1u << (10 + (g & 3))) | (1u << (26 + (g & 3)));
  // per-lane offsets, computed once: the k-steps and the m-blocks of one rebuild add compile-time constants (or XOR
  // them, for the dzT swizzle)
  const int pos_g = g < 4 ? 2 * g : 2 * (g - 4) + 1;   // pair g of a k-step sits next to pair g + 4
  const uint32_t* xpg = my_xp + g * SM::NGP;   // rebuild fragment rows g, g + 8: pixel pair g of each m-block
  const float* dy0 = my_dy + dy_off(2 * g, t);
  const float* dy1 = my_dy + dy_off(2 * g + 1, t);
  // dzt_word(4t + k, mb, pos_g) = (dzs ^ ((k ^ mb) << 3)) + 32 k, dzt_word(8h + g, ks, 2t) = (dzl ^ ((ks ^ 2h) << 3)) + 256 h
  const int dzs = dzt_word(4 * t, 0, pos_g), dzl = dzt_word(g, 0, 2 * t);
  const uint32_t* pa = my_pw + t * SM::NGP + 2 * (g >> 2);   // pixel pair 8ks + t: A rows (g, g + 8)
  const uint32_t* pb = pa + 4 * SM::NGP;                     // pixel pair 8ks + t + 4

  const int row_stride = gridDim.x * SM::WARPS;
  // unconditional loads from clamped addresses (rows past the end re-read the last row, lanes past the packed width
  // re-read word 0; neither is ever used): a predicated load with a default value made ptxas copy the result into the
  // loop-carried register ~125 instructions after the LDG, which stalled every warp on the load it had just issued
  // (13 % of all stall samples of the forward kernel, ncu r2m)
  auto fetch_index = [&](int r) -> int {
    const int rc = r < rows ? r : rows - 1;
    return gather ? __ldg(gather + (int64_t)seed * rows + rc) : rc;
  };
  auto fetch_obs = [&](int src) -> uint32_t {
    return __ldg(obs + ((int64_t)seed * obs_rows_per_seed + src) * Cfg::PW + (lane < Cfg::PW ? lane : 0));
  };
  auto fetch_dy = [&](int r) {  // async copy of the sample's dy row into this warp's slice
    if (r < rows) {
      const float* dsrc = DY1 + ((int64_t)seed * rows + r) * FLAT_CNN;
#pragma unroll
      for (int i = 0; i < FLAT_CNN / 4 / 32; ++i) {
        const int q = i * 32 + lane;                             // 16-byte chunk q = (pixel row, column quad)
        cp_async16(my_dy + dy_off(q >> 2, q & 3), dsrc + q * 4);
      }
    }
    cp_async_commit();
  };
  int row = blockIdx.x * SM::WARPS + warp;
  uint32_t pre = fetch_obs(fetch_index(row));
  int src_next = fetch_index(row + row_stride);
  fetch_dy(row);
  for (; row < rows; row += row_stride) {
    __syncwarp();
    if (lane < Cfg::PW) my_so[lane] = pre;
    if (lane == 0) my_so[Cfg::PW] = 0u;  // pad word read by the funnel shift of the last pixel
    __syncwarp();
    pre = fetch_obs(src_next);
    src_next = fetch_index(row + 2 * row_stride);
    {  // exponent-coded pair words of pixel pair `lane`, and from them the forward's patch words of its two pixels
      uint32_t w0[PWD], w1[PWD];
      patch_bits<C>(my_so, 2 * lane, w0);
      patch_bits<C>(my_so, 2 * lane + 1, w1);
      uint32_t gw[SM::NG];   // tap group q: taps 4q .. 4q+3 of pixel 2 lane at bits 10..13, of pixel 2 lane + 1 at 26..29
#pragma unroll
      for (int q = 0; q < SM::NG; ++q) {
        const int bit = 4 * q, wi = bit >> 5, sh = bit & 31;
        gw[q] = 0u;
        if (wi < PWD) {
          const uint32_t v0 = w0[wi < PWD ? wi : 0], v1 = w1[wi < PWD ? wi : 0];
          const uint32_t lo = sh >= 10 ? v0 >> (sh >= 10 ? sh - 10 : 0) : v0 << (sh < 10 ? 10 - sh : 0);
          const uint32_t hi = sh <= 26 ? v1 << (sh <= 26 ? 26 - sh : 0) : v1 >> (sh > 26 ? sh - 26 : 0);
          gw[q] = __byte_perm(lo, hi, 0x7610);
        }
      }
      uint32_t pw[SM::NGP];
#pragma unroll
      for (int k = 0; k < SM::NGP; ++k) pw[k] = 0u;
#pragma unroll
      for (int q = 0; q < SM::NG; ++q) {
        // memory order inside an m-tile: groups (0, 2, 1, 3), so the words of fragment rows g and g + 8 are adjacent
        const int ql = q & 3, slot = (q & ~3) + (ql == 1 ? 2 : (ql == 2 ? 1 : ql));
        pw[slot] = gw[q];
      }
      uint32_t* dstw = my_pw + lane * SM::NGP;
#pragma unroll
      for (int k = 0; k < SM::NGP / 4; ++k)
        *reinterpret_cast<uint4*>(dstw + 4 * k) = make_uint4(pw[4 * k], pw[4 * k + 1], pw[4 * k + 2], pw[4 * k + 3]);
      // the forward's patch word of byte b of a pixel holds taps 8b .. 8b+3 at bits 10..13 and 8b+4 .. 8b+7 at 26..29
      // (build_patch16): groups 2b and 2b+1, the low halves of their pair words for pixel 2 lane, the high halves for
      // 2 lane + 1.  Row `lane` of XP: per k-step s (bytes 2s, 2s+1) pixel 2 lane's two words, then 2 lane + 1's.
      uint32_t* dstx = my_xp + lane * SM::NGP;
#pragma unroll
      for (int s = 0; s < Conv16<C>::KS; ++s)
        *reinterpret_cast<uint4*>(dstx + 4 * s) =
            make_uint4(__byte_perm(gw[4 * s], gw[4 * s + 1], 0x5410), __byte_perm(gw[4 * s + 2], gw[4 * s + 3], 0x5410),
                       __byte_perm(gw[4 * s], gw[4 * s + 1], 0x7632), __byte_perm(gw[4 * s + 2], gw[4 * s + 3], 0x7632));
    }
    cp_async_wait_all();
    __syncwarp();
    // ---- phase A: LayerNorm backward of the pixel pair (16 mb + 2g, + 1) in channels 4t .. 4t+3; dz * gs -> fp16
    // (hi, lo) planes.  Every rounding is the one the former [pixel pair][channels 2t, 2t+1, 8+2t, 9+2t] layout made,
    // and the per-channel sums add the same pixels in the same order, so dz and all gradients keep their bits.
#pragma unroll 1   // unrolled, ptxas hoists the next rebuild's loads and spills
    for (int mp = 0; mp < 4 / SM::NBR; ++mp) {
      float zc[SM::NBR][2][4];
      const float4 cbv = *reinterpret_cast<const float4*>(cb + 4 * t);   // conv bias of channels 4t .. 4t+3
      const float cb4[4] = {cbv.x, cbv.y, cbv.z, cbv.w};
      conv16_blocks_rows<C, SM::NBR, 8 * SM::NGP, true>(xpg + 8 * SM::NBR * mp * SM::NGP, nullptr, wb, cb4, lane, zc);
#pragma unroll
      for (int i = 0; i < SM::NBR; ++i) {
        const int mb = SM::NBR * mp + i;
        float x[2][4], rs[2];   // [pixel 16 mb + 2g + p][channel 4t + k]
        conv16_xhat(zc[i], x[0], x[1], rs[0], rs[1]);
        const float4 d0 = *reinterpret_cast<const float4*>(dy0 + 256 * mb);
        const float4 d1 = *reinterpret_cast<const float4*>(dy1 + 256 * mb);
        const float dy[2][4] = {{d0.x, d0.y, d0.z, d0.w}, {d1.x, d1.y, d1.z, d1.w}};
        const float4 scv = *reinterpret_cast<const float4*>(sc + 4 * t);   // LayerNorm scale of channels 4t .. 4t+3
        const float sc4[4] = {scv.x, scv.y, scv.z, scv.w};
        float dxh[2][4];
#pragma unroll
        for (int p = 0; p < 2; ++p)
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            a_dsc[k] = fmaf(dy[p][k], x[p][k], a_dsc[k]);
            a_dbi[k] = __fadd_rn(a_dbi[k], dy[p][k]);
            dxh[p][k] = __fmul_rn(dy[p][k], sc4[k]);
          }
        // m1 = sum_ch dxh, m2 = sum_ch dxh * xhat over the 16 channels of each pixel, associated as
        // (P0 + P1) + (P2 + P3) with P_u = ((ch 2u + ch 2u+1) + ch 8+2u) + ch 9+2u: lanes 0, 1 start the chains of
        // their channel pairs, lanes 2, 3 (channels 8 .. 15) continue them, add P_2v + P_2v+1 and swap the result
        float m1[2], m2[2];
#pragma unroll
        for (int p = 0; p < 2; ++p) {
          float s1[2], s2[2];
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            s1[j] = __fadd_rn(__fadd_rn(0.f, dxh[p][2 * j]), dxh[p][2 * j + 1]);
            s2[j] = fmaf(dxh[p][2 * j + 1], x[p][2 * j + 1], fmaf(dxh[p][2 * j], x[p][2 * j], 0.f));
          }
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const float r1 = __shfl_xor_sync(0xffffffffu, s1[j], 2), r2 = __shfl_xor_sync(0xffffffffu, s2[j], 2);
            s1[j] = __fadd_rn(__fadd_rn(r1, dxh[p][2 * j]), dxh[p][2 * j + 1]);
            s2[j] = fmaf(dxh[p][2 * j + 1], x[p][2 * j + 1], fmaf(dxh[p][2 * j], x[p][2 * j], r2));
          }
          float q1 = __fadd_rn(s1[0], s1[1]), q2 = __fadd_rn(s2[0], s2[1]);
          q1 = __fadd_rn(q1, __shfl_xor_sync(0xffffffffu, q1, 1));
          q2 = __fadd_rn(q2, __shfl_xor_sync(0xffffffffu, q2, 1));
          m1[p] = __shfl_sync(0xffffffffu, q1, lane | 2);
          m2[p] = __fmul_rn(__shfl_sync(0xffffffffu, q2, lane | 2), 1.0f / CONV_O);
        }
        // dz = rstd gs (dxh - m1 / 16 - xhat m2 / 16): rstd * gs makes dz come out pre-scaled for the fp16 planes (gs
        // is a power of two; the conv-bias sum is unscaled at the end)
        float dz[2][4];
#pragma unroll
        for (int p = 0; p < 2; ++p) {
          const float rsg = __fmul_rn(rs[p], gs);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            dz[p][k] = __fmul_rn(rsg, fmaf(-x[p][k], m2[p], fmaf(m1[p], -1.0f / CONV_O, dxh[p][k])));
            a_dcb[k] = __fadd_rn(a_dcb[k], dz[p][k]);
          }
        }
        // B words: (pixel 16 mb + 2g, + 1) of channel 4t + k; k-step mb, pair g
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t hw = cvt_f16x2_satfinite(dz[0][k], dz[1][k]);
          const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw));
          const __half2 lw = __floats2half2_rn(dz[0][k] - hf.x, dz[1][k] - hf.y);
          const int wd = (dzs ^ ((k ^ mb) << 3)) + 32 * k;
          my_dzt[wd] = hw;
          my_dzt[CONV_O * 32 + wd] = *reinterpret_cast<const uint32_t*>(&lw);
        }
      }
    }
    __syncwarp();
    fetch_dy(row + row_stride);    // overlaps phase B
    // ---- phase B: dW[tap][o] += sum_pixels x[pixel, tap] * dz[pixel][o]   (fresh accumulators per sample)
    float wacc[M::MT][2][4];
#pragma unroll
    for (int mt = 0; mt < M::MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 4; ++j) wacc[mt][h][j] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      // B fragments: b0 = dz[pixels 16ks + 2t, + 1][o = 8h + g], b1 = the same of pixels + 8: one LDS.64 per plane
      uint2 bhi[2], blo[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int wd = (dzl ^ ((ks ^ 2 * h) << 3)) + 256 * h;
        bhi[h] = *reinterpret_cast<const uint2*>(my_dzt + wd);
        blo[h] = *reinterpret_cast<const uint2*>(my_dzt + CONV_O * 32 + wd);
      }
#pragma unroll
      for (int mt = 0; mt < M::MT; ++mt) {
        const uint2 wa = *reinterpret_cast<const uint2*>(pa + 8 * ks * SM::NGP + 4 * mt);
        const uint2 wb2 = *reinterpret_cast<const uint2*>(pb + 8 * ks * SM::NGP + 4 * mt);
        uint32_t a[4];
        a[0] = wa.x & amask; a[1] = wa.y & amask; a[2] = wb2.x & amask; a[3] = wb2.y & amask;
        // lo pass of both column halves, then the hi pass: no back-to-back MMAs on one accumulator
        mma_f16_16n8k16(wacc[mt][0], a, blo[0].x, blo[0].y);
        mma_f16_16n8k16(wacc[mt][1], a, blo[1].x, blo[1].y);
        mma_f16_16n8k16(wacc[mt][0], a, bhi[0].x, bhi[0].y);
        mma_f16_16n8k16(wacc[mt][1], a, bhi[1].x, bhi[1].y);
      }
    }
#pragma unroll
    for (int mt = 0; mt < M::MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 4; ++j) wrun[mt][h][j] += wacc[mt][h][j];
  }
  cp_async_wait_all();
  // ---- reduce and publish (deterministic), as in conv_bwd_mma_kernel; the A coding 2^(2^(g%4) - 15) of this thread's
  // accumulator rows and the dz scale gs are undone here (exact powers of two)
  const float inv_gs = 1.0f / gs;
  const float unscale = __uint_as_float((uint32_t)(127 + 15 - (1 << (g & 3))) << 23) * inv_gs;
  __syncthreads();  // all warps are done with their slices
  for (int w = 0; w < SM::WARPS; ++w) {
    if (warp == w) {
#pragma unroll
      for (int mt = 0; mt < M::MT; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int tap = 16 * mt + g + (j >= 2 ? 8 : 0);
            float* dst = &s_w[tap * CONV_O + 8 * h + 2 * t + (j & 1)];   // tap < 16 * MT: inside the buffer
            *dst = (w == 0 ? 0.f : *dst) + wrun[mt][h][j] * unscale;
          }
    }
    __syncthreads();
  }
  // per-channel sums: lanes with the same t hold the same channels 4t .. 4t+3 -> xor-shuffle tree over g (fixed),
  // then warps in order
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float v0 = a_dsc[k], v1 = a_dbi[k], v2 = a_dcb[k];
#pragma unroll
    for (int sft = 4; sft <= 16; sft <<= 1) {
      v0 += __shfl_xor_sync(0xffffffffu, v0, sft);
      v1 += __shfl_xor_sync(0xffffffffu, v1, sft);
      v2 += __shfl_xor_sync(0xffffffffu, v2, sft);
    }
    a_dsc[k] = v0; a_dbi[k] = v1; a_dcb[k] = v2;
  }
  for (int w = 0; w < SM::WARPS; ++w) {
    if (warp == w && g == 0) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int o = 4 * t + k;
        s_red[o] = (w == 0 ? 0.f : s_red[o]) + a_dsc[k];
        s_red[CONV_O + o] = (w == 0 ? 0.f : s_red[CONV_O + o]) + a_dbi[k];
        s_red[2 * CONV_O + o] = (w == 0 ? 0.f : s_red[2 * CONV_O + o]) + a_dcb[k] * inv_gs;
      }
    }
    __syncthreads();
  }
  float* __restrict__ o = part + ((int64_t)seed * gridDim.x + blockIdx.x) * (M::TAPS * CONV_O + 3 * CONV_O);
  for (int i = tid; i < M::TAPS * CONV_O; i += blockDim.x) o[i] = s_w[i] * (1.0f / 255.0f);
  if (tid < 3 * CONV_O) o[M::TAPS * CONV_O + tid] = s_red[tid];
}

// Sums conv_bwd_mma_kernel's per-CTA partials in a fixed order into the gradients.
// grid = (ceil(n / (256 / SL)), S), block = 256
template <int SL>
__global__ void conv_bwd_final_kernel(const float* __restrict__ part, int nctas, int taps16, float* __restrict__ grads,
                                      int64_t P, pqn_net_layout_t L) {
  const int seed = blockIdx.y;
  const int stride = taps16 + 3 * CONV_O;
  const int i = blockIdx.x * (256 / SL) + threadIdx.x % (256 / SL);
  const float v = ordered_partial_sum<SL>(part + (int64_t)seed * nctas * stride + i, nctas, stride, i < stride);
  if (i >= stride || threadIdx.x >= 256 / SL) return;
  float* __restrict__ gout = grads + (int64_t)seed * P;
  if (i < taps16) gout[L.conv_w + i] = v;
  else if (i < taps16 + CONV_O) gout[L.ln0_scale + (i - taps16)] = v;
  else if (i < taps16 + 2 * CONV_O) gout[L.ln0_bias + (i - taps16 - CONV_O)] = v;
  else gout[L.conv_b + (i - taps16 - 2 * CONV_O)] = v;
}

// MLP input gather (minibatch rows of float obs); the input BatchNorm sums come from nrm::colsum2 of the result.
__global__ void gather_rows_kernel(const float* __restrict__ obs, int64_t obs_rows_per_seed,
                                   const int32_t* __restrict__ gather, float* __restrict__ out, int rows, int D) {
  const int seed = blockIdx.y;
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (int64_t)rows * D) return;
  const int r = (int)(g / D), j = (int)(g - (int64_t)r * D);
  const int64_t src = gather ? gather[(int64_t)seed * rows + r] : r;
  const float v = __ldg(obs + ((int64_t)seed * obs_rows_per_seed + src) * D + j);
  out[((int64_t)seed * rows + r) * D + j] = v;
}

// ---------------------------------------------------------------------------
// host-side orchestration
// ---------------------------------------------------------------------------
struct Workspace {
  // CNN
  float *h1, *h2, *xhat2, *rstd2, *dz2;
  float *h1_lo, *dz2_lo, *w1_lo;  // 3xTF32 "lo" operands of the TF32 path; regions of the fp16-split planes (Planes16)
  float *cxhat, *crstd;           // conv LayerNorm xhat / rstd saved by the training forward (tf32 conv path 3 only)
  uint32_t* relu_bits;            // packed (h1 > 0) mask, 1024 bits per row (MMA conv path -> tensor-core dgrad epilogue)
  float *rb_part, *cb_part;       // per-CTA partial vectors of the deterministic row_bwd / conv_bwd reductions
  float* wg_part;                 // split-K partial outputs of the tensor-core weight gradient (small S: few output tiles)
  // MLP: per hidden layer l the output h, LayerNorm xhat and rstd; dz / dh of the layer being differentiated
  float *xg, *h[PQN_MAX_LAYERS], *xhat[PQN_MAX_LAYERS], *rstd[PQN_MAX_LAYERS], *dzl, *dh0;
  // fp16 (hi, lo') planes for the tensor-core hidden layers l >= 1: of h_{l-1} and of Dense_l's kernel (one block per
  // hidden layer each, see mlp_planes), and of dz of the layer being differentiated
  float *m16_h0, *m16_w, *m16_dz;
};

// split-K of the tensor-core weight gradient: when S * m_tiles * n_tiles output tiles cannot fill the SMs (one seed of
// the MLP has 4 tiles, of the CNN 8), the K = rows range is divided so that one CTA per SM runs; the partial tiles
// (at most wgrad_split_tiles() of them) are added in split order by wgrad_split_reduce_kernel (deterministic)
// tensor-core split-K: <= SMs tiles; FFMA row splits: tiles * S * splits < 4 * SMs
static int64_t wgrad_split_tiles() { return 4 * (int64_t)device_sm_count() + 16; }
static int wgrad_ksplit(int tiles_total, int k_blocks) {
  const int sms = device_sm_count();                 // persistent kernel, one CTA per SM: one wave of split tiles
  if (tiles_total >= sms) return 1;
  int ks = sms / tiles_total;
  if (ks > k_blocks / 8) ks = k_blocks / 8;          // keep >= 8 k-blocks per CTA
  if (ks < 1) ks = 1;
  while (ks > 1 && (int64_t)(ks - 1) * ((k_blocks + ks - 1) / ks) >= k_blocks) --ks;   // no empty split
  return ks;
}
template <int SL>
__global__ void wgrad_split_reduce_kernel(const float* __restrict__ part, int ksplit, int64_t split_stride, int64_t n_per_seed,
                                          float* __restrict__ out, int64_t out_seed_stride) {
  const int seed = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * (256 / SL) + threadIdx.x % (256 / SL);
  const float v = ordered_partial_sum<SL>(part + (int64_t)seed * n_per_seed + i, ksplit, split_stride, i < n_per_seed);
  if (i < n_per_seed && threadIdx.x < 256 / SL) out[(int64_t)seed * out_seed_stride + i] = v;
}
// out[seed][i] = sum over k < ksplit of part[k * split_stride + seed * n + i], in k-slice order
static void launch_split_reduce(const float* part, int ksplit, int64_t split_stride, int64_t n, int S, float* out,
                                int64_t out_seed_stride, cudaStream_t st) {
  LaunchScope _ls(K_GRAD_FINAL, st);
  if (final_slices(ksplit) == 32)
    wgrad_split_reduce_kernel<32><<<dim3((unsigned)((n + 7) / 8), S), 256, 0, st>>>(part, ksplit, split_stride, n, out, out_seed_stride);
  else
    wgrad_split_reduce_kernel<8><<<dim3((unsigned)((n + 31) / 32), S), 256, 0, st>>>(part, ksplit, split_stride, n, out, out_seed_stride);
}

// N tile of the FFMA gradient kernels: 128, or 64 for a 64-wide layer; output tiles of a [Kin][N] weight gradient
static inline int ffma_ntile(int N) { return N % 128 == 0 ? 128 : 64; }
static inline int ffma_tiles(int Kin, int N) { return (Kin + 127) / 128 * (N / ffma_ntile(N)); }

// The register-tiled FFMA weight gradient + (splits > 1) its ordered reduction.  `part` needs splits * S * Kin * N floats
// (<= wgrad_split_tiles() tiles of 128 x 128: wgrad_splits keeps tiles * S * splits below 4 * SMs).
static void run_wgrad_ffma(const float* X, int64_t x_seed_stride, int ldx, const float* DZ, int64_t dz_seed_stride, int N,
                           float* grads, int64_t P, int64_t off_w, int rows, int Kin, int S, int splits, float* part,
                           cudaStream_t st) {
  { LaunchScope _ls(K_WGRAD, st);
    const dim3 grid((unsigned)((Kin + 127) / 128), (unsigned)(N / ffma_ntile(N)), (unsigned)(S * splits));
    if (ffma_ntile(N) == 128)
      wgrad_kernel<128><<<grid, GT, 0, st>>>(X, x_seed_stride, ldx, DZ, dz_seed_stride, N, grads, P, off_w, rows, Kin, splits, part);
    else
      wgrad_kernel<64><<<grid, GT, 0, st>>>(X, x_seed_stride, ldx, DZ, dz_seed_stride, N, grads, P, off_w, rows, Kin, splits, part); }
  if (splits > 1) {
    const int64_t n = (int64_t)Kin * N;
    launch_split_reduce(part, splits, (int64_t)S * n, n, S, grads + off_w, P, st);
  }
}

// Weight gradient of a layer with a *thin* input (the first MLP layer: Kin = observation features <= 8):
// dW[k][n] = sum_rows X[row][k] * dZ[row][n].  A 128 x 128 register tile would spend 94 % of its FFMAs on padding, so
// here every thread owns four output columns (256 / (N/4) row groups) and Kin float4 accumulators, streams its rows
// of dZ coalesced (16-byte loads) and reads the X rows of the CTA's tile from shared memory (broadcast).  Per-CTA partials
// part[chunk][seed][Kin][N] are then added in chunk order by wgrad_split_reduce_kernel: no float atomics.
// grid = (chunks, S), block = 256
constexpr int THIN_KMAX = 8, THIN_ROWS = 128;
__global__ void __launch_bounds__(256) wgrad_thin_kernel(const float* __restrict__ X, int64_t x_seed_stride, int Kin,
                                                         const float* __restrict__ DZ, int64_t dz_seed_stride, int N,
                                                         float* __restrict__ part, int rows, int rows_per_chunk) {
  __shared__ float xs[THIN_ROWS * THIN_KMAX];
  __shared__ float4 red[256];
  const int seed = blockIdx.y, S = gridDim.y;
  const int cols4 = N >> 2;                                             // threads per row (float4 columns); N in 64..512
  const int groups = 256 / cols4, c4 = threadIdx.x % cols4, grp = threadIdx.x / cols4;
  const float* __restrict__ Xs = X + (int64_t)seed * x_seed_stride;
  const float4* __restrict__ Zs = reinterpret_cast<const float4*>(DZ + (int64_t)seed * dz_seed_stride);
  const int r_begin = blockIdx.x * rows_per_chunk, r_end = min(rows, r_begin + rows_per_chunk);
  float4 acc[THIN_KMAX];
#pragma unroll
  for (int k = 0; k < THIN_KMAX; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r0 = r_begin; r0 < r_end; r0 += THIN_ROWS) {
    const int nr = min(THIN_ROWS, r_end - r0);
    __syncthreads();
    for (int i = threadIdx.x; i < nr * Kin; i += 256) {
      const int r = i / Kin, k = i - r * Kin;
      xs[r * THIN_KMAX + k] = __ldg(Xs + (int64_t)(r0 + r) * Kin + k);
    }
    __syncthreads();
#pragma unroll 4
    for (int r = grp; r < nr; r += groups) {
      const float4 z = __ldg(Zs + (int64_t)(r0 + r) * cols4 + c4);
#pragma unroll
      for (int k = 0; k < THIN_KMAX; ++k)
        if (k < Kin) {
          const float x = xs[r * THIN_KMAX + k];
          acc[k].x = fmaf(x, z.x, acc[k].x); acc[k].y = fmaf(x, z.y, acc[k].y);
          acc[k].z = fmaf(x, z.z, acc[k].z); acc[k].w = fmaf(x, z.w, acc[k].w);
        }
    }
  }
  // add the row groups in group order (one k at a time through shared memory), then store this CTA's partial
  float4* __restrict__ out = reinterpret_cast<float4*>(part + ((int64_t)blockIdx.x * S + seed) * Kin * N);
#pragma unroll
  for (int k = 0; k < THIN_KMAX; ++k) {
    if (k >= Kin) break;
    __syncthreads();
    red[threadIdx.x] = acc[k];
    __syncthreads();
    if (grp == 0) {
      float4 v = red[c4];
      for (int g = 1; g < groups; ++g) {
        const float4 o = red[g * cols4 + c4];
        v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
      }
      out[k * cols4 + c4] = v;
    }
  }
}

// upper bound of the CTAs (all seeds) of the wave-sized grids of conv_mma_ctas(): <= 6 waves of <= 4 CTAs/SM, + S
static int64_t part_ctas(int S) { return 6 * 4 * (int64_t)device_sm_count() + 2 * (int64_t)S; }
static int64_t row_bwd_part_floats(int N, int A);
static int wgrad_splits(int tiles, int S, int rows);
static inline unsigned cdiv(int64_t a, int64_t b) { return (unsigned)((a + b - 1) / b); }

// first-layer weight gradient dW0[D][H] = X^T . dZ: the thin deterministic kernel when D <= 8 (every shipped classic-control
// env), the register-tiled FFMA kernel otherwise.  `part` is the row_bwd partial buffer (free again at this point of
// the stream; chunks * S * D * H floats are far below its size).
static void run_wgrad_first(const float* X, const float* DZ, float* grads, int64_t P, int64_t off_w, int S, int rows,
                            int D, int H, float* part, float* wg_part, cudaStream_t st) {
  if (D <= THIN_KMAX) {
    int chunks = (2 * device_sm_count()) / S;
    const int max_chunks = (rows + THIN_ROWS - 1) / THIN_ROWS;
    if (chunks > max_chunks) chunks = max_chunks;
    if (chunks < 1) chunks = 1;
    int per = (rows + chunks - 1) / chunks;
    per = (per + THIN_ROWS - 1) / THIN_ROWS * THIN_ROWS;
    chunks = (rows + per - 1) / per;
    const int64_t n = (int64_t)D * H;
    { LaunchScope _ls(K_WGRAD, st);
      wgrad_thin_kernel<<<dim3(chunks, S), 256, 0, st>>>(X, (int64_t)rows * D, D, DZ, (int64_t)rows * H, H, part, rows, per); }
    launch_split_reduce(part, chunks, (int64_t)S * n, n, S, grads + off_w, P, st);
    return;
  }
  run_wgrad_ffma(X, (int64_t)rows * D, D, DZ, (int64_t)rows * H, H, grads, P, off_w, rows, D, S,
                 wgrad_splits(ffma_tiles(D, H), S, rows), wg_part, st);
}

// OUT[S][rows][Kprev] (=, or += with accumulate) relu_mask(HPREV) * (DZ[S][rows][N] . W[Kprev][N]^T) on the FFMA kernel
static void launch_dgrad(const float* DZ, int64_t dz_seed_stride, int N, const float* params, int64_t P, int64_t off_w,
                         const float* HPREV, float* OUT, int64_t h_seed_stride, int rows, int Kprev, int accumulate, int S,
                         cudaStream_t st) {
  LaunchScope _ls(K_DGRAD, st);
  const dim3 grid(cdiv(rows, 128), (unsigned)(Kprev / ffma_ntile(Kprev)), (unsigned)S);
  if (ffma_ntile(Kprev) == 128)
    dgrad_kernel<128><<<grid, GT, 0, st>>>(DZ, dz_seed_stride, N, params, P, off_w, HPREV, OUT, h_seed_stride, rows, Kprev, accumulate);
  else
    dgrad_kernel<64><<<grid, GT, 0, st>>>(DZ, dz_seed_stride, N, params, P, off_w, HPREV, OUT, h_seed_stride, rows, Kprev, accumulate);
}

#include "pqn_bits.cuh"

static int64_t carve(const pqn_net_desc_t* d, int32_t S, int64_t rows, char* base, Workspace* w) {
  int64_t off = 0;
  auto take = [&](int64_t nfloats) -> float* {
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += (nfloats * 4 + 255) / 256 * 256;
    return p;
  };
  const int64_t R = (int64_t)S * rows;
  Workspace tmp;
  Workspace* ww = w ? w : &tmp;
  if (d->kind == PQN_NET_MINATAR_CNN) {
    ww->h1 = take(R * FLAT_CNN);
    ww->h2 = take(R * HID_CNN);
    ww->xhat2 = take(R * HID_CNN);
    ww->rstd2 = take(R);
    ww->dz2 = take(R * HID_CNN);
    ww->h1_lo = take(R * FLAT_CNN);
    ww->dz2_lo = take(R * HID_CNN);
    ww->w1_lo = take((int64_t)S * FLAT_CNN * HID_CNN);
    ww->cxhat = take(R * FLAT_CNN);
    ww->crstd = take(R * CONV_PIX);
    ww->relu_bits = reinterpret_cast<uint32_t*>(take(R * (FLAT_CNN / 32)));
    ww->rb_part = take(part_ctas(S) * row_bwd_part_floats(HID_CNN, d->num_actions));
    ww->cb_part = take(part_ctas(S) * (int64_t)(9 * d->in_c * CONV_O + 3 * CONV_O));
    ww->wg_part = take(wgrad_split_tiles() * 128 * 128);
  } else {
    const int H = d->hidden, nl = d->layers > 2 ? d->layers : 2, nh = nl - 1;
    ww->xg = take(R * d->in_c);
    for (int l = 0; l < nl; ++l) { ww->h[l] = take(R * H); ww->xhat[l] = take(R * H); ww->rstd[l] = take(R); }
    ww->dzl = take(R * H);
    ww->dh0 = take(R * H);
    ww->rb_part = take(part_ctas(S) * row_bwd_part_floats(H, d->num_actions));
    ww->cb_part = nullptr;
    ww->wg_part = take(wgrad_split_tiles() * 128 * 128);
    ww->m16_h0 = take(nh * R * H);                  // 2 planes x 2 bytes = 4 bytes per element
    ww->m16_w = take(nh * (int64_t)S * H * H);
    ww->m16_dz = take(R * H);
  }
  return off;
}

// BN = the layer's width: 64, 128 or 256, and 512 for MODE 3 only (two 256-column tiles; dense_ln_fwd adds the
// LayerNorm at 512).  Any other combination is refused, not launched with a narrower tile.
template <int MODE>
static int launch_dense(int BN, dim3 grid, cudaStream_t st, const float* X, int64_t xss, int ldx, const float* params,
                         int64_t P, int64_t ow, int64_t ob, int64_t osc, int64_t obi, int64_t ohw, int64_t ohb, int A,
                         float* H, float* XH, float* RS, float* Q, int rows, int K) {
  if (BN != 64 && BN != 128 && BN != 256 && !(MODE == 3 && BN == 512))
    return set_error(PQN_E_UNSUPPORTED, "dense_fwd: width %d is not built for mode %d", BN, MODE);
  if (BN == 64)
    { LaunchScope _ls(K_DENSE_FWD, st); dense_fwd_kernel<64, MODE><<<grid, GT, 0, st>>>(X, xss, ldx, params, P, ow, ob, osc, obi, ohw, ohb, A, H, XH, RS, Q, rows, K); }
  else if (MODE == 3 && BN == 512)
    { LaunchScope _ls(K_DENSE_FWD, st); dense_fwd_kernel<256, 3><<<dim3(grid.x, grid.y, 2), GT, 0, st>>>(X, xss, ldx, params, P, ow, ob, osc, obi, ohw, ohb, A, H, XH, RS, Q, rows, K); }
  else if (BN == 128)
    { LaunchScope _ls(K_DENSE_FWD, st); dense_fwd_kernel<128, MODE><<<grid, GT, 0, st>>>(X, xss, ldx, params, P, ow, ob, osc, obi, ohw, ohb, A, H, XH, RS, Q, rows, K); }
  else
    { LaunchScope _ls(K_DENSE_FWD, st); dense_fwd_kernel<256, MODE><<<grid, GT, 0, st>>>(X, xss, ldx, params, P, ow, ob, osc, obi, ohw, ohb, A, H, XH, RS, Q, rows, K); }
  return 0;
}


template <int C>
static int launch_conv_bwd_mma(dim3 grid, cudaStream_t st, const uint32_t* obs, int64_t orps, const int32_t* gather,
                               const float* params, int64_t P, const pqn_net_layout_t& L, const float* dy1,
                               const float* xh1, const float* rs1, float* grads, float* part, int rows) {
  auto kfn = conv_bwd_mma_kernel<C>;
  if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, ConvBwdSmem<C>::BYTES) != cudaSuccess)
    return check_launch("conv_bwd_mma(cudaFuncSetAttribute)");
  kfn<<<grid, ConvBwdSmem<C>::WARPS * 32, ConvBwdSmem<C>::BYTES, st>>>(obs, orps, gather, params, P, L, dy1, xh1, rs1,
                                                                       part, rows);
  const int n = 9 * C * CONV_O + 3 * CONV_O;
  if (final_slices((int)grid.x) == 32)
    conv_bwd_final_kernel<32><<<dim3(cdiv(n, 8), grid.y), 256, 0, st>>>(part, (int)grid.x, 9 * C * CONV_O, grads, P, L);
  else
    conv_bwd_final_kernel<8><<<dim3(cdiv(n, 32), grid.y), 256, 0, st>>>(part, (int)grid.x, 9 * C * CONV_O, grads, P, L);
  return 0;
}

// the fp16 variant (conv path 1); gs = power-of-two scale of dz before the fp16 split
template <int C>
static int launch_conv_bwd_mma16(dim3 grid, cudaStream_t st, const uint32_t* obs, int64_t orps, const int32_t* gather,
                                 const float* params, int64_t P, const pqn_net_layout_t& L, const float* dy1,
                                 float* grads, float* part, int rows, float gs) {
  auto kfn = conv_bwd_mma16_kernel<C>;
  if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, ConvBwd16<C>::BYTES) != cudaSuccess)
    return check_launch("conv_bwd_mma16(cudaFuncSetAttribute)");
  kfn<<<grid, ConvBwd16<C>::WARPS * 32, ConvBwd16<C>::BYTES, st>>>(obs, orps, gather, params, P, L, dy1, part, rows, gs);
  const int n = 9 * C * CONV_O + 3 * CONV_O;
  if (final_slices((int)grid.x) == 32)
    conv_bwd_final_kernel<32><<<dim3(cdiv(n, 8), grid.y), 256, 0, st>>>(part, (int)grid.x, 9 * C * CONV_O, grads, P, L);
  else
    conv_bwd_final_kernel<8><<<dim3(cdiv(n, 32), grid.y), 256, 0, st>>>(part, (int)grid.x, 9 * C * CONV_O, grads, P, L);
  return 0;
}

// dynamic shared memory of row_bwd_kernel<N, HEAD> (floats: eight warp-private [3N] reduction slices; HEAD: [A][N]
// weights, eight warp-private [A][N] gradient slices, [8][A] + [8][2] scalars)
static size_t row_bwd_smem(int N, int A, bool head) {
  return (size_t)(24 * N + (head ? A * N + 8 * A + 16 + 8 * A * N : 0)) * sizeof(float);
}
static int64_t row_bwd_part_floats(int N, int A) { return 3 * (int64_t)N + (int64_t)A * N + A + 2; }

template <int N, bool HEAD, typename... Args>
static int launch_row_bwd(dim3 grid, int A, cudaStream_t st, Args... args) {
  const size_t sm = row_bwd_smem(N, A, HEAD);
  if (sm > 48 * 1024 &&
      cudaFuncSetAttribute(row_bwd_kernel<N, HEAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm) != cudaSuccess)
    return check_launch("row_bwd(cudaFuncSetAttribute)");
  LaunchScope _ls(K_ROW_BWD, st);
  row_bwd_kernel<N, HEAD><<<grid, 256, sm, st>>>(args...);
  return 0;
}
static void launch_row_bwd_final(const float* part, dim3 rbg, int N, int A, bool head, float* grads, int64_t P,
                                 int64_t off_dscale, int64_t off_dbias, int64_t off_db, int64_t off_hw, int64_t off_hb,
                                 float* loss_sum, float* qsa_sum, cudaStream_t st) {
  const int stride = 3 * N + (head ? A * N + A + 2 : 0);
  LaunchScope _ls(K_GRAD_FINAL, st);
  if (final_slices((int)rbg.x) == 32)
    row_bwd_final_kernel<32><<<dim3(cdiv(stride, 8), rbg.y), 256, 0, st>>>(part, (int)rbg.x, N, A, head ? 1 : 0, grads, P, off_dscale,
                                                                           off_dbias, off_db, off_hw, off_hb, loss_sum, qsa_sum);
  else
    row_bwd_final_kernel<8><<<dim3(cdiv(stride, 32), rbg.y), 256, 0, st>>>(part, (int)rbg.x, N, A, head ? 1 : 0, grads, P, off_dscale,
                                                                           off_dbias, off_db, off_hw, off_hb, loss_sum, qsa_sum);
}

// row_bwd + its fixed-order finalize.  off_scale = LayerNorm scale of this layer (also where d scale goes), off_bias its
// bias slot, off_db the bias of the dense layer before it.
static int run_row_bwd(int N, bool head, dim3 rbg, int A, cudaStream_t st, const float* Hh, const float* XHAT,
                       const float* RSTD, const float* DH, float* DZ, float* DZLO, __half* DZ16H, __half* DZ16L,
                       float gscale, const float* params, float* grads, int64_t P, int64_t off_scale, int64_t off_bias,
                       int64_t off_db, int64_t off_hw, int64_t off_hb, const int32_t* gather, const int32_t* action,
                       const float* target, int64_t trps, float* loss_sum, float* qsa_sum, float* part, int rows) {
  int rc = 0;
#define PQN_RB(NN, HH)                                                                                              \
  rc = launch_row_bwd<NN, HH>(rbg, A, st, Hh, XHAT, RSTD, DH, DZ, DZLO, DZ16H, DZ16L, gscale, params, grads, P,     \
                              off_scale, off_scale, off_bias, off_db, off_hw, off_hb, A, gather, action, target, trps, \
                              part, rows)
  if (N == 64 && head) PQN_RB(64, true);
  else if (N == 64) PQN_RB(64, false);
  else if (N == 128 && head) PQN_RB(128, true);
  else if (N == 128) PQN_RB(128, false);
  else if (N == 256 && head) PQN_RB(256, true);
  else if (N == 256) PQN_RB(256, false);
  else if (N == 512 && head) PQN_RB(512, true);
  else if (N == 512) PQN_RB(512, false);
  else return set_error(PQN_E_UNSUPPORTED, "row_bwd width %d", N);
#undef PQN_RB
  if (rc) return rc;
  launch_row_bwd_final(part, rbg, N, A, head, grads, P, off_scale, off_bias, off_db, off_hw, off_hb, loss_sum, qsa_sum, st);
  return 0;
}

// CTAs per seed for the warp-per-sample conv kernels (grid = per_seed x S).  `resident` = CTAs the GPU holds at once
// (SMs x CTAs/SM): the grid is sized to fill whole waves of that many CTAs -- 1280 CTAs on 296 slots would run a
// fifth, 32%-full wave -- while staying near 4 waves so that per-CTA setup (weight fragments) stays amortised.
static unsigned conv_mma_ctas(int S, int rows, int ctas_per_sm) {
  const int sms = device_sm_count();
  const int resident = sms * ctas_per_sm;
  const int maxc = (rows + CONV_MMA_WARPS - 1) / CONV_MMA_WARPS;
  int best = 1;
  double best_eff = 0.0;
  const int lim = (6 * resident + S - 1) / S;
  for (int per_seed = 1; per_seed <= lim && per_seed <= maxc; ++per_seed) {
    const int total = per_seed * S;
    const int waves = (total + resident - 1) / resident;
    if (waves > 6) break;
    const double eff = (double)total / ((double)waves * resident);
    if (eff > best_eff + 0.01 || (eff > best_eff - 0.01 && waves <= 4)) { best_eff = eff > best_eff ? eff : best_eff; best = per_seed; }
  }
  return (unsigned)best;
}

template <bool TRAIN>
static int launch_conv_fwd(int C, dim3 grid, cudaStream_t st, const uint32_t* obs, int64_t orps, const int32_t* gather,
                           const float* params, int64_t P, const pqn_net_layout_t& L, float* h1, float* h1lo, float* bn,
                           int rows, float* xh1 = nullptr, float* rs1 = nullptr, uint32_t* rb = nullptr,
                           bool h16 = false) {
  if (g_conv_mma == 1) {  // fp16 mma.sync conv (default); h16: h1 / h1lo are the fp16 (hi, lo') planes
    const dim3 mg(conv_mma_ctas((int)grid.y, rows, CONV16_CTAS_PER_SM), grid.y);
    LaunchScope _ls(TRAIN ? K_CONV_FWD : K_CONV_FWD_INFER, st);
#define PQN_CONV16(CC)                                                                                              \
  if (h16) conv_fwd_mma16_kernel<CC, TRAIN, true><<<mg, CONV16_WARPS * 32, 0, st>>>(obs, orps, gather, params, P, L, h1, h1lo, rb, bn, rows); \
  else conv_fwd_mma16_kernel<CC, TRAIN, false><<<mg, CONV16_WARPS * 32, 0, st>>>(obs, orps, gather, params, P, L, h1, h1lo, rb, bn, rows)
    switch (C) {
      case 4: PQN_CONV16(4); break;
      case 6: PQN_CONV16(6); break;
      case 7: PQN_CONV16(7); break;
      case 10: PQN_CONV16(10); break;
      default: return -1;
    }
#undef PQN_CONV16
    return 0;
  }
  if (g_conv_mma == 3) {  // the round-1 tf32 mma.sync conv (kept as an A/B reference)
    const dim3 mg(conv_mma_ctas((int)grid.y, rows, 3), grid.y);
    LaunchScope _ls(TRAIN ? K_CONV_FWD : K_CONV_FWD_INFER, st);
    switch (C) {
      case 4: conv_fwd_mma_kernel<4, TRAIN><<<mg, CONV_MMA_WARPS * 32, 0, st>>>(obs, orps, gather, params, P, L, h1, h1lo, xh1, rs1, rb, bn, rows); break;
      case 6: conv_fwd_mma_kernel<6, TRAIN><<<mg, CONV_MMA_WARPS * 32, 0, st>>>(obs, orps, gather, params, P, L, h1, h1lo, xh1, rs1, rb, bn, rows); break;
      case 7: conv_fwd_mma_kernel<7, TRAIN><<<mg, CONV_MMA_WARPS * 32, 0, st>>>(obs, orps, gather, params, P, L, h1, h1lo, xh1, rs1, rb, bn, rows); break;
      case 10: conv_fwd_mma_kernel<10, TRAIN><<<mg, CONV_MMA_WARPS * 32, 0, st>>>(obs, orps, gather, params, P, L, h1, h1lo, xh1, rs1, rb, bn, rows); break;
      default: return -1;
    }
    return 0;
  }
  switch (C) {
    case 4: { LaunchScope _ls(TRAIN ? K_CONV_FWD : K_CONV_FWD_INFER, st); conv_fwd_kernel<4, TRAIN><<<grid, 256, 0, st>>>(obs, orps, gather, params, P, L, h1, h1lo, bn, rows); } break;
    case 6: { LaunchScope _ls(TRAIN ? K_CONV_FWD : K_CONV_FWD_INFER, st); conv_fwd_kernel<6, TRAIN><<<grid, 256, 0, st>>>(obs, orps, gather, params, P, L, h1, h1lo, bn, rows); } break;
    case 7: { LaunchScope _ls(TRAIN ? K_CONV_FWD : K_CONV_FWD_INFER, st); conv_fwd_kernel<7, TRAIN><<<grid, 256, 0, st>>>(obs, orps, gather, params, P, L, h1, h1lo, bn, rows); } break;
    case 10: { LaunchScope _ls(TRAIN ? K_CONV_FWD : K_CONV_FWD_INFER, st); conv_fwd_kernel<10, TRAIN><<<grid, 256, 0, st>>>(obs, orps, gather, params, P, L, h1, h1lo, bn, rows); } break;
    default: return -1;
  }
  return 0;
}

// CTAs per seed for conv_bwd: ~4 waves of 2 CTAs/SM over all seeds, at most one sample-group per CTA
static unsigned conv_bwd_ctas(int S, int rows) {
  int per_seed = (device_sm_count() * 2 * 4 + S - 1) / S;
  const int maxc = (rows + CONV_BWD_WARPS - 1) / CONV_BWD_WARPS;
  if (per_seed > maxc) per_seed = maxc;
  if (per_seed < 1) per_seed = 1;
  return (unsigned)per_seed;
}

static int wgrad_splits(int tiles, int S, int rows) {
  int s = (2 * device_sm_count() + tiles * S - 1) / (tiles * S);
  const int maxs = (rows + 255) / 256;
  if (s > maxs) s = maxs;
  if (s < 1) s = 1;
  return s;
}

// lo = x - trunc_tf32(x) for the per-seed weight block W1 (source rows at stride P)
__global__ void split_lo_strided_kernel(const float* __restrict__ src, int64_t src_seed_stride, float* __restrict__ lo,
                                        int64_t n_per_seed) {
  const int seed = blockIdx.y;
  const int64_t i4 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 * 4 >= n_per_seed) return;
  const float4 v = __ldg(reinterpret_cast<const float4*>(src + (int64_t)seed * src_seed_stride) + i4);
  reinterpret_cast<float4*>(lo + (int64_t)seed * n_per_seed)[i4] =
      make_float4(tc::tf32_lo(v.x), tc::tf32_lo(v.y), tc::tf32_lo(v.z), tc::tf32_lo(v.w));
}

static void launch_split_w1(const float* params, int64_t P, int64_t off_w, float* w1_lo, int S, cudaStream_t st) {
  const int64_t n = (int64_t)FLAT_CNN * HID_CNN;
  LaunchScope _ls(K_TC_SPLIT, st);
  split_lo_strided_kernel<<<dim3(cdiv(n / 4, 256), S), 256, 0, st>>>(params + off_w, P, w1_lo, n);
}

// ---- fp16-split tensor-core path (g_use_tc == 2) ------------------------------------------------------------------
// planes inside the workspace (no extra memory: they alias the fp32 "lo" tensors of the tf32 path, same byte size):
//   h1 planes  : w.h1_lo  region  -> __half hi[R][1024], lo'[R][1024]
//   dz2 planes : w.dz2_lo region  -> __half hi[R][128],  lo'[R][128]      (dz2 * gscale)
//   W1 planes  : w.w1_lo  region  -> __half hi[S][1024][128], lo'[S][1024][128]
struct Planes16 { __half *h1_hi, *h1_lo, *dz_hi, *dz_lo, *w1_hi, *w1_lo; };
static Planes16 planes16(const Workspace& w, int S, int64_t rows) {
  const int64_t R = (int64_t)S * rows;
  Planes16 p;
  p.h1_hi = reinterpret_cast<__half*>(w.h1_lo); p.h1_lo = p.h1_hi + R * FLAT_CNN;
  p.dz_hi = reinterpret_cast<__half*>(w.dz2_lo); p.dz_lo = p.dz_hi + R * HID_CNN;
  p.w1_hi = reinterpret_cast<__half*>(w.w1_lo); p.w1_lo = p.w1_hi + (int64_t)S * FLAT_CNN * HID_CNN;
  return p;
}
// dz2 is pre-scaled by a power of two so that gradient-sized values (|dz2| ~ |diff| / rows) sit in the middle of the
// fp16 range: gscale = 16 * 2^ceil(log2(rows)); the GEMM epilogues multiply by 1 / gscale (exact).
static float grad_scale(int64_t rows) {
  float s = 16.f;
  while (rows > 1) { s *= 2.f; rows = (rows + 1) >> 1; }
  return s;
}

__global__ void split16_strided_kernel(const float* __restrict__ src, int64_t src_seed_stride, __half* __restrict__ hi,
                                       __half* __restrict__ lo, int64_t n_per_seed) {
  const int seed = blockIdx.y;
  const int64_t i4 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 * 4 >= n_per_seed) return;
  const float4 v = __ldg(reinterpret_cast<const float4*>(src + (int64_t)seed * src_seed_stride) + i4);
  __half2 h0, h1, l0, l1;
  tc::split16x2(v.x, v.y, h0, l0);
  tc::split16x2(v.z, v.w, h1, l1);
  reinterpret_cast<uint2*>(hi + (int64_t)seed * n_per_seed)[i4] =
      make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
  reinterpret_cast<uint2*>(lo + (int64_t)seed * n_per_seed)[i4] =
      make_uint2(*reinterpret_cast<uint32_t*>(&l0), *reinterpret_cast<uint32_t*>(&l1));
}

static void launch_split16_w1(const float* params, int64_t P, int64_t off_w, const Planes16& pl, int S, cudaStream_t st) {
  const int64_t n = (int64_t)FLAT_CNN * HID_CNN;
  LaunchScope _ls(K_TC_SPLIT, st);
  split16_strided_kernel<<<dim3(cdiv(n / 4, 256), S), 256, 0, st>>>(params + off_w, P, pl.w1_hi, pl.w1_lo, n);
}
// fp32 h1 (conv paths that do not write planes themselves) -> planes
static void launch_split16_h1(const float* h1, const Planes16& pl, int64_t n, cudaStream_t st) {
  LaunchScope _ls(K_TC_SPLIT, st);
  split16_strided_kernel<<<dim3(cdiv(n / 4, 256), 1), 256, 0, st>>>(h1, 0, pl.h1_hi, pl.h1_lo, n);
}

static int tc16_dense_fwd(int epi, const float* params, int64_t P, const pqn_net_layout_t& L, const Workspace& w,
                          const Planes16& pl, int A, float* q, int S, int rows, cudaStream_t st) {
  CUtensorMap t[4];
  int rc;
  if ((rc = tc::make_tmap16(&t[0], pl.h1_hi, FLAT_CNN, rows, S, FLAT_CNN, (uint64_t)rows * FLAT_CNN, 128))) return rc;
  if ((rc = tc::make_tmap16(&t[1], pl.h1_lo, FLAT_CNN, rows, S, FLAT_CNN, (uint64_t)rows * FLAT_CNN, 128))) return rc;
  if ((rc = tc::make_tmap16(&t[2], pl.w1_hi, HID_CNN, FLAT_CNN, S, HID_CNN, (uint64_t)FLAT_CNN * HID_CNN, 64))) return rc;
  if ((rc = tc::make_tmap16(&t[3], pl.w1_lo, HID_CNN, FLAT_CNN, S, HID_CNN, (uint64_t)FLAT_CNN * HID_CNN, 64))) return rc;
  tc::GemmShape gs = {};
  gs.S = S; gs.M = rows; gs.m_tiles = (rows + 127) / 128; gs.n_tiles = 1; gs.k_blocks = FLAT_CNN / tc::TC_BK16;
  tc::EpiParams ep = {};
  ep.params = params; ep.P = P; ep.off_b = L.d0_b; ep.off_scale = L.ln1_scale; ep.off_bias = L.ln1_bias;
  ep.off_hw = L.head_w; ep.off_hb = L.head_b; ep.A = A; ep.rows = rows;
  ep.H = w.h2; ep.XHAT = w.xhat2; ep.RSTD = w.rstd2; ep.Q = q;
  return tc::launch_gemm16(0, 1, epi, t, gs, ep, st, epi == tc::EPI_LN_HEAD ? K_TC_FWD_HEAD : K_TC_FWD);
}

// the same product and Q-head epilogue with H1 computed in the GEMM from the packed observations (tc_conv_gemm_kernel):
// the h1 planes are neither written nor read
static int tc16_conv_dense_fwd(int epi, int C, const uint32_t* obs, int64_t obs_rows_per_seed, const int32_t* gather,
                               const float* params, int64_t P, const pqn_net_layout_t& L, const Workspace& w,
                               const Planes16& pl, int A, float* q, int S, int rows, cudaStream_t st) {
  CUtensorMap t[2];
  int rc;
  if ((rc = tc::make_tmap16(&t[0], pl.w1_hi, HID_CNN, FLAT_CNN, S, HID_CNN, (uint64_t)FLAT_CNN * HID_CNN, 64))) return rc;
  if ((rc = tc::make_tmap16(&t[1], pl.w1_lo, HID_CNN, FLAT_CNN, S, HID_CNN, (uint64_t)FLAT_CNN * HID_CNN, 64))) return rc;
  tc::GemmShape gs = {};
  gs.S = S; gs.M = rows; gs.m_tiles = (rows + 127) / 128; gs.n_tiles = 1; gs.k_blocks = FLAT_CNN / tc::TC_BK16;
  tc::EpiParams ep = {};
  ep.params = params; ep.P = P; ep.off_b = L.d0_b; ep.off_scale = L.ln1_scale; ep.off_bias = L.ln1_bias;
  ep.off_hw = L.head_w; ep.off_hb = L.head_b; ep.A = A; ep.rows = rows;
  ep.H = w.h2; ep.XHAT = w.xhat2; ep.RSTD = w.rstd2; ep.Q = q;
  tc::ConvIn ci;
  ci.obs = obs; ci.obs_rows_per_seed = obs_rows_per_seed; ci.gather = gather; ci.L = L;
  return tc::launch_conv_gemm16(C, epi, t, gs, ep, ci, st, epi == tc::EPI_LN_HEAD ? K_TC_FWD_HEAD : K_TC_FWD);
}

static int tc16_wgrad(float* grads, int64_t P, const pqn_net_layout_t& L, const Planes16& pl, int S, int rows,
                      float gscale, float* wg_part, cudaStream_t st) {
  CUtensorMap t[4];
  int rc;
  if ((rc = tc::make_tmap16(&t[0], pl.h1_hi, FLAT_CNN, rows, S, FLAT_CNN, (uint64_t)rows * FLAT_CNN, 64))) return rc;
  if ((rc = tc::make_tmap16(&t[1], pl.h1_lo, FLAT_CNN, rows, S, FLAT_CNN, (uint64_t)rows * FLAT_CNN, 64))) return rc;
  if ((rc = tc::make_tmap16(&t[2], pl.dz_hi, HID_CNN, rows, S, HID_CNN, (uint64_t)rows * HID_CNN, 64))) return rc;
  if ((rc = tc::make_tmap16(&t[3], pl.dz_lo, HID_CNN, rows, S, HID_CNN, (uint64_t)rows * HID_CNN, 64))) return rc;
  tc::GemmShape gs = {};
  gs.S = S; gs.M = FLAT_CNN; gs.m_tiles = FLAT_CNN / 128; gs.n_tiles = 1;
  gs.k_blocks = (rows + tc::TC_BK16 - 1) / tc::TC_BK16;
  gs.k_split = wgrad_ksplit(S * gs.m_tiles * gs.n_tiles, gs.k_blocks);
  tc::EpiParams ep = {};
  ep.ld_out = HID_CNN; ep.out_scale = 1.0f / gscale;
  const int64_t n = (int64_t)FLAT_CNN * HID_CNN;
  if (gs.k_split > 1) { ep.out = wg_part; ep.out_seed_stride = n; ep.split_stride = (int64_t)S * n; }
  else { ep.out = grads + L.d0_w; ep.out_seed_stride = P; }
  if ((rc = tc::launch_gemm16(1, 1, tc::EPI_STORE, t, gs, ep, st, K_TC_WGRAD))) return rc;
  if (gs.k_split > 1) {
    launch_split_reduce(wg_part, gs.k_split, (int64_t)S * n, n, S, grads + L.d0_w, P, st);
  }
  return 0;
}

// dY1 = relu_mask * (dZ2 . W1^T) into w.h1 (fp32; the fp16 path has no fp32 h1, so this is not in place unless the
// mask itself is the fp32 h1 of a conv path that wrote one)
static int tc16_dgrad(const Workspace& w, const Planes16& pl, int S, int rows, bool have_bits, float gscale,
                      cudaStream_t st) {
  CUtensorMap t[4];
  int rc;
  if ((rc = tc::make_tmap16(&t[0], pl.dz_hi, HID_CNN, rows, S, HID_CNN, (uint64_t)rows * HID_CNN, 128))) return rc;
  if ((rc = tc::make_tmap16(&t[1], pl.dz_lo, HID_CNN, rows, S, HID_CNN, (uint64_t)rows * HID_CNN, 128))) return rc;
  if ((rc = tc::make_tmap16(&t[2], pl.w1_hi, HID_CNN, FLAT_CNN, S, HID_CNN, (uint64_t)FLAT_CNN * HID_CNN, 128))) return rc;
  if ((rc = tc::make_tmap16(&t[3], pl.w1_lo, HID_CNN, FLAT_CNN, S, HID_CNN, (uint64_t)FLAT_CNN * HID_CNN, 128))) return rc;
  tc::GemmShape gs = {};
  gs.S = S; gs.M = rows; gs.m_tiles = (rows + 127) / 128; gs.n_tiles = FLAT_CNN / 128; gs.k_blocks = HID_CNN / tc::TC_BK16;
 
  tc::EpiParams ep = {};
  ep.out = w.h1; ep.mask = w.h1; ep.ld_out = FLAT_CNN; ep.out_seed_stride = (int64_t)rows * FLAT_CNN;
  ep.relu_bits = w.relu_bits; ep.rows = rows; ep.out_scale = 1.0f / gscale;
  return tc::launch_gemm16(0, 0, have_bits ? tc::EPI_RELU_BITS : tc::EPI_RELU_MASK, t, gs, ep, st, K_TC_DGRAD);
}

// ---- generic fp16-split GEMMs on planes (hi at p, lo' at p + plane_elems), used by the MLP hidden layer --------------
// out[S][rows][N] = A[S][rows][K] . B[S][K][N]          (A K-major, B MN-major; raw store, no bias)
static int tc16_mm_store(const __half* a, int64_t a_plane, const __half* b, int64_t b_plane, float* out, int S, int rows, int K,
                         int N, cudaStream_t st, int kid) {
  CUtensorMap t[4];
  int rc;
  if ((rc = tc::make_tmap16(&t[0], a, K, rows, S, K, (uint64_t)rows * K, 128))) return rc;
  if ((rc = tc::make_tmap16(&t[1], a + a_plane, K, rows, S, K, (uint64_t)rows * K, 128))) return rc;
  if ((rc = tc::make_tmap16(&t[2], b, N, K, S, N, (uint64_t)K * N, 64))) return rc;
  if ((rc = tc::make_tmap16(&t[3], b + b_plane, N, K, S, N, (uint64_t)K * N, 64))) return rc;
  tc::GemmShape gs = {};
  gs.S = S; gs.M = rows; gs.m_tiles = (rows + 127) / 128; gs.n_tiles = N / 128; gs.k_blocks = (K + tc::TC_BK16 - 1) / tc::TC_BK16;
 
  tc::EpiParams ep = {};
  ep.out = out; ep.ld_out = N; ep.out_seed_stride = (int64_t)rows * N;
  return tc::launch_gemm16(0, 1, tc::EPI_STORE, t, gs, ep, st, kid);
}
// dW[S(P)][M][N] = A[S][rows][M]^T . DZ[S][rows][N] * out_scale      (both operands MN-major, K = rows)
static int tc16_mm_wgrad(const __half* a, int64_t a_plane, const __half* dz, int64_t dz_plane, float* out, int64_t out_seed_stride,
                         int S, int rows, int M, int N, float out_scale, float* wg_part, cudaStream_t st) {
  CUtensorMap t[4];
  int rc;
  if ((rc = tc::make_tmap16(&t[0], a, M, rows, S, M, (uint64_t)rows * M, 64))) return rc;
  if ((rc = tc::make_tmap16(&t[1], a + a_plane, M, rows, S, M, (uint64_t)rows * M, 64))) return rc;
  if ((rc = tc::make_tmap16(&t[2], dz, N, rows, S, N, (uint64_t)rows * N, 64))) return rc;
  if ((rc = tc::make_tmap16(&t[3], dz + dz_plane, N, rows, S, N, (uint64_t)rows * N, 64))) return rc;
  tc::GemmShape gs = {};
  gs.S = S; gs.M = M; gs.m_tiles = M / 128; gs.n_tiles = N / 128; gs.k_blocks = (rows + tc::TC_BK16 - 1) / tc::TC_BK16;
  gs.k_split = wgrad_ksplit(S * gs.m_tiles * gs.n_tiles, gs.k_blocks);
  tc::EpiParams ep = {};
  ep.ld_out = N; ep.out_scale = out_scale;
  const int64_t n = (int64_t)M * N;
  if (gs.k_split > 1) { ep.out = wg_part; ep.out_seed_stride = n; ep.split_stride = (int64_t)S * n; }
  else { ep.out = out; ep.out_seed_stride = out_seed_stride; }
  if ((rc = tc::launch_gemm16(1, 1, tc::EPI_STORE, t, gs, ep, st, K_TC_WGRAD))) return rc;
  if (gs.k_split > 1) {
    launch_split_reduce(wg_part, gs.k_split, (int64_t)S * n, n, S, out, out_seed_stride, st);
  }
  return 0;
}
// out[S][rows][Kp] = (mask > 0) * (DZ[S][rows][N] . W[S][Kp][N]^T) * out_scale       (both K-major, K = N)
static int tc16_mm_dgrad(const __half* dz, int64_t dz_plane, const __half* wgt, int64_t w_plane, const float* mask, float* out,
                         int S, int rows, int N, int Kp, float out_scale, cudaStream_t st) {
  CUtensorMap t[4];
  int rc;
  if ((rc = tc::make_tmap16(&t[0], dz, N, rows, S, N, (uint64_t)rows * N, 128))) return rc;
  if ((rc = tc::make_tmap16(&t[1], dz + dz_plane, N, rows, S, N, (uint64_t)rows * N, 128))) return rc;
  if ((rc = tc::make_tmap16(&t[2], wgt, N, Kp, S, N, (uint64_t)Kp * N, 128))) return rc;
  if ((rc = tc::make_tmap16(&t[3], wgt + w_plane, N, Kp, S, N, (uint64_t)Kp * N, 128))) return rc;
  tc::GemmShape gs = {};
  gs.S = S; gs.M = rows; gs.m_tiles = (rows + 127) / 128; gs.n_tiles = Kp / 128; gs.k_blocks = (N + tc::TC_BK16 - 1) / tc::TC_BK16;
 
  tc::EpiParams ep = {};
  ep.out = out; ep.mask = mask; ep.ld_out = Kp; ep.out_seed_stride = (int64_t)rows * Kp; ep.rows = rows; ep.out_scale = out_scale;
  return tc::launch_gemm16(0, 0, tc::EPI_RELU_MASK, t, gs, ep, st, K_TC_DGRAD);
}
static void split16_rows(const float* src, int64_t src_seed_stride, int64_t n_per_seed, int S, __half* hi, __half* lo,
                         cudaStream_t st) {
  LaunchScope _ls(K_TC_SPLIT, st);
  split16_strided_kernel<<<dim3(cdiv(n_per_seed / 4, 256), S), 256, 0, st>>>(src, src_seed_stride, hi, lo, n_per_seed);
}

// ---- 3xTF32 tensor-core path (g_use_tc == 1): mma.sync.tf32 on the TMA ring of the GEMM kernel -------------------
// Z = H1 . W1 with the LayerNorm/ReLU(/head) epilogue.  epi = EPI_LN_TRAIN or EPI_LN_HEAD.
static int tc_dense_fwd(int epi, const float* params, int64_t P, const pqn_net_layout_t& L, const Workspace& w, int A,
                        float* q, int S, int rows, cudaStream_t st) {
  CUtensorMap t[4];
  int rc;
  if ((rc = tc::make_tmap(&t[0], w.h1, FLAT_CNN, rows, S, FLAT_CNN, (uint64_t)rows * FLAT_CNN, 128))) return rc;
  if ((rc = tc::make_tmap(&t[1], w.h1_lo, FLAT_CNN, rows, S, FLAT_CNN, (uint64_t)rows * FLAT_CNN, 128))) return rc;
  if ((rc = tc::make_tmap(&t[2], params + L.d0_w, HID_CNN, FLAT_CNN, S, HID_CNN, (uint64_t)P, 32))) return rc;
  if ((rc = tc::make_tmap(&t[3], w.w1_lo, HID_CNN, FLAT_CNN, S, HID_CNN, (uint64_t)FLAT_CNN * HID_CNN, 32))) return rc;
  tc::GemmShape gs = {};
  gs.S = S; gs.M = rows; gs.m_tiles = (rows + 127) / 128; gs.n_tiles = 1; gs.k_blocks = FLAT_CNN / tc::TC_BK; gs.split3 = 2;
  tc::EpiParams ep = {};
  ep.params = params; ep.P = P; ep.off_b = L.d0_b; ep.off_scale = L.ln1_scale; ep.off_bias = L.ln1_bias;
  ep.off_hw = L.head_w; ep.off_hb = L.head_b; ep.A = A; ep.rows = rows;
  ep.H = w.h2; ep.XHAT = w.xhat2; ep.RSTD = w.rstd2; ep.Q = q;
  return tc::launch_gemm(0, 1, epi, t, gs, ep, st, epi == tc::EPI_LN_HEAD ? K_TC_FWD_HEAD : K_TC_FWD);
}

// dW1 = H1^T . dZ2  -> grads[d0_w]
static int tc_wgrad(float* grads, int64_t P, const pqn_net_layout_t& L, const Workspace& w, int S, int rows,
                    cudaStream_t st) {
  CUtensorMap t[4];
  int rc;
  if ((rc = tc::make_tmap(&t[0], w.h1, FLAT_CNN, rows, S, FLAT_CNN, (uint64_t)rows * FLAT_CNN, 32))) return rc;
  if ((rc = tc::make_tmap(&t[1], w.h1_lo, FLAT_CNN, rows, S, FLAT_CNN, (uint64_t)rows * FLAT_CNN, 32))) return rc;
  if ((rc = tc::make_tmap(&t[2], w.dz2, HID_CNN, rows, S, HID_CNN, (uint64_t)rows * HID_CNN, 32))) return rc;
  if ((rc = tc::make_tmap(&t[3], w.dz2_lo, HID_CNN, rows, S, HID_CNN, (uint64_t)rows * HID_CNN, 32))) return rc;
  tc::GemmShape gs = {};
  gs.S = S; gs.M = FLAT_CNN; gs.m_tiles = FLAT_CNN / 128; gs.n_tiles = 1; gs.k_blocks = (rows + tc::TC_BK - 1) / tc::TC_BK;
  gs.split3 = 2;
  tc::EpiParams ep = {};
  ep.out = grads + L.d0_w; ep.ld_out = HID_CNN; ep.out_seed_stride = P;
  return tc::launch_gemm(1, 1, tc::EPI_STORE, t, gs, ep, st, K_TC_WGRAD);
}

// dY1 = relu_mask(H1) * (dZ2 . W1^T), written in place over H1
static int tc_dgrad(const float* params, int64_t P, const pqn_net_layout_t& L, const Workspace& w, int S, int rows,
                    bool have_bits, cudaStream_t st) {
  CUtensorMap t[4];
  int rc;
  if ((rc = tc::make_tmap(&t[0], w.dz2, HID_CNN, rows, S, HID_CNN, (uint64_t)rows * HID_CNN, 128))) return rc;
  if ((rc = tc::make_tmap(&t[1], w.dz2_lo, HID_CNN, rows, S, HID_CNN, (uint64_t)rows * HID_CNN, 128))) return rc;
  if ((rc = tc::make_tmap(&t[2], params + L.d0_w, HID_CNN, FLAT_CNN, S, HID_CNN, (uint64_t)P, 128))) return rc;
  if ((rc = tc::make_tmap(&t[3], w.w1_lo, HID_CNN, FLAT_CNN, S, HID_CNN, (uint64_t)FLAT_CNN * HID_CNN, 128))) return rc;
  tc::GemmShape gs = {};
  gs.S = S; gs.M = rows; gs.m_tiles = (rows + 127) / 128; gs.n_tiles = FLAT_CNN / 128; gs.k_blocks = HID_CNN / tc::TC_BK;
  gs.split3 = 1;   // A_lo = dz2_lo, written by row_bwd
  tc::EpiParams ep = {};
  ep.out = w.h1; ep.mask = w.h1; ep.ld_out = FLAT_CNN; ep.out_seed_stride = (int64_t)rows * FLAT_CNN;
  ep.relu_bits = w.relu_bits; ep.rows = rows;
  // the packed mask (16 B per row and tile) replaces re-reading the 2 GB of activations it was derived from
  return tc::launch_gemm(0, 0, have_bits ? tc::EPI_RELU_BITS : tc::EPI_RELU_MASK, t, gs, ep, st, K_TC_DGRAD);
}

#include "pqn_norm.cuh"

// Dense -> LayerNorm -> ReLU (MODE 0: h; MODE 1: h, xhat, rstd) or Dense -> LayerNorm -> ReLU -> Q head (MODE 2) on the
// FFMA kernels, at every built width.  Up to 256 columns this is dense_fwd_kernel with the fused epilogue.  A 512-wide
// row does not fit its register tile, so the raw product (MODE 3, two 256-column tiles) goes to H and ln_fwd_kernel<512>
// normalises it in place (MODE 2: H is scratch, head_fwd_kernel adds the head).
template <int MODE>
static int dense_ln_fwd(int N, dim3 grid, cudaStream_t st, const float* X, int64_t xss, int ldx, const float* params,
                         int64_t P, const DenseOff& o, int64_t ohw, int64_t ohb, int A, float* H, float* XH, float* RS,
                         float* Q, int rows, int K) {
  if (N != 512)
    return launch_dense<MODE>(N, grid, st, X, xss, ldx, params, P, o.w, o.b, o.g, o.bi, ohw, ohb, A, H, XH, RS, Q, rows, K);
  int rc = launch_dense<3>(N, grid, st, X, xss, ldx, params, P, o.w, o.b, 0, 0, 0, 0, A, H, nullptr, nullptr, nullptr, rows, K);
  if (rc) return rc;
  { LaunchScope _ls(K_DENSE_FWD, st);
    nrm::ln_fwd_kernel<512><<<dim3(cdiv(rows, 8), grid.y), 256, 0, st>>>(H, rows, params, P, o.g, o.bi, MODE == 1 ? XH : nullptr,
                                                                        MODE == 1 ? RS : nullptr, H); }
  if (MODE == 2) {
    LaunchScope _ls(K_DENSE_FWD, st);
    nrm::head_fwd_kernel<<<dim3(cdiv(rows, 8), grid.y), 256, 0, st>>>(H, rows, N, params, P, ohw, ohb, A, Q);
  }
  return 0;
}

#include "pqn_rnn.cuh"

// HH = H (64, 128, 256 or 512) as a constant for the one-thread-per-feature kernels
#define PQN_H_DISPATCH(H_, ...)                                         \
  switch (H_) {                                                         \
    case 64: { constexpr int HH = 64; __VA_ARGS__; } break;             \
    case 128: { constexpr int HH = 128; __VA_ARGS__; } break;           \
    case 256: { constexpr int HH = 256; __VA_ARGS__; } break;           \
    case 512: { constexpr int HH = 512; __VA_ARGS__; } break;           \
    default: return set_error(PQN_E_UNSUPPORTED, "GRU hidden=%d", H_);  \
  }

static inline bool modular_net(const pqn_net_desc_t* d) { return d->norm_type != PQN_NORM_LAYER || d->norm_input != 0; }

// The default MLP's hidden layers l >= 1 (K = N = H) run on the wgmma fp16-split GEMMs from H = 128 up; a 64-wide
// layer would fill half of the GEMM's 128-wide N tile, so H = 64 stays on the FFMA kernels (64-wide N tiles).
static inline bool mlp_hidden_tc(int H) { return g_use_tc == 2 && H >= 128; }
// fp16 (hi, lo') planes of hidden layer l >= 1: its input h_{l-1} ([R][H] each) and its kernel ([S][H][H] each)
static inline __half* mlp_h_planes(const Workspace& w, int64_t R, int H, int l) {
  return reinterpret_cast<__half*>(w.m16_h0) + (int64_t)(l - 1) * 2 * R * H;
}
static inline __half* mlp_w_planes(const Workspace& w, int S, int H, int l) {
  return reinterpret_cast<__half*>(w.m16_w) + (int64_t)(l - 1) * 2 * S * H * H;
}
// Z = h_{l-1} . W_l on wgmma (planes of both operands written here), then bias + LayerNorm + ReLU in place
static int mlp_hidden_tc_fwd(const Workspace& w, const pqn_net_layout_t& L, const float* params, int64_t P, int H, int l, int S,
                             int rows, float* xhat, float* rstd, int kid, cudaStream_t st) {
  const int64_t R = (int64_t)S * rows;
  const DenseOff o = dense_off(L, H, l);
  __half* hp = mlp_h_planes(w, R, H, l);
  __half* wp = mlp_w_planes(w, S, H, l);
  split16_rows(w.h[l - 1], 0, R * H, 1, hp, hp + R * H, st);
  split16_rows(params + o.w, P, (int64_t)H * H, S, wp, wp + (int64_t)S * H * H, st);
  int rc = tc16_mm_store(hp, R * H, wp, (int64_t)S * H * H, w.h[l], S, rows, H, H, st, kid);
  if (rc) return rc;
  LaunchScope _ls(K_NORM_FWD, st);
  const dim3 g(cdiv(rows, 8), S);
  switch (H) {
    case 128: nrm::ln_fwd_kernel<128><<<g, 256, 0, st>>>(w.h[l], rows, params, P, o.g, o.bi, xhat, rstd, w.h[l], o.b); break;
    case 256: nrm::ln_fwd_kernel<256><<<g, 256, 0, st>>>(w.h[l], rows, params, P, o.g, o.bi, xhat, rstd, w.h[l], o.b); break;
    case 512: nrm::ln_fwd_kernel<512><<<g, 256, 0, st>>>(w.h[l], rows, params, P, o.g, o.bi, xhat, rstd, w.h[l], o.b); break;
    default: return set_error(PQN_E_UNSUPPORTED, "tensor-core hidden layer width %d", H);
  }
  return 0;
}

// Layer 0 of the default MLP on packed bits (PQN_NET_MLP_BITS, tensor-core path 2): w.h[0] = ReLU(LayerNorm(bits . W0 +
// b0)), with xhat / rstd for the backward when given
static int bits_layer0_ln(const pqn_net_desc_t* d, const pqn_net_layout_t& L, const float* params, const uint32_t* obs,
                          int64_t orps, const int32_t* gather, int S, int rows, const Workspace& w, const bits::BitsWs& bw,
                          float* xhat, float* rstd, cudaStream_t st) {
  const int D = d->in_c, H = d->hidden;
  const int64_t P = L.total;
  bits::launch_wfrag(params, P, L.d0_w, nullptr, nullptr, D, H, S, bw.wf, st);
  int rc = bits::launch_fwd(obs, orps, gather, rows, D, H, bw.wf, params + L.d0_b, P, nullptr, w.h[0], S, st);
  if (rc) return rc;
  LaunchScope _ls(K_NORM_FWD, st);
  const dim3 g(cdiv(rows, 8), S);
  switch (H) {
    case 64: nrm::ln_fwd_kernel<64><<<g, 256, 0, st>>>(w.h[0], rows, params, P, L.ln0_scale, L.ln0_bias, xhat, rstd, w.h[0]); break;
    case 128: nrm::ln_fwd_kernel<128><<<g, 256, 0, st>>>(w.h[0], rows, params, P, L.ln0_scale, L.ln0_bias, xhat, rstd, w.h[0]); break;
    case 256: nrm::ln_fwd_kernel<256><<<g, 256, 0, st>>>(w.h[0], rows, params, P, L.ln0_scale, L.ln0_bias, xhat, rstd, w.h[0]); break;
    case 512: nrm::ln_fwd_kernel<512><<<g, 256, 0, st>>>(w.h[0], rows, params, P, L.ln0_scale, L.ln0_bias, xhat, rstd, w.h[0]); break;
    default: return set_error(PQN_E_UNSUPPORTED, "hidden=%d", H);
  }
  return 0;
}

// pqn_rnn_step / pqn_rnn_step_stats after their descriptor checks (batch_stats read-only: train=False)
static int rnn_step(const pqn_net_desc_t* d, const float* params, const float* batch_stats, float* hs, const float* obs,
                    int64_t obs_rows_per_seed, const uint8_t* last_done, const int32_t* last_action, float* q, int32_t S,
                    int32_t E, void* workspace, void* stream, const char* who) {
  int rc;
  if (!params || !hs || !obs || !last_done || !last_action || !q || !workspace || S <= 0 || E <= 0 || S > 65535)
    return set_error(PQN_E_INVALID, "%s: bad argument", who);
  cudaStream_t st = (cudaStream_t)stream;
  pqn_net_layout_t L;
  make_layout(d, &L);
  rnn::RnnWs w;
  rnn::carve_rnn(d, S, E, (char*)workspace, &w);
  if ((rc = rnn::rnn_trunk(d, L, params, const_cast<float*>(batch_stats), obs, obs_rows_per_seed, S, E, false, w, st)))
    return rc;
  if ((rc = rnn::rnn_scan_fwd<false>(d, L, params, last_action, last_done, hs, hs, S, 1, E, w, st))) return rc;
  { LaunchScope _ls(K_RNN_MISC, st);
    nrm::head_fwd_kernel<<<dim3(cdiv(E, 8), S), 256, 0, st>>>(w.y, E, d->hidden, params, L.total, L.head_w, L.head_b,
                                                               d->num_actions, q); }
  return check_launch(who);
}

// pqn_rnn_loss_grad / pqn_rnn_loss_grad_stats after their descriptor checks (batch_stats updated in place)
static int rnn_loss_grad(const pqn_net_desc_t* d, const float* params, float* batch_stats, const float* hs0,
                         const float* obs, const uint8_t* last_done, const int32_t* last_action, const int32_t* action,
                         const float* reward, const uint8_t* done, float* grads, float* loss_sum, float* qsa_sum, int32_t S,
                         int32_t T, int32_t B, SeedScalar gamma, SeedScalar lambda, void* workspace, void* stream,
                         const char* who) {
  int rc;
  if (!params || !hs0 || !obs || !last_done || !last_action || !action || !reward || !done || !grads || !loss_sum ||
      !qsa_sum || !workspace || S <= 0 || T < 2 || B <= 0 || B > 1024 || S > 65535)
    return set_error(PQN_E_INVALID, "%s: bad argument (T >= 2, B <= 1024)", who);
  cudaStream_t st = (cudaStream_t)stream;
  pqn_net_layout_t L;
  make_layout(d, &L);
  const int64_t P = L.total;
  const int H = d->hidden, A = d->num_actions, D = d->in_c, rows = T * B;
  rnn::RnnWs w;
  rnn::carve_rnn(d, S, rows, (char*)workspace, &w);
  if (cudaMemsetAsync(grads, 0, (size_t)S * P * sizeof(float), st) != cudaSuccess)
    return check_launch(who);
  const int64_t gs = (int64_t)S * rows * H;
  // ---- forward over the window
  if ((rc = rnn::rnn_trunk(d, L, params, batch_stats, obs, rows, S, rows, true, w, st))) return rc;
  if ((rc = rnn::rnn_scan_fwd<true>(d, L, params, last_action, last_done, hs0, w.dhl /*scratch carry out*/, S, T, B, w, st)))
    return rc;
  { LaunchScope _ls(K_RNN_MISC, st);
    nrm::head_fwd_kernel<<<dim3(cdiv(rows, 8), S), 256, 0, st>>>(w.y, rows, H, params, P, L.head_w, L.head_b, A, w.q); }
  // ---- targets, loss, dq
  { LaunchScope _ls(K_RNN_MISC, st);
    const int bt = ((B + 31) / 32) * 32;
    rnn::rnn_targets_kernel<<<S, bt, 2 * bt * sizeof(float), st>>>(w.q, action, reward, done, T, B, A, gamma, lambda, w.dq,
                                                                    loss_sum, qsa_sum); }
  // ---- head backward
  { LaunchScope _ls(K_RNN_MISC, st);
    PQN_H_DISPATCH(H, rnn::rnn_head_bwd_kernel<HH><<<dim3(nrm::RED_BLOCKS, S), HH, 0, st>>>(w.y, w.dq, rows, A, params, P, L.head_w, w.dy, w.part)); }
  { LaunchScope _ls(K_RNN_MISC, st);
    rnn::rnn_head_bwd_final_kernel<<<S, 256, 0, st>>>(w.part, nrm::RED_BLOCKS, H, A, grads, P, L.head_w, L.head_b); }
  // ---- BPTT through the GRU
  const int64_t wts = (int64_t)S * H * H;
  { LaunchScope _ls(K_RNN_MISC, st);
    rnn::gru_transpose_kernel<<<dim3(32, S, 3), 256, 0, st>>>(params, P, L, H, w.wt, wts); }
  { LaunchScope _ls(K_RNN_SCAN, st);
    const dim3 grid(cdiv(B, rnn::RB), S);
    PQN_H_DISPATCH(H, rnn::gru_scan_bwd_kernel<HH><<<grid, HH, 0, st>>>(w.dy, last_done, w.h0, w.rg, w.zg, w.ng, w.hn, w.wt, wts, w.da, gs, w.dhn, T, B)); }
  // ---- weight gradients of the GRU (batched over the window)
  const float* xl = w.h[d->layers - 1];   // trunk output = first H columns of the GRU input
  const int64_t iw[3] = {L.gru_ir_w, L.gru_iz_w, L.gru_in_w}, ib[3] = {L.gru_ir_b, L.gru_iz_b, L.gru_in_b};
  const int64_t hw[3] = {L.gru_hr_w, L.gru_hz_w, L.gru_hn_w};
  const int sp = wgrad_splits(ffma_tiles(H, H), S, rows);
  nrm::NormWs nw = {};
  nw.part = w.part;
  for (int g = 0; g < 3; ++g) {
    const float* da = w.da + g * gs;
    run_wgrad_ffma(xl, (int64_t)rows * H, H, da, (int64_t)rows * H, H, grads, P, iw[g], rows, H, S, sp, w.wgp, st);
    nrm::colsum2(da, da, S, rows, H, H, nw, w.sums, grads, P, ib[g], -1, st);                         // d b_ig
    const float* dh = g == 2 ? w.dhn : da;                                                             // hn uses d(hn)
    run_wgrad_ffma(w.h0, (int64_t)rows * H, H, dh, (int64_t)rows * H, H, grads, P, hw[g], rows, H, S, sp, w.wgp, st);
    // d x_L (+)= da_g W_ig[:H]^T, masked by the trunk's ReLU
    launch_dgrad(da, (int64_t)rows * H, H, params, P, iw[g], xl, w.dx, (int64_t)rows * H, rows, H, g > 0 ? 1 : 0, S, st);
  }
  nrm::colsum2(w.dhn, w.dhn, S, rows, H, H, nw, w.sums, grads, P, L.gru_hn_b, -1, st);                 // d b_hn
  { LaunchScope _ls(K_RNN_MISC, st);
    PQN_H_DISPATCH(H, rnn::rnn_onehot_grad_kernel<HH><<<dim3(S, 3), HH, 0, st>>>(w.da, gs, last_action, rows, A, grads, P, L)); }
  if (rnn::modular_rnn(d)) {
    if ((rc = rnn::rnn_trunk_bwd_modular(d, L, params, obs, grads, S, rows, w, st))) return rc;
    return check_launch(who);
  }
  // ---- trunk backward (LayerNorm backward -> weight gradient -> input gradient of the layer below)
  const dim3 rbg(conv_mma_ctas(S, rows, 4), S);
  float* dcur = w.dx;
  for (int l = d->layers - 1; l >= 0; --l) {
    const DenseOff o = dense_off(L, H, l);
    if ((rc = run_row_bwd(H, false, rbg, A, st, nullptr, w.xh[l], w.rs[l], dcur, dcur, nullptr, nullptr, nullptr, 1.0f, params,
                          grads, P, o.g, o.bi, o.b, 0, 0, nullptr, nullptr, nullptr, 0, nullptr, nullptr, w.rbp,
                          rows))) return rc;
    const float* xprev = l == 0 ? obs : w.h[l - 1];
    const int kin = l == 0 ? D : H;
    const int spl = wgrad_splits(ffma_tiles(kin, H), S, rows);
    run_wgrad_ffma(xprev, (int64_t)rows * kin, kin, dcur, (int64_t)rows * H, H, grads, P, o.w, rows, kin, S, spl, w.wgp, st);
    if (l > 0) {
      // dh_{l-1} goes to the buffer dcur does not use (dx and dhl alternate): dgrad reads all of dz_l while it writes
      float* dnext = dcur == w.dhl ? w.dx : w.dhl;
      launch_dgrad(dcur, (int64_t)rows * H, H, params, P, o.w, w.h[l - 1], dnext, (int64_t)rows * H, rows, H, 0, S, st);
      dcur = dnext;
    }
  }
  return check_launch(who);
}

}  // namespace pqn

using namespace pqn;

extern "C" {

int64_t pqn_net_stats_floats(const pqn_net_desc_t* d) {
  if (check_desc(d, "pqn_net_stats_floats")) return -1;
  return nrm::stats_floats(d);
}

int pqn_rnn_step(const pqn_net_desc_t* d, const float* params, float* hs, const float* obs, int64_t obs_rows_per_seed,
                 const uint8_t* last_done, const int32_t* last_action, float* q, int32_t S, int32_t E, void* workspace,
                 void* stream) {
  int rc = check_desc(d, "pqn_rnn_step");
  if (rc) return rc;
  if ((rc = rnn::check_rnn(d, "pqn_rnn_step"))) return rc;
  return rnn_step(d, params, nullptr, hs, obs, obs_rows_per_seed, last_done, last_action, q, S, E, workspace, stream,
                  "pqn_rnn_step");
}

int pqn_rnn_step_stats(const pqn_net_desc_t* d, const float* params, const float* batch_stats, float* hs, const float* obs,
                       int64_t obs_rows_per_seed, const uint8_t* last_done, const int32_t* last_action, float* q, int32_t S,
                       int32_t E, void* workspace, void* stream) {
  int rc = check_desc(d, "pqn_rnn_step_stats");
  if (rc) return rc;
  if ((rc = rnn::check_rnn_stats(d, batch_stats, "pqn_rnn_step_stats"))) return rc;
  return rnn_step(d, params, batch_stats, hs, obs, obs_rows_per_seed, last_done, last_action, q, S, E, workspace, stream,
                  "pqn_rnn_step_stats");
}

int pqn_rnn_loss_grad(const pqn_net_desc_t* d, const float* params, const float* hs0, const float* obs,
                      const uint8_t* last_done, const int32_t* last_action, const int32_t* action, const float* reward,
                      const uint8_t* done, float* grads, float* loss_sum, float* qsa_sum, int32_t S, int32_t T, int32_t B,
                      float gamma, float lambda, void* workspace, void* stream) {
  int rc = check_desc(d, "pqn_rnn_loss_grad");
  if (rc) return rc;
  if ((rc = rnn::check_rnn(d, "pqn_rnn_loss_grad"))) return rc;
  return rnn_loss_grad(d, params, nullptr, hs0, obs, last_done, last_action, action, reward, done, grads, loss_sum, qsa_sum,
                       S, T, B, SeedScalar{nullptr, gamma}, SeedScalar{nullptr, lambda}, workspace, stream,
                       "pqn_rnn_loss_grad");
}

int pqn_rnn_loss_grad_stats(const pqn_net_desc_t* d, const float* params, float* batch_stats, const float* hs0,
                            const float* obs, const uint8_t* last_done, const int32_t* last_action, const int32_t* action,
                            const float* reward, const uint8_t* done, float* grads, float* loss_sum, float* qsa_sum,
                            int32_t S, int32_t T, int32_t B, float gamma, float lambda, void* workspace, void* stream) {
  int rc = check_desc(d, "pqn_rnn_loss_grad_stats");
  if (rc) return rc;
  if ((rc = rnn::check_rnn_stats(d, batch_stats, "pqn_rnn_loss_grad_stats"))) return rc;
  return rnn_loss_grad(d, params, batch_stats, hs0, obs, last_done, last_action, action, reward, done, grads, loss_sum,
                       qsa_sum, S, T, B, SeedScalar{nullptr, gamma}, SeedScalar{nullptr, lambda}, workspace, stream,
                       "pqn_rnn_loss_grad_stats");
}

int pqn_rnn_loss_grad_seeds(const pqn_net_desc_t* d, const float* params, float* batch_stats, const float* hs0,
                            const float* obs, const uint8_t* last_done, const int32_t* last_action, const int32_t* action,
                            const float* reward, const uint8_t* done, float* grads, float* loss_sum, float* qsa_sum,
                            int32_t S, int32_t T, int32_t B, const float* gamma, const float* lambda, void* workspace,
                            void* stream) {
  int rc = check_desc(d, "pqn_rnn_loss_grad_seeds");
  if (rc) return rc;
  if ((rc = rnn::check_rnn_stats(d, batch_stats, "pqn_rnn_loss_grad_seeds"))) return rc;
  if (!gamma || !lambda) return set_error(PQN_E_INVALID, "pqn_rnn_loss_grad_seeds: gamma / lambda is NULL");
  return rnn_loss_grad(d, params, batch_stats, hs0, obs, last_done, last_action, action, reward, done, grads, loss_sum,
                       qsa_sum, S, T, B, SeedScalar{gamma, 0.f}, SeedScalar{lambda, 0.f}, workspace, stream,
                       "pqn_rnn_loss_grad_seeds");
}

int pqn_set_conv_mma_path(int on) {
  if (on != 0 && on != 1 && on != 3) return set_error(PQN_E_UNSUPPORTED, "pqn_set_conv_mma_path: no conv path %d", on);
  g_conv_mma = on;
  return PQN_OK;
}

int pqn_set_conv_fusion(int on) {
  if (on != 0 && on != 1) return set_error(PQN_E_UNSUPPORTED, "pqn_set_conv_fusion: no mode %d", on);
  g_conv_fuse = on;
  return PQN_OK;
}

int pqn_set_tensor_core_path(int on) {
  if (on < 0 || on > 2) return set_error(PQN_E_UNSUPPORTED, "pqn_set_tensor_core_path: no tensor-core path %d", on);
  g_use_tc = on;
  return PQN_OK;
}

int pqn_net_layout(const pqn_net_desc_t* d, pqn_net_layout_t* out) {
  int rc = check_desc(d, "pqn_net_layout");
  if (rc) return rc;
  if (!out) return set_error(PQN_E_INVALID, "pqn_net_layout: out is NULL");
  make_layout(d, out);
  return PQN_OK;
}

int pqn_net_dense_layer(const pqn_net_desc_t* d, int32_t layer, int64_t* offsets_host) {
  int rc = check_desc(d, "pqn_net_dense_layer");
  if (rc) return rc;
  if (d->kind != PQN_NET_MLP && d->kind != PQN_NET_RNN && d->kind != PQN_NET_MLP_BITS)
    return set_error(PQN_E_INVALID, "pqn_net_dense_layer: only the MLP and GRU networks have hidden dense layers");
  if (!offsets_host || layer < 0 || layer >= d->layers)
    return set_error(PQN_E_INVALID, "pqn_net_dense_layer: layer=%d out of [0,%d) or offsets NULL", layer, d->layers);
  pqn_net_layout_t L;
  make_layout(d, &L);
  const DenseOff o = dense_off(L, d->hidden, layer);
  offsets_host[0] = o.w; offsets_host[1] = o.b; offsets_host[2] = o.g; offsets_host[3] = o.bi;
  return PQN_OK;
}

int64_t pqn_net_workspace_bytes(const pqn_net_desc_t* d, int32_t S, int64_t rows) {
  if (check_desc(d, "pqn_net_workspace_bytes")) return -1;
  if (d->kind == PQN_NET_RNN) return rnn::carve_rnn(d, S, rows, nullptr, nullptr);
  if (modular_net(d)) return nrm::carve_norm(d, S, rows, nullptr, nullptr);
  return carve(d, S, rows, nullptr, nullptr) +
         (d->kind == PQN_NET_MLP_BITS ? bits::carve_bits(d, S, rows, nullptr, nullptr) : 0);
}

int pqn_qnet_forward(const pqn_net_desc_t* d, const float* params, const float* batch_stats, const void* obs,
                     const int32_t* gather, int64_t obs_rows_per_seed, float* q, int32_t S, int64_t rows, void* workspace,
                     void* stream) {
  int rc = check_desc(d, "pqn_qnet_forward");
  if (rc) return rc;
  if (!params || !obs || !q || !workspace || S <= 0 || rows <= 0 || S > 65535)
    return set_error(PQN_E_INVALID, "pqn_qnet_forward: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  pqn_net_layout_t L;
  make_layout(d, &L);
  if (modular_net(d)) {
    nrm::NormWs nw;
    nrm::carve_norm(d, S, rows, (char*)workspace, &nw);
    return nrm::norm_forward(d, L, params, const_cast<float*>(batch_stats), obs, gather, obs_rows_per_seed, q, S, (int)rows,
                            0, nullptr, nw, st);
  }
  Workspace w;
  carve(d, S, rows, (char*)workspace, &w);
  const int A = d->num_actions;
  if (d->kind == PQN_NET_MINATAR_CNN) {
    const bool use_tc = g_use_tc && A <= PQN_TC_MAX_A;
    const bool f16 = use_tc && g_use_tc == 2;
    const Planes16 pl = planes16(w, S, rows);
    const bool conv16 = f16 && g_conv_mma == 1;   // the mma.sync conv writes the fp16 planes itself
    const bool fused = conv16 && g_conv_fuse;   // ... or runs inside the dense GEMM
    if (!fused)
      launch_conv_fwd<false>(d->in_c, dim3(cdiv(rows, 4), S), st, (const uint32_t*)obs, obs_rows_per_seed, gather, params,
                             L.total, L, conv16 ? (float*)pl.h1_hi : w.h1, conv16 ? (float*)pl.h1_lo : nullptr, nullptr,
                             (int)rows, nullptr, nullptr, nullptr, conv16);
    if (fused) {
      launch_split16_w1(params, L.total, L.d0_w, pl, S, st);
      if ((rc = tc16_conv_dense_fwd(tc::EPI_LN_HEAD, d->in_c, (const uint32_t*)obs, obs_rows_per_seed, gather, params,
                                    L.total, L, w, pl, A, q, S, (int)rows, st))) return rc;
    } else if (f16) {
      if (!conv16) launch_split16_h1(w.h1, pl, (int64_t)S * rows * FLAT_CNN, st);
      launch_split16_w1(params, L.total, L.d0_w, pl, S, st);
      if ((rc = tc16_dense_fwd(tc::EPI_LN_HEAD, params, L.total, L, w, pl, A, q, S, (int)rows, st))) return rc;
    } else if (use_tc) {
      launch_split_w1(params, L.total, L.d0_w, w.w1_lo, S, st);
      if ((rc = tc_dense_fwd(tc::EPI_LN_HEAD, params, L.total, L, w, A, q, S, (int)rows, st))) return rc;
    } else {
      if ((rc = launch_dense<2>(128, dim3(cdiv(rows, 128), S), st, w.h1, rows * FLAT_CNN, FLAT_CNN, params, L.total, L.d0_w,
                      L.d0_b, L.ln1_scale, L.ln1_bias, L.head_w, L.head_b, A, nullptr, nullptr, nullptr, q, (int)rows,
                      FLAT_CNN))) return rc;
    }
  } else {
    const int D = d->in_c, H = d->hidden;
    const bool bits = d->kind == PQN_NET_MLP_BITS, bits_tc = bits && g_use_tc == 2;
    const float* x = (const float*)obs;
    int64_t xss = obs_rows_per_seed * D;
    if (bits && !bits_tc) {   // packed bits with the tensor-core path off: gathered fp32 rows for the FFMA kernels
      bits::launch_expand((const uint32_t*)obs, obs_rows_per_seed, gather, (int)rows, D, w.xg, S, st);
      x = w.xg;
      xss = rows * D;
    } else if (gather && !bits) {
      { LaunchScope _ls(K_GATHER_ROWS, st); gather_rows_kernel<<<dim3(cdiv(rows * D, 256), S), 256, 0, st>>>(x, obs_rows_per_seed, gather, w.xg,
                                                                      (int)rows, D); }
      x = w.xg;
      xss = rows * D;
    }
    const int BM = (H == 128) ? 128 : 64;
    const dim3 grid(cdiv(rows, BM), S);
    const int last = d->layers - 1;
    if (bits_tc) {
      bits::BitsWs bw;
      bits::carve_bits(d, S, rows, (char*)workspace + carve(d, S, rows, nullptr, nullptr), &bw);
      if ((rc = bits_layer0_ln(d, L, params, (const uint32_t*)obs, obs_rows_per_seed, gather, S, (int)rows, w, bw, nullptr,
                               nullptr, st))) return rc;
      if (last == 0) {
        LaunchScope _ls(K_NORM_FWD, st);
        nrm::head_fwd_kernel<<<dim3(cdiv(rows, 8), S), 256, 0, st>>>(w.h[0], (int)rows, H, params, L.total, L.head_w, L.head_b, A, q);
      }
    } else if (last == 0) {
      if ((rc = dense_ln_fwd<2>(H, grid, st, x, xss, D, params, L.total, dense_off(L, H, 0), L.head_w, L.head_b, A, w.h[0], nullptr,
                      nullptr, q, (int)rows, D))) return rc;
    } else {
      if ((rc = dense_ln_fwd<0>(H, grid, st, x, xss, D, params, L.total, dense_off(L, H, 0), 0, 0, A, w.h[0], nullptr, nullptr, nullptr,
                      (int)rows, D))) return rc;
    }
    {
      for (int l = 1; l <= last; ++l) {
        if (mlp_hidden_tc(H)) {
          // hidden layer (K = N = H) on wgmma: fp16-split planes of h_{l-1} and of the Dense_l kernel, raw product, then
          // bias + LayerNorm + ReLU (and, after the last, the Q head) in row kernels
          if ((rc = mlp_hidden_tc_fwd(w, L, params, L.total, H, l, S, (int)rows, nullptr, nullptr,
                                      l == last ? K_TC_FWD_HEAD : K_TC_FWD, st))) return rc;
          if (l == last) {
            LaunchScope _ls(K_NORM_FWD, st);
            nrm::head_fwd_kernel<<<dim3(cdiv(rows, 8), S), 256, 0, st>>>(w.h[l], (int)rows, H, params, L.total, L.head_w, L.head_b, A, q);
          }
        } else if (l == last) {
          if ((rc = dense_ln_fwd<2>(H, grid, st, w.h[l - 1], rows * H, H, params, L.total, dense_off(L, H, l), L.head_w, L.head_b, A,
                          w.h[l], nullptr, nullptr, q, (int)rows, H))) return rc;
        } else {
          if ((rc = dense_ln_fwd<0>(H, grid, st, w.h[l - 1], rows * H, H, params, L.total, dense_off(L, H, l), 0, 0, A, w.h[l], nullptr,
                          nullptr, nullptr, (int)rows, H))) return rc;
        }
      }
    }
  }
  return check_launch("pqn_qnet_forward");
}

int pqn_qnet_loss_grad(const pqn_net_desc_t* d, const float* params, float* batch_stats, const void* obs,
                       const int32_t* gather, int64_t obs_rows_per_seed, const int32_t* action, const float* target,
                       int64_t tr_rows_per_seed, float* grads, float* loss_sum, float* qsa_sum, float* bn_sums,
                       int32_t S, int64_t rows, void* workspace, void* stream) {
  int rc = check_desc(d, "pqn_qnet_loss_grad");
  if (rc) return rc;
  if (!params || !obs || !action || !target || !grads || !loss_sum || !qsa_sum || !workspace || S <= 0 || rows <= 0 ||
      S > 65535)
    return set_error(PQN_E_INVALID, "pqn_qnet_loss_grad: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  pqn_net_layout_t L;
  make_layout(d, &L);
  const int64_t P = L.total;
  Workspace w;
  carve(d, S, rows, (char*)workspace, &w);
  const int A = d->num_actions;
  const int R = (int)rows;
  if (cudaMemsetAsync(grads, 0, (size_t)S * P * sizeof(float), st) != cudaSuccess)
    return check_launch("pqn_qnet_loss_grad(memset)");
  if (modular_net(d)) {
    nrm::NormWs nw;
    nrm::carve_norm(d, S, rows, (char*)workspace, &nw);
    return nrm::norm_loss_grad(d, L, params, batch_stats, obs, gather, obs_rows_per_seed, action, target, tr_rows_per_seed,
                              grads, loss_sum, qsa_sum, bn_sums, S, R, nw, st);
  }

  if (d->kind == PQN_NET_MINATAR_CNN) {
    const uint32_t* ob = (const uint32_t*)obs;
    const bool use_tc = g_use_tc && A <= PQN_TC_MAX_A;
    const bool f16 = use_tc && g_use_tc == 2;
    const Planes16 pl = planes16(w, S, rows);
    const bool conv16 = f16 && g_conv_mma == 1;
    const float gscale = f16 ? grad_scale(rows) : 1.0f;
    launch_conv_fwd<true>(d->in_c, dim3(cdiv(rows, 4), S), st, ob, obs_rows_per_seed, gather, params, P, L,
                          conv16 ? (float*)pl.h1_hi : w.h1, conv16 ? (float*)pl.h1_lo : nullptr, bn_sums, R,
                          g_conv_mma == 3 ? w.cxhat : nullptr, g_conv_mma == 3 ? w.crstd : nullptr,
                          (g_conv_mma == 1 || g_conv_mma == 3) ? w.relu_bits : nullptr, conv16);
    if (f16) {
      if (!conv16) launch_split16_h1(w.h1, pl, (int64_t)S * rows * FLAT_CNN, st);
      launch_split16_w1(params, P, L.d0_w, pl, S, st);
      if ((rc = tc16_dense_fwd(tc::EPI_LN_TRAIN, params, P, L, w, pl, A, nullptr, S, R, st))) return rc;
    } else if (use_tc) {
      launch_split_w1(params, P, L.d0_w, w.w1_lo, S, st);
      if ((rc = tc_dense_fwd(tc::EPI_LN_TRAIN, params, P, L, w, A, nullptr, S, R, st))) return rc;
    } else {
      if ((rc = launch_dense<1>(128, dim3(cdiv(rows, 128), S), st, w.h1, rows * FLAT_CNN, FLAT_CNN, params, P, L.d0_w, L.d0_b,
                      L.ln1_scale, L.ln1_bias, 0, 0, A, w.h2, w.xhat2, w.rstd2, nullptr, R, FLAT_CNN))) return rc;
    }
    const dim3 rbg(conv_mma_ctas(S, R, 4), S);
    if ((rc = run_row_bwd(128, true, rbg, A, st, w.h2, w.xhat2, w.rstd2, nullptr, w.dz2, (use_tc && !f16) ? w.dz2_lo : nullptr,
                          f16 ? pl.dz_hi : nullptr, f16 ? pl.dz_lo : nullptr, gscale, params, grads, P, L.ln1_scale,
                          L.ln1_bias, L.d0_b, L.head_w, L.head_b, gather, action, target, tr_rows_per_seed, loss_sum,
                          qsa_sum, w.rb_part, R))) return rc;
    if (f16) {
      if ((rc = tc16_wgrad(grads, P, L, pl, S, R, gscale, w.wg_part, st))) return rc;
      if ((rc = tc16_dgrad(w, pl, S, R, g_conv_mma == 1 || g_conv_mma == 3, gscale, st))) return rc;
    } else if (use_tc) {
      if ((rc = tc_wgrad(grads, P, L, w, S, R, st))) return rc;
      if ((rc = tc_dgrad(params, P, L, w, S, R, g_conv_mma == 1 || g_conv_mma == 3, st))) return rc;
    } else {
      const int splits = wgrad_splits(FLAT_CNN / 128, S, R);
      run_wgrad_ffma(w.h1, rows * FLAT_CNN, FLAT_CNN, w.dz2, rows * HID_CNN, HID_CNN, grads, P, L.d0_w, R, FLAT_CNN, S, splits, w.wg_part, st);
      launch_dgrad(w.dz2, rows * HID_CNN, HID_CNN, params, P, L.d0_w, w.h1, w.h1, rows * FLAT_CNN, R, FLAT_CNN, 0, S, st);
    }
    dim3 cg(conv_bwd_ctas(S, R), S);
    if (g_conv_mma) {
      const dim3 mg(conv_mma_ctas(S, R, 2), S);
      LaunchScope _ls(K_CONV_BWD, st);
      // dz of the conv is rstd times a dense-layer-sized gradient, and rstd reaches 1 / sqrt(LN_EPS) = 1000 on the empty
      // 3x3 patches of the initial parameters (conv bias 0: z = 0, var = 0).  One sixteenth of the dense gradient scale,
      // 2^ceil(log2 rows), keeps it above the subnormals; the headroom below the fp16 maximum (conversions saturate) is
      // small: test_gpu_cnn_grads.py measures max |dz * gs| = 3.96e4 at init with TD errors of scale 30 (1.65x below),
      // test_gpu_cnn_grads_tiles.py 4.02e4 at C = 7 (1.63x below)
      const float gs16 = grad_scale((int)rows) * (1.0f / 16.0f);
      if (g_conv_mma == 1) {
        switch (d->in_c) {
          case 4: rc = launch_conv_bwd_mma16<4>(mg, st, ob, obs_rows_per_seed, gather, params, P, L, w.h1, grads, w.cb_part, R, gs16); break;
          case 6: rc = launch_conv_bwd_mma16<6>(mg, st, ob, obs_rows_per_seed, gather, params, P, L, w.h1, grads, w.cb_part, R, gs16); break;
          case 7: rc = launch_conv_bwd_mma16<7>(mg, st, ob, obs_rows_per_seed, gather, params, P, L, w.h1, grads, w.cb_part, R, gs16); break;
          case 10: rc = launch_conv_bwd_mma16<10>(mg, st, ob, obs_rows_per_seed, gather, params, P, L, w.h1, grads, w.cb_part, R, gs16); break;
        }
      } else
      switch (d->in_c) {
        case 4: rc = launch_conv_bwd_mma<4>(mg, st, ob, obs_rows_per_seed, gather, params, P, L, w.h1, w.cxhat, w.crstd, grads, w.cb_part, R); break;
        case 6: rc = launch_conv_bwd_mma<6>(mg, st, ob, obs_rows_per_seed, gather, params, P, L, w.h1, w.cxhat, w.crstd, grads, w.cb_part, R); break;
        case 7: rc = launch_conv_bwd_mma<7>(mg, st, ob, obs_rows_per_seed, gather, params, P, L, w.h1, w.cxhat, w.crstd, grads, w.cb_part, R); break;
        case 10: rc = launch_conv_bwd_mma<10>(mg, st, ob, obs_rows_per_seed, gather, params, P, L, w.h1, w.cxhat, w.crstd, grads, w.cb_part, R); break;
      }
      if (rc) return rc;
    } else
    switch (d->in_c) {
      case 4: { LaunchScope _ls(K_CONV_BWD, st); conv_bwd_kernel<4><<<cg, 256, 0, st>>>(ob, obs_rows_per_seed, gather, params, P, L, w.h1, grads, R); } break;
      case 6: { LaunchScope _ls(K_CONV_BWD, st); conv_bwd_kernel<6><<<cg, 256, 0, st>>>(ob, obs_rows_per_seed, gather, params, P, L, w.h1, grads, R); } break;
      case 7: { LaunchScope _ls(K_CONV_BWD, st); conv_bwd_kernel<7><<<cg, 256, 0, st>>>(ob, obs_rows_per_seed, gather, params, P, L, w.h1, grads, R); } break;
      case 10: { LaunchScope _ls(K_CONV_BWD, st); conv_bwd_kernel<10><<<cg, 256, 0, st>>>(ob, obs_rows_per_seed, gather, params, P, L, w.h1, grads, R); } break;
    }
  } else {
    const int D = d->in_c, H = d->hidden;
    const int BM = (H == 128) ? 128 : 64;
    const bool bits = d->kind == PQN_NET_MLP_BITS, bits_tc = bits && g_use_tc == 2;
    const uint32_t* ob = (const uint32_t*)obs;
    bits::BitsWs bw = {};
    if (bits) bits::carve_bits(d, S, rows, (char*)workspace + carve(d, S, rows, nullptr, nullptr), &bw);
    if (bits && !bits_tc) {   // packed bits with the tensor-core path off: gathered fp32 rows for the FFMA kernels
      bits::launch_expand(ob, obs_rows_per_seed, gather, R, D, w.xg, S, st);
    } else if (!bits) {
      LaunchScope _ls(K_GATHER_ROWS, st); gather_rows_kernel<<<dim3(cdiv(rows * D, 256), S), 256, 0, st>>>((const float*)obs, obs_rows_per_seed, gather, w.xg, R, D);
    }
    if (bn_sums && bits) {
      // BatchNorm_0 statistics of {0,1} inputs: sum x = sum x^2 = the per-feature popcount of the minibatch
      bits::launch_counts(ob, obs_rows_per_seed, gather, R, D, bw, nullptr, bn_sums, S, st);
    } else if (bn_sums) {
      // input BatchNorm statistics (sum x, sum x^2 per feature): deterministic two-stage column sums of the gathered
      // rows (the per-element float atomics this replaces were 18 % of an Acrobot update at 65,536 envs)
      nrm::NormWs nw = {};
      nw.part = w.rb_part;
      nrm::colsum2(w.xg, w.xg, S, R, D, D, nw, bn_sums, nullptr, 0, -1, -1, st);
    }
    const dim3 grid(cdiv(rows, BM), S);
    const int last = d->layers - 1;
    const bool tcl = mlp_hidden_tc(H);
    const int64_t RR = (int64_t)S * rows;
    // ---- forward, keeping every layer's h, xhat and rstd
    if (bits_tc) {
      if ((rc = bits_layer0_ln(d, L, params, ob, obs_rows_per_seed, gather, S, R, w, bw, w.xhat[0], w.rstd[0], st))) return rc;
    } else if ((rc = dense_ln_fwd<1>(H, grid, st, w.xg, rows * D, D, params, P, dense_off(L, H, 0), 0, 0, A, w.h[0], w.xhat[0],
                                     w.rstd[0], nullptr, R, D))) return rc;
    for (int l = 1; l <= last; ++l) {
      if (tcl) {
        if ((rc = mlp_hidden_tc_fwd(w, L, params, P, H, l, S, R, w.xhat[l], w.rstd[l], K_TC_FWD, st))) return rc;
      } else {
        if ((rc = dense_ln_fwd<1>(H, grid, st, w.h[l - 1], rows * H, H, params, P, dense_off(L, H, l), 0, 0, A, w.h[l], w.xhat[l],
                        w.rstd[l], nullptr, R, H))) return rc;
      }
    }
    // ---- backward, last layer first.  For l >= 1, row_bwd turns dh_l (the head's, or dh0 from the layer above) into
    // dz_l: fp16 planes pre-scaled by gscale for the wgmma layers, fp32 dzl otherwise; then dW_l and dh_{l-1} (into
    // dh0, ReLU-masked by h_{l-1}).  Layer 0's dz is fp32 (in place in dh0, or dzl when it is the only layer).
    const dim3 rbg(conv_mma_ctas(S, R, 4), S);
    __half* zp = reinterpret_cast<__half*>(w.m16_dz);
    const float gscale = grad_scale(rows);
    for (int l = last; l >= 1; --l) {
      const DenseOff o = dense_off(L, H, l);
      const bool head = l == last;
      if ((rc = run_row_bwd(H, head, rbg, A, st, w.h[l], w.xhat[l], w.rstd[l], head ? nullptr : w.dh0, w.dzl, nullptr,
                            tcl ? zp : nullptr, tcl ? zp + RR * H : nullptr, tcl ? gscale : 1.0f, params, grads, P, o.g,
                            o.bi, o.b, head ? L.head_w : 0, head ? L.head_b : 0, head ? gather : nullptr,
                            head ? action : nullptr, head ? target : nullptr, head ? tr_rows_per_seed : 0,
                            head ? loss_sum : nullptr, head ? qsa_sum : nullptr, w.rb_part, R))) return rc;
      if (tcl) {
        __half* hp = mlp_h_planes(w, RR, H, l);
        __half* wp = mlp_w_planes(w, S, H, l);
        if ((rc = tc16_mm_wgrad(hp, RR * H, zp, RR * H, grads + o.w, P, S, R, H, H, 1.0f / gscale, w.wg_part, st))) return rc;
        if ((rc = tc16_mm_dgrad(zp, RR * H, wp, (int64_t)S * H * H, w.h[l - 1], w.dh0, S, R, H, H, 1.0f / gscale, st))) return rc;
      } else {
        run_wgrad_ffma(w.h[l - 1], rows * H, H, w.dzl, rows * H, H, grads, P, o.w, R, H, S,
                       wgrad_splits(ffma_tiles(H, H), S, R), w.wg_part, st);
        launch_dgrad(w.dzl, rows * H, H, params, P, o.w, w.h[l - 1], w.dh0, rows * H, R, H, 0, S, st);
      }
    }
    const DenseOff o0 = dense_off(L, H, 0);
    float* dz0 = last == 0 ? w.dzl : w.dh0;
    const bool head = last == 0;
    if ((rc = run_row_bwd(H, head, rbg, A, st, w.h[0], w.xhat[0], w.rstd[0], head ? nullptr : w.dh0, dz0, nullptr, nullptr,
                          nullptr, 1.0f, params, grads, P, o0.g, o0.bi, o0.b, head ? L.head_w : 0, head ? L.head_b : 0,
                          head ? gather : nullptr, head ? action : nullptr, head ? target : nullptr,
                          head ? tr_rows_per_seed : 0, head ? loss_sum : nullptr, head ? qsa_sum : nullptr, w.rb_part, R)))
      return rc;
    if (bits_tc) bits::launch_wgrad(ob, obs_rows_per_seed, gather, R, D, H, dz0, gscale, nullptr, grads + o0.w, P, bw, S, st);
    else run_wgrad_first(w.xg, dz0, grads, P, o0.w, S, R, D, H, w.rb_part, w.wg_part, st);
  }
  return check_launch("pqn_qnet_loss_grad");
}

}  // extern "C"
