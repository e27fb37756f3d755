// Q-network variants NORM_TYPE in {layer_norm, batch_norm, none} x NORM_INPUT in {False, True}
// (purejaxql/pqn_minatar.py:24-69, purejaxql/pqn_gymnax.py:29-58) other than the shipped default
// (layer_norm, NORM_INPUT=False), which keeps the fused kernels of pqn_net.cu / pqn_tc.cu.
//
// This is the "modular" path: one small kernel per layer op, fp32 CUDA cores, every cross-row reduction in two
// deterministic stages (per-block partials in a fixed layout, then one block per seed adds them in index order --
// no float atomics).  BatchNorm needs the two passes anyway (batch statistics before normalisation, the
// sum_dy / sum_dy_xhat terms before dz), and these configurations are not the headline workload.
//
// flax semantics restated (the test-side NumPy restatement, pqn_ref_norm, carries the reference line numbers):
//   nn.BatchNorm(use_running_average=not train): reduce over all axes but the last, eps 1e-5, momentum 0.99,
//   fast variance max(E[x^2]-E[x]^2, 0); train: batch statistics normalise, running = .99 running + .01 batch.
//   NORM_INPUT=True: the input BatchNorm replaces x/255 (CNN) or the raw observation (MLP) and gets gradients;
//   otherwise it is the dummy whose running statistics are the only thing that changes (pqn_minatar.py:61-66).
//
// Included at the end of namespace pqn in pqn_net.cu (it reuses the FFMA GEMM kernels and bit helpers there).
#pragma once

namespace nrm {

constexpr int NORM_LN = 0, NORM_BN = 1, NORM_NONE = 2;
constexpr float BN_EPS = 1e-5f;
constexpr int RED_BLOCKS = 64;   // row chunks per seed of the two-stage reductions

// ---------------------------------------------------------------------------------------------------------------
// two-stage per-channel reduction over [S][rows][ncols] (channel = col % G):  out[s][0][g] = sum A,
// out[s][1][g] = sum A*B.   A == B gives (sum x, sum x^2); (dy, xhat) gives (d beta, d gamma); (dz, dz)[0] = d bias.
// Requires 256 % G == 0, G == 512 (two channels per thread), or G == ncols <= 16 or <= 1024 (the generic paths below).
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colsum2_partial_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                              int rows, int ncols, int G, float* __restrict__ part) {
  __shared__ float sh[2][256];
  const int seed = blockIdx.y, b = blockIdx.x, nb = gridDim.x, t = threadIdx.x;
  const int chunk = (rows + nb - 1) / nb;
  const int r0 = b * chunk, r1 = min(rows, r0 + chunk);
  const float* __restrict__ a = A + (int64_t)seed * rows * ncols;
  const float* __restrict__ bb = B + (int64_t)seed * rows * ncols;
  float s = 0.f, ss = 0.f;
  if (256 % G == 0) {
    // flat index e over the chunk: channel = e % G = t % G (ncols % G == 0), fixed per thread
    const int64_t e0 = (int64_t)r0 * ncols, e1 = (int64_t)r1 * ncols;
    for (int64_t e = e0 + t; e < e1; e += 256) {
      const float x = a[e];
      s += x;
      ss = fmaf(x, bb[e], ss);
    }
    sh[0][t] = s; sh[1][t] = ss;
    __syncthreads();
    if (t < G) {
      float v0 = 0.f, v1 = 0.f;
      for (int k = t; k < 256; k += G) { v0 += sh[0][k]; v1 += sh[1][k]; }
      float* o = part + (((int64_t)seed * nb + b) * 2) * G;
      o[t] = v0; o[G + t] = v1;
    }
  } else if (G == 512) {
    // 512 channels (ncols % 512 == 0): thread t owns channels t and t + 256 of every 512-wide row segment
    const int64_t e0 = (int64_t)r0 * ncols, e1 = (int64_t)r1 * ncols;
    float s2 = 0.f, ss2 = 0.f;
    for (int64_t e = e0 + t; e < e1; e += 512) {
      const float x = a[e], y = a[e + 256];
      s += x; ss = fmaf(x, bb[e], ss);
      s2 += y; ss2 = fmaf(y, bb[e + 256], ss2);
    }
    float* o = part + (((int64_t)seed * nb + b) * 2) * G;
    o[t] = s; o[256 + t] = s2; o[G + t] = ss; o[G + 256 + t] = ss2;
  } else if (G > 16) {
    // wide G that does not divide 256 (the packed-bits MLP's input features, ncols == G <= 1024): thread t owns
    // channels t, t + 256, ..., rows in order
    float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
    for (int r = r0; r < r1; ++r) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int c = t + 256 * k;
        if (c < G) {
          const float x = a[(int64_t)r * ncols + c];
          a0[k] += x;
          a1[k] = fmaf(x, bb[(int64_t)r * ncols + c], a1[k]);
        }
      }
    }
    float* o = part + (((int64_t)seed * nb + b) * 2) * G;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = t + 256 * k;
      if (c < G) { o[c] = a0[k]; o[G + c] = a1[k]; }
    }
  } else {
    // small G that does not divide 256 (MLP input features, ncols == G <= 16): thread = row, G register accumulators,
    // then a fixed-order tree per channel (warp shuffles, warps in order)
    float acc0[16], acc1[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) acc0[c] = acc1[c] = 0.f;
    for (int r = r0 + t; r < r1; r += 256) {
#pragma unroll
      for (int c = 0; c < 16; ++c)
        if (c < G) {
          const float x = a[(int64_t)r * ncols + c];
          acc0[c] += x;
          acc1[c] = fmaf(x, bb[(int64_t)r * ncols + c], acc1[c]);
        }
    }
    float* o = part + (((int64_t)seed * nb + b) * 2) * G;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      if (c >= G) break;
      float v0 = acc0[c], v1 = acc1[c];
#pragma unroll
      for (int sft = 16; sft > 0; sft >>= 1) {
        v0 += __shfl_xor_sync(0xffffffffu, v0, sft);
        v1 += __shfl_xor_sync(0xffffffffu, v1, sft);
      }
      __syncthreads();
      if ((t & 31) == 0) { sh[0][t >> 5] = v0; sh[1][t >> 5] = v1; }
      __syncthreads();
      if (t == 0) {
        float s0 = 0.f, s1 = 0.f;
        for (int w = 0; w < 8; ++w) { s0 += sh[0][w]; s1 += sh[1][w]; }
        o[c] = s0; o[G + c] = s1;
      }
    }
  }
}

// out[s][k][g] = sum_b part[s][b][k][g]  (fixed order); optionally accumulates into a gradient slot:
//   dst0 (if >= 0): grads[s*P + dst0 + g]  = sum A      dst1 (if >= 0): grads[s*P + dst1 + g] = sum A*B
__global__ void colsum2_final_kernel(const float* __restrict__ part, int nb, int G, float* __restrict__ out,
                                     float* __restrict__ grads, int64_t P, int64_t dst0, int64_t dst1) {
  const int seed = blockIdx.x;
  for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) {
    float v = 0.f;
    for (int b = 0; b < nb; ++b) v += part[(((int64_t)seed * nb + b) * 2) * G + i];
    if (out) out[(int64_t)seed * 2 * G + i] = v;
    if (grads) {
      const int k = i / G, g = i - k * G;
      const int64_t dst = k == 0 ? dst0 : dst1;
      if (dst >= 0) grads[(int64_t)seed * P + dst + g] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// BatchNorm statistics -> (mean, rstd) table mr[S][2][G]
//   train: from sums[S][2][G] over `count` elements; also updates the running statistics run[S(stride)][2][G] when
//          run != nullptr;   eval: from the running statistics.
// ---------------------------------------------------------------------------------------------------------------
__global__ void bn_prepare_kernel(const float* __restrict__ sums, float count, float* run, int64_t run_stride, int G,
                                  int train, float momentum, float* __restrict__ mr) {
  const int seed = blockIdx.x;
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float mean, var;
    float* rm = run ? run + (int64_t)seed * run_stride : nullptr;
    if (train) {
      mean = sums[(int64_t)seed * 2 * G + g] / count;
      var = fmaxf(sums[(int64_t)seed * 2 * G + G + g] / count - mean * mean, 0.f);
      if (rm) {
        rm[g] = momentum * rm[g] + (1.0f - momentum) * mean;
        rm[G + g] = momentum * rm[G + g] + (1.0f - momentum) * var;
      }
    } else {
      mean = rm[g];
      var = rm[G + g];
    }
    mr[(int64_t)seed * 2 * G + g] = mean;
    mr[(int64_t)seed * 2 * G + G + g] = 1.0f / sqrtf(var + BN_EPS);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// normalisation + ReLU forward, elementwise flavours (channel = col % G):
//   BN  : xhat = (z - mean) * rstd ; h = relu(xhat * gamma + beta)          NONE: xhat aliases z ; h = relu(z)
//   AFF : y = (x - mean) * rstd * gamma + beta, no ReLU (the input BatchNorm of the MLP)
// ---------------------------------------------------------------------------------------------------------------
template <int MODE /*0 BN+ReLU, 1 none+ReLU, 2 affine only*/>
__global__ void norm_elem_fwd_kernel(const float* __restrict__ Z, int64_t n_per_seed, int ncols, int G,
                                     const float* __restrict__ mr, const float* __restrict__ params, int64_t P,
                                     int64_t off_g, int64_t off_b, float* __restrict__ XH, float* __restrict__ H) {
  const int seed = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_per_seed) return;
  const int g = (int)((i % ncols) % G);
  const float z = Z[(int64_t)seed * n_per_seed + i];
  if (MODE == 1) {
    H[(int64_t)seed * n_per_seed + i] = fmaxf(z, 0.f);
    return;
  }
  const float xh = (z - mr[(int64_t)seed * 2 * G + g]) * mr[(int64_t)seed * 2 * G + G + g];
  const float y = xh * params[(int64_t)seed * P + off_g + g] + params[(int64_t)seed * P + off_b + g];
  if (XH) XH[(int64_t)seed * n_per_seed + i] = xh;
  H[(int64_t)seed * n_per_seed + i] = MODE == 0 ? fmaxf(y, 0.f) : y;
}

// LayerNorm over groups of G consecutive values + ReLU: one warp per group for G in {64, 128, 256, 512} (lane-strided),
// one thread per group for G == 16.  rstd[S][groups]
template <int G>
__global__ void ln_fwd_kernel(const float* Z, int64_t groups_per_seed, const float* __restrict__ params,
                              int64_t P, int64_t off_g, int64_t off_b, float* XH, float* RS, float* H,
                              int64_t off_zbias = -1) {
  // off_zbias >= 0: Z is a raw product (tensor-core GEMM with a plain store epilogue), the dense bias is added here.
  // H may alias Z (every thread reads its elements before it writes them).
  const int seed = blockIdx.y;
  const float* __restrict__ gam = params + (int64_t)seed * P + off_g;
  const float* __restrict__ bet = params + (int64_t)seed * P + off_b;
  const float* __restrict__ zb = off_zbias >= 0 ? params + (int64_t)seed * P + off_zbias : nullptr;
  if constexpr (G == 16) {
    const int64_t grp = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (grp >= groups_per_seed) return;
    const int64_t base = ((int64_t)seed * groups_per_seed + grp) * 16;
    float z[16];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = *reinterpret_cast<const float4*>(Z + base + 4 * q);
      z[4 * q] = v.x; z[4 * q + 1] = v.y; z[4 * q + 2] = v.z; z[4 * q + 3] = v.w;
    }
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) { if (zb) z[j] += zb[j]; s1 += z[j]; s2 = fmaf(z[j], z[j], s2); }
    const float mean = s1 * (1.0f / 16), var = fmaxf(s2 * (1.0f / 16) - mean * mean, 0.f);
    const float rstd = 1.0f / sqrtf(var + LN_EPS);
    if (RS) RS[(int64_t)seed * groups_per_seed + grp] = rstd;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float xh = (z[j] - mean) * rstd;
      if (XH) XH[base + j] = xh;
      H[base + j] = fmaxf(xh * gam[j] + bet[j], 0.f);
    }
  } else {
    const int lane = threadIdx.x & 31;
    const int64_t grp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (grp >= groups_per_seed) return;
    const int64_t base = ((int64_t)seed * groups_per_seed + grp) * G;
    float z[G >= 32 ? G / 32 : 1];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < G / 32; ++j) {
      z[j] = Z[base + j * 32 + lane] + (zb ? zb[j * 32 + lane] : 0.f);
      s1 += z[j];
      s2 = fmaf(z[j], z[j], s2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const float mean = s1 * (1.0f / G), var = fmaxf(s2 * (1.0f / G) - mean * mean, 0.f);
    const float rstd = 1.0f / sqrtf(var + LN_EPS);
    if (lane == 0 && RS) RS[(int64_t)seed * groups_per_seed + grp] = rstd;
#pragma unroll
    for (int j = 0; j < G / 32; ++j) {
      const int c = j * 32 + lane;
      const float xh = (z[j] - mean) * rstd;
      if (XH) XH[base + c] = xh;
      H[base + c] = fmaxf(xh * gam[c] + bet[c], 0.f);
    }
  }
}

// LayerNorm backward: dz = rstd * (dxh - mean_g(dxh) - xhat * mean_g(dxh * xhat)), dxh = dy * gamma.  In place (DZ may
// alias DY).
template <int G>
__global__ void ln_bwd_kernel(const float* DY, const float* __restrict__ XH, const float* __restrict__ RS,
                              int64_t groups_per_seed, const float* __restrict__ params, int64_t P, int64_t off_g,
                              float* DZ) {
  const int seed = blockIdx.y;
  const float* __restrict__ gam = params + (int64_t)seed * P + off_g;
  if constexpr (G == 16) {
    const int64_t grp = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (grp >= groups_per_seed) return;
    const int64_t base = ((int64_t)seed * groups_per_seed + grp) * 16;
    float dxh[16], xh[16];
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      xh[j] = XH[base + j];
      dxh[j] = DY[base + j] * gam[j];
      m1 += dxh[j];
      m2 = fmaf(dxh[j], xh[j], m2);
    }
    m1 *= (1.0f / 16); m2 *= (1.0f / 16);
    const float rstd = RS[(int64_t)seed * groups_per_seed + grp];
#pragma unroll
    for (int j = 0; j < 16; ++j) DZ[base + j] = rstd * (dxh[j] - m1 - xh[j] * m2);
  } else {
    const int lane = threadIdx.x & 31;
    const int64_t grp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (grp >= groups_per_seed) return;
    const int64_t base = ((int64_t)seed * groups_per_seed + grp) * G;
    float dxh[G >= 32 ? G / 32 : 1], xh[G >= 32 ? G / 32 : 1];
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int j = 0; j < G / 32; ++j) {
      const int c = j * 32 + lane;
      xh[j] = XH[base + c];
      dxh[j] = DY[base + c] * gam[c];
      m1 += dxh[j];
      m2 = fmaf(dxh[j], xh[j], m2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      m1 += __shfl_xor_sync(0xffffffffu, m1, o);
      m2 += __shfl_xor_sync(0xffffffffu, m2, o);
    }
    m1 *= (1.0f / G); m2 *= (1.0f / G);
    const float rstd = RS[(int64_t)seed * groups_per_seed + grp];
#pragma unroll
    for (int j = 0; j < G / 32; ++j) DZ[base + j * 32 + lane] = rstd * (dxh[j] - m1 - xh[j] * m2);
  }
}

// BatchNorm backward (train mode): dz = rstd * gamma * (dy - dbeta / N - xhat * dgamma / N);  dg[S][2][G] = (dbeta,
// dgamma) from colsum2(dy, xhat).  In place allowed.
__global__ void bn_bwd_kernel(const float* DY, const float* __restrict__ XH, int64_t n_per_seed, int ncols, int G,
                              const float* __restrict__ mr, const float* __restrict__ dg, float invN,
                              const float* __restrict__ params, int64_t P, int64_t off_g, float* DZ) {
  const int seed = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_per_seed) return;
  const int g = (int)((i % ncols) % G);
  const float rstd = mr[(int64_t)seed * 2 * G + G + g], gam = params[(int64_t)seed * P + off_g + g];
  const float dbeta = dg[(int64_t)seed * 2 * G + g], dgamma = dg[(int64_t)seed * 2 * G + G + g];
  const int64_t e = (int64_t)seed * n_per_seed + i;
  DZ[e] = rstd * gam * (DY[e] - dbeta * invN - XH[e] * dgamma * invN);
}

// dz = dy * (h > 0)   (NORM_TYPE none: ReLU directly on the pre-activation; also the ReLU mask of the other variants)
__global__ void relu_mask_kernel(const float* DY, const float* __restrict__ Hh, int64_t n, float* DZ) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) DZ[i] = Hh[i] > 0.f ? DY[i] : 0.f;
}

// ---------------------------------------------------------------------------------------------------------------
// Q head: q = h @ Wh + bh (forward), and its loss backward:
//   dy[row][n] = dq_row * Wh[n][a_row] * (h[row][n] > 0)       dq_row = (q_sa - target) / rows
//   per-block partials of loss, mean q_sa, d bh[A], d Wh[N][A]  ->  head_bwd_final_kernel adds them in order.
// One thread per feature n (blockDim = max(N, 256)), the block walks its chunk of rows.
// ---------------------------------------------------------------------------------------------------------------
__global__ void head_fwd_kernel(const float* __restrict__ Hh, int rows, int N, const float* __restrict__ params,
                                int64_t P, int64_t off_w, int64_t off_b, int A, float* __restrict__ Q) {
  const int seed = blockIdx.y, lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* __restrict__ h = Hh + ((int64_t)seed * rows + row) * N;
  const float* __restrict__ W = params + (int64_t)seed * P + off_w;
  for (int a = 0; a < A; ++a) {
    float acc = 0.f;
    for (int n = lane; n < N; n += 32) acc = fmaf(h[n], W[(int64_t)n * A + a], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) Q[((int64_t)seed * rows + row) * A + a] = acc + params[(int64_t)seed * P + off_b + a];
  }
}

constexpr int HEAD_MAX_A = 32;
__global__ void __launch_bounds__(512) head_bwd_kernel(
    const float* __restrict__ Hh, const float* __restrict__ Q, int rows, int N, const float* __restrict__ params,
    int64_t P, int64_t off_w, int A, const int32_t* __restrict__ gather, const int32_t* __restrict__ action,
    const float* __restrict__ target, int64_t tr_rows_per_seed, float* __restrict__ DY, float* __restrict__ part) {
  // part[S][nb][ 2 + A + N*A ]
  const int seed = blockIdx.y, b = blockIdx.x, nb = gridDim.x, n = threadIdx.x;
  const int chunk = (rows + nb - 1) / nb;
  const int r0 = b * chunk, r1 = min(rows, r0 + chunk);
  const float* __restrict__ W = params + (int64_t)seed * P + off_w;
  const float invB = 1.0f / (float)rows;
  float dw[HEAD_MAX_A];
#pragma unroll
  for (int a = 0; a < HEAD_MAX_A; ++a) dw[a] = 0.f;
  float loss = 0.f, qsa = 0.f, dbh_mine = 0.f;   // thread n < A also accumulates d bh[n]
  for (int row = r0; row < r1; ++row) {
    const int64_t grow = (int64_t)seed * rows + row;
    const int src = gather ? gather[grow] : row;
    const int act = action[(int64_t)seed * tr_rows_per_seed + src];
    const float q_sa = Q[grow * A + act];
    const float diff = q_sa - target[(int64_t)seed * tr_rows_per_seed + src];
    const float dq = diff * invB;
    if (n == 0) { loss = fmaf(0.5f * diff, diff * invB, loss); qsa = fmaf(q_sa, invB, qsa); }
    if (n == act) dbh_mine += dq;
    if (n < N) {
      const float h = Hh[grow * N + n];
#pragma unroll
      for (int a = 0; a < HEAD_MAX_A; ++a)
        if (a == act) dw[a] = fmaf(h, dq, dw[a]);
      DY[grow * N + n] = h > 0.f ? dq * W[(int64_t)n * A + act] : 0.f;
    }
  }
  float* o = part + ((int64_t)seed * nb + b) * (2 + A + (int64_t)N * A);
  if (n == 0) { o[0] = loss; o[1] = qsa; }
  if (n < A) o[2 + n] = dbh_mine;
  if (n < N)
    for (int a = 0; a < A; ++a) o[2 + A + (int64_t)n * A + a] = dw[a];
}

__global__ void head_bwd_final_kernel(const float* __restrict__ part, int nb, int N, int A, float* __restrict__ grads,
                                      int64_t P, int64_t off_w, int64_t off_b, float* __restrict__ loss_sum,
                                      float* __restrict__ qsa_sum) {
  const int seed = blockIdx.x;
  const int64_t stride = 2 + A + (int64_t)N * A;
  for (int64_t i = threadIdx.x; i < stride; i += blockDim.x) {
    float v = 0.f;
    for (int b = 0; b < nb; ++b) v += part[((int64_t)seed * nb + b) * stride + i];
    if (i == 0) loss_sum[seed] += v;
    else if (i == 1) qsa_sum[seed] += v;
    else if (i < 2 + A) grads[(int64_t)seed * P + off_b + (i - 2)] = v;
    else grads[(int64_t)seed * P + off_w + (i - 2 - A)] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// CNN pieces: input affine / effective conv weights, raw conv forward, conv weight gradient from dz1, gradient finish
// ---------------------------------------------------------------------------------------------------------------
// per-channel set-bit counts of the (gathered) packed observations: part[S][nb][C]  (integers, exact in float)
template <int C>
__global__ void __launch_bounds__(256) obs_counts_kernel(const uint32_t* __restrict__ obs, int64_t orps,
                                                         const int32_t* __restrict__ gather, int rows,
                                                         float* __restrict__ part) {
  using Cfg = ConvCfg<C>;
  __shared__ uint32_t cmask[C][Cfg::PW];
  __shared__ int sh[C][8];
  const int seed = blockIdx.y, b = blockIdx.x, nb = gridDim.x, t = threadIdx.x;
  for (int i = t; i < C * Cfg::PW; i += 256) {
    const int c = i / Cfg::PW, wi = i % Cfg::PW;
    uint32_t m = 0u;
    for (int bit = 0; bit < 32; ++bit) {
      const int f = wi * 32 + bit;
      if (f < Cfg::OBS_BITS && f % C == c) m |= 1u << bit;
    }
    cmask[c][wi] = m;
  }
  __syncthreads();
  const int chunk = (rows + nb - 1) / nb;
  const int r0 = b * chunk, r1 = min(rows, r0 + chunk);
  int cnt[C];
#pragma unroll
  for (int c = 0; c < C; ++c) cnt[c] = 0;
  for (int row = r0 + t; row < r1; row += 256) {
    const int64_t src = gather ? gather[(int64_t)seed * rows + row] : row;
    const uint32_t* __restrict__ o = obs + ((int64_t)seed * orps + src) * Cfg::PW;
    for (int wi = 0; wi < Cfg::OBS_WORDS; ++wi) {
      const uint32_t w = __ldg(o + wi);
#pragma unroll
      for (int c = 0; c < C; ++c) cnt[c] += __popc(w & cmask[c][wi]);
    }
  }
#pragma unroll
  for (int c = 0; c < C; ++c) {
    int v = cnt[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((t & 31) == 0) sh[c][t >> 5] = v;
  }
  __syncthreads();
  if (t < C) {
    int v = 0;
    for (int w = 0; w < 8; ++w) v += sh[t][w];
    part[((int64_t)seed * nb + b) * C + t] = (float)v;
  }
}

// aff[S][2][C] = (d_c, a0_c): the network input is x_c = a0_c + bit * d_c.
//   NORM_INPUT: d = rstd * gamma, a0 = beta - mean * d, with (mean, var) the batch statistics of the bits (train: from
//   the counts; x in {0,1} => E[x^2] = E[x]) or the running ones (eval);  else d = 1/255, a0 = 0 (pqn_minatar.py:66).
// Also writes bn_sums[S][2][C] = (count, count) for the running-statistics update of the engine (train).
// weff[S][9C][16] = W * d_c ; beff[S][16] = b + sum_{tap,c} W[tap,c,:] * a0_c
template <int C>
__global__ void conv_eff_kernel(const float* __restrict__ params, int64_t P, pqn_net_layout_t L,
                                const float* __restrict__ cnt_part, int nb, float count, const float* __restrict__ run,
                                int64_t run_stride, int norm_input, int train, float* __restrict__ aff,
                                float* __restrict__ bn_sums, float* __restrict__ weff, float* __restrict__ beff) {
  __shared__ float d[C], a0[C];
  const int seed = blockIdx.x, t = threadIdx.x;
  const float* __restrict__ prm = params + (int64_t)seed * P;
  if (t < C) {
    float cn = 0.f;
    if (cnt_part)
      for (int b = 0; b < nb; ++b) cn += cnt_part[((int64_t)seed * nb + b) * C + t];
    if (bn_sums && cnt_part) { bn_sums[(int64_t)seed * 2 * C + t] += cn; bn_sums[(int64_t)seed * 2 * C + C + t] += cn; }
    float dd = 1.0f / 255.0f, aa = 0.f, mean = 0.f, rstd = 0.f;
    if (norm_input) {
      float var;
      if (train) { mean = cn / count; var = fmaxf(mean - mean * mean, 0.f); }
      else { mean = run[(int64_t)seed * run_stride + t]; var = run[(int64_t)seed * run_stride + C + t]; }
      rstd = 1.0f / sqrtf(var + BN_EPS);
      dd = rstd * prm[L.bn_scale + t];
      aa = prm[L.bn_bias + t] - mean * dd;
    }
    d[t] = dd; a0[t] = aa;
    aff[(int64_t)seed * 4 * C + t] = dd;
    aff[(int64_t)seed * 4 * C + C + t] = aa;
    aff[(int64_t)seed * 4 * C + 2 * C + t] = mean;
    aff[(int64_t)seed * 4 * C + 3 * C + t] = rstd;
  }
  __syncthreads();
  for (int i = t; i < 9 * C * CONV_O; i += blockDim.x) {
    const int c = (i / CONV_O) % C;
    weff[(int64_t)seed * 9 * C * CONV_O + i] = prm[L.conv_w + i] * d[c];
  }
  if (t < CONV_O) {
    float bsum = prm[L.conv_b + t];
    for (int k = 0; k < 9 * C; ++k) bsum = fmaf(prm[L.conv_w + k * CONV_O + t], a0[k % C], bsum);
    beff[(int64_t)seed * CONV_O + t] = bsum;
  }
}

// raw conv: Z1[S][rows][64][16] = conv_bits(x; weff) + beff.  thread = (sample, output pixel), 4 samples per block.
template <int C>
__global__ void __launch_bounds__(256) conv_raw_kernel(const uint32_t* __restrict__ obs, int64_t orps,
                                                       const int32_t* __restrict__ gather, const float* __restrict__ weff,
                                                       const float* __restrict__ beff, float* __restrict__ Z1, int rows) {
  using Cfg = ConvCfg<C>;
  __shared__ __align__(16) float ws[Cfg::TAPS * CONV_O];
  __shared__ float cb[CONV_O];
  __shared__ uint32_t so[4][Cfg::SW];
  const int tid = threadIdx.x, sl = tid >> 6, pix = tid & 63;
  const int seed = blockIdx.y;
  const int row = blockIdx.x * 4 + sl;
  const bool valid = row < rows;
  for (int i = tid; i < Cfg::TAPS * CONV_O; i += 256) ws[i] = weff[(int64_t)seed * Cfg::TAPS * CONV_O + i];
  if (tid < CONV_O) cb[tid] = beff[(int64_t)seed * CONV_O + tid];
  if (pix < Cfg::SW) {
    uint32_t w = 0u;
    if (valid && pix < Cfg::PW) {
      const int64_t src = gather ? gather[(int64_t)seed * rows + row] : row;
      w = __ldg(obs + ((int64_t)seed * orps + src) * Cfg::PW + pix);
    }
    so[sl][pix] = w;
  }
  __syncthreads();
  float acc[CONV_O];
  conv_pixel<C>(so[sl], ws, cb, pix >> 3, pix & 7, acc);
  if (valid) {
    float4* __restrict__ out = reinterpret_cast<float4*>(Z1 + ((int64_t)seed * rows + row) * FLAT_CNN + pix * CONV_O);
#pragma unroll
    for (int o4 = 0; o4 < CONV_O / 4; ++o4) out[o4] = make_float4(acc[4 * o4], acc[4 * o4 + 1], acc[4 * o4 + 2], acc[4 * o4 + 3]);
  }
}

// raw conv weight gradient from dz1: one warp per sample, set-bit driven (MinAtar observations are sparse):
//   dWraw[tap][c][o] = sum_{samples, pixels} bit[pixel + tap][c] * dz1[pixel][o]     (NOT yet scaled by d_c)
// lane = (tap parity, o); warps reduce through shared memory in warp order, blocks through part[S][nb][9C*16].
template <int C>
__global__ void __launch_bounds__(256) conv_dw_kernel(const uint32_t* __restrict__ obs, int64_t orps,
                                                      const int32_t* __restrict__ gather, const float* __restrict__ DZ1,
                                                      int rows, float* __restrict__ part) {
  using Cfg = ConvCfg<C>;
  constexpr int TAPS = Cfg::TAPS;
  __shared__ uint32_t so[8][Cfg::SW];
  __shared__ __align__(16) float sdz[8][CONV_PIX * SDZ_LD];
  float* s_w = &sdz[0][0];  // [C][5][32] block accumulator, aliases the dz stage once the row loop is done
  static_assert(5 * C * 32 <= 8 * CONV_PIX * SDZ_LD, "block dW accumulator fits the dz stage");
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int seed = blockIdx.y, b = blockIdx.x, nb = gridDim.x;
  const int o_b = lane & 15, tpar = lane >> 4;
  int t_di[5], t_dj[5];
#pragma unroll
  for (int it = 0; it < 5; ++it) {
    const int tap = it * 2 + tpar;
    t_di[it] = tap < 9 ? tap / 3 : 100;
    t_dj[it] = tap < 9 ? tap % 3 : 0;
  }
  float wacc[C][5];
#pragma unroll
  for (int c = 0; c < C; ++c)
#pragma unroll
    for (int it = 0; it < 5; ++it) wacc[c][it] = 0.f;
  uint32_t* __restrict__ my_so = so[warp];
  float* __restrict__ my_dz = sdz[warp];
  const int chunk = (rows + nb - 1) / nb;
  const int r0 = b * chunk, r1 = min(rows, r0 + chunk);
  for (int row = r0 + warp; row < r1; row += 8) {
    __syncwarp();
    {
      const int64_t src = gather ? gather[(int64_t)seed * rows + row] : row;
      const uint32_t* __restrict__ orow = obs + ((int64_t)seed * orps + src) * Cfg::PW;
      for (int wi = lane; wi < Cfg::SW; wi += 32) my_so[wi] = wi < Cfg::PW ? __ldg(orow + wi) : 0u;
      const float* __restrict__ dzr = DZ1 + ((int64_t)seed * rows + row) * FLAT_CNN;
      for (int i = lane; i < FLAT_CNN; i += 32) my_dz[(i >> 4) * SDZ_LD + (i & 15)] = dzr[i];
    }
    __syncwarp();
#pragma unroll
    for (int c = 0; c < C; ++c) {
      for (int wi = 0; wi < Cfg::OBS_WORDS; ++wi) {
        uint32_t bits = my_so[wi];
        if (C == 4) bits &= 0x11111111u << c;
        while (bits) {
          const int bpos = __ffs(bits) - 1;
          bits &= bits - 1u;
          const int f = wi * 32 + bpos;
          const int q = f / C;
          if (f - q * C != c || f >= Cfg::OBS_BITS) continue;
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
  __syncthreads();
  // the 8 warps add their registers to the block accumulator one after the other (fixed order => deterministic)
  for (int w = 0; w < 8; ++w) {
    if (warp == w) {
#pragma unroll
      for (int c = 0; c < C; ++c)
#pragma unroll
        for (int it = 0; it < 5; ++it) {
          float* dst = &s_w[(c * 5 + it) * 32 + lane];
          *dst = (w == 0 ? 0.f : *dst) + wacc[c][it];
        }
    }
    __syncthreads();
  }
  for (int i = tid; i < TAPS * CONV_O; i += 256) {
    const int o = i % CONV_O, k = i / CONV_O, c = k % C, tap = k / C;
    const int it = tap >> 1, ln = (tap & 1) * 16 + o;
    part[((int64_t)seed * nb + b) * TAPS * CONV_O + i] = s_w[(c * 5 + it) * 32 + ln];
  }
}

// d conv kernel / bias (and, with NORM_INPUT, d of the input BatchNorm's scale / bias) from the raw reductions:
//   dW[tap,c,o] = dWraw * d_c + a0_c * sdz[o]           d b[o] = sdz[o] = sum dz1[:, o]
//   d gamma_c   = sum_{tap,o} W[tap,c,o] * rstd_c * (dWraw[tap,c,o] - mean_c * sdz[o])
//   d beta_c    = sum_{tap,o} W[tap,c,o] * sdz[o]
template <int C>
__global__ void conv_grad_finish_kernel(const float* __restrict__ dw_part, int nb, const float* __restrict__ sdz /*[S][2][16]*/,
                                        const float* __restrict__ aff, const float* __restrict__ params, int64_t P,
                                        pqn_net_layout_t L, int norm_input, float* __restrict__ grads) {
  constexpr int TAPS = 9 * C;
  __shared__ float raw[TAPS * CONV_O];
  __shared__ float sd[CONV_O];
  const int seed = blockIdx.x, t = threadIdx.x;
  const float* __restrict__ prm = params + (int64_t)seed * P;
  float* __restrict__ g = grads + (int64_t)seed * P;
  const float* __restrict__ af = aff + (int64_t)seed * 4 * C;
  for (int i = t; i < TAPS * CONV_O; i += blockDim.x) {
    float v = 0.f;
    for (int b = 0; b < nb; ++b) v += dw_part[((int64_t)seed * nb + b) * TAPS * CONV_O + i];
    raw[i] = v;
  }
  if (t < CONV_O) sd[t] = sdz[(int64_t)seed * 2 * CONV_O + t];
  __syncthreads();
  for (int i = t; i < TAPS * CONV_O; i += blockDim.x) {
    const int o = i % CONV_O, c = (i / CONV_O) % C;
    g[L.conv_w + i] = raw[i] * af[c] + af[C + c] * sd[o];
  }
  if (t < CONV_O) g[L.conv_b + t] = sd[t];
  if (norm_input && t < C) {
    float dgam = 0.f, dbet = 0.f;
    const float mean = af[2 * C + t], rstd = af[3 * C + t];
    for (int tap = 0; tap < 9; ++tap)
      for (int o = 0; o < CONV_O; ++o) {
        const int i = (tap * C + t) * CONV_O + o;
        const float w = prm[L.conv_w + i];
        dgam = fmaf(w, rstd * (raw[i] - mean * sd[o]), dgam);
        dbet = fmaf(w, sd[o], dbet);
      }
    g[L.bn_scale + t] = dgam;
    g[L.bn_bias + t] = dbet;
  }
}

// MLP / GRU input: d x_n[row][j] = sum_n dz0[row][n] * W0[j][n], one warp per row and the D input features in turn.
// Built for narrow inputs (classic control, bsuite: D <= 50); any D runs, at D shuffle reductions per row.
__global__ void dgrad_small_kernel(const float* __restrict__ DZ, int rows, int H, const float* __restrict__ params,
                                   int64_t P, int64_t off_w, int D, float* __restrict__ DX) {
  const int seed = blockIdx.y, lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* __restrict__ dz = DZ + ((int64_t)seed * rows + row) * H;
  const float* __restrict__ W = params + (int64_t)seed * P + off_w;
  for (int j = 0; j < D; ++j) {
    float acc = 0.f;
    for (int n = lane; n < H; n += 32) acc = fmaf(dz[n], W[(int64_t)j * H + n], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) DX[((int64_t)seed * rows + row) * D + j] = acc;
  }
}

// xhat of the MLP input BatchNorm: (x - mean) * rstd  (for d gamma = sum dxn * xhat)
__global__ void in_xhat_kernel(const float* __restrict__ X, int64_t n_per_seed, int D, const float* __restrict__ mr,
                               float* __restrict__ XH) {
  const int seed = blockIdx.y;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_per_seed) return;
  const int j = (int)(i % D);
  XH[(int64_t)seed * n_per_seed + i] = (X[(int64_t)seed * n_per_seed + i] - mr[(int64_t)seed * 2 * D + j]) * mr[(int64_t)seed * 2 * D + D + j];
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
struct NormWs {
  // shared small buffers; mr[l]: (mean, rstd) of hidden norm l, mr_in: of the MLP's input BatchNorm
  float *part, *sums, *dg, *mr[PQN_MAX_LAYERS], *mr_in, *aff, *weff, *beff, *cntp, *q;
  float* wgp;   // per-split partials of the FFMA weight gradient (run_wgrad_ffma)
  bits::BitsWs bw;   // PQN_NET_MLP_BITS: Dense_0 on packed bits
  // CNN
  float *z1, *xh1, *h1, *rs1, *z2, *xh2, *h2, *rs2, *d2, *d1;
  // MLP
  float *xg, *xn, *xhin, *dxn, *z[PQN_MAX_LAYERS], *xh[PQN_MAX_LAYERS], *h[PQN_MAX_LAYERS], *rs[PQN_MAX_LAYERS],
      *d[PQN_MAX_LAYERS];
};

// channels per seed of the (sum, sum of squares) / (mean, rstd) tables: every per-channel reduction of the network
static int64_t chan_floats(const pqn_net_desc_t* d) {
  int64_t m = d->kind != PQN_NET_MINATAR_CNN && d->hidden > 256 ? d->hidden : 256;
  // the input features' statistics
  if ((d->kind == PQN_NET_MLP_BITS || d->kind == PQN_NET_RNN) && d->in_c > m) m = d->in_c;
  return 2 * m;
}

static int64_t part_floats(const pqn_net_desc_t* d) {
  const int A = d->num_actions;
  const int N = d->kind == PQN_NET_MINATAR_CNN ? HID_CNN : d->hidden;
  int64_t m = chan_floats(d);
  if (2 + A + (int64_t)N * A > m) m = 2 + A + (int64_t)N * A;
  if (d->kind == PQN_NET_MINATAR_CNN && 9 * d->in_c * CONV_O > m) m = 9 * d->in_c * CONV_O;
  return m * RED_BLOCKS;
}

static int64_t carve_norm(const pqn_net_desc_t* d, int32_t S, int64_t rows, char* base, NormWs* w) {
  int64_t off = 0;
  auto take = [&](int64_t nfloats) -> float* {
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += (nfloats * 4 + 255) / 256 * 256;
    return p;
  };
  NormWs tmp;
  NormWs* ww = w ? w : &tmp;
  const int64_t R = (int64_t)S * rows;
  const int A = d->num_actions;
  ww->part = take((int64_t)S * part_floats(d));
  ww->wgp = take(wgrad_split_tiles() * 128 * 128);
  const int nl = d->kind != PQN_NET_MINATAR_CNN && d->layers > 2 ? d->layers : 2;   // hidden norms (CNN: 2)
  ww->sums = take((int64_t)S * chan_floats(d));
  ww->dg = take((int64_t)S * chan_floats(d));
  ww->mr_in = take((int64_t)S * chan_floats(d));
  for (int l = 0; l < nl; ++l) ww->mr[l] = take((int64_t)S * chan_floats(d));
  ww->q = take(R * A);
  if (d->kind == PQN_NET_MINATAR_CNN) {
    const int C = d->in_c;
    ww->aff = take((int64_t)S * 4 * C);
    ww->weff = take((int64_t)S * 9 * C * CONV_O);
    ww->beff = take((int64_t)S * CONV_O);
    ww->cntp = take((int64_t)S * RED_BLOCKS * C);
    ww->z1 = take(R * FLAT_CNN); ww->xh1 = take(R * FLAT_CNN); ww->h1 = take(R * FLAT_CNN); ww->rs1 = take(R * CONV_PIX);
    ww->z2 = take(R * HID_CNN); ww->xh2 = take(R * HID_CNN); ww->h2 = take(R * HID_CNN); ww->rs2 = take(R);
    ww->d2 = take(R * HID_CNN); ww->d1 = take(R * FLAT_CNN);
  } else {
    const int D = d->in_c, H = d->hidden;
    ww->xg = take(R * D); ww->xn = take(R * D); ww->xhin = take(R * D); ww->dxn = take(R * D);
    for (int l = 0; l < nl; ++l) {
      ww->z[l] = take(R * H); ww->xh[l] = take(R * H); ww->h[l] = take(R * H); ww->rs[l] = take(R); ww->d[l] = take(R * H);
    }
    if (d->kind == PQN_NET_MLP_BITS) off += bits::carve_bits(d, S, rows, base ? base + off : nullptr, &ww->bw);
  }
  return off;
}

// floats per seed of the batch_stats block: [in mean F][in var F] then, for NORM_TYPE=batch_norm, (mean, var) of every
// hidden BatchNorm in network order
static int64_t stats_floats(const pqn_net_desc_t* d) {
  int64_t n = 2 * d->in_c;
  if (d->norm_type == NORM_BN) {
    if (d->kind == PQN_NET_MINATAR_CNN) n += 2 * CONV_O + 2 * HID_CNN;
    else n += 2 * (int64_t)d->hidden * d->layers;
  }
  return n;
}
// offset of hidden BatchNorm `layer` (CNN: 0 or 1; MLP: 0 .. NUM_LAYERS-1) in the batch_stats block
static int64_t stats_off(const pqn_net_desc_t* d, int layer) {
  const int64_t n = 2 * d->in_c;
  if (d->kind == PQN_NET_MINATAR_CNN) return layer == 0 ? n : n + 2 * CONV_O;
  return n + 2 * (int64_t)d->hidden * layer;
}

static inline void colsum2(const float* A, const float* B, int S, int rows, int ncols, int G, NormWs& w, float* out,
                           float* grads, int64_t P, int64_t dst0, int64_t dst1, cudaStream_t st) {
  { LaunchScope _ls(K_NORM_REDUCE, st); colsum2_partial_kernel<<<dim3(RED_BLOCKS, S), 256, 0, st>>>(A, B, rows, ncols, G, w.part); }
  { LaunchScope _ls(K_NORM_REDUCE, st); colsum2_final_kernel<<<S, 256, 0, st>>>(w.part, RED_BLOCKS, G, out, grads, P, dst0, dst1); }
}

// normalisation + ReLU of one layer: Z [S][rows][ncols] (channel = col % G) -> XH, H.  LN: G-wide groups.
// `train`: BatchNorm uses (and returns in mr) the batch statistics and updates run (may be null); eval: running ones.
static int norm_layer_fwd(int norm, const float* Z, int S, int rows, int ncols, int G, const float* params, int64_t P,
                          int64_t off_g, int64_t off_b, float* run, int64_t run_stride, int train, NormWs& w, float* mr,
                          float* XH, float* RS, float* H, cudaStream_t st) {
  const int64_t n = (int64_t)rows * ncols;
  if (norm == NORM_LN) {
    const int64_t groups = n / G;
    LaunchScope _ls(K_NORM_FWD, st);
    if (G == 16) ln_fwd_kernel<16><<<dim3(cdiv(groups, 256), S), 256, 0, st>>>(Z, groups, params, P, off_g, off_b, XH, RS, H);
    else if (G == 64) ln_fwd_kernel<64><<<dim3(cdiv(groups, 8), S), 256, 0, st>>>(Z, groups, params, P, off_g, off_b, XH, RS, H);
    else if (G == 512) ln_fwd_kernel<512><<<dim3(cdiv(groups, 8), S), 256, 0, st>>>(Z, groups, params, P, off_g, off_b, XH, RS, H);
    else if (G == 128) ln_fwd_kernel<128><<<dim3(cdiv(groups, 8), S), 256, 0, st>>>(Z, groups, params, P, off_g, off_b, XH, RS, H);
    else if (G == 256) ln_fwd_kernel<256><<<dim3(cdiv(groups, 8), S), 256, 0, st>>>(Z, groups, params, P, off_g, off_b, XH, RS, H);
    else return set_error(PQN_E_UNSUPPORTED, "LayerNorm width %d", G);
  } else if (norm == NORM_BN) {
    if (train) colsum2(Z, Z, S, rows, ncols, G, w, w.sums, nullptr, 0, -1, -1, st);
    { LaunchScope _ls(K_NORM_FWD, st); bn_prepare_kernel<<<S, 256, 0, st>>>(w.sums, (float)((double)rows * (ncols / G)), run, run_stride, G, train, 0.99f, mr); }
    { LaunchScope _ls(K_NORM_FWD, st); norm_elem_fwd_kernel<0><<<dim3(cdiv(n, 256), S), 256, 0, st>>>(Z, n, ncols, G, mr, params, P, off_g, off_b, XH, H); }
  } else {
    LaunchScope _ls(K_NORM_FWD, st);
    norm_elem_fwd_kernel<1><<<dim3(cdiv(n, 256), S), 256, 0, st>>>(Z, n, ncols, G, nullptr, params, P, 0, 0, nullptr, H);
  }
  return 0;
}

// backward of one normalisation layer: D holds dy (already ReLU-masked) on entry and dz on exit; writes d gamma / d beta
// into grads (LN / BN) and the preceding layer's bias gradient (= per-channel sum of dz) to off_db.
static int norm_layer_bwd(int norm, float* D, const float* XH, const float* RS, int S, int rows, int ncols, int G,
                          const float* params, float* grads, int64_t P, int64_t off_g, int64_t off_b, int64_t off_db,
                          NormWs& w, const float* mr, cudaStream_t st) {
  const int64_t n = (int64_t)rows * ncols;
  if (norm != NORM_NONE) colsum2(D, XH, S, rows, ncols, G, w, w.dg, grads, P, off_b, off_g, st);   // (d beta, d gamma)
  if (norm == NORM_LN) {
    const int64_t groups = n / G;
    LaunchScope _ls(K_NORM_BWD, st);
    if (G == 16) ln_bwd_kernel<16><<<dim3(cdiv(groups, 256), S), 256, 0, st>>>(D, XH, RS, groups, params, P, off_g, D);
    else if (G == 64) ln_bwd_kernel<64><<<dim3(cdiv(groups, 8), S), 256, 0, st>>>(D, XH, RS, groups, params, P, off_g, D);
    else if (G == 128) ln_bwd_kernel<128><<<dim3(cdiv(groups, 8), S), 256, 0, st>>>(D, XH, RS, groups, params, P, off_g, D);
    else if (G == 256) ln_bwd_kernel<256><<<dim3(cdiv(groups, 8), S), 256, 0, st>>>(D, XH, RS, groups, params, P, off_g, D);
    else if (G == 512) ln_bwd_kernel<512><<<dim3(cdiv(groups, 8), S), 256, 0, st>>>(D, XH, RS, groups, params, P, off_g, D);
    else return set_error(PQN_E_UNSUPPORTED, "LayerNorm width %d", G);
  } else if (norm == NORM_BN) {
    LaunchScope _ls(K_NORM_BWD, st);
    bn_bwd_kernel<<<dim3(cdiv(n, 256), S), 256, 0, st>>>(D, XH, n, ncols, G, mr, w.dg, (float)(1.0 / ((double)rows * (ncols / G))),
                                                         params, P, off_g, D);
  }
  colsum2(D, D, S, rows, ncols, G, w, w.sums, grads, P, off_db, -1, st);   // d bias of the conv / dense before it
  return 0;
}

template <int C>
static int cnn_norm_conv(const pqn_net_desc_t* d, const pqn_net_layout_t& L, const float* params, float* batch_stats,
                         int64_t sstride, const uint32_t* obs, int64_t orps, const int32_t* gather, int S, int rows,
                         int train, float* bn_sums, NormWs& w, cudaStream_t st) {
  const int64_t P = L.total;
  if (train) { LaunchScope _ls(K_NORM_REDUCE, st); obs_counts_kernel<C><<<dim3(RED_BLOCKS, S), 256, 0, st>>>(obs, orps, gather, rows, w.cntp); }
  { LaunchScope _ls(K_NORM_FWD, st);
    conv_eff_kernel<C><<<S, 256, 0, st>>>(params, P, L, train ? w.cntp : nullptr, RED_BLOCKS, (float)((double)rows * 100.0),
                                           batch_stats, sstride, d->norm_input, train, w.aff, train ? bn_sums : nullptr,
                                           w.weff, w.beff); }
  { LaunchScope _ls(train ? K_CONV_FWD : K_CONV_FWD_INFER, st);
    conv_raw_kernel<C><<<dim3(cdiv(rows, 4), S), 256, 0, st>>>(obs, orps, gather, w.weff, w.beff, w.z1, rows); }
  return 0;
}

template <int C>
static int cnn_norm_conv_bwd(const pqn_net_desc_t* d, const pqn_net_layout_t& L, const float* params, const uint32_t* obs,
                             int64_t orps, const int32_t* gather, int S, int rows, float* grads, NormWs& w, cudaStream_t st) {
  { LaunchScope _ls(K_CONV_BWD, st); conv_dw_kernel<C><<<dim3(RED_BLOCKS, S), 256, 0, st>>>(obs, orps, gather, w.d1, rows, w.part); }
  // w.sums holds (sum dz1, .) per conv channel from norm_layer_bwd's last colsum2
  { LaunchScope _ls(K_CONV_BWD, st); conv_grad_finish_kernel<C><<<S, 256, 0, st>>>(w.part, RED_BLOCKS, w.sums, w.aff, params, L.total, L, d->norm_input, grads); }
  return 0;
}

#define PQN_C_DISPATCH(C_, ...)                                    \
  switch (C_) {                                                    \
    case 4: { constexpr int CC = 4; __VA_ARGS__; } break;          \
    case 6: { constexpr int CC = 6; __VA_ARGS__; } break;          \
    case 7: { constexpr int CC = 7; __VA_ARGS__; } break;          \
    case 10: { constexpr int CC = 10; __VA_ARGS__; } break;        \
    default: return set_error(PQN_E_UNSUPPORTED, "CNN in_c=%d", C_); \
  }

// q = network.apply({params, batch_stats}, obs, train=False) for the non-default norm configurations; with
// `train` != 0 it is the training forward of the loss (batch statistics, running statistics updated in place).
static int norm_forward(const pqn_net_desc_t* d, const pqn_net_layout_t& L, const float* params, float* batch_stats,
                        const void* obs, const int32_t* gather, int64_t orps, float* q, int S, int rows, int train,
                        float* bn_sums, NormWs& w, cudaStream_t st) {
  const int64_t P = L.total, sstride = stats_floats(d);
  const int A = d->num_actions, norm = d->norm_type;
  int rc = 0;
  if ((norm == NORM_BN || d->norm_input) && !batch_stats)
    return set_error(PQN_E_INVALID, "this NORM_TYPE / NORM_INPUT needs the batch_stats block");
  if (d->kind == PQN_NET_MINATAR_CNN) {
    PQN_C_DISPATCH(d->in_c, rc = cnn_norm_conv<CC>(d, L, params, batch_stats, sstride, (const uint32_t*)obs, orps, gather,
                                                   S, rows, train, bn_sums, w, st));
    if (rc) return rc;
    float* run0 = norm == NORM_BN ? batch_stats + stats_off(d, 0) : nullptr;
    float* run1 = norm == NORM_BN ? batch_stats + stats_off(d, 1) : nullptr;
    if ((rc = norm_layer_fwd(norm, w.z1, S, rows, FLAT_CNN, CONV_O, params, P, L.ln0_scale, L.ln0_bias, run0, sstride, train,
                             w, w.mr[0], norm == NORM_NONE ? nullptr : w.xh1, w.rs1, w.h1, st))) return rc;
    if ((rc = launch_dense<3>(128, dim3(cdiv(rows, 128), S), st, w.h1, (int64_t)rows * FLAT_CNN, FLAT_CNN, params, P, L.d0_w, L.d0_b,
                    0, 0, 0, 0, A, w.z2, nullptr, nullptr, nullptr, rows, FLAT_CNN))) return rc;
    if ((rc = norm_layer_fwd(norm, w.z2, S, rows, HID_CNN, HID_CNN, params, P, L.ln1_scale, L.ln1_bias, run1, sstride, train,
                             w, w.mr[1], norm == NORM_NONE ? nullptr : w.xh2, w.rs2, w.h2, st))) return rc;
    { LaunchScope _ls(K_NORM_FWD, st); head_fwd_kernel<<<dim3(cdiv(rows, 8), S), 256, 0, st>>>(w.h2, rows, HID_CNN, params, P, L.head_w, L.head_b, A, q); }
  } else {
    const int D = d->in_c, H = d->hidden;
    const bool bits = d->kind == PQN_NET_MLP_BITS, bits_tc = bits && g_use_tc == 2;
    const uint32_t* ob = (const uint32_t*)obs;
    const float* x = (const float*)obs;
    int64_t xss = orps * D;
    if (bits) {
      if (!bits_tc) {   // tensor-core path off: the gathered bits as fp32 rows, then the fp32 MLP path below
        bits::launch_expand(ob, orps, gather, rows, D, w.xg, S, st);
        x = w.xg;
      }
      xss = (int64_t)rows * D;
    } else if (gather || train) {   // training also needs the input sums for the (dummy or real) input BatchNorm
      { LaunchScope _ls(K_GATHER_ROWS, st); gather_rows_kernel<<<dim3(cdiv((int64_t)rows * D, 256), S), 256, 0, st>>>(x, orps, gather, w.xg, rows, D); }
      x = w.xg;
      xss = (int64_t)rows * D;
    }
    if (xss != (int64_t)rows * D) {  // strided rollout rows: make them dense for the elementwise kernels
      { LaunchScope _ls(K_GATHER_ROWS, st); gather_rows_kernel<<<dim3(cdiv((int64_t)rows * D, 256), S), 256, 0, st>>>(x, orps, nullptr, w.xg, rows, D); }
      x = w.xg;
    }
    if (train || d->norm_input) {
      if (train && bits_tc) {
        bits::launch_counts(ob, orps, gather, rows, D, w.bw, w.sums, bn_sums, S, st);
      } else if (train) {
        colsum2(x, x, S, rows, D, D, w, w.sums, nullptr, 0, -1, -1, st);
        if (bn_sums) cudaMemcpyAsync(bn_sums, w.sums, (size_t)S * 2 * D * sizeof(float), cudaMemcpyDeviceToDevice, st);
      }
      // running statistics of the input BatchNorm are updated by pqn_bn_stats_update (engine) from bn_sums
      { LaunchScope _ls(K_NORM_FWD, st); bn_prepare_kernel<<<S, 256, 0, st>>>(w.sums, (float)rows, train ? nullptr : batch_stats, sstride, D, train, 0.99f, w.mr_in); }
    }
    const float* xin = x;
    const float* b0 = params + L.d0_b;   // bits_tc: Dense_0's bias, per seed at stride b0_stride
    int64_t b0_stride = P;
    const uint32_t* fl = nullptr;   // NORM_INPUT: features folded around 1 (bits flipped)
    if (bits_tc) {
      // NORM_INPUT: BN(x_f) = a0_f + bit * d_f folded into Dense_0' = diag(d) W0 and b0' = b0 + a0^T W0 per call
      const float* dv = nullptr;
      if (d->norm_input) {
        { LaunchScope _ls(K_NORM_FWD, st);
          bits::eff_kernel<<<dim3(cdiv(H, 128), S), 128, 0, st>>>(params, P, L.bn_scale, L.bn_bias, L.d0_w, L.d0_b, w.mr_in, D, H,
                                                                  w.bw.aff, w.bw.flip, w.bw.beff); }
        dv = w.bw.aff;
        fl = w.bw.flip;
        b0 = w.bw.beff;
        b0_stride = H;
      }
      bits::launch_wfrag(params, P, L.d0_w, dv, fl, D, H, S, w.bw.wf, st);
    } else if (d->norm_input) {
      { LaunchScope _ls(K_NORM_FWD, st); norm_elem_fwd_kernel<2><<<dim3(cdiv((int64_t)rows * D, 256), S), 256, 0, st>>>(x, (int64_t)rows * D, D, D, w.mr_in, params, P, L.bn_scale, L.bn_bias, nullptr, w.xn); }
      xin = w.xn;
    }
    const int BM = (H == 128) ? 128 : 64;
    const float* cur = xin;
    int kin = D;
    for (int l = 0; l < d->layers; ++l) {
      const DenseOff o = dense_off(L, H, l);
      if (l == 0 && bits_tc) {
        if ((rc = bits::launch_fwd(ob, orps, gather, rows, D, H, w.bw.wf, b0, b0_stride, fl, w.z[0], S, st))) return rc;
      } else if ((rc = launch_dense<3>(H, dim3(cdiv(rows, BM), S), st, cur, (int64_t)rows * kin, kin, params, P, o.w, o.b, 0, 0, 0, 0,
                                       A, w.z[l], nullptr, nullptr, nullptr, rows, kin))) return rc;
      float* run = norm == NORM_BN ? batch_stats + stats_off(d, l) : nullptr;
      if ((rc = norm_layer_fwd(norm, w.z[l], S, rows, H, H, params, P, o.g, o.bi, run, sstride, train, w, w.mr[l],
                               norm == NORM_NONE ? nullptr : w.xh[l], w.rs[l], w.h[l], st))) return rc;
      cur = w.h[l];
      kin = H;
    }
    { LaunchScope _ls(K_NORM_FWD, st); head_fwd_kernel<<<dim3(cdiv(rows, 8), S), 256, 0, st>>>(cur, rows, H, params, P, L.head_w, L.head_b, A, q); }
  }
  return check_launch("norm_forward");
}

static int norm_loss_grad(const pqn_net_desc_t* d, const pqn_net_layout_t& L, const float* params, float* batch_stats,
                          const void* obs, const int32_t* gather, int64_t orps, const int32_t* action, const float* target,
                          int64_t trps, float* grads, float* loss_sum, float* qsa_sum, float* bn_sums, int S, int rows,
                          NormWs& w, cudaStream_t st) {
  const int64_t P = L.total;
  const int A = d->num_actions, norm = d->norm_type;
  int rc = norm_forward(d, L, params, batch_stats, obs, gather, orps, w.q, S, rows, 1, bn_sums, w, st);
  if (rc) return rc;
  const bool cnn = d->kind == PQN_NET_MINATAR_CNN;
  const int N = cnn ? HID_CNN : d->hidden;
  const int last = cnn ? 1 : d->layers - 1;
  float* hl = cnn ? w.h2 : w.h[last];
  float* dl = cnn ? w.d2 : w.d[last];
  { LaunchScope _ls(K_ROW_BWD, st); head_bwd_kernel<<<dim3(RED_BLOCKS, S), N > 256 ? N : 256, 0, st>>>(hl, w.q, rows, N, params, P, L.head_w, A, gather, action, target, trps, dl, w.part); }
  { LaunchScope _ls(K_GRAD_FINAL, st); head_bwd_final_kernel<<<S, 256, 0, st>>>(w.part, RED_BLOCKS, N, A, grads, P, L.head_w, L.head_b, loss_sum, qsa_sum); }
  if (cnn) {
    if ((rc = norm_layer_bwd(norm, w.d2, w.xh2, w.rs2, S, rows, HID_CNN, HID_CNN, params, grads, P, L.ln1_scale, L.ln1_bias,
                             L.d0_b, w, w.mr[1], st))) return rc;
    const int splits = wgrad_splits(FLAT_CNN / 128, S, rows);
    run_wgrad_ffma(w.h1, (int64_t)rows * FLAT_CNN, FLAT_CNN, w.d2, (int64_t)rows * HID_CNN, HID_CNN, grads, P, L.d0_w, rows, FLAT_CNN, S, splits, w.wgp, st);
    launch_dgrad(w.d2, (int64_t)rows * HID_CNN, HID_CNN, params, P, L.d0_w, w.h1, w.d1, (int64_t)rows * FLAT_CNN, rows, FLAT_CNN, 0, S, st);
    if ((rc = norm_layer_bwd(norm, w.d1, w.xh1, w.rs1, S, rows, FLAT_CNN, CONV_O, params, grads, P, L.ln0_scale, L.ln0_bias,
                             -1, w, w.mr[0], st))) return rc;
    PQN_C_DISPATCH(d->in_c, rc = cnn_norm_conv_bwd<CC>(d, L, params, (const uint32_t*)obs, orps, gather, S, rows, grads, w, st));
    if (rc) return rc;
  } else {
    const int D = d->in_c, H = d->hidden;
    const bool bits_tc = d->kind == PQN_NET_MLP_BITS && g_use_tc == 2;
    const uint32_t* ob = (const uint32_t*)obs;
    const float* xin = d->norm_input ? w.xn : w.xg;
    for (int l = last; l >= 0; --l) {
      const DenseOff o = dense_off(L, H, l);
      if ((rc = norm_layer_bwd(norm, w.d[l], w.xh[l], w.rs[l], S, rows, H, H, params, grads, P, o.g, o.bi, o.b, w,
                               w.mr[l], st))) return rc;
      const float* xprev = l == 0 ? xin : w.h[l - 1];
      const int kin = l == 0 ? D : H;
      // dz of a batch-normalised layer carries rstd (up to ~316): one sixteenth of the dense gradient scale keeps it far
      // below the fp16 maximum
      const float gs = grad_scale(rows) * (1.0f / 16.0f);
      if (l == 0 && bits_tc && !d->norm_input) {
        bits::launch_wgrad(ob, orps, gather, rows, D, H, w.d[0], gs, nullptr, grads + o.w, P, w.bw, S, st);
      } else if (l == 0 && bits_tc) {
        // G = bits^T dz0, then every NORM_INPUT gradient from G and sum_r dz0 (w.sums, left by norm_layer_bwd)
        bits::launch_wgrad(ob, orps, gather, rows, D, H, w.d[0], gs, w.bw.flip, w.bw.G, (int64_t)D * H, w.bw, S, st);
        LaunchScope _ls(K_NORM_BWD, st);
        bits::grad_finish_kernel<<<dim3(cdiv(D, 8), S), 256, 0, st>>>(w.bw.G, w.sums, 2 * (int64_t)H, w.bw.aff, w.bw.flip, w.mr_in, params, P,
                                                                      o.w, L.bn_scale, L.bn_bias, D, H, grads);
      } else {
        const int sp = wgrad_splits(ffma_tiles(kin, H), S, rows);
        run_wgrad_ffma(xprev, (int64_t)rows * kin, kin, w.d[l], (int64_t)rows * H, H, grads, P, o.w, rows, kin, S, sp, w.wgp, st);
      }
      if (l > 0) launch_dgrad(w.d[l], (int64_t)rows * H, H, params, P, o.w, w.h[l - 1], w.d[l - 1], (int64_t)rows * H, rows, H, 0, S, st);
    }
    if (d->norm_input && !bits_tc) {   // the input BatchNorm is on the path: gradients of its scale / bias
      { LaunchScope _ls(K_DGRAD, st); dgrad_small_kernel<<<dim3(cdiv(rows, 8), S), 256, 0, st>>>(w.d[0], rows, H, params, P, L.d0_w, D, w.dxn); }
      { LaunchScope _ls(K_NORM_BWD, st); in_xhat_kernel<<<dim3(cdiv((int64_t)rows * D, 256), S), 256, 0, st>>>(w.xg, (int64_t)rows * D, D, w.mr_in, w.xhin); }
      colsum2(w.dxn, w.xhin, S, rows, D, D, w, w.dg, grads, P, L.bn_bias, L.bn_scale, st);
    }
  }
  return check_launch("norm_loss_grad");
}

}  // namespace nrm
