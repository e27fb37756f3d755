// Recurrent PQN Q-network (GRU variant) of purejaxql/pqn_rnn_gymnax.py:26-105 and its loss (:295-366):
//   dummy input BatchNorm; NUM_LAYERS x {Dense(H) -> LayerNorm -> ReLU}; one-hot(last_action) appended; ScannedRNN =
//   flax GRUCell scanned over time with the carry reset to zeros where last_done is set; Dense(A) Q head;
//   loss = 0.5 * mean((q[t, a_t] - Q(lambda) target_t)^2) over t = 0 .. T-2 of the window, targets from stop-gradient
//   q values of the same forward pass (bootstrap max_a q[T-1]).
// flax.linen.GRUCell (restated from its published source; the test-side NumPy restatement pins it against
// torch.nn.GRUCell):   r = sigmoid(x W_ir + b_ir + h W_hr)      z = sigmoid(x W_iz + b_iz + h W_hz)
//                      n = tanh(x W_in + b_in + r * (h W_hn + b_hn))       h' = (1 - z) n + z h
// NORM_TYPE in {layer_norm, batch_norm, none} x NORM_INPUT (:65-76).  The default (layer_norm, NORM_INPUT=False, the
// shipped pqn_rnn_*.yaml) runs its trunk on the fused dense + LayerNorm kernels; every other combination runs the
// modular trunk of pqn_norm.cuh (raw dense, then one normalisation kernel per layer), whose BatchNorms reduce over
// every row of the [T][B] window and keep running statistics in the caller's batch_stats block.
//
// Structure (fp32 CUDA cores; these runs are small and launch-bound: 32 envs x 64 steps per update in the shipped
// preset): the time-independent parts (trunk MLP, input-side gate products x W_i*, Q head, all weight gradients) are
// batched GEMMs over the whole [T][B] window with the FFMA kernels of pqn_net.cu; the recurrence itself is ONE launch
// per direction -- rows of the batch are independent, so a CTA owns a few rows and loops over time internally
// (gru_scan_fwd / gru_scan_bwd), no grid-wide synchronisation per step.
//
// Included at the end of namespace pqn in pqn_net.cu.
#pragma once

namespace rnn {

constexpr int RB = 4;   // batch rows per CTA of the scan kernels

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }
__device__ __forceinline__ float sigmoid_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

// One GRU scan over T steps for the rows [b0, b0 + RB) of seed blockIdx.y.  thread j = hidden feature.
//   AI[g][S][T*B][H]  input-side pre-activations x W_ig[:H] + b_ig (g = r, z, n), rows time-major (t * B + b)
//   la[S][T*B] last action (one-hot rows W_ig[H + a] are added here), reset[S][T*B] (last_done)
//   hs[S][B][H] carry in / out (hs_out may alias);  Y[S][T*B][H] outputs
//   TRAIN: caches H0, R, Z, N, HN [S][T*B][H] for the backward scan
template <int H, bool TRAIN>
__global__ void __launch_bounds__(H) gru_scan_fwd_kernel(
    const float* __restrict__ AI, int64_t ai_gate_stride, const int32_t* __restrict__ la, const uint8_t* __restrict__ reset,
    const float* hs_in, float* hs_out, const float* __restrict__ params, int64_t P, pqn_net_layout_t L, int A,
    float* __restrict__ Y, float* __restrict__ H0, float* __restrict__ Rg, float* __restrict__ Zg, float* __restrict__ Ng,
    float* __restrict__ HN, int T, int B) {
  __shared__ float sh[RB][H];
  const int seed = blockIdx.y, j = threadIdx.x;
  const int b0 = blockIdx.x * RB;
  const float* __restrict__ prm = params + (int64_t)seed * P;
  const float* __restrict__ Whr = prm + L.gru_hr_w;
  const float* __restrict__ Whz = prm + L.gru_hz_w;
  const float* __restrict__ Whn = prm + L.gru_hn_w;
  const float bhn = prm[L.gru_hn_b + j];
  float h[RB];
#pragma unroll
  for (int r = 0; r < RB; ++r) h[r] = (b0 + r < B) ? hs_in[((int64_t)seed * B + b0 + r) * H + j] : 0.f;
  for (int t = 0; t < T; ++t) {
    bool rs[RB];
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const int64_t row = (int64_t)seed * T * B + (int64_t)t * B + min(b0 + r, B - 1);
      rs[r] = reset[row] != 0;
      if (rs[r]) h[r] = 0.f;                       // carry reset where last_done (pqn_rnn_gymnax.py:41-45)
      sh[r][j] = h[r];
    }
    __syncthreads();
    float ar[RB], az[RB], an[RB];
#pragma unroll
    for (int r = 0; r < RB; ++r) ar[r] = az[r] = an[r] = 0.f;
#pragma unroll 4
    for (int k = 0; k < H; ++k) {
      const float wr = Whr[(int64_t)k * H + j], wz = Whz[(int64_t)k * H + j], wn = Whn[(int64_t)k * H + j];
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        const float hk = sh[r][k];
        ar[r] = fmaf(hk, wr, ar[r]); az[r] = fmaf(hk, wz, az[r]); an[r] = fmaf(hk, wn, an[r]);
      }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      if (b0 + r >= B) continue;
      const int64_t row = (int64_t)seed * T * B + (int64_t)t * B + b0 + r;
      const int a = la[row];
      const float xr = AI[row * H + j] + prm[L.gru_ir_w + (int64_t)(H + a) * H + j];
      const float xz = AI[ai_gate_stride + row * H + j] + prm[L.gru_iz_w + (int64_t)(H + a) * H + j];
      const float xn = AI[2 * ai_gate_stride + row * H + j] + prm[L.gru_in_w + (int64_t)(H + a) * H + j];
      const float rg = sigmoid_acc(xr + ar[r]);
      const float zg = sigmoid_acc(xz + az[r]);
      const float hn = an[r] + bhn;
      const float ng = tanhf(xn + rg * hn);
      const float hnew = (1.0f - zg) * ng + zg * h[r];
      if (TRAIN) {
        H0[row * H + j] = h[r]; Rg[row * H + j] = rg; Zg[row * H + j] = zg; Ng[row * H + j] = ng; HN[row * H + j] = hn;
      }
      Y[row * H + j] = hnew;
      h[r] = hnew;
    }
  }
#pragma unroll
  for (int r = 0; r < RB; ++r)
    if (b0 + r < B) hs_out[((int64_t)seed * B + b0 + r) * H + j] = h[r];
}

// Reverse scan (BPTT through the GRU).  WT = transposed recurrent kernels [3][S][H][H] (WT[g][j][k] = W_hg[k][j]).
//   dY[S][T*B][H] gradient of the outputs; writes DA[3][S][T*B][H] = (da_r, da_z, da_n) and DHN = d(h W_hn + b_hn)
template <int H>
__global__ void __launch_bounds__(H) gru_scan_bwd_kernel(
    const float* __restrict__ dY, const uint8_t* __restrict__ reset, const float* __restrict__ H0,
    const float* __restrict__ Rg, const float* __restrict__ Zg, const float* __restrict__ Ng, const float* __restrict__ HN,
    const float* __restrict__ WT, int64_t wt_gate_stride, float* __restrict__ DA, int64_t da_gate_stride,
    float* __restrict__ DHN, int T, int B) {
  __shared__ float sh[RB][3][H];
  const int seed = blockIdx.y, j = threadIdx.x;
  const int b0 = blockIdx.x * RB;
  const float* __restrict__ WrT = WT + (int64_t)seed * H * H;
  const float* __restrict__ WzT = WT + wt_gate_stride + (int64_t)seed * H * H;
  const float* __restrict__ WnT = WT + 2 * wt_gate_stride + (int64_t)seed * H * H;
  float dh[RB];
#pragma unroll
  for (int r = 0; r < RB; ++r) dh[r] = 0.f;
  for (int t = T - 1; t >= 0; --t) {
    float keep[RB];   // dh * z : the direct path to the carry
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      float da_r = 0.f, da_z = 0.f, dhn = 0.f;
      keep[r] = 0.f;
      if (b0 + r < B) {
        const int64_t row = (int64_t)seed * T * B + (int64_t)t * B + b0 + r;
        const float rg = Rg[row * H + j], zg = Zg[row * H + j], ng = Ng[row * H + j], hn = HN[row * H + j],
                    h0 = H0[row * H + j];
        const float d = dh[r] + dY[row * H + j];
        const float dn = d * (1.0f - zg);
        const float dzg = d * (h0 - ng);
        keep[r] = d * zg;
        const float da_n = dn * (1.0f - ng * ng);
        const float dr = da_n * hn;
        dhn = da_n * rg;
        da_r = dr * rg * (1.0f - rg);
        da_z = dzg * zg * (1.0f - zg);
        DA[row * H + j] = da_r;
        DA[da_gate_stride + row * H + j] = da_z;
        DA[2 * da_gate_stride + row * H + j] = da_n;
        DHN[row * H + j] = dhn;
      }
      sh[r][0][j] = da_r; sh[r][1][j] = da_z; sh[r][2][j] = dhn;
    }
    __syncthreads();
    // dh0[k = j] = keep + sum_m da_r[m] W_hr[j][m] + da_z[m] W_hz[j][m] + dhn[m] W_hn[j][m]   (transposed: coalesced)
    float acc[RB];
#pragma unroll
    for (int r = 0; r < RB; ++r) acc[r] = keep[r];
#pragma unroll 4
    for (int m = 0; m < H; ++m) {
      const float wr = WrT[(int64_t)m * H + j], wz = WzT[(int64_t)m * H + j], wn = WnT[(int64_t)m * H + j];
#pragma unroll
      for (int r = 0; r < RB; ++r)
        acc[r] = fmaf(sh[r][0][m], wr, fmaf(sh[r][1][m], wz, fmaf(sh[r][2][m], wn, acc[r])));
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const int64_t row = (int64_t)seed * T * B + (int64_t)t * B + min(b0 + r, B - 1);
      dh[r] = reset[row] ? 0.f : acc[r];          // the reset cuts the carry
    }
  }
}

// WT[g][seed][j][k] = W_hg[k][j]
__global__ void gru_transpose_kernel(const float* __restrict__ params, int64_t P, pqn_net_layout_t L, int H,
                                     float* __restrict__ WT, int64_t wt_gate_stride) {
  const int seed = blockIdx.y, g = blockIdx.z;
  const int64_t off = g == 0 ? L.gru_hr_w : (g == 1 ? L.gru_hz_w : L.gru_hn_w);
  const float* __restrict__ W = params + (int64_t)seed * P + off;
  float* __restrict__ o = WT + g * wt_gate_stride + (int64_t)seed * H * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < H * H; i += gridDim.x * blockDim.x) {
    const int jj = i / H, k = i - jj * H;
    o[i] = W[(int64_t)k * H + jj];
  }
}

// In-loss Q(lambda) targets (:295-323), the loss and d loss / d q.  One block per seed, thread = batch column b.
//   q[S][T*B][A]; action/reward/done [S][T*B];  dq[S][T*B][A] (zero outside the chosen actions and at t = T-1)
//   part[S][2] = (loss, mean chosen q) of this minibatch, summed over the columns in thread order
__global__ void rnn_targets_kernel(const float* __restrict__ q, const int32_t* __restrict__ action,
                                   const float* __restrict__ reward, const uint8_t* __restrict__ done, int T, int B, int A,
                                   SeedScalar gamma_s, SeedScalar lam_s, float* __restrict__ dq,
                                   float* __restrict__ loss_sum, float* __restrict__ qsa_sum) {
  extern __shared__ float red[];   // [2][32] warp sums (blockDim is a multiple of 32, so at least 64 floats)
  const int seed = blockIdx.x, b = threadIdx.x;
  const float gamma = gamma_s.at(seed), lam = lam_s.at(seed);
  float l_acc = 0.f, q_acc = 0.f;
  const float inv = 1.0f / (float)((T - 1) * B);
  if (b < B) {
    const int64_t base = (int64_t)seed * T * B;
    auto maxq = [&](int t) {
      const float* qq = q + (base + (int64_t)t * B + b) * A;
      float m = qq[0];
      for (int a = 1; a < A; ++a) m = fmaxf(m, qq[a]);
      return m;
    };
    for (int t = 0; t < T; ++t)
      for (int a = 0; a < A; ++a) dq[(base + (int64_t)t * B + b) * A + a] = 0.f;
    const float last_q = maxq(T - 1);                                            // stop_gradient (:341-342)
    // arrays of the scan are the first T-1 steps; index -1 of them is t = T-2
    const int64_t r2 = base + (int64_t)(T - 2) * B + b;
    float lam_ret = reward[r2] + gamma * (1.0f - (float)done[r2]) * last_q;      // :315
    float next_q = maxq(T - 2);                                                  // :316
    auto emit = [&](int t, float target) {
      const int64_t row = base + (int64_t)t * B + b;
      const int a = action[row];
      const float qsa = q[row * A + a];
      const float diff = qsa - target;
      l_acc = fmaf(0.5f * diff, diff * inv, l_acc);
      q_acc = fmaf(qsa, inv, q_acc);
      dq[row * A + a] = diff * inv;
    };
    emit(T - 2, lam_ret);
    for (int t = T - 3; t >= 0; --t) {                                           // :299-313, reverse scan
      const int64_t row = base + (int64_t)t * B + b;
      const float d = (float)done[row], r = reward[row];
      const float boot = r + gamma * (1.0f - d) * next_q;
      float lr = boot + gamma * lam * (lam_ret - next_q);
      lr = (1.0f - d) * lr + d * r;
      next_q = maxq(t);
      lam_ret = lr;
      emit(t, lr);
    }
  }
  // deterministic reduction over the columns: a butterfly within each warp, then thread 0 adds the warp sums in order.
  // (a serial sum over the columns drifts with B: ~8 fp32 ulps at B = 1024).  For B <= 2 the result is the serial
  // sum's, bit for bit: the other lanes add zeros.
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    l_acc += __shfl_xor_sync(0xffffffffu, l_acc, o);
    q_acc += __shfl_xor_sync(0xffffffffu, q_acc, o);
  }
  if ((b & 31) == 0) { red[b >> 5] = l_acc; red[32 + (b >> 5)] = q_acc; }
  __syncthreads();
  if (b == 0) {
    float l = 0.f, qs = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { l += red[i]; qs += red[32 + i]; }
    loss_sum[seed] += l;
    qsa_sum[seed] += qs;
  }
}

// Q head backward from a dense dq: dY = dq W^T; per-block partials of dW[H][A], db[A] (two-stage, deterministic)
constexpr int RNN_MAX_A = 32;
template <int H>
__global__ void __launch_bounds__(H) rnn_head_bwd_kernel(const float* __restrict__ Y, const float* __restrict__ dq, int rows,
                                                         int A, const float* __restrict__ params, int64_t P, int64_t off_w,
                                                         float* __restrict__ dY, float* __restrict__ part) {
  const int seed = blockIdx.y, b = blockIdx.x, nb = gridDim.x, j = threadIdx.x;
  const int chunk = (rows + nb - 1) / nb;
  const int r0 = b * chunk, r1 = min(rows, r0 + chunk);
  const float* __restrict__ W = params + (int64_t)seed * P + off_w;
  float dw[RNN_MAX_A], wrow[RNN_MAX_A], db_mine = 0.f;
#pragma unroll
  for (int a = 0; a < RNN_MAX_A; ++a) { dw[a] = 0.f; wrow[a] = a < A ? W[(int64_t)j * A + a] : 0.f; }
  for (int row = r0; row < r1; ++row) {
    const int64_t g = (int64_t)seed * rows + row;
    const float y = Y[g * H + j];
    float acc = 0.f;
#pragma unroll
    for (int a = 0; a < RNN_MAX_A; ++a)
      if (a < A) {
        const float d = dq[g * A + a];
        dw[a] = fmaf(y, d, dw[a]);
        acc = fmaf(d, wrow[a], acc);
        if (j == a) db_mine += d;
      }
    dY[g * H + j] = acc;
  }
  float* o = part + ((int64_t)seed * nb + b) * (A + (int64_t)H * A);
  if (j < A) o[j] = db_mine;
  for (int a = 0; a < A; ++a) o[A + (int64_t)j * A + a] = dw[a];
}

__global__ void rnn_head_bwd_final_kernel(const float* __restrict__ part, int nb, int H, int A, float* __restrict__ grads,
                                          int64_t P, int64_t off_w, int64_t off_b) {
  const int seed = blockIdx.x;
  const int64_t stride = A + (int64_t)H * A;
  for (int64_t i = threadIdx.x; i < stride; i += blockDim.x) {
    float v = 0.f;
    for (int b = 0; b < nb; ++b) v += part[((int64_t)seed * nb + b) * stride + i];
    if (i < A) grads[(int64_t)seed * P + off_b + i] = v;
    else grads[(int64_t)seed * P + off_w + (i - A)] = v;
  }
}

// gradient of the one-hot rows of the input-side gate kernels: dW_ig[H + a][j] = sum over rows with last_action == a of
// DA_g[row][j].  One block per (seed, gate), thread = feature, rows in order (deterministic).
template <int H>
__global__ void __launch_bounds__(H) rnn_onehot_grad_kernel(const float* __restrict__ DA, int64_t da_gate_stride,
                                                            const int32_t* __restrict__ la, int rows, int A,
                                                            float* __restrict__ grads, int64_t P, pqn_net_layout_t L) {
  const int seed = blockIdx.x, g = blockIdx.y, j = threadIdx.x;
  const int64_t off = g == 0 ? L.gru_ir_w : (g == 1 ? L.gru_iz_w : L.gru_in_w);
  float acc[RNN_MAX_A];
#pragma unroll
  for (int a = 0; a < RNN_MAX_A; ++a) acc[a] = 0.f;
  for (int row = 0; row < rows; ++row) {
    const int64_t gr = (int64_t)seed * rows + row;
    const int a = la[gr];
    const float d = DA[g * da_gate_stride + gr * H + j];
#pragma unroll
    for (int q = 0; q < RNN_MAX_A; ++q)
      if (q == a) acc[q] += d;
  }
  for (int a = 0; a < A; ++a) grads[(int64_t)seed * P + off + (int64_t)(H + a) * H + j] = acc[a];
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
struct RnnWs {
  float *h[PQN_MAX_LAYERS], *xh[PQN_MAX_LAYERS], *rs[PQN_MAX_LAYERS], *ai, *y, *h0, *rg, *zg, *ng, *hn, *q, *dq, *dy, *da, *dhn, *dx, *dhl, *wt, *part, *sums, *rbp, *wgp;
  // modular trunk only: (mean, rstd) of hidden BatchNorm l and of the input BatchNorm, (d beta, d gamma) sums, the
  // dense obs rows, the normalised input, its xhat and its gradient
  float *mr[PQN_MAX_LAYERS], *mr_in, *dg, *xg, *xn, *xhin, *dxn;
};

static inline bool modular_rnn(const pqn_net_desc_t* d) { return d->norm_type != PQN_NORM_LAYER || d->norm_input != 0; }

static int64_t carve_rnn(const pqn_net_desc_t* d, int32_t S, int64_t rows, char* base, RnnWs* w) {
  int64_t off = 0;
  auto take = [&](int64_t nfloats) -> float* {
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += (nfloats * 4 + 255) / 256 * 256;
    return p;
  };
  RnnWs tmp;
  RnnWs* ww = w ? w : &tmp;
  const int64_t R = (int64_t)S * rows;
  const int H = d->hidden, A = d->num_actions;
  const int nl = d->layers > 2 ? d->layers : 2;
  for (int l = 0; l < nl; ++l) { ww->h[l] = take(R * H); ww->xh[l] = take(R * H); ww->rs[l] = take(R); }
  ww->ai = take(3 * R * H);
  ww->y = take(R * H); ww->h0 = take(R * H); ww->rg = take(R * H); ww->zg = take(R * H); ww->ng = take(R * H);
  ww->hn = take(R * H);
  ww->q = take(R * A); ww->dq = take(R * A);
  ww->dy = take(R * H); ww->da = take(3 * R * H); ww->dhn = take(R * H); ww->dx = take(R * H); ww->dhl = take(R * H);
  ww->wt = take(3 * (int64_t)S * H * H);
  const int64_t chan = nrm::chan_floats(d);   // the colsum2 tables of the GRU biases (H channels)
  ww->part = take((int64_t)S * nrm::RED_BLOCKS * (chan > A + H * A ? chan : A + H * A));
  ww->sums = take((int64_t)S * chan);
  ww->wgp = take(wgrad_split_tiles() * 128 * 128);   // per-split partials of the FFMA weight gradient
  ww->rbp = take(part_ctas(S) * row_bwd_part_floats(H, A));
  if (modular_rnn(d)) {   // appended, so the default network's workspace does not change
    const int D = d->in_c;
    for (int l = 0; l < d->layers; ++l) ww->mr[l] = take((int64_t)S * chan);
    ww->mr_in = take((int64_t)S * chan);
    ww->dg = take((int64_t)S * chan);
    ww->xg = take(R * D); ww->xn = take(R * D); ww->xhin = take(R * D); ww->dxn = take(R * D);
  }
  return off;
}

static int check_rnn(const pqn_net_desc_t* d, const char* who) {
  if (d->kind != PQN_NET_RNN) return set_error(PQN_E_INVALID, "%s: not an RNN descriptor", who);
  if (modular_rnn(d))
    return set_error(PQN_E_UNSUPPORTED, "%s: the GRU network is built for NORM_TYPE=layer_norm, NORM_INPUT=False here; "
                     "the other NORM_TYPE / NORM_INPUT take batch_stats (pqn_rnn_step_stats / pqn_rnn_loss_grad_stats)", who);
  return PQN_OK;
}

// the *_stats entry points: every NORM_TYPE / NORM_INPUT; batch_stats may be NULL only for the default network.  The
// input BatchNorm's statistics are colsum2 column sums over G == D features, which it builds for D <= 1024; the
// per-channel tables (nrm::chan_floats) grow with D beyond 256.
static int check_rnn_stats(const pqn_net_desc_t* d, const float* batch_stats, const char* who) {
  if (d->kind != PQN_NET_RNN) return set_error(PQN_E_INVALID, "%s: not an RNN descriptor", who);
  if (modular_rnn(d) && !batch_stats)
    return set_error(PQN_E_INVALID, "%s: NORM_TYPE=%s, NORM_INPUT=%d needs the batch_stats block (NULL given)", who,
                     d->norm_type == PQN_NORM_BATCH ? "batch_norm" : (d->norm_type == PQN_NORM_LAYER ? "layer_norm" : "none"),
                     d->norm_input);
  if (batch_stats && d->in_c > 1024)
    return set_error(PQN_E_UNSUPPORTED, "%s: input BatchNorm over %d features (at most 1024 built)", who, d->in_c);
  return PQN_OK;
}

// trunk (NUM_LAYERS x Dense -> normalize -> ReLU) + input-side gate products over `rows` rows per seed.
//   x: float obs rows, row r of seed s at s * orps + r.  batch_stats: running statistics (NULL for the default network).
//   train: the modular trunk's BatchNorms use the batch statistics of the rows and update batch_stats in place; the
//   input BatchNorm's statistics are updated whenever batch_stats is given (also for the default network, whose
//   fused trunk does not read them).  Eval: the running statistics normalise.
static int rnn_trunk(const pqn_net_desc_t* d, const pqn_net_layout_t& L, const float* params, float* batch_stats,
                     const float* x, int64_t orps, int S, int rows, bool train, RnnWs& w, cudaStream_t st) {
  const int D = d->in_c, H = d->hidden, A = d->num_actions;
  const int64_t P = L.total;
  const int BM = (H == 128) ? 128 : 64;
  const float* cur = x;
  int64_t css = orps * D;
  int kin = D;
  nrm::NormWs nw = {};
  nw.part = w.part; nw.sums = w.sums; nw.dg = w.dg;
  if (!modular_rnn(d)) {
    if (train && batch_stats) {
      // BatchNorm_0 is applied and its output discarded (:75-76); train mode still moves its running statistics.
      // bn_prepare turns the sums into (mean, rstd) in place: each thread reads its two sums before it writes them.
      nrm::colsum2(x, x, S, rows, D, D, nw, w.sums, nullptr, 0, -1, -1, st);
      LaunchScope _ls(K_NORM_FWD, st);
      nrm::bn_prepare_kernel<<<S, 256, 0, st>>>(w.sums, (float)rows, batch_stats, nrm::stats_floats(d), D, 1, 0.99f, w.sums);
    }
    for (int l = 0; l < d->layers; ++l) {
      const DenseOff o = dense_off(L, H, l);
      const int rc = train ? dense_ln_fwd<1>(H, dim3(cdiv(rows, BM), S), st, cur, css, kin, params, P, o, 0, 0, A, w.h[l],
                                             w.xh[l], w.rs[l], nullptr, rows, kin)
                           : dense_ln_fwd<0>(H, dim3(cdiv(rows, BM), S), st, cur, css, kin, params, P, o, 0, 0, A, w.h[l],
                                             nullptr, nullptr, nullptr, rows, kin);
      if (rc) return rc;
      cur = w.h[l]; css = (int64_t)rows * H; kin = H;
    }
  } else {
    const int norm = d->norm_type;
    const int64_t sstride = nrm::stats_floats(d);
    if (orps != rows) {   // strided rollout rows: make them dense for the column sums and the elementwise kernels
      LaunchScope _ls(K_GATHER_ROWS, st);
      gather_rows_kernel<<<dim3(cdiv((int64_t)rows * D, 256), S), 256, 0, st>>>(x, orps, nullptr, w.xg, rows, D);
      cur = w.xg; css = (int64_t)rows * D;
    }
    const float* xd = cur;
    if (train || d->norm_input) {
      if (train) nrm::colsum2(xd, xd, S, rows, D, D, nw, w.sums, nullptr, 0, -1, -1, st);
      LaunchScope _ls(K_NORM_FWD, st);
      nrm::bn_prepare_kernel<<<S, 256, 0, st>>>(w.sums, (float)rows, batch_stats, sstride, D, train, 0.99f, w.mr_in);
    }
    if (d->norm_input) {
      LaunchScope _ls(K_NORM_FWD, st);
      nrm::norm_elem_fwd_kernel<2><<<dim3(cdiv((int64_t)rows * D, 256), S), 256, 0, st>>>(
          xd, (int64_t)rows * D, D, D, w.mr_in, params, P, L.bn_scale, L.bn_bias, nullptr, w.xn);
      cur = w.xn;
    }
    for (int l = 0; l < d->layers; ++l) {
      const DenseOff o = dense_off(L, H, l);
      // raw pre-activation into h[l], normalised + ReLU in place
      int rc = launch_dense<3>(H, dim3(cdiv(rows, BM), S), st, cur, css, kin, params, P, o.w, o.b, 0, 0, 0, 0, A, w.h[l],
                               nullptr, nullptr, nullptr, rows, kin);
      if (rc) return rc;
      float* run = norm == nrm::NORM_BN ? batch_stats + nrm::stats_off(d, l) : nullptr;
      if ((rc = nrm::norm_layer_fwd(norm, w.h[l], S, rows, H, H, params, P, o.g, o.bi, run, sstride, train, nw, w.mr[l],
                                    train && norm != nrm::NORM_NONE ? w.xh[l] : nullptr, train ? w.rs[l] : nullptr, w.h[l],
                                    st))) return rc;
      cur = w.h[l]; css = (int64_t)rows * H; kin = H;
    }
  }
  const int64_t gs = (int64_t)S * rows * H;
  const int64_t iw[3] = {L.gru_ir_w, L.gru_iz_w, L.gru_in_w}, ib[3] = {L.gru_ir_b, L.gru_iz_b, L.gru_in_b};
  for (int g = 0; g < 3; ++g) {
    const int rc = launch_dense<3>(H, dim3(cdiv(rows, BM), S), st, cur, css, H, params, P, iw[g], ib[g], 0, 0, 0, 0, A,
                                   w.ai + g * gs, nullptr, nullptr, nullptr, rows, H);
    if (rc) return rc;
  }
  return 0;
}

// Backward of the modular trunk.  On entry w.dx holds d x_L, the gate input-gradients under the trunk's ReLU mask.
// Per layer, last first: normalisation backward (LN / BN with the batch statistics' terms / none) with d scale, d bias
// of the norm and of the dense, the FFMA weight gradient, the masked input gradient of the layer below.  With
// NORM_INPUT, d scale / d bias of BatchNorm_0 from the input gradient of Dense_0 (nrm::norm_loss_grad's recipe).
//   x: the dense float obs rows [S][rows][D] of the forward.
static int rnn_trunk_bwd_modular(const pqn_net_desc_t* d, const pqn_net_layout_t& L, const float* params, const float* x,
                                 float* grads, int S, int rows, RnnWs& w, cudaStream_t st) {
  const int D = d->in_c, H = d->hidden;
  const int64_t P = L.total;
  nrm::NormWs nw = {};
  nw.part = w.part; nw.sums = w.sums; nw.dg = w.dg;
  const float* xin = d->norm_input ? w.xn : x;
  float* dcur = w.dx;
  for (int l = d->layers - 1; l >= 0; --l) {
    const DenseOff o = dense_off(L, H, l);
    int rc = nrm::norm_layer_bwd(d->norm_type, dcur, w.xh[l], w.rs[l], S, rows, H, H, params, grads, P, o.g, o.bi, o.b, nw,
                                 w.mr[l], st);
    if (rc) return rc;
    const float* xprev = l == 0 ? xin : w.h[l - 1];
    const int kin = l == 0 ? D : H;
    run_wgrad_ffma(xprev, (int64_t)rows * kin, kin, dcur, (int64_t)rows * H, H, grads, P, o.w, rows, kin, S,
                   wgrad_splits(ffma_tiles(kin, H), S, rows), w.wgp, st);
    if (l > 0) {
      float* dnext = dcur == w.dhl ? w.dx : w.dhl;   // dgrad reads all of dz_l while it writes dh_{l-1}
      launch_dgrad(dcur, (int64_t)rows * H, H, params, P, o.w, w.h[l - 1], dnext, (int64_t)rows * H, rows, H, 0, S, st);
      dcur = dnext;
    }
  }
  if (d->norm_input) {
    { LaunchScope _ls(K_DGRAD, st);
      nrm::dgrad_small_kernel<<<dim3(cdiv(rows, 8), S), 256, 0, st>>>(dcur, rows, H, params, P, L.d0_w, D, w.dxn); }
    { LaunchScope _ls(K_NORM_BWD, st);
      nrm::in_xhat_kernel<<<dim3(cdiv((int64_t)rows * D, 256), S), 256, 0, st>>>(x, (int64_t)rows * D, D, w.mr_in, w.xhin); }
    nrm::colsum2(w.dxn, w.xhin, S, rows, D, D, nw, w.dg, grads, P, L.bn_bias, L.bn_scale, st);
  }
  return 0;
}

template <bool TRAIN>
static int rnn_scan_fwd(const pqn_net_desc_t* d, const pqn_net_layout_t& L, const float* params, const int32_t* la,
                        const uint8_t* reset, const float* hs_in, float* hs_out, int S, int T, int B, RnnWs& w,
                        cudaStream_t st) {
  const int H = d->hidden, A = d->num_actions;
  const int64_t gs = (int64_t)S * T * B * H;
  const dim3 grid(cdiv(B, RB), S);
  LaunchScope _ls(K_RNN_SCAN, st);
#define PQN_GRU_FWD(HH)                                                                                                     \
  gru_scan_fwd_kernel<HH, TRAIN><<<grid, HH, 0, st>>>(w.ai, gs, la, reset, hs_in, hs_out, params, L.total, L, A, w.y, w.h0, \
                                                      w.rg, w.zg, w.ng, w.hn, T, B)
  switch (H) {
    case 64: PQN_GRU_FWD(64); break;
    case 128: PQN_GRU_FWD(128); break;
    case 256: PQN_GRU_FWD(256); break;
    case 512: PQN_GRU_FWD(512); break;
    default: return set_error(PQN_E_UNSUPPORTED, "GRU hidden=%d (64, 128, 256 or 512 built)", H);
  }
#undef PQN_GRU_FWD
  return 0;
}

}  // namespace rnn
