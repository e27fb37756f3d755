// optax.chain(clip_by_global_norm(max_norm), radam(lr)) + apply_updates, batched
// over S independent seeds (one flat parameter block per seed).
//
// Reference: purejaxql/pqn_minatar.py:159-162 (optimizer wiring), :292
// (apply_gradients), :140-147 (linear lr schedule).  optax defaults restated
// (third party): radam b1=.9 b2=.999 eps=1e-8 eps_root=0 threshold=5;
//   clip: g <- g                     if ||g|| <  max_norm
//         g <- (g / ||g||) * max_norm otherwise          (global norm over ALL leaves)
//   mu <- b1 mu + (1-b1) g ; nu <- b2 nu + (1-b2) g^2 ; t <- t+1
//   mu_hat = mu / (1-b1^t) ; nu_hat = nu / (1-b2^t)
//   rho_t >= 5 : u = r_t * mu_hat / (sqrt(nu_hat) + eps)   else  u = mu_hat
//   p <- p - lr_t * u
// The per-step scalars (lr_t, 1-b1^t, 1-b2^t, r_t or 0) come from a device table
// indexed by a device step counter so that the whole update can live in a CUDA graph.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/pqn_b200.h"
#include "api_common.h"
#include "threefry.cuh"

namespace pqn {

constexpr int NORM_BLOCKS = 64;  // blocks per seed in the squared-norm reduction

__global__ void __launch_bounds__(256) sqnorm_kernel(const float* __restrict__ grads, int64_t P,
                                                     float* __restrict__ gn) {
  const int seed = blockIdx.y;
  const float4* __restrict__ g = reinterpret_cast<const float4*>(grads + (int64_t)seed * P);
  const int64_t n4 = P / 4;  // P is a multiple of 4 by construction of the layout
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (int64_t)gridDim.x * 256) {
    const float4 v = __ldg(g + i);
    acc = fmaf(v.x, v.x, acc); acc = fmaf(v.y, v.y, acc); acc = fmaf(v.z, v.z, acc); acc = fmaf(v.w, v.w, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w];
    gn[(int64_t)seed * NORM_BLOCKS + blockIdx.x] = t;   // block partial; radam_kernel adds them in block order
  }
}

// PBT (population-based training): seed s reads the table of seed sched_src[s] and scales its lr_t by lr_mult[s]
template <bool PBT>
__global__ void __launch_bounds__(256) radam_kernel(float* __restrict__ params, const float* __restrict__ grads,
                                                    float* __restrict__ mu, float* __restrict__ nu,
                                                    const float* __restrict__ sched, int64_t sched_stride,
                                                    const int32_t* __restrict__ sched_src,
                                                    const float* __restrict__ lr_mult,
                                                    const int32_t* __restrict__ step_counter,
                                                    const float* __restrict__ gn, int64_t P, SeedScalar max_norm_s,
                                                    float b1, float b2, float eps) {
  const int seed = blockIdx.y;
  const int64_t i4 = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int t = step_counter[0];
  const int64_t table = PBT ? (int64_t)__ldg(sched_src + seed) : (int64_t)seed;
  const float* __restrict__ row = sched + table * sched_stride + 4 * t;   // this seed's table (stride 0: shared)
  const float lr = PBT ? __fmul_rn(__ldg(row + 0), __ldg(lr_mult + seed)) : __ldg(row + 0);
  const float bc1 = __ldg(row + 1);
  const float bc2 = __ldg(row + 2);
  const float rect = __ldg(row + 3);
  const float max_norm = max_norm_s.at(seed);
  // squared gradient norm = the NORM_BLOCKS (64) block partials of sqnorm_kernel, added in a FIXED order (xor-shuffle
  // tree inside each of the first two warps, then warp 0 + warp 1) and broadcast through shared memory: deterministic,
  // and one pass over the 64 partials per block instead of one per thread
  static_assert(NORM_BLOCKS == 64, "two warps reduce the block partials");
  __shared__ float s_half[2];
  if (threadIdx.x < 64) {
    float v = gn[(int64_t)seed * NORM_BLOCKS + threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_half[threadIdx.x >> 5] = v;
  }
  __syncthreads();
  const float g_norm = sqrtf(s_half[0] + s_half[1]);
  if (i4 * 4 >= P) return;   // (after the block-wide barrier above)
  const bool no_clip = g_norm < max_norm;
  const int64_t off = (int64_t)seed * P + i4 * 4;
  float4 p = *reinterpret_cast<float4*>(params + off);
  const float4 g = __ldg(reinterpret_cast<const float4*>(grads + off));
  float4 m = *reinterpret_cast<float4*>(mu + off);
  float4 v = *reinterpret_cast<float4*>(nu + off);
  float* pp = reinterpret_cast<float*>(&p);
  const float* gp = reinterpret_cast<const float*>(&g);
  float* mp = reinterpret_cast<float*>(&m);
  float* vp = reinterpret_cast<float*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float gc = no_clip ? gp[j] : (gp[j] / g_norm) * max_norm;
    mp[j] = b1 * mp[j] + (1.0f - b1) * gc;
    vp[j] = b2 * vp[j] + (1.0f - b2) * (gc * gc);
    const float mhat = mp[j] / bc1;
    float u;
    if (rect > 0.f) u = rect * mhat / (sqrtf(vp[j] / bc2) + eps);
    else u = mhat;
    pp[j] = pp[j] - lr * u;
  }
  *reinterpret_cast<float4*>(params + off) = p;
  *reinterpret_cast<float4*>(mu + off) = m;
  *reinterpret_cast<float4*>(nu + off) = v;
}

__global__ void advance_kernel(int32_t* step_counter) { step_counter[0] += 1; }

__global__ void bn_update_kernel(float* __restrict__ batch_stats, float* __restrict__ bn_sums, int F, int64_t stride,
                                 float count, float momentum) {
  const int seed = blockIdx.x;
  const int f = threadIdx.x;
  if (f >= F) return;
  float* bs = batch_stats + (int64_t)seed * stride;
  float* sm = bn_sums + (int64_t)seed * 2 * F;
  const float mean = sm[f] / count;
  const float var = fmaxf(sm[F + f] / count - mean * mean, 0.f);
  bs[f] = momentum * bs[f] + (1.0f - momentum) * mean;
  bs[F + f] = momentum * bs[F + f] + (1.0f - momentum) * var;
  sm[f] = 0.f;
  sm[F + f] = 0.f;
}

// Parameter initialisation on the device (network.init, purejaxql/pqn_minatar.py:156-170): flax defaults —
// Conv/Dense kernels variance_scaling(scale, "fan_in", "truncated_normal") with scale 2 (he_normal) or 1
// (lecun_normal), i.e. N(0,1) truncated to [-2,2] times sqrt(scale/fan_in)/0.87962566; biases 0; norm scales 1.
// Draws are counter-based (threefry block (element, attempt) under a per-tensor key derived from the seed key)
// with Box-Muller + rejection: deterministic in the seed key, same distribution as flax, not the same draws
// (flax folds module paths into the key).
// Entry t < MAX_INIT draws under split(seed key, MAX_INIT)[t]; the split's width enters every value, so it stays 16 and
// the entries past it (deep networks only) draw under split(split(seed key, 2)[1], MAX_INIT)[t - MAX_INIT].
struct InitEntry {
  long long off, n;
  float std;   // > 0: truncated normal * std ; 0: zeros ; < 0: ones
};
constexpr int MAX_INIT = 16;
constexpr int MAX_INIT_ENTRIES = 2 * MAX_INIT;
struct InitTable {
  int count;
  InitEntry e[MAX_INIT_ENTRIES];
};

__global__ void net_init_kernel(const uint32_t* __restrict__ keys, float* __restrict__ params, int64_t P, InitTable tab) {
  const int seed = blockIdx.y;
  const Key sk{keys[2 * seed], keys[2 * seed + 1]};
  for (int t = 0; t < tab.count; ++t) {
    const InitEntry en = tab.e[t];
    const Key kt = t < MAX_INIT ? split_at(sk, (uint32_t)MAX_INIT, (uint32_t)t, 0)
                                : split_at(split_at(sk, 2u, 1u, 0), (uint32_t)MAX_INIT, (uint32_t)(t - MAX_INIT), 0);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < en.n; i += (long long)gridDim.x * blockDim.x) {
      float v;
      if (en.std == 0.f) v = 0.f;
      else if (en.std < 0.f) v = 1.f;
      else {
        float z = 0.f;
        for (uint32_t a = 0; a < 32u; ++a) {
          uint32_t x0 = (uint32_t)i, x1 = a;
          threefry2x32(kt.k0, kt.k1, x0, x1);
          const float u1 = ((float)(x0 >> 8) + 0.5f) * (1.0f / 16777216.0f);   // (0,1)
          const float u2 = ((float)(x1 >> 8) + 0.5f) * (1.0f / 16777216.0f);
          z = sqrtf(-2.0f * logf(u1)) * cosf(6.283185307179586f * u2);
          if (fabsf(z) <= 2.0f) break;
          z = fminf(fmaxf(z, -2.0f), 2.0f);
        }
        v = z * en.std;
      }
      params[(int64_t)seed * P + en.off + i] = v;
    }
  }
}

}  // namespace pqn

using namespace pqn;

static int radam_clip_step(float* params, const float* grads, float* mu, float* nu, const float* sched,
                           int64_t sched_stride, const int32_t* sched_src, const float* lr_mult,
                           int32_t* step_counter, float* gnorm_scratch, int32_t S, int64_t P,
                           SeedScalar max_norm, float b1, float b2, float eps, void* stream, const char* who) {
  if (!params || !grads || !mu || !nu || !sched || sched_stride < 0 || !step_counter || !gnorm_scratch || S <= 0 ||
      P <= 0 || (P & 3) || S > 65535)
    return set_error(PQN_E_INVALID, "%s: bad argument (P must be a multiple of 4)", who);
  cudaStream_t st = (cudaStream_t)stream;
  { LaunchScope _ls(K_SQNORM, st); sqnorm_kernel<<<dim3(NORM_BLOCKS, S), 256, 0, st>>>(grads, P, gnorm_scratch); }
  const unsigned nb = (unsigned)((P / 4 + 255) / 256);
  if (sched_src) {
    LaunchScope _ls(K_RADAM, st);
    radam_kernel<true><<<dim3(nb, S), 256, 0, st>>>(params, grads, mu, nu, sched, sched_stride, sched_src, lr_mult,
                                                    step_counter, gnorm_scratch, P, max_norm, b1, b2, eps);
  } else {
    LaunchScope _ls(K_RADAM, st);
    radam_kernel<false><<<dim3(nb, S), 256, 0, st>>>(params, grads, mu, nu, sched, sched_stride, nullptr, nullptr,
                                                     step_counter, gnorm_scratch, P, max_norm, b1, b2, eps);
  }
  { LaunchScope _ls(K_ADVANCE, st); advance_kernel<<<1, 1, 0, st>>>(step_counter); }
  return check_launch(who);
}

extern "C" {

int pqn_radam_clip_step(float* params, const float* grads, float* mu, float* nu, const float* sched,
                        int32_t* step_counter, float* gnorm_scratch, int32_t S, int64_t P, float max_norm, float b1,
                        float b2, float eps, void* stream) {
  return radam_clip_step(params, grads, mu, nu, sched, 0, nullptr, nullptr, step_counter, gnorm_scratch, S, P,
                         SeedScalar{nullptr, max_norm},
                         b1, b2, eps, stream, "pqn_radam_clip_step");
}

int pqn_radam_clip_step_seeds(float* params, const float* grads, float* mu, float* nu, const float* sched,
                              int64_t sched_seed_stride, int32_t* step_counter, float* gnorm_scratch, int32_t S,
                              int64_t P, const float* max_norm, float b1, float b2, float eps, void* stream) {
  if (!max_norm) return set_error(PQN_E_INVALID, "pqn_radam_clip_step_seeds: max_norm is NULL");
  return radam_clip_step(params, grads, mu, nu, sched, sched_seed_stride, nullptr, nullptr, step_counter, gnorm_scratch,
                         S, P, SeedScalar{max_norm, 0.f}, b1, b2, eps, stream, "pqn_radam_clip_step_seeds");
}

int pqn_radam_clip_step_pbt(float* params, const float* grads, float* mu, float* nu, const float* sched,
                            int64_t sched_seed_stride, const int32_t* sched_src, const float* lr_mult,
                            int32_t* step_counter, float* gnorm_scratch, int32_t S, int64_t P, const float* max_norm,
                            float b1, float b2, float eps, void* stream) {
  if (!max_norm || !sched_src || !lr_mult)
    return set_error(PQN_E_INVALID, "pqn_radam_clip_step_pbt: max_norm, sched_src and lr_mult are required");
  return radam_clip_step(params, grads, mu, nu, sched, sched_seed_stride, sched_src, lr_mult, step_counter,
                         gnorm_scratch, S, P, SeedScalar{max_norm, 0.f}, b1, b2, eps, stream, "pqn_radam_clip_step_pbt");
}

int pqn_net_init(const pqn_net_desc_t* d, const uint32_t* keys, float* params, int32_t S, void* stream) {
  pqn_net_layout_t L;
  int rc = pqn_net_layout(d, &L);
  if (rc) return rc;
  if (!keys || !params || S <= 0 || S > 65535) return set_error(PQN_E_INVALID, "pqn_net_init: bad argument");
  InitTable tab;
  tab.count = 0;
  bool overflow = false;
  auto add = [&](int64_t off, int64_t n, float std) {
    if (off < 0) return;
    if (tab.count == MAX_INIT_ENTRIES) { overflow = true; return; }
    tab.e[tab.count++] = InitEntry{(long long)off, (long long)n, std};
  };
  auto tn = [](double scale, double fan_in) { return (float)(sqrt(scale / fan_in) / 0.87962566103423978); };
  const int A = d->num_actions;
  cudaStream_t st = (cudaStream_t)stream;
  if (d->kind == PQN_NET_MINATAR_CNN) {
    const int C = d->in_c;
    add(L.bn_scale, C, -1.f);
    add(L.conv_w, 9 * C * 16, tn(2.0, 9.0 * C));            // he_normal (pqn_minatar.py:43)
    add(L.ln0_scale, 16, -1.f);
    add(L.d0_w, 1024 * 128, tn(2.0, 1024.0));               // he_normal (:48)
    add(L.ln1_scale, 128, -1.f);
    add(L.head_w, 128 * A, tn(1.0, 128.0));                 // lecun_normal default (:68)
  } else {
    const int D = d->in_c, H = d->hidden;
    add(L.bn_scale, D, -1.f);
    add(L.d0_w, (int64_t)D * H, tn(1.0, D));
    add(L.ln0_scale, H, -1.f);
    for (int l = 1; l < d->layers; ++l) {
      int64_t o[4];
      if ((rc = pqn_net_dense_layer(d, l, o))) return rc;
      add(o[0], (int64_t)H * H, tn(1.0, H));
      add(o[2], H, -1.f);
    }
    if (d->kind == PQN_NET_RNN) {   // GRUCell input denses: lecun_normal over fan_in = H + A; the orthogonal recurrent
      add(L.gru_ir_w, (int64_t)(H + A) * H, tn(1.0, H + A));   // kernels are drawn on the host (networks.py)
      add(L.gru_iz_w, (int64_t)(H + A) * H, tn(1.0, H + A));
      add(L.gru_in_w, (int64_t)(H + A) * H, tn(1.0, H + A));
    }
    add(L.head_w, (int64_t)H * A, tn(1.0, H));
  }
  if (overflow) return set_error(PQN_E_UNSUPPORTED, "pqn_net_init: more than %d initialised tensors", MAX_INIT_ENTRIES);
  if (cudaMemsetAsync(params, 0, (size_t)S * L.total * sizeof(float), st) != cudaSuccess) return check_launch("pqn_net_init(memset)");
  { LaunchScope _ls(K_NET_INIT, st); net_init_kernel<<<dim3(64, S), 256, 0, st>>>(keys, params, L.total, tab); }
  return check_launch("pqn_net_init");
}

int pqn_bn_stats_update(float* batch_stats, float* bn_sums, int32_t S, int32_t F, int64_t stats_seed_stride, float count,
                        float momentum, void* stream) {
  if (!batch_stats || !bn_sums || S <= 0 || F <= 0 || F > 1024 || count <= 0.f ||
      (stats_seed_stride != 0 && stats_seed_stride < 2 * F))
    return set_error(PQN_E_INVALID, "pqn_bn_stats_update: bad argument");
  const int64_t stride = stats_seed_stride ? stats_seed_stride : 2 * (int64_t)F;
  { LaunchScope _ls(K_BN_UPDATE, (cudaStream_t)stream); bn_update_kernel<<<S, ((F + 31) / 32) * 32, 0, (cudaStream_t)stream>>>(batch_stats, bn_sums, F, stride, count, momentum); }
  return check_launch("pqn_bn_stats_update");
}

}  // extern "C"
