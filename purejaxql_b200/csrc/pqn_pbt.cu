// Population-based training: one truncation-selection exploit/explore event over the seed axis, on the device.
//
//   fitness   f[s] = (sum_{c < cols} fit[s * stride + c]) / cols, summed in float64 in column order
//   order     descending f; ties by the lower seed index; NaN last (also by index).  top = order[0, m),
//             bottom = order[S - m, S)
//   keys      kp, ke = split(kp);  ka, kf = split(ke);  a = randint(ka, (m,), 0, m);
//             b = randint(kf, (m, n_perturb), 0, 2)
//   exploit   child bottom[j] takes the rows of parent top[a[j]]: params, mu, nu, batch_stats, eps rows
//             [eps_from, eps_rows), sched_src, lr_mult, gamma, lambda, max_norm, rew_scale
//   explore   phi = factors[b[j][i]] for key perturb[i]: lr_mult and max_norm / rew_scale *= phi;
//             gamma / lambda <- clamp(1 - (1 - x) * phi, 0, 1), each operation rounded once in fp32
//
// m <= S / 2, so the parents (top) and the children (bottom) are disjoint: every launch reads parents' rows and
// writes children's rows only, and the row copies of every array go in one launch.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pqn_b200.h"
#include "api_common.h"
#include "threefry.cuh"

namespace pqn {

constexpr int PBT_THREADS = 256;
constexpr int PBT_MAX_PERTURB = 5;

// workspace layout: order keys uint64[S] | src int32[m] | factors float32[m][PBT_MAX_PERTURB]
static int64_t ws_src_off(int64_t S) { return ((8 * S + 255) / 256) * 256; }
static int64_t ws_fac_off(int64_t S, int64_t m) { return ws_src_off(S) + ((4 * m + 255) / 256) * 256; }
static int64_t ws_bytes(int64_t S, int64_t m) { return ws_fac_off(S, m) + 4 * m * PBT_MAX_PERTURB; }

// order-preserving key of a fitness: larger key = earlier in the order; -0 ties +0; NaN is the smallest key
__device__ __forceinline__ unsigned long long fitness_key(double f) {
  if (f != f) return 0ull;
  if (f == 0.0) f = 0.0;
  const unsigned long long u = (unsigned long long)__double_as_longlong(f);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

__global__ void __launch_bounds__(PBT_THREADS) pbt_fitness_kernel(const double* __restrict__ fit, int64_t stride,
                                                                  int cols, int S, double* __restrict__ fitness,
                                                                  unsigned long long* __restrict__ keys) {
  const int s = blockIdx.x * PBT_THREADS + threadIdx.x;
  if (s >= S) return;
  double acc = 0.0;
  for (int c = 0; c < cols; ++c) acc += fit[(int64_t)s * stride + c];
  const double f = acc / (double)cols;
  fitness[s] = f;
  keys[s] = fitness_key(f);
}

// rank by counting: seed i's position is the number of seeds that precede it.  Each block stages the keys in
// tiles of PBT_THREADS through shared memory; the count is exact, so the order does not depend on the launch shape.
__global__ void __launch_bounds__(PBT_THREADS) pbt_rank_kernel(const unsigned long long* __restrict__ keys, int S,
                                                               int32_t* __restrict__ order) {
  __shared__ unsigned long long tile[PBT_THREADS];
  const int i = blockIdx.x * PBT_THREADS + threadIdx.x;
  const unsigned long long ki = i < S ? keys[i] : 0ull;
  int rank = 0;
  for (int t0 = 0; t0 < S; t0 += PBT_THREADS) {
    const int j = t0 + threadIdx.x;
    tile[threadIdx.x] = j < S ? keys[j] : 0ull;
    __syncthreads();
    const int n = min(PBT_THREADS, S - t0);
    for (int jj = 0; jj < n; ++jj) {
      const unsigned long long kj = tile[jj];
      rank += (kj > ki) || (kj == ki && t0 + jj < i);
    }
    __syncthreads();
  }
  if (i < S) order[rank] = i;
}

struct PbtPerturb {
  int n;
  int code[PBT_MAX_PERTURB];
  float factor[2];
};

// one block: advances the event key, draws the parents and the factors, writes parent[] and the plan
__global__ void __launch_bounds__(1024) pbt_plan_kernel(int32_t* __restrict__ kp, int part, int S, int m,
                                                       const int32_t* __restrict__ order, int32_t* __restrict__ parent,
                                                       int32_t* __restrict__ src,
                                                       float* __restrict__ fac, PbtPerturb pt) {
  __shared__ Key s_ka, s_kf;
  if (threadIdx.x == 0) {
    const Key k{(uint32_t)kp[0], (uint32_t)kp[1]};
    Key kn, ke, ka, kf;
    split2(k, part, kn, ke);
    split2(ke, part, ka, kf);
    kp[0] = (int32_t)kn.k0;
    kp[1] = (int32_t)kn.k1;
    s_ka = ka;
    s_kf = kf;
  }
  for (int s = threadIdx.x; s < S; s += blockDim.x) parent[s] = s;
  __syncthreads();
  const uint32_t nb = (uint32_t)m * (uint32_t)pt.n;
  for (int j = threadIdx.x; j < m; j += blockDim.x) {
    const int a = randint_at(s_ka, (uint32_t)m, (uint32_t)j, 0, m, part);
    const int p = order[a];
    src[j] = p;
    parent[order[S - m + j]] = p;
    for (int i = 0; i < pt.n; ++i)
      fac[j * PBT_MAX_PERTURB + i] = pt.factor[randint_at(s_kf, nb, (uint32_t)(j * pt.n + i), 0, 2, part)];
  }
}

struct PbtRows {
  float* ptr[4];
  int64_t len[4];
};

// grid (x: row chunks, y: child j, z: array): child bottom[j] <- parent src[j], row by row of every array
__global__ void __launch_bounds__(PBT_THREADS) pbt_copy_rows_kernel(PbtRows rows, const int32_t* __restrict__ order,
                                                                    const int32_t* __restrict__ src, int S, int m) {
  const int j = blockIdx.y;
  float* base = rows.ptr[0];
  int64_t len = rows.len[0];
  switch (blockIdx.z) {   // constant indices: a dynamic index would copy the kernel parameters to local memory
    case 1: base = rows.ptr[1]; len = rows.len[1]; break;
    case 2: base = rows.ptr[2]; len = rows.len[2]; break;
    case 3: base = rows.ptr[3]; len = rows.len[3]; break;
    default: break;
  }
  const int64_t c = order[S - m + j], p = src[j];
  for (int64_t i = (int64_t)blockIdx.x * PBT_THREADS + threadIdx.x; i < len; i += (int64_t)gridDim.x * PBT_THREADS)
    base[c * len + i] = base[p * len + i];
}

__device__ __forceinline__ float toward_one(float x, float phi) {   // 1 - (1 - x) * phi, clamped to [0, 1]
  const float y = __fsub_rn(1.0f, __fmul_rn(__fsub_rn(1.0f, x), phi));
  return fminf(fmaxf(y, 0.0f), 1.0f);
}

// grid (x: eps row chunks, y: child j): the eps rows [eps_from, eps_rows) of column bottom[j]; block x == 0 also
// copies and perturbs the child's scalars
__global__ void __launch_bounds__(PBT_THREADS) pbt_tables_kernel(
    const int32_t* __restrict__ order, const int32_t* __restrict__ src, const float* __restrict__ fac, int S, int m,
    float* __restrict__ eps, int eps_rows, int eps_from, int32_t* __restrict__ sched_src, float* __restrict__ lr_mult,
    float* __restrict__ gamma, float* __restrict__ lam, float* __restrict__ max_norm, float* __restrict__ rew_scale,
    PbtPerturb pt) {
  const int j = blockIdx.y;
  const int c = order[S - m + j], p = src[j];
  for (int r = eps_from + blockIdx.x * PBT_THREADS + threadIdx.x; r < eps_rows; r += gridDim.x * PBT_THREADS)
    eps[(int64_t)r * S + c] = eps[(int64_t)r * S + p];
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  float lr = lr_mult[p], g = gamma[p], l = lam[p], mn = max_norm[p], rs = rew_scale[p];
  for (int i = 0; i < pt.n; ++i) {
    const float phi = fac[j * PBT_MAX_PERTURB + i];
    switch (pt.code[i]) {
      case PQN_PBT_LR: lr = __fmul_rn(lr, phi); break;
      case PQN_PBT_MAX_GRAD_NORM: mn = __fmul_rn(mn, phi); break;
      case PQN_PBT_REW_SCALE: rs = __fmul_rn(rs, phi); break;
      case PQN_PBT_GAMMA: g = toward_one(g, phi); break;
      case PQN_PBT_LAMBDA: l = toward_one(l, phi); break;
    }
  }
  sched_src[c] = sched_src[p];
  lr_mult[c] = lr;
  gamma[c] = g;
  lam[c] = l;
  max_norm[c] = mn;
  rew_scale[c] = rs;
}

}  // namespace pqn

using namespace pqn;

extern "C" {

int64_t pqn_pbt_workspace_bytes(int32_t S, int32_t m) {
  if (S <= 0 || m <= 0) return 0;
  return ws_bytes(S, m);
}

int pqn_pbt_event(const pqn_pbt_event_t* e, void* stream) {
  if (!e) return set_error(PQN_E_INVALID, "pqn_pbt_event: NULL arguments");
  const int S = e->S, m = e->m;
  if (S < 2 || S > 65535 || m < 1 || 2 * m > S)
    return set_error(PQN_E_INVALID, "pqn_pbt_event: need 2 <= S <= 65535 and 1 <= m <= S/2 (S=%d, m=%d)", S, m);
  if (!e->fit || e->fit_cols < 1 || e->fit_stride < e->fit_cols || !e->key || !e->fitness || !e->order ||
      !e->parent || !e->workspace)
    return set_error(PQN_E_INVALID, "pqn_pbt_event: bad fitness, key, output or workspace argument");
  if (e->n_perturb < 0 || e->n_perturb > PBT_MAX_PERTURB || !(e->factors[0] > 0.f) || !(e->factors[1] > 0.f))
    return set_error(PQN_E_INVALID, "pqn_pbt_event: bad perturbation (n_perturb=%d)", e->n_perturb);
  PbtPerturb pt;
  pt.n = e->n_perturb;
  pt.factor[0] = e->factors[0];
  pt.factor[1] = e->factors[1];
  int seen = 0;
  for (int i = 0; i < PBT_MAX_PERTURB; ++i) pt.code[i] = -1;
  for (int i = 0; i < pt.n; ++i) {
    const int c = e->perturb[i];
    if (c < 0 || c >= PBT_MAX_PERTURB || (seen >> c & 1))
      return set_error(PQN_E_INVALID, "pqn_pbt_event: perturb[%d]=%d is not a distinct PQN_PBT_* key", i, c);
    seen |= 1 << c;
    pt.code[i] = c;
  }
  PbtRows rows;
  int narr = 0;
  float* arr[4] = {e->params, e->mu, e->nu, e->batch_stats};
  const int64_t len[4] = {e->P, e->P, e->P, e->stats_floats};
  for (int a = 0; a < 4; ++a) {
    if (a < 3 && (!arr[a] || len[a] <= 0))
      return set_error(PQN_E_INVALID, "pqn_pbt_event: params, mu and nu are required (P=%lld)", (long long)e->P);
    if (a == 3 && (!arr[a] || len[a] <= 0)) continue;
    rows.ptr[narr] = arr[a];
    rows.len[narr] = len[a];
    ++narr;
  }
  if (!e->eps || e->eps_rows < 0 || e->eps_from < 0 || !e->sched_src || !e->lr_mult || !e->gamma || !e->lambda_ ||
      !e->max_norm || !e->rew_scale)
    return set_error(PQN_E_INVALID, "pqn_pbt_event: a per-seed table is missing");
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)e->workspace;
  unsigned long long* keys = (unsigned long long*)ws;
  int32_t* src = (int32_t*)(ws + ws_src_off(S));
  float* fac = (float*)(ws + ws_fac_off(S, m));
  const unsigned nbs = (unsigned)((S + PBT_THREADS - 1) / PBT_THREADS);
  { LaunchScope _ls(K_PBT, st); pbt_fitness_kernel<<<nbs, PBT_THREADS, 0, st>>>(e->fit, e->fit_stride, e->fit_cols, S, e->fitness, keys); }
  { LaunchScope _ls(K_PBT, st); pbt_rank_kernel<<<nbs, PBT_THREADS, 0, st>>>(keys, S, e->order); }
  { LaunchScope _ls(K_PBT, st); pbt_plan_kernel<<<1, 1024, 0, st>>>(e->key, e->rng_mode ? 1 : 0, S, m, e->order, e->parent, src, fac, pt); }
  int64_t longest = 0;
  for (int a = 0; a < narr; ++a) longest = rows.len[a] > longest ? rows.len[a] : longest;
  const unsigned nbr = (unsigned)((longest + PBT_THREADS * 4 - 1) / (PBT_THREADS * 4));
  { LaunchScope _ls(K_PBT, st); pbt_copy_rows_kernel<<<dim3(nbr, m, narr), PBT_THREADS, 0, st>>>(rows, e->order, src, S, m); }
  const int eps_n = e->eps_rows > e->eps_from ? e->eps_rows - e->eps_from : 0;
  const unsigned nbe = (unsigned)((eps_n + PBT_THREADS - 1) / PBT_THREADS) > 0 ? (unsigned)((eps_n + PBT_THREADS - 1) / PBT_THREADS) : 1u;
  { LaunchScope _ls(K_PBT, st); pbt_tables_kernel<<<dim3(nbe, m), PBT_THREADS, 0, st>>>(
        e->order, src, fac, S, m, e->eps, e->eps_rows, e->eps_from, e->sched_src, e->lr_mult, e->gamma, e->lambda_,
        e->max_norm, e->rew_scale, pt); }
  return check_launch("pqn_pbt_event");
}

}  // extern "C"
