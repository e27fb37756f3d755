// libpqn_b200.so: version, error slot, launch counter and per-kernel event timing.
#include <stdarg.h>
#include <stdio.h>

#include <vector>

#include "../../include/pqn_b200.h"
#include "api_common.h"

namespace pqn {
static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int check_launch(const char* what) {
  const cudaError_t e = cudaPeekAtLastError();
  if (e == cudaSuccess) return PQN_OK;
  cudaGetLastError();  // clear the sticky launch error so later calls report their own
  return set_error(PQN_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

int device_sm_count() {
  static int cache[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && cache[dev] > 0) return cache[dev];
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  if (dev >= 0 && dev < 64) cache[dev] = n;
  return n;
}

static const char* const kNames[K_COUNT] = {
    "env_reset", "env_step", "env_obs", "eps_greedy", "rollout_act_step", "rollout_keys", "qlambda", "rng",
    "conv_fwd", "dense_fwd", "row_bwd", "wgrad", "dgrad", "conv_bwd", "gather_rows", "sqnorm", "radam", "advance",
    "bn_update", "tc_gemm", "tc_split", "tc_dense_fwd", "tc_wgrad", "tc_dgrad", "net_init",
    "conv_fwd_infer", "tc_dense_fwd_head", "norm_fwd", "norm_bwd", "norm_reduce", "rnn_scan", "rnn_misc",
    "grad_finalize", "permutation", "bits_dense_fwd", "bits_wgrad", "pbt"};

struct Span { int id; cudaEvent_t a, b; };
static long long g_launches = 0;
static bool g_prof = false;
static std::vector<Span> g_spans;
static std::vector<cudaEvent_t> g_pool;
static cudaEvent_t g_cur = nullptr;

static cudaEvent_t get_event() {
  if (!g_pool.empty()) { cudaEvent_t e = g_pool.back(); g_pool.pop_back(); return e; }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}

void prof_begin(int id, cudaStream_t st) {
  ++g_launches;
  if (!g_prof) return;
  g_cur = get_event();
  cudaEventRecord(g_cur, st);
}
void prof_end(int id, cudaStream_t st) {
  if (!g_prof || !g_cur) return;
  cudaEvent_t b = get_event();
  cudaEventRecord(b, st);
  g_spans.push_back(Span{id, g_cur, b});
  g_cur = nullptr;
}
}  // namespace pqn

using namespace pqn;

extern "C" {
const char* pqn_last_error(void) { return g_err; }
int pqn_version(void) { return 100; }  // 0.1.0

long long pqn_launch_count(void) { return g_launches; }
int pqn_num_kernels(void) { return K_COUNT; }
const char* pqn_kernel_name(int id) { return (id >= 0 && id < K_COUNT) ? kNames[id] : ""; }

int pqn_profile_enable(int on) {
  g_prof = on != 0;
  return PQN_OK;
}

int pqn_profile_read(double* ms_host, long long* count_host, int reset) {
  if (!ms_host || !count_host) return set_error(PQN_E_INVALID, "pqn_profile_read: NULL output");
  for (int i = 0; i < K_COUNT; ++i) { ms_host[i] = 0.0; count_host[i] = 0; }
  for (const Span& s : g_spans) {
    if (cudaEventSynchronize(s.b) != cudaSuccess) return check_launch("pqn_profile_read");
    float ms = 0.f;
    cudaEventElapsedTime(&ms, s.a, s.b);
    ms_host[s.id] += ms;
    count_host[s.id] += 1;
  }
  if (reset) {
    for (const Span& s : g_spans) { g_pool.push_back(s.a); g_pool.push_back(s.b); }
    g_spans.clear();
  }
  return PQN_OK;
}
}
