// Error plumbing + launch accounting shared by the translation units of
// libpqn_b200.so.
#pragma once
#include <cuda_runtime.h>

namespace pqn {
// records a printf-style message in the thread-local error slot and returns `code`
int set_error(int code, const char* fmt, ...);
// cudaPeekAtLastError() after a launch: 0 or PQN_E_CUDA (message recorded)
int check_launch(const char* what);

// kernel ids for the launch counter / per-kernel CUDA-event timing (pqn_profile_*)
enum KernelId : int {
  K_ENV_RESET = 0, K_ENV_STEP, K_ENV_OBS, K_EPS_GREEDY, K_ROLLOUT_ACT_STEP, K_ROLLOUT_KEYS, K_QLAMBDA, K_RNG,
  K_CONV_FWD, K_DENSE_FWD, K_ROW_BWD, K_WGRAD, K_DGRAD, K_CONV_BWD, K_GATHER_ROWS, K_SQNORM, K_RADAM, K_ADVANCE,
  K_BN_UPDATE, K_TC_GEMM, K_TC_SPLIT, K_TC_FWD, K_TC_WGRAD, K_TC_DGRAD, K_NET_INIT,
  K_CONV_FWD_INFER /* rollout / evaluation variant */, K_TC_FWD_HEAD /* forward GEMM with the Q-head epilogue */,
  K_NORM_FWD, K_NORM_BWD, K_NORM_REDUCE /* modular NORM_TYPE / NORM_INPUT path (pqn_norm.cuh) */,
  K_RNN_SCAN, K_RNN_MISC /* GRU network (pqn_rnn.cuh) */,
  K_GRAD_FINAL /* fixed-order second stage of the deterministic gradient reductions */,
  K_PERM /* jax.random.permutation bucket + rank sort (pqn_perm.cu) */,
  K_BITS_FWD, K_BITS_WGRAD /* Dense_0 of the MLP on packed MinAtar bits (pqn_bits.cuh) */,
  K_PBT /* population-based training event (pqn_pbt.cu) */, K_COUNT
};

// A hyperparameter that may differ between seeds: v[seed] when v is given (the *_seeds entry points), else the value c
// every seed shares (the scalar entry points).  Passed by value to the kernel that reads it.
struct SeedScalar {
  const float* v;
  float c;
#ifdef __CUDACC__
  __device__ __forceinline__ float at(int seed) const { return v ? __ldg(v + seed) : c; }
#endif
};

// SM count of the CURRENT device (cached per device ordinal, not per process)
int device_sm_count();

void prof_begin(int id, cudaStream_t st);
void prof_end(int id, cudaStream_t st);

// Wrap exactly one kernel launch: counts it and, when profiling is on, brackets
// it with CUDA events on the launching stream.
struct LaunchScope {
  int id;
  cudaStream_t st;
  LaunchScope(int id_, cudaStream_t st_) : id(id_), st(st_) { prof_begin(id, st); }
  ~LaunchScope() { prof_end(id, st); }
};
}  // namespace pqn
