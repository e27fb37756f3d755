// CPU logic harness of the bsuite envs — TEST INFRASTRUCTURE ONLY (built by tests/test_memory_chain_host.py).
// Compiles the same __host__ __device__ per-env functions the CUDA kernels use (env_bsuite.cuh, rollout_logic.cuh)
// with g++, in the order the kernels of pqn_env.cu call them, so that MemoryChain-bsuite can be checked bit for bit
// against the oracle without a GPU.  The product never calls this.
#include <stdint.h>

#include "../purejaxql_b200/csrc/env_bsuite.cuh"
#include "../purejaxql_b200/csrc/rollout_logic.cuh"

using namespace pqn;
using Env = MemoryChainEnv;

static void obs_out(const Env::State& s, float* obs, int64_t i) {
  float o[Env::OBS_DIM];
  Env::obs_float(s, o);
  for (int f = 0; f < Env::OBS_DIM; ++f) obs[i * Env::OBS_DIM + f] = o[f];
}

extern "C" {
int h_mc_state_words(void) { return Env::STATE_WORDS; }

// env_reset_kernel
void h_mc_reset(const uint32_t* keys, uint32_t* state, float* obs, int64_t N, int memory_length, int part) {
  for (int64_t i = 0; i < N; ++i) {
    Env::State s;
    env_set_params(s, EnvParams{memory_length});
    Env::reset_env(Key{keys[2 * i], keys[2 * i + 1]}, part, Env::DEFAULT_MAX_STEPS, s);
    Env::store(s, state, N, i);
    LogState lg;
    log_reset(lg);
    log_store(lg, state, N, i, Env::CORE_WORDS);
    obs_out(s, obs, i);
  }
}

// env_step_kernel
void h_mc_step(const uint32_t* keys, uint32_t* state, const int32_t* action, float* obs, float* reward, uint8_t* done,
               int64_t N, int part) {
  for (int64_t i = 0; i < N; ++i) {
    Env::State s;
    Env::load(s, state, N, i);
    LogState lg;
    log_load(lg, state, N, i, Env::CORE_WORDS);
    float r;
    bool d;
    env_step_full<Env>(Key{keys[2 * i], keys[2 * i + 1]}, part, Env::DEFAULT_MAX_STEPS, s, lg, action[i], r, d);
    Env::store(s, state, N, i);
    log_store(lg, state, N, i, Env::CORE_WORDS);
    reward[i] = r;
    done[i] = d;
    obs_out(s, obs, i);
  }
}

// env_obs_kernel
void h_mc_obs(const uint32_t* state, float* obs, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    Env::State s;
    Env::load(s, state, N, i);
    obs_out(s, obs, i);
  }
}
}
