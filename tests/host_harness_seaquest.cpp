// CPU logic harness of Seaquest-MinAtar — TEST INFRASTRUCTURE ONLY (built by tests/test_seaquest_host.py).  Compiles
// the same __host__ __device__ functions the CUDA kernels use (env_seaquest.cuh, rollout_logic.cuh) with g++, in the
// order the kernels of pqn_env.cu call them, so that the env can be checked against tests/seaquest_oracle.py without
// a GPU.  The product never calls this.
#include <stdint.h>

#include "../purejaxql_b200/csrc/env_seaquest.cuh"
#include "../purejaxql_b200/csrc/rollout_logic.cuh"

using namespace pqn;
using Env = SeaquestEnv;

static void obs_out(const Env::State& s, float* obs, int64_t i) {
  uint32_t bits[Env::OBS_WORDS_PAD];
  for (int w = 0; w < Env::OBS_WORDS_PAD; ++w) bits[w] = 0u;
  Env::obs_bits_mem(s, bits, 1);
  for (int f = 0; f < Env::OBS_DIM; ++f) obs[i * Env::OBS_DIM + f] = (float)((bits[f >> 5] >> (f & 31)) & 1u);
}

extern "C" {
int h_sq_state_words(void) { return Env::STATE_WORDS; }
int h_sq_obs_dim(void) { return Env::OBS_DIM; }
int h_sq_max_steps(void) { return Env::DEFAULT_MAX_STEPS; }

// env_reset_kernel
void h_sq_reset(const uint32_t* keys, uint32_t* state, float* obs, int64_t N, int max_steps, int part) {
  for (int64_t i = 0; i < N; ++i) {
    Env::State s;
    Env::reset_env(Key{keys[2 * i], keys[2 * i + 1]}, part, max_steps, s);
    Env::store(s, state, N, i);
    LogState lg;
    log_reset(lg);
    log_store(lg, state, N, i, Env::CORE_WORDS);
    obs_out(s, obs, i);
  }
}

// env_step_kernel
void h_sq_step(const uint32_t* keys, uint32_t* state, const int32_t* action, float* obs, float* reward, uint8_t* done,
               int64_t N, int max_steps, int part) {
  for (int64_t i = 0; i < N; ++i) {
    Env::State s;
    Env::load(s, state, N, i);
    LogState lg;
    log_load(lg, state, N, i, Env::CORE_WORDS);
    float r;
    bool d;
    env_step_full<Env>(Key{keys[2 * i], keys[2 * i + 1]}, part, max_steps, s, lg, action[i], r, d);
    Env::store(s, state, N, i);
    log_store(lg, state, N, i, Env::CORE_WORDS);
    reward[i] = r;
    done[i] = d;
    obs_out(s, obs, i);
  }
}

// env_obs_kernel
void h_sq_obs(const uint32_t* state, float* out, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    Env::State s;
    Env::load(s, state, N, i);
    obs_out(s, out, i);
  }
}
}
