// CPU logic harness of SimpleBandit-bsuite, BernoulliBandit-misc, FourRooms-misc and MetaMaze-misc — TEST
// INFRASTRUCTURE ONLY (built by tests/test_misc_envs_host.py).  Compiles the same __host__ __device__ per-env functions
// the CUDA kernels use (env_bsuite.cuh, env_misc.cuh, rollout_logic.cuh) with g++, in the order the kernels of
// pqn_env.cu call them, so that the four envs can be checked against the oracles without a GPU.  The product never
// calls this.
#include <stdint.h>

#include "../purejaxql_b200/csrc/env_bsuite.cuh"
#include "../purejaxql_b200/csrc/env_misc.cuh"
#include "../purejaxql_b200/csrc/rollout_logic.cuh"

using namespace pqn;

template <class Env>
static void obs_out(const typename Env::State& s, float* obs, int64_t i) {
  float o[Env::OBS_DIM];
  Env::obs_float(s, o);
  for (int f = 0; f < Env::OBS_DIM; ++f) obs[i * Env::OBS_DIM + f] = o[f];
}

// env_reset_kernel
template <class Env>
static void reset(const uint32_t* keys, uint32_t* state, float* obs, int64_t N, int max_steps, int part) {
  for (int64_t i = 0; i < N; ++i) {
    typename Env::State s;
    Env::reset_env(Key{keys[2 * i], keys[2 * i + 1]}, part, max_steps, s);
    Env::store(s, state, N, i);
    LogState lg;
    log_reset(lg);
    log_store(lg, state, N, i, Env::CORE_WORDS);
    obs_out<Env>(s, obs, i);
  }
}

// env_step_kernel
template <class Env>
static void step(const uint32_t* keys, uint32_t* state, const int32_t* action, float* obs, float* reward,
                 uint8_t* done, int64_t N, int max_steps, int part) {
  for (int64_t i = 0; i < N; ++i) {
    typename Env::State s;
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
    obs_out<Env>(s, obs, i);
  }
}

// env_obs_kernel
template <class Env>
static void obs(const uint32_t* state, float* out, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    typename Env::State s;
    Env::load(s, state, N, i);
    obs_out<Env>(s, out, i);
  }
}

#define PQN_HARNESS(prefix, Env)                                                                                   \
  int h_##prefix##_state_words(void) { return Env::STATE_WORDS; }                                                  \
  int h_##prefix##_obs_dim(void) { return Env::OBS_DIM; }                                                          \
  int h_##prefix##_max_steps(void) { return Env::DEFAULT_MAX_STEPS; }                                              \
  void h_##prefix##_reset(const uint32_t* keys, uint32_t* state, float* o, int64_t N, int max_steps, int part) {   \
    reset<Env>(keys, state, o, N, max_steps, part);                                                                \
  }                                                                                                                \
  void h_##prefix##_step(const uint32_t* keys, uint32_t* state, const int32_t* action, float* o, float* reward,     \
                         uint8_t* done, int64_t N, int max_steps, int part) {                                      \
    step<Env>(keys, state, action, o, reward, done, N, max_steps, part);                                           \
  }                                                                                                                \
  void h_##prefix##_obs(const uint32_t* state, float* o, int64_t N) { obs<Env>(state, o, N); }

extern "C" {
PQN_HARNESS(simple_bandit, SimpleBanditEnv)
PQN_HARNESS(bernoulli_bandit, BernoulliBanditEnv)
PQN_HARNESS(four_rooms, FourRoomsEnv)
PQN_HARNESS(meta_maze, MetaMazeEnv)
}
