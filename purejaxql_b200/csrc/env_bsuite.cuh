// bsuite memory tasks as gymnax builds them (MemoryChain-bsuite), one env per thread.
//
// Restates gymnax==0.0.6 gymnax/environments/bsuite/memory_chain.py (third party; call sites
// purejaxql/pqn_rnn_gymnax.py:134-139) with num_bits = 1, the only value `gymnax.make("MemoryChain-bsuite")` builds:
//   reset_env:  k_ctx, k_q = split(key); context = bernoulli(k_ctx, 0.5, (1,)); query = randint(k_q, (), 0, 1) = 0
//   get_obs:    [1 - time / memory_length,  query if time == memory_length - 1 else 0,
//                2 context - 1 if time == 0 else 0]
//   step_env:   obs = get_obs(state) BEFORE time += 1; full = time - 1 >= memory_length (after the increment);
//               reward = (full & correct) - (full & !correct), correct = action == context[query];
//               done = time - 1 == memory_length, so an episode lasts memory_length + 1 steps.
// Integer logic plus one fp32 division: bit-exact against the reference.
//
// memory_length is an env parameter (EnvParams.memory_length, gymnax default 5).  It lives in a word of the state
// block: the reset kernels write it (env_set_params below), step_env leaves it alone and the auto-reset inside
// env_step_full keeps it, so pqn_env_step / pqn_env_obs / pqn_rollout_act_step need no extra argument.
#pragma once
#include "env_common.cuh"

namespace pqn {

struct MemoryChainEnv {
  static constexpr int ID = ENV_MEMORY_CHAIN;
  static constexpr int CORE_WORDS = 6;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 2;
  static constexpr int OBS_DIM = 3;  // num_bits + 2, flattened from (1, 3)
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 1000;  // EnvParams.max_steps_in_episode; episodes end on memory_length
  static constexpr int DEFAULT_MEMORY_LENGTH = 5;

  // words: context, query, total_perfect, total_regret, time, memory_length
  struct State {
    int context, query, total_perfect, total_regret, time, memory_length;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    s.context = (int)st[i]; s.query = (int)st[N + i]; s.total_perfect = (int)st[2 * N + i];
    s.total_regret = (int)st[3 * N + i]; s.time = (int)st[4 * N + i]; s.memory_length = (int)st[5 * N + i];
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = (uint32_t)s.context; st[N + i] = (uint32_t)s.query; st[2 * N + i] = (uint32_t)s.total_perfect;
    st[3 * N + i] = (uint32_t)s.total_regret; st[4 * N + i] = (uint32_t)s.time;
    st[5 * N + i] = (uint32_t)s.memory_length;
  }

  // Leaves s.memory_length as it is: the reset kernels set it first, the auto-reset carries the pre-step value.
  PQN_HD static void reset_env(Key key, int part, int /*max_steps*/, State& s) {
    Key k_ctx, k_q;
    split2(key, part, k_ctx, k_q);
    // bernoulli(k_ctx, 0.5, (1,)) = uniform(k_ctx, (1,)) < 0.5
    s.context = uniform_from_bits(bits_at(k_ctx, 1u, 0u, part), 0.0f, 1.0f) < 0.5f ? 1 : 0;
    s.query = 0;  // randint(k_q, (), 0, num_bits) with num_bits = 1 draws from a span of one value
    s.total_perfect = 0; s.total_regret = 0; s.time = 0;
  }

  PQN_HD static void step_env(Key /*key*/, int /*part*/, int /*max_steps*/, State& s, int action, float& reward,
                              bool& done) {
    s.time = s.time + 1;
    const bool full = s.time - 1 >= s.memory_length;
    const bool correct = action == s.context;  // context[query], query = 0
    const bool win = full && correct, lose = full && !correct;
    reward = (win ? 1.f : 0.f) - (lose ? 1.f : 0.f);
    s.total_perfect += win ? 1 : 0;
    s.total_regret += lose ? 2 : 0;
    done = s.time - 1 == s.memory_length;
  }

  // get_obs at time t (fp32 IEEE division: this TU is built with -fmad=false and the division is not fast-math).
  PQN_HD static void obs_at(const State& s, int t, float (&o)[OBS_DIM]) {
    o[0] = 1.0f - (float)t / (float)s.memory_length;
    o[1] = t == s.memory_length - 1 ? (float)s.query : 0.f;
    o[2] = t == 0 ? (float)(2 * s.context - 1) : 0.f;
  }

  // The observation returned together with `s`: step_env's obs is get_obs of the PRE-step state, i.e. at time - 1,
  // and reset's (also after an auto-reset) is get_obs at time 0.
  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) { obs_at(s, s.time > 0 ? s.time - 1 : 0, o); }
};

// Env parameters other than max_steps, stored in the state by the reset kernels.
PQN_HD void env_set_params(MemoryChainEnv::State& s, const EnvParams& p) { s.memory_length = p.memory_length; }

// gymnax bsuite/catch.py (Catch-bsuite) with the 10 x 5 board `gymnax.make` builds.  Restated from recollection of
// gymnax 0.0.6:
//   reset_env:  ball_x = randint(key, (), 0, 5), ball_y = 0, paddle_x = 2, paddle_y = 9, prev_done = False, time = 0
//   step_env:   paddle_x = clip(paddle_x + action - 1, 0, 4); ball_y += 1; prev_done = ball_y == paddle_y;
//               reward = prev_done * (1.0 * caught + -1.0 * (1 - caught)), caught = paddle_x == ball_x (so -0.0 on
//               the steps before the last where the paddle is not under the ball); time += 1;
//               done = ball_y == paddle_y || time >= max_steps, so an episode lasts 9 steps
//   get_obs:    zeros (10, 5), 1 set at (ball_y, ball_x) and at (paddle_y, paddle_x) (set, not added)
// gymnax's step_env also draws a fresh initial state from the step key and selects it where the incoming state has
// prev_done = True.  A state with prev_done = True is always terminal, so Environment.step's auto-reset replaces it
// before step_env can see it: the draw can never matter, and this step does not make it.  Integer work, bit-exact.
struct CatchEnv {
  static constexpr int ID = ENV_CATCH;
  static constexpr int ROWS = 10, COLUMNS = 5;
  static constexpr int CORE_WORDS = 2;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 3;
  static constexpr int OBS_DIM = ROWS * COLUMNS;
  static constexpr int OBS_ROWS = ROWS, OBS_COLS = COLUMNS;  // gymnax's (10, 5) board, unflattened
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 1000;  // EnvParams.max_steps_in_episode; episodes end on the last row

  // word 0: ball_x | ball_y << 4 | paddle_x << 8 | paddle_y << 12 | prev_done << 16;  word 1: time
  struct State {
    int ball_x, ball_y, paddle_x, paddle_y, prev_done, time;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    const uint32_t w = (uint32_t)st[i];
    s.ball_x = (int)(w & 15u); s.ball_y = (int)((w >> 4) & 15u); s.paddle_x = (int)((w >> 8) & 15u);
    s.paddle_y = (int)((w >> 12) & 15u); s.prev_done = (int)((w >> 16) & 1u); s.time = (int)st[N + i];
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = (uint32_t)s.ball_x | ((uint32_t)s.ball_y << 4) | ((uint32_t)s.paddle_x << 8) |
            ((uint32_t)s.paddle_y << 12) | ((uint32_t)s.prev_done << 16);
    st[N + i] = (uint32_t)s.time;
  }

  PQN_HD static void reset_env(Key key, int part, int /*max_steps*/, State& s) {
    s.ball_x = randint_scalar(key, (uint32_t)COLUMNS, part);
    s.ball_y = 0; s.paddle_x = COLUMNS / 2; s.paddle_y = ROWS - 1; s.prev_done = 0; s.time = 0;
  }

  PQN_HD static void step_env(Key /*key*/, int /*part*/, int max_steps, State& s, int action, float& reward,
                              bool& done) {
    const int px = s.paddle_x + action - 1;
    s.paddle_x = px < 0 ? 0 : (px > COLUMNS - 1 ? COLUMNS - 1 : px);
    s.ball_y = s.ball_y + 1;
    s.prev_done = s.ball_y == s.paddle_y ? 1 : 0;
    const bool caught = s.paddle_x == s.ball_x;
    reward = (float)s.prev_done * (caught ? 1.0f : -1.0f);
    s.time = s.time + 1;
    done = s.prev_done != 0 || s.time >= max_steps;
  }

  // compares instead of indexed writes, so that `o` stays in registers
  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) {
    const int ball = s.ball_y * COLUMNS + s.ball_x, paddle = s.paddle_y * COLUMNS + s.paddle_x;
#pragma unroll
    for (int j = 0; j < OBS_DIM; ++j) o[j] = (j == ball || j == paddle) ? 1.f : 0.f;
  }
};

}  // namespace pqn
