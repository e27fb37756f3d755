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

// gymnax bsuite/deep_sea.py (DeepSea-bsuite) with the constructor's size 8 and the default EnvParams
// (deterministic = True, unscaled_move_cost = 0.01).  Restated from recollection of gymnax 0.0.6:
//   reset_env:  row = column = 0, bad_episode = False, total_bad_episodes = denoised_return = 0,
//               optimal_no_cost = 1.0, optimal_return = optimal_no_cost - unscaled_move_cost, time = 0;
//               action_mapping = ones((8, 8)) under deterministic = True (a per-env bernoulli draw otherwise)
//   step_env:   right = action == action_mapping[row, column];
//               reward = 0.0 + (right & row == 7 & column == 7) - right * unscaled_move_cost / 8;
//               a left move at row == column sets bad_episode; column = clip(column +- 1, 0, 7); row += 1;
//               total_bad_episodes += bad_episode at row == 8; time += 1;
//               done = row == 8 || time >= max_steps_in_episode, so an episode lasts 8 steps
//   get_obs:    the (8, 8) one-hot of (row, column), all zeros once row == 8
// gymnax's step_env also draws a uniform (a right move succeeds when it exceeds 1 / size, or under deterministic) and
// a normal (reward noise, multiplied by 1 - deterministic) from its key.  At deterministic = True the uniform's
// condition is or-ed with True, and the noise term is 0 * finite = +-0.0 (jax.random.normal is finite: it maps a
// uniform in (-1, 1) through erfinv).  Adding +-0.0 to a reward that starts as +0.0 + bool leaves it bit for bit as
// it is (+0 + -0 = +0 in round-to-nearest), so neither draw can reach an output and this step does not make them.
// Integer work plus fp32 constants: bit-exact.
struct DeepSeaEnv {
  static constexpr int ID = ENV_DEEP_SEA;
  static constexpr int SIZE = 8;
  static constexpr int CORE_WORDS = 8;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 2;
  static constexpr int OBS_DIM = SIZE * SIZE;
  static constexpr int OBS_ROWS = SIZE, OBS_COLS = SIZE;  // gymnax's (8, 8) board, unflattened
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 2000;  // EnvParams.max_steps_in_episode; episodes end on the last row
  static constexpr float UNSCALED_MOVE_COST = 0.01f;
  static constexpr float MOVE_COST = UNSCALED_MOVE_COST / SIZE;  // exact: a power-of-two divisor

  // word 0: row | column << 8 | bad_episode << 16;  1: total_bad_episodes;  2: denoised_return;
  // 3, 4: optimal_return, optimal_no_cost (fp32 bits);  5, 6: action_mapping, bit 8 * row + column;  7: time
  struct State {
    int row, column, bad_episode, total_bad_episodes, denoised_return;
    float optimal_return, optimal_no_cost;
    uint32_t map_lo, map_hi;
    int time;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    const uint32_t w = (uint32_t)st[i];
    s.row = (int)(w & 255u); s.column = (int)((w >> 8) & 255u); s.bad_episode = (int)((w >> 16) & 1u);
    s.total_bad_episodes = (int)st[N + i]; s.denoised_return = (int)st[2 * N + i];
    s.optimal_return = u2f((uint32_t)st[3 * N + i]); s.optimal_no_cost = u2f((uint32_t)st[4 * N + i]);
    s.map_lo = (uint32_t)st[5 * N + i]; s.map_hi = (uint32_t)st[6 * N + i]; s.time = (int)st[7 * N + i];
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = (uint32_t)s.row | ((uint32_t)s.column << 8) | ((uint32_t)s.bad_episode << 16);
    st[N + i] = (uint32_t)s.total_bad_episodes; st[2 * N + i] = (uint32_t)s.denoised_return;
    st[3 * N + i] = f2u(s.optimal_return); st[4 * N + i] = f2u(s.optimal_no_cost);
    st[5 * N + i] = s.map_lo; st[6 * N + i] = s.map_hi; st[7 * N + i] = (uint32_t)s.time;
  }

  PQN_HD static void reset_env(Key /*key*/, int /*part*/, int /*max_steps*/, State& s) {
    s.row = 0; s.column = 0; s.bad_episode = 0; s.total_bad_episodes = 0; s.denoised_return = 0;
    s.optimal_no_cost = 1.0f;
    s.optimal_return = s.optimal_no_cost - UNSCALED_MOVE_COST;
    s.map_lo = 0xFFFFFFFFu; s.map_hi = 0xFFFFFFFFu;  // ones((8, 8)): deterministic = True
    s.time = 0;
  }

  PQN_HD static void step_env(Key /*key*/, int /*part*/, int max_steps, State& s, int action, float& reward,
                              bool& done) {
    const int bit = s.row * SIZE + s.column;
    const uint32_t map_word = bit < 32 ? s.map_lo : s.map_hi;
    const bool right = action == (int)((map_word >> (bit & 31)) & 1u);
    const bool treasure = right && s.row == SIZE - 1 && s.column == SIZE - 1;
    reward = (treasure ? 1.f : 0.f) - (right ? MOVE_COST : 0.f);
    s.denoised_return += treasure ? 1 : 0;
    if (!right && s.row == s.column) s.bad_episode = 1;
    s.column = right ? (s.column + 1 > SIZE - 1 ? SIZE - 1 : s.column + 1) : (s.column - 1 < 0 ? 0 : s.column - 1);
    s.row = s.row + 1;
    if (s.row == SIZE) s.total_bad_episodes += s.bad_episode;
    s.time = s.time + 1;
    done = s.row == SIZE || s.time >= max_steps;
  }

  // compares instead of an indexed write, so that `o` stays in registers
  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) {
    const int hot = s.row < SIZE ? s.row * SIZE + s.column : -1;
#pragma unroll
    for (int j = 0; j < OBS_DIM; ++j) o[j] = j == hot ? 1.f : 0.f;
  }
};

// gymnax bsuite/umbrella_chain.py (UmbrellaChain-bsuite) with n_distractor = 0, as `gymnax.make` builds it, and
// chain_length = 10.  Restated from recollection of gymnax 0.0.6:
//   reset_env:  k_need, k_has, k_obs = split(key, 3); need_umbrella = bernoulli(k_need, 0.5, ()),
//               has_umbrella = bernoulli(k_has, 0.5, ()), total_regret = 0, time = 0 (k_obs feeds the distractors)
//   step_env:   k_reward, k_obs = split(key); has_umbrella = action if time == 0;
//               chain_full = time + 1 == chain_length;
//               reward = +-1 by has_umbrella == need_umbrella if chain_full, else 2 * bernoulli(k_reward, 0.5, ()) - 1;
//               total_regret += 2 * (chain_full & !match); time += 1;
//               done = time == chain_length || time >= max_steps_in_episode, so an episode lasts 10 steps
//   get_obs:    [need_umbrella, has_umbrella, 1 - time / chain_length]
// Integer logic plus one fp32 division: bit-exact.
struct UmbrellaChainEnv {
  static constexpr int ID = ENV_UMBRELLA_CHAIN;
  static constexpr int CHAIN_LENGTH = 10;
  static constexpr int CORE_WORDS = 4;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 2;
  static constexpr int OBS_DIM = 3;  // 3 + n_distractor, flattened from (1, 3)
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 100;  // EnvParams.max_steps_in_episode; episodes end on chain_length

  // words: need_umbrella, has_umbrella, total_regret, time
  struct State {
    int need_umbrella, has_umbrella, total_regret, time;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    s.need_umbrella = (int)st[i]; s.has_umbrella = (int)st[N + i]; s.total_regret = (int)st[2 * N + i];
    s.time = (int)st[3 * N + i];
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = (uint32_t)s.need_umbrella; st[N + i] = (uint32_t)s.has_umbrella;
    st[2 * N + i] = (uint32_t)s.total_regret; st[3 * N + i] = (uint32_t)s.time;
  }

  PQN_HD static int coin(Key k, int part) { return uniform_scalar(k, part) < 0.5f ? 1 : 0; }  // bernoulli(k, 0.5, ())

  PQN_HD static void reset_env(Key key, int part, int /*max_steps*/, State& s) {
    Key k_need, k_has, k_obs;
    split3(key, part, k_need, k_has, k_obs);
    s.need_umbrella = coin(k_need, part);
    s.has_umbrella = coin(k_has, part);
    s.total_regret = 0; s.time = 0;
  }

  PQN_HD static void step_env(Key key, int part, int max_steps, State& s, int action, float& reward, bool& done) {
    if (s.time == 0) s.has_umbrella = action;
    const bool chain_full = s.time + 1 == CHAIN_LENGTH;
    const bool match = s.has_umbrella == s.need_umbrella;
    if (chain_full) {
      reward = match ? 1.f : -1.f;
    } else {
      Key k_reward, k_obs;
      split2(key, part, k_reward, k_obs);
      reward = (float)(2 * coin(k_reward, part) - 1);
    }
    s.total_regret += (chain_full && !match) ? 2 : 0;
    s.time = s.time + 1;
    done = s.time == CHAIN_LENGTH || s.time >= max_steps;
  }

  // fp32 IEEE division (this TU is built with -fmad=false and the division is not fast-math)
  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) {
    o[0] = (float)s.need_umbrella;
    o[1] = (float)s.has_umbrella;
    o[2] = 1.0f - (float)s.time / (float)CHAIN_LENGTH;
  }
};

// gymnax bsuite/discounting_chain.py (DiscountingChain-bsuite) with mapping_seed = None, as `gymnax.make` builds it.
// Restated from recollection of gymnax 0.0.6:
//   reset_env:  context = -1, time = 0; rewards = ones(5).at[randint(key, (), 0, 5)].set(1.1)
//   step_env:   context = action if time == 0; time += 1;
//               reward = rewards[context] if time == reward_timestep[context] else 0.0,
//               reward_timestep = [1, 3, 10, 30, 100]; done = time >= max_steps_in_episode (100)
//   get_obs:    [context, time / max_steps_in_episode]
// The state keeps the index of the 1.1 reward (mapped_action) rather than the five rewards, so a mapping fixed by
// mapping_seed fits the same word.  It also keeps max_steps_in_episode, the observation's divisor: the reset kernels
// pass it to reset_env, and the auto-reset inside a step passes the same value.  Integer logic plus one fp32 division:
// bit-exact.
struct DiscountingChainEnv {
  static constexpr int ID = ENV_DISCOUNTING_CHAIN;
  static constexpr int CORE_WORDS = 4;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 5;
  static constexpr int OBS_DIM = 2;  // flattened from (1, 2)
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 100;  // EnvParams.max_steps_in_episode: every episode lasts this long
  static constexpr float MAPPED_REWARD = 1.1f;

  PQN_HD static int reward_timestep(int context) {
    return context == 0 ? 1 : context == 1 ? 3 : context == 2 ? 10 : context == 3 ? 30 : 100;
  }

  // words: context (-1 until the first step), mapped_action, time, max_steps_in_episode
  struct State {
    int context, mapped_action, time, max_steps;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    s.context = (int)st[i]; s.mapped_action = (int)st[N + i]; s.time = (int)st[2 * N + i];
    s.max_steps = (int)st[3 * N + i];
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = (uint32_t)s.context; st[N + i] = (uint32_t)s.mapped_action; st[2 * N + i] = (uint32_t)s.time;
    st[3 * N + i] = (uint32_t)s.max_steps;
  }

  PQN_HD static void reset_env(Key key, int part, int max_steps, State& s) {
    s.context = -1;
    s.mapped_action = randint_scalar(key, (uint32_t)NUM_ACTIONS, part);
    s.time = 0;
    s.max_steps = max_steps;
  }

  PQN_HD static void step_env(Key /*key*/, int /*part*/, int max_steps, State& s, int action, float& reward,
                              bool& done) {
    if (s.time == 0) s.context = action;
    s.time = s.time + 1;
    reward = s.time == reward_timestep(s.context) ? (s.context == s.mapped_action ? MAPPED_REWARD : 1.0f) : 0.f;
    done = s.time >= max_steps;
  }

  // fp32 IEEE division (this TU is built with -fmad=false and the division is not fast-math)
  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) {
    o[0] = (float)s.context;
    o[1] = (float)s.time / (float)s.max_steps;
  }
};

// gymnax bsuite/bandit.py (SimpleBandit-bsuite) with the constructor's num_actions = 11 and the default EnvParams
// (optimal_return = 1).  Restated from recollection of gymnax 0.0.6:
//   reset_env:  action_mask = choice(key, arange(11), (11,), replace=False), which is permutation(key, arange(11));
//               rewards = linspace(0, 1, 11)[action_mask], total_regret = 0.0, time = 0
//   step_env:   reward = rewards[action]; total_regret += optimal_return - reward; time += 1;
//               done = is_terminal = True: every step ends the episode, so every step auto-resets and redraws
//   get_obs:    ones((1, 1))
// permutation is jax's _shuffle: ceil(3 ln 11 / ln(2^32 - 1)) = 1 round, a stable sort of arange(11) by
// random_bits(sub, 32, (11,)) with (key, sub) = split(key).  jnp.linspace in jax 0.4.x computes
// start * (1 - step) + stop * step with step = iota / 10 in fp32, which at start 0 and stop 1 is the quotient k / 10.
// The state keeps action_mask (4 bits per action), so reward = action_mask[action] / 10.  Integer work plus one fp32
// division: bit-exact.
struct SimpleBanditEnv {
  static constexpr int ID = ENV_SIMPLE_BANDIT;
  static constexpr int CORE_WORDS = 5;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 11;
  static constexpr int OBS_DIM = 1;
  static constexpr int OBS_ROWS = 1, OBS_COLS = 1;  // gymnax's (1, 1) observation, unflattened
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 100;  // EnvParams.max_steps_in_episode; every step is terminal anyway
  static constexpr float OPTIMAL_RETURN = 1.0f;

  // words 0, 1: action_mask, entry j in bits 4 (j mod 8) of word j / 8;  2: total_regret (fp32 bits);  3: time;
  // 4: optimal_return (fp32 bits, the EnvParams word the step reads)
  struct State {
    uint32_t mask_lo, mask_hi;
    float total_regret;
    int time;
    float optimal_return;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    s.mask_lo = (uint32_t)st[i]; s.mask_hi = (uint32_t)st[N + i]; s.total_regret = u2f((uint32_t)st[2 * N + i]);
    s.time = (int)st[3 * N + i]; s.optimal_return = u2f((uint32_t)st[4 * N + i]);
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = s.mask_lo; st[N + i] = s.mask_hi; st[2 * N + i] = f2u(s.total_regret); st[3 * N + i] = (uint32_t)s.time;
    st[4 * N + i] = f2u(s.optimal_return);
  }

  PQN_HD static void reset_env(Key key, int part, int /*max_steps*/, State& s) {
    Key k_next, sub;
    split2(key, part, k_next, sub);
    uint32_t sk[NUM_ACTIONS];
#pragma unroll
    for (int j = 0; j < NUM_ACTIONS; ++j) sk[j] = bits_at(sub, (uint32_t)NUM_ACTIONS, (uint32_t)j, part);
    // stable sort: element j lands at its rank, the number of keys below it plus the equal keys before it
    uint32_t lo = 0u, hi = 0u;
#pragma unroll
    for (int j = 0; j < NUM_ACTIONS; ++j) {
      int rank = 0;
#pragma unroll
      for (int i = 0; i < NUM_ACTIONS; ++i) rank += (sk[i] < sk[j] || (sk[i] == sk[j] && i < j)) ? 1 : 0;
      if (rank < 8) lo |= (uint32_t)j << (4 * rank); else hi |= (uint32_t)j << (4 * (rank - 8));
    }
    s.mask_lo = lo; s.mask_hi = hi;
    s.total_regret = 0.f; s.time = 0;
    s.optimal_return = OPTIMAL_RETURN;
  }

  PQN_HD static int mask_at(const State& s, int j) {
    return (int)(((j < 8 ? s.mask_lo : s.mask_hi) >> (4 * (j & 7))) & 15u);
  }

  PQN_HD static void step_env(Key /*key*/, int /*part*/, int /*max_steps*/, State& s, int action, float& reward,
                              bool& done) {
    reward = (float)mask_at(s, action) / 10.0f;
    s.total_regret = s.total_regret + s.optimal_return - reward;
    s.time = s.time + 1;
    done = true;
  }

  PQN_HD static void obs_float(const State& /*s*/, float (&o)[OBS_DIM]) { o[0] = 1.f; }
};

}  // namespace pqn
