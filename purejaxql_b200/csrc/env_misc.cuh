// gymnax's discrete-action misc environments that need nothing external (BernoulliBandit-misc, GaussianBandit-misc,
// FourRooms-misc, MetaMaze-misc), one env per thread, with gymnax's default constructor arguments and EnvParams.
//
// Restated from recollection of gymnax==0.0.6 gymnax/environments/misc/ (third party; call sites
// purejaxql/pqn_gymnax.py:92 and purejaxql/pqn_rnn_gymnax.py:133-139, `gymnax.make(config["ENV_NAME"])`).
// tests/misc_envs_oracle.py and tests/gaussian_bandit_oracle.py list every recollected point;
// tests/golden/make_misc_golden_from_ref.py and make_gaussian_bandit_golden_from_ref.py record gymnax trajectories
// that check them.
#pragma once
#include "env_common.cuh"

namespace pqn {

// gymnax's time_normalization(t) = (max_lim - min_lim) * t / t_max + min_lim with its defaults (-1, 1, t_max = 100),
// as get_obs calls it under normalize_time = True; fp32, left to right (this TU is built with -fmad=false)
PQN_HD float misc_time_normalization(int t) { return 2.0f * (float)t / 100.0f + -1.0f; }

// misc/bernoulli_bandit.py (BernoulliBandit-misc) with num_arms = 2 and the default EnvParams
// (sample_probs = [0.1, 0.9], normalize_time = True):
//   reset_env:  p1 = choice(key, sample_probs, (1,)) = sample_probs[randint(key, (1,), 0, 2)];
//               reward_probs = [p1, 1 - p1], exp_reward_best = max(reward_probs), last_action = 0, last_reward = 0,
//               time = 0
//   step_env:   reward = bernoulli(key, reward_probs[action]) = uniform(key, ()) < reward_probs[action];
//               last_action = action, last_reward = reward, time += 1; done = time >= max_steps_in_episode (100)
//   get_obs:    [one_hot(last_action, 2), last_reward, time_normalization(time)]
// The reward probabilities are state, drawn at reset; sample_probs is read only there.  Bit-exact.
struct BernoulliBanditEnv {
  static constexpr int ID = ENV_BERNOULLI_BANDIT;
  static constexpr int CORE_WORDS = 6;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 2;
  static constexpr int OBS_DIM = 4;
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 100;  // EnvParams.max_steps_in_episode: every episode lasts this long
  PQN_HD static float sample_prob(int k) { return k == 0 ? 0.1f : 0.9f; }

  // words: last_action, last_reward, reward_probs[0], reward_probs[1], exp_reward_best (fp32 bits), time
  struct State {
    int last_action, last_reward;
    float p0, p1, exp_reward_best;
    int time;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    s.last_action = (int)st[i]; s.last_reward = (int)st[N + i];
    s.p0 = u2f((uint32_t)st[2 * N + i]); s.p1 = u2f((uint32_t)st[3 * N + i]);
    s.exp_reward_best = u2f((uint32_t)st[4 * N + i]); s.time = (int)st[5 * N + i];
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = (uint32_t)s.last_action; st[N + i] = (uint32_t)s.last_reward;
    st[2 * N + i] = f2u(s.p0); st[3 * N + i] = f2u(s.p1); st[4 * N + i] = f2u(s.exp_reward_best);
    st[5 * N + i] = (uint32_t)s.time;
  }

  PQN_HD static void reset_env(Key key, int part, int /*max_steps*/, State& s) {
    const float p = sample_prob(randint_scalar(key, 2u, part));
    s.p0 = p;
    s.p1 = 1.0f - p;
    s.exp_reward_best = s.p0 > s.p1 ? s.p0 : s.p1;
    s.last_action = 0; s.last_reward = 0; s.time = 0;
  }

  PQN_HD static void step_env(Key key, int part, int max_steps, State& s, int action, float& reward, bool& done) {
    const int r = uniform_scalar(key, part) < (action == 0 ? s.p0 : s.p1) ? 1 : 0;
    reward = (float)r;
    s.last_action = action; s.last_reward = r;
    s.time = s.time + 1;
    done = s.time >= max_steps;
  }

  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) {
    o[0] = s.last_action == 0 ? 1.f : 0.f;
    o[1] = s.last_action == 1 ? 1.f : 0.f;
    o[2] = (float)s.last_reward;
    o[3] = misc_time_normalization(s.time);
  }
};

// misc/gaussian_bandit.py (GaussianBandit-misc), two arms, with the default EnvParams (mu1 = 0.0, sigma_p = 1.0,
// sigma_l = 1.0, normalize_time = True):
//   reset_env:  mu2 = sigma_p * normal(key, ()), drawn from the reset key itself; exp_reward_best = max(mu1, mu2),
//               last_action = 0, last_reward = 0.0, time = 0
//   step_env:   reward = mu1 if action == 0 else mu2 + sigma_l * normal(key, ()), drawn from the step key itself;
//               last_action = action, last_reward = reward, time += 1; done = time >= max_steps_in_episode (100)
//   get_obs:    [one_hot(last_action, 2), last_reward, time_normalization(time)]
// Arm 0 pays mu1 and arm 1 a normal around its mean mu2.  gymnax draws the step's normal for both arms and selects it
// away for arm 0, so this env draws it only for arm 1.  mu1 and sigma_l are kept in state words (the step reads them
// from EnvParams).  The step's mu2 + sigma_l * n is one fma, as the Horner steps of erf_inv (threefry.cuh); at
// sigma_l = 1 the product is exact and the fma and the rounded add agree.  The normal's log1pf makes the rewards and
// mu2 depend on the math library: libdevice's on the device, as XLA:GPU's jax.random.normal.
struct GaussianBanditEnv {
  static constexpr int ID = ENV_GAUSSIAN_BANDIT;
  static constexpr int CORE_WORDS = 7;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 2;
  static constexpr int OBS_DIM = 4;
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 100;  // EnvParams.max_steps_in_episode: every episode lasts this long
  static constexpr float MU1 = 0.0f, SIGMA_P = 1.0f, SIGMA_L = 1.0f;

  // words: last_action, last_reward, mu2, exp_reward_best (fp32 bits), time, then the EnvParams words mu1 and
  // sigma_l (fp32 bits)
  struct State {
    int last_action;
    float last_reward, mu2, exp_reward_best;
    int time;
    float mu1, sigma_l;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    s.last_action = (int)st[i]; s.last_reward = u2f((uint32_t)st[N + i]);
    s.mu2 = u2f((uint32_t)st[2 * N + i]); s.exp_reward_best = u2f((uint32_t)st[3 * N + i]);
    s.time = (int)st[4 * N + i];
    s.mu1 = u2f((uint32_t)st[5 * N + i]); s.sigma_l = u2f((uint32_t)st[6 * N + i]);
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = (uint32_t)s.last_action; st[N + i] = f2u(s.last_reward);
    st[2 * N + i] = f2u(s.mu2); st[3 * N + i] = f2u(s.exp_reward_best);
    st[4 * N + i] = (uint32_t)s.time;
    st[5 * N + i] = f2u(s.mu1); st[6 * N + i] = f2u(s.sigma_l);
  }

  PQN_HD static void reset_env(Key key, int part, int /*max_steps*/, State& s) {
    s.mu1 = MU1; s.sigma_l = SIGMA_L;
    s.mu2 = mul_rn(SIGMA_P, normal_scalar(key, part));
    s.exp_reward_best = s.mu2 > s.mu1 ? s.mu2 : s.mu1;
    s.last_action = 0; s.last_reward = 0.f; s.time = 0;
  }

  PQN_HD static void step_env(Key key, int part, int max_steps, State& s, int action, float& reward, bool& done) {
    reward = action == 0 ? s.mu1 : fmaf(s.sigma_l, normal_scalar(key, part), s.mu2);
    s.last_action = action; s.last_reward = reward;
    s.time = s.time + 1;
    done = s.time >= max_steps;
  }

  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) {
    o[0] = s.last_action == 0 ? 1.f : 0.f;
    o[1] = s.last_action == 1 ? 1.f : 0.f;
    o[2] = s.last_reward;
    o[3] = misc_time_normalization(s.time);
  }
};

// misc/rooms.py (FourRooms-misc) with the constructor's defaults (use_visual_obs = False, goal_fixed = [8, 9],
// pos_fixed = [4, 1]) and the default EnvParams (fail_prob = 1/3, resample_init_pos = resample_goal_pos = False):
//   the 13 x 13 four-rooms map below; directions [[-1, 0], [0, 1], [1, 0], [0, -1]]
//   reset_env:  rng_goal, rng_pos = split(key); goal and pos are drawn from them but selected away (resample_* is
//               False), so goal = [8, 9], pos = [4, 1], time = 0
//   step_env:   key_random, key_action = split(key);
//               action = randint(key_action, (), 0, 4) if uniform(key_random, ()) < fail_prob * 4 / 3 else action;
//               p = pos + directions[action]; pos = p if the map is open at p else pos;
//               reward = pos == goal; time += 1; done = pos == goal || time >= max_steps_in_episode (500)
//   get_obs:    [pos[0], pos[1], goal[0], goal[1]]
// The reset's draws cannot reach an output, and the random action matters only where the uniform is below the
// threshold, so this env skips the reset's draws and draws the random action only there.  fail_prob is kept in a
// state word (the step reads it from EnvParams).  Integer work plus fp32 constants: bit-exact.
struct FourRoomsEnv {
  static constexpr int ID = ENV_FOUR_ROOMS;
  static constexpr int SIZE = 13;
  static constexpr int CORE_WORDS = 3;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 4;
  static constexpr int OBS_DIM = 4;
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 500;  // EnvParams.max_steps_in_episode
  static constexpr int GOAL_R = 8, GOAL_C = 9, START_R = 4, START_C = 1;

  // walls of map row r, bit c:  xxxxxxxxxxxxx / x     x     x (x2) / x           x / x     x     x (x2) /
  // xx xxxx     x / x     xxx xxx / x     x     x (x2) / x           x / x     x     x / xxxxxxxxxxxxx
  PQN_HD static uint32_t wall_row(int r) {
    switch (r) {
      case 3: case 10: return 0x1001u;
      case 6: return 0x107Bu;
      case 7: return 0x1DC1u;
      case 0: case 12: return 0x1FFFu;
      default: return 0x1041u;
    }
  }
  PQN_HD static bool open(int r, int c) { return ((wall_row(r) >> c) & 1u) == 0u; }

  // word 0: pos[0] | pos[1] << 8 | goal[0] << 16 | goal[1] << 24;  1: time;  2: fail_prob (fp32 bits)
  struct State {
    int pos_r, pos_c, goal_r, goal_c, time;
    float fail_prob;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    const uint32_t w = (uint32_t)st[i];
    s.pos_r = (int)(w & 255u); s.pos_c = (int)((w >> 8) & 255u);
    s.goal_r = (int)((w >> 16) & 255u); s.goal_c = (int)(w >> 24);
    s.time = (int)st[N + i]; s.fail_prob = u2f((uint32_t)st[2 * N + i]);
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = (uint32_t)s.pos_r | ((uint32_t)s.pos_c << 8) | ((uint32_t)s.goal_r << 16) | ((uint32_t)s.goal_c << 24);
    st[N + i] = (uint32_t)s.time; st[2 * N + i] = f2u(s.fail_prob);
  }

  PQN_HD static void reset_env(Key /*key*/, int /*part*/, int /*max_steps*/, State& s) {
    s.pos_r = START_R; s.pos_c = START_C; s.goal_r = GOAL_R; s.goal_c = GOAL_C; s.time = 0;
    s.fail_prob = 1.0f / 3.0f;
  }

  PQN_HD static void step_env(Key key, int part, int max_steps, State& s, int action, float& reward, bool& done) {
    Key k_random, k_action;
    split2(key, part, k_random, k_action);
    if (uniform_scalar(k_random, part) < s.fail_prob * 4.0f / 3.0f) action = randint_scalar(k_action, 4u, part);
    const int r = s.pos_r + (action == 0 ? -1 : action == 2 ? 1 : 0);
    const int c = s.pos_c + (action == 1 ? 1 : action == 3 ? -1 : 0);
    if (open(r, c)) { s.pos_r = r; s.pos_c = c; }
    const bool at_goal = s.pos_r == s.goal_r && s.pos_c == s.goal_c;
    reward = at_goal ? 1.f : 0.f;
    s.time = s.time + 1;
    done = at_goal || s.time >= max_steps;
  }

  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) {
    o[0] = (float)s.pos_r; o[1] = (float)s.pos_c; o[2] = (float)s.goal_r; o[3] = (float)s.goal_c;
  }
};

// misc/meta_maze.py (MetaMaze-misc) with the constructor's maze_size = 9, rf_size = 3 and the default EnvParams
// (reward = 10.0, normalize_time = True):
//   the map: walls on the border and at every (even row, even column) inside, except the centre (4, 4); coords are
//   its 41 free cells in row-major order; directions [[-1, 0], [0, 1], [1, 0], [0, -1]]
//   reset_pos(key, coords, goal): k = randint(key, (), 0, 40); coords[40] if coords[k] == goal else coords[k]
//   reset_env:  rng_goal, rng_pos = split(key); goal = coords[randint(rng_goal, (), 0, 41)];
//               pos = reset_pos(rng_pos, coords, goal); last_action = 0, last_reward = 0.0, time = 0
//   step_env:   p = pos + directions[action]; pos = pos if p is a wall else p; goal_reached = pos == goal;
//               reward = goal_reached * reward; pos = reset_pos(key, coords, goal) where goal_reached;
//               last_action = action, last_reward = reward, time += 1; done = time >= max_steps_in_episode (200)
//   get_obs:    [the 3 x 3 map around pos (1 = wall), one_hot(last_action, 4), last_reward,
//                time_normalization(time)]
// The step's reset_pos draw is selected only where the goal is reached, so this env draws it only there.  The reward
// parameter is kept in a state word (the step reads it from EnvParams).  Integer work plus fp32 constants: bit-exact.
struct MetaMazeEnv {
  static constexpr int ID = ENV_META_MAZE;
  static constexpr int SIZE = 9;
  static constexpr int RF = 3;
  static constexpr int FREE_CELLS = 41;
  static constexpr int CORE_WORDS = 5;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 4;
  static constexpr int OBS_DIM = RF * RF + NUM_ACTIONS + 2;
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 200;  // EnvParams.max_steps_in_episode: every episode lasts this long
  static constexpr float GOAL_REWARD = 10.0f;

  PQN_HD static bool wall(int r, int c) {
    return r == 0 || r == SIZE - 1 || c == 0 || c == SIZE - 1 ||
           ((r & 1) == 0 && (c & 1) == 0 && !(r == SIZE / 2 && c == SIZE / 2));
  }
  // coords[k]: free cells per row are 7 on odd rows, 4 on rows 2 and 6 and 5 on row 4 (the free centre)
  PQN_HD static void coord(int k, int& r, int& c) {
    r = 1;
    for (;;) {
      const int n = (r & 1) ? SIZE - 2 : (r == SIZE / 2 ? (SIZE - 1) / 2 + 1 : (SIZE - 1) / 2);
      if (k < n) break;
      k -= n;
      ++r;
    }
    for (c = 1; c < SIZE - 1; ++c) {
      if (!wall(r, c)) {
        if (k == 0) return;
        --k;
      }
    }
  }
  PQN_HD static void reset_pos(Key key, int part, int goal_r, int goal_c, int& r, int& c) {
    coord(randint_scalar(key, (uint32_t)(FREE_CELLS - 1), part), r, c);
    if (r == goal_r && c == goal_c) coord(FREE_CELLS - 1, r, c);
  }

  // words: last_action, last_reward (fp32 bits), pos[0] | pos[1] << 8 | goal[0] << 16 | goal[1] << 24, time,
  // reward (fp32 bits, the EnvParams word the step reads)
  struct State {
    int last_action;
    float last_reward;
    int pos_r, pos_c, goal_r, goal_c, time;
    float reward;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    s.last_action = (int)st[i]; s.last_reward = u2f((uint32_t)st[N + i]);
    const uint32_t w = (uint32_t)st[2 * N + i];
    s.pos_r = (int)(w & 255u); s.pos_c = (int)((w >> 8) & 255u);
    s.goal_r = (int)((w >> 16) & 255u); s.goal_c = (int)(w >> 24);
    s.time = (int)st[3 * N + i]; s.reward = u2f((uint32_t)st[4 * N + i]);
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = (uint32_t)s.last_action; st[N + i] = f2u(s.last_reward);
    st[2 * N + i] = (uint32_t)s.pos_r | ((uint32_t)s.pos_c << 8) | ((uint32_t)s.goal_r << 16) |
                    ((uint32_t)s.goal_c << 24);
    st[3 * N + i] = (uint32_t)s.time; st[4 * N + i] = f2u(s.reward);
  }

  PQN_HD static void reset_env(Key key, int part, int /*max_steps*/, State& s) {
    Key rng_goal, rng_pos;
    split2(key, part, rng_goal, rng_pos);
    coord(randint_scalar(rng_goal, (uint32_t)FREE_CELLS, part), s.goal_r, s.goal_c);
    reset_pos(rng_pos, part, s.goal_r, s.goal_c, s.pos_r, s.pos_c);
    s.last_action = 0; s.last_reward = 0.f; s.time = 0;
    s.reward = GOAL_REWARD;
  }

  PQN_HD static void step_env(Key key, int part, int max_steps, State& s, int action, float& reward, bool& done) {
    const int r = s.pos_r + (action == 0 ? -1 : action == 2 ? 1 : 0);
    const int c = s.pos_c + (action == 1 ? 1 : action == 3 ? -1 : 0);
    if (!wall(r, c)) { s.pos_r = r; s.pos_c = c; }
    const bool goal_reached = s.pos_r == s.goal_r && s.pos_c == s.goal_c;
    reward = (goal_reached ? 1.f : 0.f) * s.reward;
    if (goal_reached) reset_pos(key, part, s.goal_r, s.goal_c, s.pos_r, s.pos_c);
    s.last_action = action; s.last_reward = reward;
    s.time = s.time + 1;
    done = s.time >= max_steps;
  }

  // compares instead of indexed writes, so that `o` stays in registers
  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) {
#pragma unroll
    for (int j = 0; j < RF * RF; ++j) o[j] = wall(s.pos_r - 1 + j / RF, s.pos_c - 1 + j % RF) ? 1.f : 0.f;
#pragma unroll
    for (int a = 0; a < NUM_ACTIONS; ++a) o[RF * RF + a] = s.last_action == a ? 1.f : 0.f;
    o[RF * RF + NUM_ACTIONS] = s.last_reward;
    o[RF * RF + NUM_ACTIONS + 1] = misc_time_normalization(s.time);
  }
};

}  // namespace pqn
