// gymnax classic-control dynamics (CartPole-v1, Acrobot-v1), one env per thread.
//
// Restates gymnax==0.0.6 gymnax/environments/classic_control/{cartpole,acrobot}.py
// (third party; call sites purejaxql/pqn_gymnax.py:92-104,192-194).  fp32
// physics: agreement with the reference is to a few ulp per step (sin/cos
// implementations and FMA contraction differ between XLA and CUDA), not bitwise.
// This translation unit is compiled with -fmad=false so that the expression
// trees below round exactly as written.
#pragma once
#include <math.h>
#include "env_common.cuh"

namespace pqn {

struct CartPoleEnv {
  static constexpr int ID = ENV_CARTPOLE;
  static constexpr int CORE_WORDS = 5;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 2;
  static constexpr int OBS_DIM = 4;
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 500;

  struct State {
    float x, x_dot, theta, theta_dot;
    int time;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    s.x = u2f(st[i]); s.x_dot = u2f(st[N + i]); s.theta = u2f(st[2 * N + i]);
    s.theta_dot = u2f(st[3 * N + i]); s.time = (int)st[4 * N + i];
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = f2u(s.x); st[N + i] = f2u(s.x_dot); st[2 * N + i] = f2u(s.theta);
    st[3 * N + i] = f2u(s.theta_dot); st[4 * N + i] = (uint32_t)s.time;
  }

  PQN_HD static bool is_terminal(const State& s, int max_steps) {
    const float x_threshold = 2.4f;
    const float theta_threshold = (float)(12.0 * 2.0 * 3.141592653589793 / 360.0);
    const bool d1 = s.x < -x_threshold || s.x > x_threshold;
    const bool d2 = s.theta < -theta_threshold || s.theta > theta_threshold;
    return d1 || d2 || s.time >= max_steps;
  }

  PQN_HD static void reset_env(Key key, int part, int /*max_steps*/, State& s) {
    // jax.random.uniform(key, minval=-0.05, maxval=0.05, shape=(4,))
    float u[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = uniform_from_bits(bits_at(key, 4u, j, part), -0.05f, 0.05f);
    s.x = u[0]; s.x_dot = u[1]; s.theta = u[2]; s.theta_dot = u[3]; s.time = 0;
  }

  PQN_HD static void step_env(Key /*key*/, int /*part*/, int max_steps, State& s, int action,
                              float& reward, bool& done) {
    const float gravity = 9.8f, masspole = 0.1f, total_mass = (float)(1.0 + 0.1), length = 0.5f;
    const float polemass_length = 0.05f, force_mag = 10.0f, tau = 0.02f;
    const bool prev_terminal = is_terminal(s, max_steps);
    const float af = (float)action;
    const float force = force_mag * af - force_mag * (1.0f - af);
    const float costheta = cosf(s.theta);
    const float sintheta = sinf(s.theta);
    const float temp = (force + polemass_length * (s.theta_dot * s.theta_dot) * sintheta) / total_mass;
    const float thetaacc = (gravity * sintheta - costheta * temp) /
                           (length * ((float)(4.0 / 3.0) - masspole * (costheta * costheta) / total_mass));
    const float xacc = temp - polemass_length * thetaacc * costheta / total_mass;
    const float x = s.x + tau * s.x_dot;
    const float x_dot = s.x_dot + tau * xacc;
    const float theta = s.theta + tau * s.theta_dot;
    const float theta_dot = s.theta_dot + tau * thetaacc;
    reward = 1.0f - (prev_terminal ? 1.0f : 0.0f);
    s.x = x; s.x_dot = x_dot; s.theta = theta; s.theta_dot = theta_dot; s.time = s.time + 1;
    done = is_terminal(s, max_steps);
  }

  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) {
    o[0] = s.x; o[1] = s.x_dot; o[2] = s.theta; o[3] = s.theta_dot;
  }
};

struct AcrobotEnv {
  static constexpr int ID = ENV_ACROBOT;
  static constexpr int CORE_WORDS = 5;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 3;
  static constexpr int OBS_DIM = 6;
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 500;

  struct State {
    float a1, a2, v1, v2;
    int time;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    s.a1 = u2f(st[i]); s.a2 = u2f(st[N + i]); s.v1 = u2f(st[2 * N + i]);
    s.v2 = u2f(st[3 * N + i]); s.time = (int)st[4 * N + i];
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = f2u(s.a1); st[N + i] = f2u(s.a2); st[2 * N + i] = f2u(s.v1);
    st[3 * N + i] = f2u(s.v2); st[4 * N + i] = (uint32_t)s.time;
  }

  PQN_HD static void reset_env(Key key, int part, int /*max_steps*/, State& s) {
    float u[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = uniform_from_bits(bits_at(key, 4u, j, part), -0.1f, 0.1f);
    s.a1 = u[0]; s.a2 = u[1]; s.v1 = u[2]; s.v2 = u[3]; s.time = 0;
  }

  // dsdt(s_augmented): unit masses/lengths, com 0.5, moi 1, g 9.8.
  PQN_HD static void dsdt(const float (&y)[5], float (&d)[5]) {
    const float m1 = 1.f, m2 = 1.f, l1 = 1.f, lc1 = 0.5f, lc2 = 0.5f, I1 = 1.f, I2 = 1.f, g = 9.8f;
    const float pi = 3.14159265358979323846f;
    const float th1 = y[0], th2 = y[1], dth1 = y[2], dth2 = y[3], a = y[4];
    const float c2 = cosf(th2), s2 = sinf(th2);
    const float d1 = m1 * (lc1 * lc1) + m2 * (l1 * l1 + lc2 * lc2 + 2.f * l1 * lc2 * c2) + I1 + I2;
    const float d2 = m2 * (lc2 * lc2 + l1 * lc2 * c2) + I2;
    const float phi2 = m2 * lc2 * g * cosf(th1 + th2 - pi / 2.0f);
    const float phi1 = -m2 * l1 * lc2 * (dth2 * dth2) * s2 - 2.f * m2 * l1 * lc2 * dth2 * dth1 * s2 +
                       (m1 * lc1 + m2 * l1) * g * cosf(th1 - pi / 2.f) + phi2;
    const float ddth2 = (a + d2 / d1 * phi1 - m2 * l1 * lc2 * (dth1 * dth1) * s2 - phi2) /
                        (m2 * (lc2 * lc2) + I2 - (d2 * d2) / d1);
    const float ddth1 = -(a + d2 * ddth2 + phi1) / d1;
    d[0] = dth1; d[1] = dth2; d[2] = ddth1; d[3] = ddth2; d[4] = 0.f;
  }

  PQN_HD static float wrap(float x, float m, float M) {
    const float diff = M - m;
    const float go_up = x < m ? 1.f : 0.f;
    const float go_down = x >= M ? 1.f : 0.f;
    const float how_often = go_up * ceilf((m - x) / diff) + go_down * floorf((x - m) / diff);
    return x - how_often * diff * go_down + how_often * diff * go_up;
  }

  PQN_HD static void step_env(Key key, int part, int max_steps, State& s, int action,
                              float& reward, bool& done) {
    const float dt = 0.2f, pi = 3.14159265358979323846f;
    const float max_vel_1 = (float)(4.0 * 3.141592653589793), max_vel_2 = (float)(9.0 * 3.141592653589793);
    const float torque_noise_max = 0.0f;
    float torque = (float)((action <= 0 ? 0 : (action >= 2 ? 2 : action)) - 1);
    // "always sample": uniform(key, (), -noise, +noise) with noise = 0
    torque = torque + uniform_from_bits(bits_scalar(key, part), -torque_noise_max, torque_noise_max);
    float y0[5] = {s.a1, s.a2, s.v1, s.v2, torque};
    float k1[5], k2[5], k3[5], k4[5], yt[5];
    const float dt2 = dt / 2.0f;
    dsdt(y0, k1);
#pragma unroll
    for (int j = 0; j < 5; ++j) yt[j] = y0[j] + dt2 * k1[j];
    dsdt(yt, k2);
#pragma unroll
    for (int j = 0; j < 5; ++j) yt[j] = y0[j] + dt2 * k2[j];
    dsdt(yt, k3);
#pragma unroll
    for (int j = 0; j < 5; ++j) yt[j] = y0[j] + dt * k3[j];
    dsdt(yt, k4);
    float ns[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      ns[j] = y0[j] + dt / 6.0f * (k1[j] + 2.f * k2[j] + 2.f * k3[j] + k4[j]);
    s.a1 = wrap(ns[0], -pi, pi);
    s.a2 = wrap(ns[1], -pi, pi);
    s.v1 = fminf(fmaxf(ns[2], -max_vel_1), max_vel_1);
    s.v2 = fminf(fmaxf(ns[3], -max_vel_2), max_vel_2);
    s.time = s.time + 1;
    const bool done_angle = (-cosf(s.a1) - cosf(s.a2 + s.a1)) > 1.0f;
    done = done_angle || s.time >= max_steps;
    reward = -1.0f * (1.0f - (done_angle ? 1.f : 0.f));
  }

  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) {
    o[0] = cosf(s.a1); o[1] = sinf(s.a1); o[2] = cosf(s.a2); o[3] = sinf(s.a2);
    o[4] = s.v1; o[5] = s.v2;
  }
};

// gymnax classic_control/mountain_car.py (MountainCar-v0).  Restated from recollection of gymnax 0.0.6: the EnvParams
// defaults below, the uniform(-0.6, -0.4) reset, the step order and the wall rule
// `velocity *= 1 - (position == min_position) * (velocity < 0)`, which gives -0.0 for a negative velocity.
struct MountainCarEnv {
  static constexpr int ID = ENV_MOUNTAIN_CAR;
  static constexpr int CORE_WORDS = 3;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 3;
  static constexpr int OBS_DIM = 2;
  static constexpr bool BINARY_OBS = false;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 1, OBS_WORDS_PAD = 1;
  static constexpr int DEFAULT_MAX_STEPS = 200;

  struct State {
    float position, velocity;
    int time;
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    s.position = u2f(st[i]); s.velocity = u2f(st[N + i]); s.time = (int)st[2 * N + i];
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = f2u(s.position); st[N + i] = f2u(s.velocity); st[2 * N + i] = (uint32_t)s.time;
  }

  PQN_HD static void reset_env(Key key, int part, int /*max_steps*/, State& s) {
    // jax.random.uniform(key, shape=(), minval=-0.6, maxval=-0.4)
    s.position = uniform_from_bits(bits_scalar(key, part), -0.6f, -0.4f);
    s.velocity = 0.f;
    s.time = 0;
  }

  PQN_HD static void step_env(Key /*key*/, int /*part*/, int max_steps, State& s, int action, float& reward,
                              bool& done) {
    const float min_position = -1.2f, max_position = 0.6f, max_speed = 0.07f;
    const float goal_position = 0.5f, goal_velocity = 0.0f, force = 0.001f, gravity = 0.0025f;
    float velocity = s.velocity + (float)(action - 1) * force - cosf(3.0f * s.position) * gravity;
    velocity = fminf(fmaxf(velocity, -max_speed), max_speed);
    float position = s.position + velocity;
    position = fminf(fmaxf(position, min_position), max_position);
    velocity = velocity * (float)(1 - ((position == min_position && velocity < 0.f) ? 1 : 0));
    reward = -1.0f;
    s.position = position; s.velocity = velocity; s.time = s.time + 1;
    done = (position >= goal_position && velocity >= goal_velocity) || s.time >= max_steps;
  }

  PQN_HD static void obs_float(const State& s, float (&o)[OBS_DIM]) { o[0] = s.position; o[1] = s.velocity; }
};

}  // namespace pqn
