// MinAtar Seaquest dynamics, one env per thread.
//
// Restated from MinAtar's own minatar/environments/seaquest.py (Young & Tian 2019) in gymnax's conventions: gymnax==0.0.6
// does not register "Seaquest-MinAtar" (DESIGN.md section 8), so there is no JAX port to follow.  Reset and step are
// Environment.reset_env / step_env under the auto-reset of env_common.cuh; MinAtar's numpy draws become jax.random
// draws on fixed subkeys of the step key.  PARITY UNPINNED: the tests pin this kernel bit-exactly to the NumPy
// restatement in tests/seaquest_oracle.py, whose closing list numbers every rule, constant and draw that could not
// be checked against MinAtar here.
//
// MinAtar keeps bullets, fish, subs and divers in Python lists, walks each list backwards and removes entries as it
// goes.  Here every list is a fixed-capacity array in list order (entry k of a list = list[k]; removal shifts the tail
// down, appends go to the end), so the same walk visits the same entries in the same order.  An append to a full list
// is dropped (oracle assumption S14).
//
// State words (word-major SoA, 19 core + 5 LogWrapper words = 96 bytes per env):
//   w0  sub_x[0:4) sub_y[4:8) sub_or[8] shot_timer[9:12) diver_count[12:15) surface[15] terminal[16]
//       move_speed[17:20) ramp_index[20:25)
//   w1  oxygen+1[0:8) e_spawn_speed[8:13) e_spawn_timer[13:18) d_spawn_timer[18:24)
//   w2  list lengths: f_bullets[0:2) e_fish[2:6) e_subs[6:10) e_bullets[10:14) divers[14:17)
//   w3  time
//   w4  f_bullets (2 x 16 bits)   w5..w8 e_fish (8)   w9..w12 e_subs (8)   w13..w16 e_bullets (8)   w17..w18 divers (4)
// An entry is x[0:4) y[4:8) lr[8] move_timer[9:12) shot_timer[12:16); slots past a list's length are zero.
#pragma once
#include "env_minatar_more.cuh"

namespace pqn {

namespace sq {
PQN_HD int ex(uint32_t e) { return (int)(e & 15u); }
PQN_HD int ey(uint32_t e) { return (int)((e >> 4) & 15u); }
PQN_HD int elr(uint32_t e) { return (int)((e >> 8) & 1u); }
PQN_HD int emt(uint32_t e) { return (int)((e >> 9) & 7u); }
PQN_HD int est(uint32_t e) { return (int)((e >> 12) & 15u); }
PQN_HD uint32_t emake(int x, int y, int lr, int mt, int st) {
  return (uint32_t)x | ((uint32_t)y << 4) | ((uint32_t)lr << 8) | ((uint32_t)mt << 9) | ((uint32_t)st << 12);
}
// list.pop(idx) on a fixed-capacity list (unrolled: the array stays in registers)
template <int CAP>
PQN_HD void remove_at(uint32_t (&a)[CAP], int& n, int idx) {
#pragma unroll
  for (int k = 0; k < CAP - 1; ++k)
    if (k >= idx) a[k] = a[k + 1];
  a[CAP - 1] = 0u;
  n -= 1;
}
// list.append(v); dropped when the list is full
template <int CAP>
PQN_HD void append(uint32_t (&a)[CAP], int& n, uint32_t v) {
#pragma unroll
  for (int k = 0; k < CAP; ++k)
    if (k == n) a[k] = v;
  n += n < CAP ? 1 : 0;
}
template <int CAP, typename W>
PQN_HD void load_list(uint32_t (&a)[CAP], const W* __restrict__ st, int64_t N, int64_t i, int w0) {
#pragma unroll
  for (int k = 0; k < CAP; k += 2) {
    const uint32_t v = st[(int64_t)(w0 + k / 2) * N + i];
    a[k] = v & 0xFFFFu;
    a[k + 1] = v >> 16;
  }
}
template <int CAP>
PQN_HD void store_list(const uint32_t (&a)[CAP], uint32_t* __restrict__ st, int64_t N, int64_t i, int w0) {
#pragma unroll
  for (int k = 0; k < CAP; k += 2) st[(int64_t)(w0 + k / 2) * N + i] = a[k] | (a[k + 1] << 16);
}
}  // namespace sq

struct SeaquestEnv {
  static constexpr int ID = ENV_SEAQUEST;
  static constexpr int CORE_WORDS = 19;
  static constexpr int STATE_WORDS = CORE_WORDS + LOG_WORDS;
  static constexpr int NUM_ACTIONS = 6;  // MinAtar's minimal set = full set: n, l, u, r, d, f
  static constexpr int OBS_H = 10, OBS_W = 10, OBS_C = 10;
  static constexpr int OBS_DIM = 1000;
  static constexpr bool BINARY_OBS = true;
  static constexpr bool OBS_IN_REGS = false;
  static constexpr int OBS_WORDS = 32;
  static constexpr int OBS_WORDS_PAD = 32;
  static constexpr int DEFAULT_MAX_STEPS = 1000;
  // minatar/environments/seaquest.py module constants
  static constexpr int RAMP_INTERVAL = 100;  // defined there but unused by Seaquest: its ramp steps at each surfacing
  static constexpr int MAX_OXYGEN = 200, INIT_SPAWN_SPEED = 20, DIVER_SPAWN_SPEED = 30, INIT_MOVE_INTERVAL = 5;
  static constexpr int SHOT_COOL_DOWN = 5, ENEMY_SHOT_INTERVAL = 10, ENEMY_MOVE_INTERVAL = 5, DIVER_MOVE_INTERVAL = 5;
  // list capacities (oracle assumption S14)
  static constexpr int FB_CAP = 2, EF_CAP = 8, ES_CAP = 8, EB_CAP = 8, DV_CAP = 4;

  struct State {
    int sub_x, sub_y, sub_or, shot_timer, diver_count, move_speed, ramp_index;
    int oxygen, e_spawn_speed, e_spawn_timer, d_spawn_timer, time;
    bool surface, terminal;
    int nfb, nef, nes, neb, ndv;
    uint32_t fb[FB_CAP], ef[EF_CAP], es[ES_CAP], eb[EB_CAP], dv[DV_CAP];
  };

  template <typename W>
  PQN_HD static void load(State& s, const W* __restrict__ st, int64_t N, int64_t i) {
    const uint32_t w0 = st[i], w1 = st[N + i], w2 = st[2 * N + i];
    s.sub_x = w0 & 15u; s.sub_y = (w0 >> 4) & 15u; s.sub_or = (w0 >> 8) & 1u; s.shot_timer = (w0 >> 9) & 7u;
    s.diver_count = (w0 >> 12) & 7u; s.surface = (w0 >> 15) & 1u; s.terminal = (w0 >> 16) & 1u;
    s.move_speed = (w0 >> 17) & 7u; s.ramp_index = (w0 >> 20) & 31u;
    s.oxygen = (int)(w1 & 255u) - 1; s.e_spawn_speed = (w1 >> 8) & 31u; s.e_spawn_timer = (w1 >> 13) & 31u;
    s.d_spawn_timer = (w1 >> 18) & 63u;
    s.nfb = w2 & 3u; s.nef = (w2 >> 2) & 15u; s.nes = (w2 >> 6) & 15u; s.neb = (w2 >> 10) & 15u; s.ndv = (w2 >> 14) & 7u;
    s.time = (int)st[3 * N + i];
    sq::load_list(s.fb, st, N, i, 4);
    sq::load_list(s.ef, st, N, i, 5);
    sq::load_list(s.es, st, N, i, 9);
    sq::load_list(s.eb, st, N, i, 13);
    sq::load_list(s.dv, st, N, i, 17);
  }
  PQN_HD static void store(const State& s, uint32_t* __restrict__ st, int64_t N, int64_t i) {
    st[i] = (uint32_t)s.sub_x | ((uint32_t)s.sub_y << 4) | ((uint32_t)s.sub_or << 8) | ((uint32_t)s.shot_timer << 9) |
            ((uint32_t)s.diver_count << 12) | ((uint32_t)s.surface << 15) | ((uint32_t)s.terminal << 16) |
            ((uint32_t)s.move_speed << 17) | ((uint32_t)s.ramp_index << 20);
    st[N + i] = (uint32_t)(s.oxygen + 1) | ((uint32_t)s.e_spawn_speed << 8) | ((uint32_t)s.e_spawn_timer << 13) |
                ((uint32_t)s.d_spawn_timer << 18);
    st[2 * N + i] = (uint32_t)s.nfb | ((uint32_t)s.nef << 2) | ((uint32_t)s.nes << 6) | ((uint32_t)s.neb << 10) |
                    ((uint32_t)s.ndv << 14);
    st[3 * N + i] = (uint32_t)s.time;
    sq::store_list(s.fb, st, N, i, 4);
    sq::store_list(s.ef, st, N, i, 5);
    sq::store_list(s.es, st, N, i, 9);
    sq::store_list(s.eb, st, N, i, 13);
    sq::store_list(s.dv, st, N, i, 17);
  }

  PQN_HD static void reset_env(Key /*key*/, int /*part*/, int /*max_steps*/, State& s) {
    s.oxygen = MAX_OXYGEN; s.diver_count = 0; s.sub_x = 5; s.sub_y = 0; s.sub_or = 0;
    s.e_spawn_speed = INIT_SPAWN_SPEED; s.e_spawn_timer = INIT_SPAWN_SPEED; s.d_spawn_timer = DIVER_SPAWN_SPEED;
    s.move_speed = INIT_MOVE_INTERVAL; s.ramp_index = 0; s.shot_timer = 0; s.surface = true; s.terminal = false;
    s.time = 0;
    s.nfb = s.nef = s.nes = s.neb = s.ndv = 0;
#pragma unroll
    for (int k = 0; k < FB_CAP; ++k) s.fb[k] = 0u;
#pragma unroll
    for (int k = 0; k < EF_CAP; ++k) { s.ef[k] = 0u; s.es[k] = 0u; s.eb[k] = 0u; }
#pragma unroll
    for (int k = 0; k < DV_CAP; ++k) s.dv[k] = 0u;
  }

  // MinAtar's (oxygen * 10) // max_oxygen, Python floor division (oxygen >= -1)
  PQN_HD static int oxygen_tenths(int oxygen) { return oxygen >= 0 ? oxygen * 10 / MAX_OXYGEN : -1; }

  // Subkeys of the step key: split(key, 5) = (enemy lr, enemy is_sub, enemy row, diver lr, diver row).  A draw is made
  // only on a step whose spawn timer is 0: on other steps nothing reads it.
  PQN_HD static void step_env(Key key, int part, int max_steps, State& s, int action, float& reward, bool& done) {
    using namespace sq;
    int r = 0;
    bool term = false;
    // ---- spawn an enemy: fish or sub, random side and row; skipped when a row-mate faces the other way
    if (s.e_spawn_timer == 0) {
      const int lr = 1 - randint_scalar(split_at(key, 5u, 0u, part), 2u, part);   // choice([True, False])
      const float c0 = (float)(1.0 / 3.0), c1 = c0 + (float)(2.0 / 3.0);          // choice([True, False], p=[1/3, 2/3])
      const float u = c1 * (1.0f - uniform_scalar(split_at(key, 5u, 1u, part), part));
      const bool is_sub = !(c0 < u);
      const int y = 1 + randint_scalar(split_at(key, 5u, 2u, part), 8u, part);    // choice(arange(1, 9))
      bool blocked = false;
#pragma unroll
      for (int k = 0; k < ES_CAP; ++k) blocked = blocked || (k < s.nes && ey(s.es[k]) == y && elr(s.es[k]) != lr);
#pragma unroll
      for (int k = 0; k < EF_CAP; ++k) blocked = blocked || (k < s.nef && ey(s.ef[k]) == y && elr(s.ef[k]) != lr);
      if (!blocked) {
        if (is_sub) append(s.es, s.nes, emake(lr ? 0 : 9, y, lr, s.move_speed, ENEMY_SHOT_INTERVAL));
        else append(s.ef, s.nef, emake(lr ? 0 : 9, y, lr, s.move_speed, 0));
      }
      s.e_spawn_timer = s.e_spawn_speed;
    }
    // ---- spawn a diver
    if (s.d_spawn_timer == 0) {
      const int lr = 1 - randint_scalar(split_at(key, 5u, 3u, part), 2u, part);
      const int y = 1 + randint_scalar(split_at(key, 5u, 4u, part), 8u, part);
      append(s.dv, s.ndv, emake(lr ? 0 : 9, y, lr, DIVER_MOVE_INTERVAL, 0));
      s.d_spawn_timer = DIVER_SPAWN_SPEED;
    }
    // ---- player: fire, or move (l / r also turn the sub)
    if (action == 5 && s.shot_timer == 0) {
      append(s.fb, s.nfb, emake(s.sub_x, s.sub_y, s.sub_or, 0, 0));
      s.shot_timer = SHOT_COOL_DOWN;
    } else if (action == 1) { s.sub_x = s.sub_x > 0 ? s.sub_x - 1 : 0; s.sub_or = 0; }
    else if (action == 3) { s.sub_x = s.sub_x < 9 ? s.sub_x + 1 : 9; s.sub_or = 1; }
    else if (action == 2) s.sub_y = s.sub_y > 0 ? s.sub_y - 1 : 0;
    else if (action == 4) s.sub_y = s.sub_y < 8 ? s.sub_y + 1 : 8;
    // ---- friendly bullets: move, then hit the first fish, else the first sub, on their cell (+1 each)
#pragma unroll
    for (int i = FB_CAP - 1; i >= 0; --i) {
      if (i >= s.nfb) continue;
      const uint32_t b = s.fb[i];
      const int x = ex(b) + (elr(b) ? 1 : -1), y = ey(b);
      if (x < 0 || x > 9) { remove_at(s.fb, s.nfb, i); continue; }
      s.fb[i] = emake(x, y, elr(b), 0, 0);
      bool hit = false;
#pragma unroll
      for (int k = 0; k < EF_CAP; ++k)
        if (!hit && k < s.nef && ex(s.ef[k]) == x && ey(s.ef[k]) == y) { remove_at(s.ef, s.nef, k); hit = true; }
#pragma unroll
      for (int k = 0; k < ES_CAP; ++k)
        if (!hit && k < s.nes && ex(s.es[k]) == x && ey(s.es[k]) == y) { remove_at(s.es, s.nes, k); hit = true; }
      if (hit) { remove_at(s.fb, s.nfb, i); r += 1; }
    }
    // ---- divers: picked up on the sub's cell while fewer than 6 are aboard, else move every DIVER_MOVE_INTERVAL + 1
#pragma unroll
    for (int i = DV_CAP - 1; i >= 0; --i) {
      if (i >= s.ndv) continue;
      const uint32_t d = s.dv[i];
      const int y = ey(d), lr = elr(d);
      if (ex(d) == s.sub_x && y == s.sub_y && s.diver_count < 6) { remove_at(s.dv, s.ndv, i); s.diver_count += 1; }
      else if (emt(d) == 0) {
        const int x = ex(d) + (lr ? 1 : -1);
        if (x < 0 || x > 9) remove_at(s.dv, s.ndv, i);
        else if (x == s.sub_x && y == s.sub_y && s.diver_count < 6) { remove_at(s.dv, s.ndv, i); s.diver_count += 1; }
        else s.dv[i] = emake(x, y, lr, DIVER_MOVE_INTERVAL, 0);
      } else {
        s.dv[i] = emake(ex(d), y, lr, emt(d) - 1, 0);
      }
    }
    // ---- enemy subs: collide, move every move_speed + 1 steps (a bullet on the new cell sinks them, +1), shoot
    //      every ENEMY_SHOT_INTERVAL + 1 steps.  A sub removed this step still fires (MinAtar updates the removed
    //      entry), so a sub that left the board appends a bullet at x = -1 or 10.  It is stored as x & 15 (15 or
    //      10), never meets the sub, and the enemy bullet pass below moves it to 14 or 11 and removes it, as MinAtar
    //      removes x = -2 or 11; until then it holds a list slot, as in MinAtar.
#pragma unroll
    for (int i = ES_CAP - 1; i >= 0; --i) {
      if (i >= s.nes) continue;
      const uint32_t e = s.es[i];
      int x = ex(e), mt = emt(e), st = est(e);
      const int y = ey(e), lr = elr(e);
      if (x == s.sub_x && y == s.sub_y) term = true;
      bool gone = false;
      if (mt == 0) {
        mt = s.move_speed;
        x += lr ? 1 : -1;
        if (x < 0 || x > 9) gone = true;
        else if (x == s.sub_x && y == s.sub_y) term = true;
        else {
#pragma unroll
          for (int k = 0; k < FB_CAP; ++k)
            if (!gone && k < s.nfb && ex(s.fb[k]) == x && ey(s.fb[k]) == y) { remove_at(s.fb, s.nfb, k); gone = true; r += 1; }
        }
      } else {
        mt -= 1;
      }
      if (st == 0) {
        st = ENEMY_SHOT_INTERVAL;
        append(s.eb, s.neb, emake(x & 15, y, lr, 0, 0));
      } else {
        st -= 1;
      }
      if (gone) remove_at(s.es, s.nes, i);
      else s.es[i] = emake(x, y, lr, mt, st);
    }
    // ---- enemy bullets: collide, move one cell, collide
#pragma unroll
    for (int i = EB_CAP - 1; i >= 0; --i) {
      if (i >= s.neb) continue;
      const uint32_t b = s.eb[i];
      const int y = ey(b), lr = elr(b);
      if (ex(b) == s.sub_x && y == s.sub_y) term = true;
      const int x = ex(b) + (lr ? 1 : -1);
      if (x < 0 || x > 9) remove_at(s.eb, s.neb, i);
      else {
        s.eb[i] = emake(x, y, lr, 0, 0);
        if (x == s.sub_x && y == s.sub_y) term = true;
      }
    }
    // ---- enemy fish: as the subs, without shots
#pragma unroll
    for (int i = EF_CAP - 1; i >= 0; --i) {
      if (i >= s.nef) continue;
      const uint32_t e = s.ef[i];
      int x = ex(e), mt = emt(e);
      const int y = ey(e), lr = elr(e);
      if (x == s.sub_x && y == s.sub_y) term = true;
      bool gone = false;
      if (mt == 0) {
        mt = s.move_speed;
        x += lr ? 1 : -1;
        if (x < 0 || x > 9) gone = true;
        else if (x == s.sub_x && y == s.sub_y) term = true;
        else {
#pragma unroll
          for (int k = 0; k < FB_CAP; ++k)
            if (!gone && k < s.nfb && ex(s.fb[k]) == x && ey(s.fb[k]) == y) { remove_at(s.fb, s.nfb, k); gone = true; r += 1; }
        }
      } else {
        mt -= 1;
      }
      if (gone) remove_at(s.ef, s.nef, i);
      else s.ef[i] = emake(x, y, lr, mt, 0);
    }
    // ---- timers, oxygen, surfacing
    s.e_spawn_timer -= s.e_spawn_timer > 0 ? 1 : 0;
    s.d_spawn_timer -= s.d_spawn_timer > 0 ? 1 : 0;
    s.shot_timer -= s.shot_timer > 0 ? 1 : 0;
    if (s.oxygen < 0) term = true;
    if (s.sub_y > 0) {
      s.oxygen -= 1;
      s.surface = false;
    } else if (!s.surface) {
      if (s.diver_count == 0) {
        term = true;
      } else {
        s.surface = true;
        if (s.diver_count == 6) { s.diver_count = 0; r += oxygen_tenths(s.oxygen); }
        else s.diver_count -= 1;
        s.oxygen = MAX_OXYGEN;
        if (s.e_spawn_speed > 1 || s.move_speed > 2) {
          if (s.move_speed > 2 && (s.ramp_index & 1)) s.move_speed -= 1;
          if (s.e_spawn_speed > 1) s.e_spawn_speed -= 1;
          s.ramp_index += 1;
        }
      }
    }
    reward = (float)r;
    s.time += 1;
    done = term || s.time >= max_steps;
    s.terminal = done;
  }

  // channels: sub_front, sub_back, friendly_bullet, trail, enemy_bullet, enemy_fish, enemy_sub, oxygen_guage,
  // diver_guage, diver
  PQN_HD static void obs_bits_mem(const State& s, uint32_t* o, int stride) {
    using namespace sq;
    obs_set_bit(o, stride, (s.sub_y * 10 + s.sub_x) * OBS_C + 0);
    const int back = s.sub_or ? s.sub_x - 1 : s.sub_x + 1;   // on the board: l / r move before they turn the sub
    obs_set_bit(o, stride, (s.sub_y * 10 + back) * OBS_C + 1);
    // state[9, 0:oxygen*10//max_oxygen]: at oxygen -1 the slice 0:-1 covers columns 0..8
    const int og = s.oxygen >= 0 ? oxygen_tenths(s.oxygen) : 9;
    for (int x = 0; x < og; ++x) obs_set_bit(o, stride, (90 + x) * OBS_C + 7);
    for (int x = 9 - s.diver_count; x < 9; ++x) obs_set_bit(o, stride, (90 + x) * OBS_C + 8);
#pragma unroll
    for (int k = 0; k < FB_CAP; ++k)
      if (k < s.nfb) obs_set_bit(o, stride, (ey(s.fb[k]) * 10 + ex(s.fb[k])) * OBS_C + 2);
#pragma unroll
    for (int k = 0; k < EB_CAP; ++k)
      if (k < s.neb) obs_set_bit(o, stride, (ey(s.eb[k]) * 10 + ex(s.eb[k])) * OBS_C + 4);
#pragma unroll
    for (int k = 0; k < EF_CAP + ES_CAP + DV_CAP; ++k) {
      const bool on = k < EF_CAP ? k < s.nef : (k < EF_CAP + ES_CAP ? k - EF_CAP < s.nes : k - EF_CAP - ES_CAP < s.ndv);
      if (!on) continue;
      const uint32_t e = k < EF_CAP ? s.ef[k] : (k < EF_CAP + ES_CAP ? s.es[k - EF_CAP] : s.dv[k - EF_CAP - ES_CAP]);
      const int ch = k < EF_CAP ? 5 : (k < EF_CAP + ES_CAP ? 6 : 9);
      const int x = ex(e), y = ey(e), bx = elr(e) ? x - 1 : x + 1;
      obs_set_bit(o, stride, (y * 10 + x) * OBS_C + ch);
      if (bx >= 0 && bx <= 9) obs_set_bit(o, stride, (y * 10 + bx) * OBS_C + 3);
    }
  }
};

}  // namespace pqn
