"""NumPy restatement of MinAtar's Seaquest (``minatar/environments/seaquest.py``, Young & Tian 2019) in gymnax 0.0.6's
conventions, test infrastructure for the Seaquest-MinAtar env operator (``purejaxql_b200/csrc/env_seaquest.cuh``).

gymnax 0.0.6 does not register ``Seaquest-MinAtar``, so there is no JAX port to restate: the game logic below follows
MinAtar's ``Env.act`` line by line, on Python lists walked backwards with removal, as MinAtar does.  It plugs into the
batched gymnax protocol of ``oracle/gymnax_envs.py`` (``Environment`` auto-reset, ``LogWrapper``), reused unchanged;
use :func:`make` below, as ``oracle.gymnax_envs.make`` does not know this env.

The state is a dict of per-env arrays, with the lists as zero-padded ``[n, capacity, fields]`` arrays plus their
lengths ``n_<list>``: ``f_bullets`` (x, y, lr), ``e_bullets`` (x, y, lr), ``e_fish`` (x, y, lr, move_timer),
``e_subs`` (x, y, lr, move_timer, shot_timer), ``divers`` (x, y, lr, move_timer).  ``purejaxql_b200.envs.
state_to_fields`` returns the same keys.

PARITY UNPINNED: neither MinAtar nor a gymnax that registers the game is installed here, and every point of the list at
the end of this file rests on recollection of MinAtar's code.  ``tests/golden/make_seaquest_golden_from_ref.py``
records real trajectories that check them.
"""
from __future__ import annotations

import numpy as np

from oracle import gymnax_envs as G
from oracle import jax_prng as jr

F32 = np.float32
I32 = np.int32

RAMP_INTERVAL = 100            # defined by MinAtar, unused by Seaquest (S9)
MAX_OXYGEN = 200
INIT_SPAWN_SPEED = 20
DIVER_SPAWN_SPEED = 30
INIT_MOVE_INTERVAL = 5
SHOT_COOL_DOWN = 5
ENEMY_SHOT_INTERVAL = 10
ENEMY_MOVE_INTERVAL = 5        # defined by MinAtar; enemies move at the ramped move_speed instead
DIVER_MOVE_INTERVAL = 5

CAPS = {"f_bullets": 2, "e_fish": 8, "e_subs": 8, "e_bullets": 8, "divers": 4}
WIDTH = {"f_bullets": 3, "e_fish": 4, "e_subs": 5, "e_bullets": 3, "divers": 4}
SCALARS = ("oxygen", "diver_count", "sub_x", "sub_y", "shot_timer", "move_speed", "ramp_index", "e_spawn_speed",
           "e_spawn_timer", "d_spawn_timer", "time")
FLAGS = ("sub_or", "surface", "terminal")
CHANNELS = ("sub_front", "sub_back", "friendly_bullet", "trail", "enemy_bullet", "enemy_fish", "enemy_sub",
            "oxygen_guage", "diver_guage", "diver")


def _unpack(s, i):
    """env i of the batched state -> MinAtar-style attributes with Python lists"""
    e = {k: int(s[k][i]) for k in SCALARS}
    e.update({k: bool(s[k][i]) for k in FLAGS})
    for name in CAPS:
        e[name] = [list(map(int, row)) for row in s[name][i, :int(s["n_" + name][i])]]
    return e


def _pack(envs):
    n = len(envs)
    s = {k: np.array([e[k] for e in envs], I32) for k in SCALARS}
    s.update({k: np.array([e[k] for e in envs], bool) for k in FLAGS})
    for name, cap in CAPS.items():
        a = np.zeros((n, cap, WIDTH[name]), I32)
        for i, e in enumerate(envs):
            if e[name]:
                a[i, :len(e[name])] = np.array(e[name], I32)
        s[name] = a
        s["n_" + name] = np.array([len(e[name]) for e in envs], I32)
    return s


def _append(e, name, entry):
    if len(e[name]) < CAPS[name]:           # S14: an append to a full list is dropped
        e[name].append(entry)


class Seaquest:
    name = "Seaquest-MinAtar"
    obs_shape = (10, 10, 10)
    num_actions = 6                        # n, l, u, r, d, f (S2)
    max_steps_in_episode = 1000            # S12

    def reset_env(self, key):
        n = key.shape[0]
        e = dict(oxygen=MAX_OXYGEN, diver_count=0, sub_x=5, sub_y=0, sub_or=False, f_bullets=[], e_bullets=[],
                 e_fish=[], e_subs=[], divers=[], e_spawn_speed=INIT_SPAWN_SPEED, e_spawn_timer=INIT_SPAWN_SPEED,
                 d_spawn_timer=DIVER_SPAWN_SPEED, move_speed=INIT_MOVE_INTERVAL, ramp_index=0, shot_timer=0,
                 surface=True, terminal=False, time=0)
        s = _pack([dict(e, **{k: [] for k in CAPS}) for _ in range(n)])
        return self.get_obs(s), s

    def get_obs(self, s):
        n = s["sub_x"].shape[0]
        obs = np.zeros((n, 10, 10, 10), bool)
        for i in range(n):
            e = _unpack(s, i)
            o = obs[i]
            o[e["sub_y"], e["sub_x"], 0] = 1
            back_x = e["sub_x"] - 1 if e["sub_or"] else e["sub_x"] + 1
            o[e["sub_y"], back_x, 1] = 1
            o[9, 0:e["oxygen"] * 10 // MAX_OXYGEN, 7] = 1          # S11: Python slice, 0:-1 at oxygen -1
            o[9, 9 - e["diver_count"]:9, 8] = 1
            for b in e["f_bullets"]:
                o[b[1], b[0], 2] = 1
            for b in e["e_bullets"]:
                o[b[1], b[0], 4] = 1
            for name, ch in (("e_fish", 5), ("e_subs", 6), ("divers", 9)):
                for z in e[name]:
                    o[z[1], z[0], ch] = 1
                    bx = z[0] - 1 if z[2] else z[0] + 1
                    if 0 <= bx <= 9:
                        o[z[1], bx, 3] = 1
        return obs.astype(F32)

    @staticmethod
    def draws(key):
        """the five draws of a step, for every env (used only where a spawn timer is 0)"""
        n = key.shape[0]
        ks = jr.split(key, 5)
        enemy_lr = (1 - jr.randint(ks[:, 0], (), 0, 2)).astype(I32)                   # choice([True, False])
        is_sub = (1 - G._choice_p(ks[:, 1], np.tile(np.array([1 / 3, 2 / 3], F32), (n, 1)))).astype(I32)
        enemy_y = (1 + jr.randint(ks[:, 2], (), 0, 8)).astype(I32)                    # choice(arange(1, 9))
        diver_lr = (1 - jr.randint(ks[:, 3], (), 0, 2)).astype(I32)
        diver_y = (1 + jr.randint(ks[:, 4], (), 0, 8)).astype(I32)
        return enemy_lr, is_sub, enemy_y, diver_lr, diver_y

    @staticmethod
    def act(e, a, enemy_lr, is_sub, enemy_y, diver_lr, diver_y):
        """MinAtar Env.act on one env (lists mutated in place) -> (reward, terminal)"""
        r = 0
        terminal = False
        pos = lambda z: z[0:2] == [e["sub_x"], e["sub_y"]]
        # spawn enemy
        if e["e_spawn_timer"] == 0:
            lr, y = bool(enemy_lr), int(enemy_y)
            if not any(z[1] == y and bool(z[2]) != lr for z in e["e_subs"] + e["e_fish"]):
                x = 0 if lr else 9
                if is_sub:
                    _append(e, "e_subs", [x, y, int(lr), e["move_speed"], ENEMY_SHOT_INTERVAL])
                else:
                    _append(e, "e_fish", [x, y, int(lr), e["move_speed"]])
            e["e_spawn_timer"] = e["e_spawn_speed"]
        # spawn diver
        if e["d_spawn_timer"] == 0:
            lr = bool(diver_lr)
            _append(e, "divers", [0 if lr else 9, int(diver_y), int(lr), DIVER_MOVE_INTERVAL])
            e["d_spawn_timer"] = DIVER_SPAWN_SPEED
        # player
        if a == 5 and e["shot_timer"] == 0:
            _append(e, "f_bullets", [e["sub_x"], e["sub_y"], int(e["sub_or"])])
            e["shot_timer"] = SHOT_COOL_DOWN
        elif a == 1:
            e["sub_x"] = max(0, e["sub_x"] - 1)
            e["sub_or"] = False
        elif a == 3:
            e["sub_x"] = min(9, e["sub_x"] + 1)
            e["sub_or"] = True
        elif a == 2:
            e["sub_y"] = max(0, e["sub_y"] - 1)
        elif a == 4:
            e["sub_y"] = min(8, e["sub_y"] + 1)
        # friendly bullets
        fb = e["f_bullets"]
        for i in reversed(range(len(fb))):
            b = fb[i]
            b[0] += 1 if b[2] else -1
            if b[0] < 0 or b[0] > 9:
                fb.pop(i)
                continue
            hit = False
            for lst in (e["e_fish"], e["e_subs"]):
                for k, z in enumerate(lst):
                    if not hit and z[0:2] == b[0:2]:
                        lst.pop(k)
                        hit = True
                        break
            if hit:
                fb.pop(i)
                r += 1
        # divers
        dv = e["divers"]
        for i in reversed(range(len(dv))):
            d = dv[i]
            if pos(d) and e["diver_count"] < 6:
                dv.pop(i)
                e["diver_count"] += 1
            elif d[3] == 0:
                d[3] = DIVER_MOVE_INTERVAL
                d[0] += 1 if d[2] else -1
                if d[0] < 0 or d[0] > 9:
                    dv.pop(i)
                elif pos(d) and e["diver_count"] < 6:
                    dv.pop(i)
                    e["diver_count"] += 1
            else:
                d[3] -= 1
        # enemy subs
        es = e["e_subs"]
        for i in reversed(range(len(es))):
            z = es[i]
            if pos(z):
                terminal = True
            gone = False
            if z[3] == 0:
                z[3] = e["move_speed"]
                z[0] += 1 if z[2] else -1
                if z[0] < 0 or z[0] > 9:
                    gone = True
                elif pos(z):
                    terminal = True
                else:
                    for k, b in enumerate(fb):
                        if z[0:2] == b[0:2]:
                            gone = True
                            fb.pop(k)
                            r += 1
                            break
            else:
                z[3] -= 1
            if z[4] == 0:
                z[4] = ENEMY_SHOT_INTERVAL
                _append(e, "e_bullets", [z[0], z[1], z[2]])
            else:
                z[4] -= 1
            if gone:
                es.pop(i)
        # enemy bullets
        eb = e["e_bullets"]
        for i in reversed(range(len(eb))):
            b = eb[i]
            if pos(b):
                terminal = True
            b[0] += 1 if b[2] else -1
            if b[0] < 0 or b[0] > 9:
                eb.pop(i)
            elif pos(b):
                terminal = True
        # enemy fish
        ef = e["e_fish"]
        for i in reversed(range(len(ef))):
            z = ef[i]
            if pos(z):
                terminal = True
            if z[3] == 0:
                z[3] = e["move_speed"]
                z[0] += 1 if z[2] else -1
                if z[0] < 0 or z[0] > 9:
                    ef.pop(i)
                elif pos(z):
                    terminal = True
                else:
                    for k, b in enumerate(fb):
                        if z[0:2] == b[0:2]:
                            ef.pop(i)
                            fb.pop(k)
                            r += 1
                            break
            else:
                z[3] -= 1
        # timers, oxygen, surfacing
        e["e_spawn_timer"] -= e["e_spawn_timer"] > 0
        e["d_spawn_timer"] -= e["d_spawn_timer"] > 0
        e["shot_timer"] -= e["shot_timer"] > 0
        if e["oxygen"] < 0:
            terminal = True
        if e["sub_y"] > 0:
            e["oxygen"] -= 1
            e["surface"] = False
        elif not e["surface"]:
            if e["diver_count"] == 0:
                terminal = True
            else:
                e["surface"] = True
                if e["diver_count"] == 6:
                    e["diver_count"] = 0
                    r += e["oxygen"] * 10 // MAX_OXYGEN
                else:
                    e["diver_count"] -= 1
                e["oxygen"] = MAX_OXYGEN
                if e["e_spawn_speed"] > 1 or e["move_speed"] > 2:
                    if e["move_speed"] > 2 and e["ramp_index"] % 2:
                        e["move_speed"] -= 1
                    if e["e_spawn_speed"] > 1:
                        e["e_spawn_speed"] -= 1
                    e["ramp_index"] += 1
        return r, terminal

    def step_env(self, key, s, action):
        n = action.shape[0]
        dr = self.draws(key)
        envs, reward, term = [], np.zeros(n, F32), np.zeros(n, bool)
        for i in range(n):
            e = _unpack(s, i)
            r, t = self.act(e, int(action[i]), *(int(d[i]) for d in dr))
            reward[i], term[i] = r, t
            envs.append(e)
        ns = _pack(envs)
        ns["time"] = (s["time"] + 1).astype(I32)
        done = term | (ns["time"] >= self.max_steps_in_episode)
        ns["terminal"] = done
        info = {"discount": np.where(done, F32(0.0), F32(1.0)).astype(F32)}
        return self.get_obs(ns), ns, reward, done, info


def make(flatten: bool = False, log: bool = True, max_steps: int | None = None):
    core = Seaquest()
    if max_steps is not None:
        core.max_steps_in_episode = max_steps
    env = G.Environment(core, flatten=flatten)
    return G.LogWrapper(env) if log else env


# Assumptions (each rests on recollection of MinAtar's seaquest.py and gymnax's MinAtar conventions):
#
#  S1. Channel order sub_front, sub_back, friendly_bullet, trail, enemy_bullet, enemy_fish, enemy_sub, oxygen_guage,
#      diver_guage, diver; the observation is bool (10, 10, 10) cast to float32, cells set, not added.
#  S2. Actions 0..5 = n, l, u, r, d, f; MinAtar's minimal action set is its full set for this game.  l and r move the
#      sub one column (clipped to 0..9) and turn it; u and d move it one row, clipped to 0..8; f fires when the shot
#      timer is 0 and then sets it to SHOT_COOL_DOWN = 5; one action per step, f taking precedence only as listed.
#  S3. Order of one step: spawn enemy, spawn diver, player, friendly bullets, divers, enemy subs, enemy bullets, enemy
#      fish, timers, oxygen and surfacing.  Each list is walked from its last entry to its first.
#  S4. Friendly bullets move one cell in their sub's facing at firing time and leave the board past 0..9; on a cell
#      with a fish the first such fish is removed, else the first sub on it, with the bullet, for +1.  MinAtar's sub
#      loop has no break; with two subs on one cell it would remove the bullet twice and raise, so one hit is taken.
#  S5. Enemies move every move_speed + 1 steps (a timer reloaded with the current move_speed), divers every
#      DIVER_MOVE_INTERVAL + 1 = 6 steps; an enemy that moves onto a friendly bullet is removed with it for +1, and
#      an enemy on the sub's cell, before or after its move, ends the episode.
#  S6. Enemy subs fire every ENEMY_SHOT_INTERVAL + 1 = 11 steps from their cell after moving, in their direction; a
#      sub removed in the same step still fires (MinAtar keeps updating the removed entry).  Enemy bullets end the
#      episode on the sub's cell before or after their one-cell move.
#  S7. Enemy spawn: every e_spawn_speed steps (timer reloaded, then decremented the same step), lr = choice([True,
#      False]), is_sub = choice([True, False], p=[1/3, 2/3]), row = choice(arange(1, 9)), x = 0 moving right or 9
#      moving left; no spawn when an enemy in that row faces the other way.  New entries take the current move_speed
#      and, for subs, ENEMY_SHOT_INTERVAL.
#  S8. Diver spawn every DIVER_SPAWN_SPEED = 30 steps (first at step 30), lr and row drawn as for enemies; a diver on
#      the sub's cell, before or after its move, is picked up while fewer than 6 are aboard.
#  S9. Oxygen starts at MAX_OXYGEN = 200 and drops by 1 each step below row 0; oxygen < 0 at the check ends the
#      episode.  Returning to row 0 after a dive: with no diver the episode ends; with 6 the reward is oxygen * 10 //
#      200 and all six leave; otherwise one diver is lost.  Either way oxygen refills and the difficulty ramps: while
#      e_spawn_speed > 1 or move_speed > 2, move_speed drops by 1 (not below 2) at odd ramp_index, e_spawn_speed by 1
#      (not below 1), ramp_index += 1.  There is no time-based ramp, so RAMP_INTERVAL is unused.
#  S10. reset: oxygen 200, sub at (x 5, row 0) facing left, no divers, empty lists, e_spawn_speed = e_spawn_timer = 20,
#      d_spawn_timer = 30, move_speed 5, ramp_index 0, shot_timer 0, surface True.  reset draws nothing.
#  S11. The oxygen gauge lights row 9, columns 0:oxygen * 10 // 200 (Python slice: at oxygen -1 that is 0:-1, columns
#      0..8); the diver gauge lights columns 9 - diver_count .. 8 of row 9.  Trails mark the cell behind each fish,
#      sub and diver when it is on the board.
#  S12. gymnax conventions: Environment.step auto-reset, LogWrapper, done = terminal or time >= max_steps_in_episode
#      with time counted per step; max_steps_in_episode defaults to 1000, as the other gymnax MinAtar ports here.  No
#      sticky actions (MinAtar's Environment wrapper has them; gymnax's ports do not).
#  S13. Draws: split(step key, 5) = (enemy lr, enemy is_sub, enemy row, diver lr, diver row); choice without p is
#      randint over the indices, choice with p the cumsum search of jax.random.choice, as in the Asterix port.
#  S14. Lists are capped: 2 friendly bullets (one shot per 5 steps, at most 10 steps on the board), 4 divers (one per
#      30 steps, at most 60 steps on the board: at most 2 alive), 8 fish, 8 subs and 8 enemy bullets; an append to a
#      full list is dropped.  Only the enemy lists can reach their caps, and only deep into the difficulty ramp.
#  S15. Entries are removed by position.  MinAtar's list.remove drops the first entry equal in every field, which
#      differs only when two entries of one list are equal in every field.
