"""NumPy restatements of gymnax==0.0.6 ``environments/misc/bernoulli_bandit.py`` (``BernoulliBandit``), ``rooms.py``
(``FourRooms``) and ``meta_maze.py`` (``MetaMaze``), test infrastructure for the BernoulliBandit-misc, FourRooms-misc
and MetaMaze-misc env operators (``purejaxql_b200/csrc/env_misc.cuh``).

They plug into the batched gymnax protocol of ``oracle/gymnax_envs.py`` (``Environment`` auto-reset, ``LogWrapper``),
which they reuse unchanged, as ``tests/bsuite_chains_oracle.py`` does; :func:`make` also builds SimpleBandit-bsuite
from ``tests/bsuite_bandit_oracle.py``.  Reference call sites: ``purejaxql/pqn_gymnax.py:92`` and
``purejaxql/pqn_rnn_gymnax.py:133-139`` (``gymnax.make(config["ENV_NAME"])`` with default ``EnvParams``).

PARITY UNPINNED: gymnax is not installable here, and every point below rests on recollection of gymnax's code.
``tests/golden/make_misc_golden_from_ref.py`` records real gymnax trajectories and ``EnvParams`` defaults that check
them.

Shared by BernoulliBandit and MetaMaze:

(T1) get_obs's time entry is time_normalization(time) = (max_lim - min_lim) * t / t_max + min_lim with its defaults
     min_lim -1, max_lim 1, t_max 100 (not max_steps_in_episode), as get_obs calls it under normalize_time = True:
     2 * t / 100 - 1 in fp32, left to right.  (The other reading, t / max_steps_in_episode, is not restated.)
(T2) one_hot(last_action) comes before last_reward in the observation.

BernoulliBandit-misc (``gymnax.make`` builds num_arms = 2):

(N1) EnvParams defaults: sample_probs [0.1, 0.9] (Wang et al.'s "easy" set; the least certain default),
     normalize_time True, max_steps_in_episode 100; 2 actions.
(N2) reset_env: p1 = choice(key, sample_probs, (1,)), which without p and with replacement is
     sample_probs[randint(key, (1,), 0, 2)]; reward_probs = [p1, 1 - p1] (fp32), exp_reward_best = max(reward_probs),
     last_action 0, last_reward 0, time 0.
(N3) step_env: reward = bernoulli(key, reward_probs[action]) = uniform(key, ()) < reward_probs[action], drawn from the
     step key itself; last_action = action, last_reward = reward, time += 1.
(N4) done = time >= max_steps_in_episode, so every episode lasts 100 steps.
(N5) the observation is [one_hot(last_action, 2), last_reward, time_normalization(time)]: 4 floats.

FourRooms-misc (``gymnax.make`` builds use_visual_obs False, goal_fixed [8, 9], pos_fixed [4, 1]):

(R1) EnvParams defaults: fail_prob 1/3, resample_init_pos False, resample_goal_pos False, max_steps_in_episode 500;
     4 actions; directions [[-1, 0], [0, 1], [1, 0], [0, -1]].
(R2) the 13 x 13 map of ``FOUR_ROOMS_MAP`` ('x' a wall), walkable where ' '.
(R3) reset_env: rng_goal, rng_pos = split(key); gymnax draws a goal and a position from them and selects them away
     (resample_* False), so goal = [8, 9], pos = [4, 1], time 0.  Neither draw reaches an output; this oracle does not
     make them.
(R4) step_env: key_random, key_action = split(key); the action is replaced by randint(key_action, (), 0, 4) where
     uniform(key_random, ()) < fail_prob * 4 / 3 (fp32); p = pos + directions[action]; pos = p if the map is open at
     p, else pos; reward = pos == goal (1.0 or 0.0); time += 1.
(R5) done = pos == goal or time >= max_steps_in_episode.
(R6) the observation is [pos[0], pos[1], goal[0], goal[1]]: 4 floats.

MetaMaze-misc (``gymnax.make`` builds maze_size 9, rf_size 3):

(M1) EnvParams defaults: reward 10.0, punishment 0.0 (not read by the step), normalize_time True,
     max_steps_in_episode 200; 4 actions; directions as (R1).
(M2) the map: walls on the border and at every (even row, even column) inside, except the centre (4, 4); coords are
     its 41 free cells in row-major order.
(M3) reset_pos(key, coords, goal): k = randint(key, (), 0, 40); coords[40] where coords[k] == goal, else coords[k].
(M4) reset_env: rng_goal, rng_pos = split(key); goal = coords[randint(rng_goal, (), 0, 41)];
     pos = reset_pos(rng_pos, coords, goal); last_action 0, last_reward 0.0, time 0.
(M5) step_env: p = pos + directions[action]; pos = pos if p is a wall, else p; goal_reached = pos == goal;
     reward = goal_reached * reward (fp32); where goal_reached, pos = reset_pos(key, coords, goal) with the step key
     itself; last_action = action, last_reward = reward, time += 1.
(M6) done = time >= max_steps_in_episode, so every episode lasts 200 steps.
(M7) the observation is [the 3 x 3 map around pos (1.0 = wall), one_hot(last_action, 4), last_reward,
     time_normalization(time)]: 15 floats.
"""
from __future__ import annotations

import numpy as np

import bsuite_bandit_oracle as BB
from oracle import gymnax_envs as G
from oracle import jax_prng as jr

F32 = np.float32
I32 = np.int32
DIRECTIONS = np.array([[-1, 0], [0, 1], [1, 0], [0, -1]], I32)


def _discount(done):
    return {"discount": np.where(done, F32(0.0), F32(1.0)).astype(F32)}


def time_normalization(t):
    """(T1): fp32 ``(1.0 - -1.0) * t / 100 + -1.0``."""
    return ((F32(2.0) * np.asarray(t).astype(F32)).astype(F32) / F32(100)).astype(F32) + F32(-1.0)


def one_hot(a, n):
    return (np.asarray(a)[:, None] == np.arange(n)[None, :]).astype(F32)


class BernoulliBandit:
    name = "BernoulliBandit-misc"
    obs_shape = (4,)
    num_actions = 2
    sample_probs = np.array([0.1, 0.9], F32)                                                # (N1)
    state_fields = ("last_action", "last_reward", "exp_reward_best", "reward_probs", "time")

    def __init__(self, max_steps_in_episode: int = 100):
        self.max_steps_in_episode = int(max_steps_in_episode)

    def get_obs(self, s):                                                                   # (N5)
        return np.concatenate([one_hot(s["last_action"], 2), s["last_reward"].astype(F32)[:, None],
                               time_normalization(s["time"])[:, None]], 1).astype(F32)

    def reset_env(self, key):
        n = key.shape[0]
        p1 = self.sample_probs[jr.randint(key, (), 0, 2)]                                  # (N2)
        probs = np.stack([p1, (F32(1) - p1).astype(F32)], 1).astype(F32)
        s = dict(last_action=np.zeros(n, I32), last_reward=np.zeros(n, I32), reward_probs=probs,
                 exp_reward_best=probs.max(1), time=np.zeros(n, I32))
        return self.get_obs(s), s

    def step_env(self, key, s, action):
        n = action.shape[0]
        p = s["reward_probs"][np.arange(n), action.astype(np.int64)]
        r = (jr.uniform(key, ()) < p).astype(I32)                                          # (N3)
        ns = dict(last_action=action.astype(I32), last_reward=r, reward_probs=s["reward_probs"].copy(),
                  exp_reward_best=s["exp_reward_best"].copy(), time=(s["time"] + 1).astype(I32))
        done = ns["time"] >= self.max_steps_in_episode                                     # (N4)
        return self.get_obs(ns), ns, r.astype(F32), done, _discount(done)


FOUR_ROOMS_MAP = """
xxxxxxxxxxxxx
x     x     x
x     x     x
x           x
x     x     x
x     x     x
xx xxxx     x
x     xxx xxx
x     x     x
x     x     x
x           x
x     x     x
xxxxxxxxxxxxx"""


class FourRooms:
    name = "FourRooms-misc"
    obs_shape = (4,)
    num_actions = 4
    env_map = np.array([[ch == " " for ch in row] for row in FOUR_ROOMS_MAP.split("\n")[1:]])   # (R2) True = open
    goal_fixed = np.array([8, 9], I32)
    pos_fixed = np.array([4, 1], I32)
    fail_prob = F32(1.0 / 3)
    state_fields = ("pos", "goal", "time")

    def __init__(self, max_steps_in_episode: int = 500):
        self.max_steps_in_episode = int(max_steps_in_episode)                                # (R1)

    def get_obs(self, s):                                                                   # (R6)
        return np.concatenate([s["pos"], s["goal"]], 1).astype(F32)

    def reset_env(self, key):
        n = key.shape[0]                                                                    # (R3)
        s = dict(pos=np.tile(self.pos_fixed, (n, 1)), goal=np.tile(self.goal_fixed, (n, 1)), time=np.zeros(n, I32),
                 fail_prob=np.full(n, self.fail_prob, F32))
        return self.get_obs(s), s

    def step_env(self, key, s, action):
        ks = jr.split(key, 2)                                                               # (R4)
        thresh = ((s["fail_prob"] * F32(4)).astype(F32) / F32(3)).astype(F32)
        rand = jr.uniform(ks[:, 0], ()) < thresh
        action = np.where(rand, jr.randint(ks[:, 1], (), 0, 4), action).astype(I32)
        p = s["pos"] + DIRECTIONS[action]
        ok = self.env_map[p[:, 0], p[:, 1]]
        pos = np.where(ok[:, None], p, s["pos"]).astype(I32)
        at_goal = (pos == s["goal"]).all(1)
        ns = dict(pos=pos, goal=s["goal"].copy(), time=(s["time"] + 1).astype(I32), fail_prob=s["fail_prob"].copy())
        done = at_goal | (ns["time"] >= self.max_steps_in_episode)                         # (R5)
        return self.get_obs(ns), ns, at_goal.astype(F32), done, _discount(done)


def _meta_maze_map(size=9):
    m = np.zeros((size, size), F32)
    m[0, :] = m[-1, :] = m[:, 0] = m[:, -1] = 1
    for r in range(1, size - 1):
        for c in range(1, size - 1):
            if r % 2 == 0 and c % 2 == 0:
                m[r, c] = 1
    m[size // 2, size // 2] = 0
    return m                                                                                # (M2)


class MetaMaze:
    name = "MetaMaze-misc"
    obs_shape = (15,)
    num_actions = 4
    env_map = _meta_maze_map()
    coords = np.argwhere(env_map == 0).astype(I32)                                         # row-major
    goal_reward = F32(10.0)
    state_fields = ("last_action", "last_reward", "pos", "goal", "time")

    def __init__(self, max_steps_in_episode: int = 200):
        self.max_steps_in_episode = int(max_steps_in_episode)                                # (M1)

    def get_obs(self, s):                                                                   # (M7)
        n = s["pos"].shape[0]
        off = np.arange(-1, 2)
        rows = s["pos"][:, 0, None, None] + off[None, :, None]
        cols = s["pos"][:, 1, None, None] + off[None, None, :]
        rf = self.env_map[rows, cols].reshape(n, 9)
        return np.concatenate([rf, one_hot(s["last_action"], 4), s["last_reward"][:, None].astype(F32),
                               time_normalization(s["time"])[:, None]], 1).astype(F32)

    def reset_pos(self, key, goal):                                                         # (M3)
        k = jr.randint(key, (), 0, len(self.coords) - 1)
        c = self.coords[k]
        hit = (c == goal).all(1)
        return np.where(hit[:, None], self.coords[-1], c).astype(I32)

    def reset_env(self, key):
        n = key.shape[0]
        ks = jr.split(key, 2)                                                               # (M4)
        goal = self.coords[jr.randint(ks[:, 0], (), 0, len(self.coords))]
        pos = self.reset_pos(ks[:, 1], goal)
        s = dict(last_action=np.zeros(n, I32), last_reward=np.zeros(n, F32), pos=pos, goal=goal.astype(I32),
                 time=np.zeros(n, I32), reward=np.full(n, self.goal_reward, F32))
        return self.get_obs(s), s

    def step_env(self, key, s, action):
        p = s["pos"] + DIRECTIONS[action]                                                   # (M5)
        blocked = self.env_map[p[:, 0], p[:, 1]] == 1
        pos = np.where(blocked[:, None], s["pos"], p).astype(I32)
        reached = (pos == s["goal"]).all(1)
        reward = (reached.astype(F32) * s["reward"]).astype(F32)
        pos = np.where(reached[:, None], self.reset_pos(key, s["goal"]), pos).astype(I32)
        ns = dict(last_action=action.astype(I32), last_reward=reward, pos=pos, goal=s["goal"].copy(),
                  time=(s["time"] + 1).astype(I32), reward=s["reward"].copy())
        done = ns["time"] >= self.max_steps_in_episode                                     # (M6)
        return self.get_obs(ns), ns, reward, done, _discount(done)


CORES = {"SimpleBandit-bsuite": BB.SimpleBandit, "BernoulliBandit-misc": BernoulliBandit, "FourRooms-misc": FourRooms,
         "MetaMaze-misc": MetaMaze}


def make(env_name: str, flatten: bool = True, log: bool = True, max_steps_in_episode: int | None = None):
    """``LogWrapper([FlattenObservationWrapper(]gymnax.make(env_name)[)])``; ``max_steps_in_episode`` overrides the
    default ``EnvParams`` field."""
    cls = CORES[env_name]
    core = cls() if max_steps_in_episode is None else cls(max_steps_in_episode)
    env = G.Environment(core, flatten=flatten)
    return G.LogWrapper(env) if log else env
