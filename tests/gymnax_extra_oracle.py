"""NumPy restatements of gymnax==0.0.6 ``environments/classic_control/mountain_car.py`` (``MountainCar``) and
``environments/bsuite/catch.py`` (``Catch``), test infrastructure for the MountainCar-v0 and Catch-bsuite env
operators (``purejaxql_b200/csrc/env_classic.cuh``, ``purejaxql_b200/csrc/env_bsuite.cuh``).

They plug into the batched gymnax protocol of ``oracle/gymnax_envs.py`` (``Environment`` auto-reset,
``LogWrapper``), which they reuse unchanged.  They live here, beside ``tests/bsuite_oracle.py``, rather than in
``oracle/gymnax_envs.py``: the ``oracle`` package is the reference the existing tests measure against and is kept as it
is.  So ``oracle.gymnax_envs.make`` does not know these two envs; use :func:`make` below, or register a class in
``oracle.gymnax_envs._REGISTRY`` for the duration of a test.  Reference call sites: ``purejaxql/pqn_gymnax.py:92`` and
``purejaxql/pqn_rnn_gymnax.py:133-139`` (``gymnax.make(config["ENV_NAME"])``).

PARITY UNPINNED: gymnax is not installable here, and every point below rests on recollection of gymnax's code.
``tests/golden/make_gymnax_extra_golden_from_ref.py`` records real gymnax trajectories and ``EnvParams`` defaults
that check them.

MountainCar-v0:

(M1) EnvParams defaults: min_position -1.2, max_position 0.6, max_speed 0.07, goal_position 0.5, goal_velocity 0.0,
     force 0.001, gravity 0.0025, max_steps_in_episode 200; 3 actions.
(M2) reset_env: position = uniform(key, (), -0.6, -0.4), velocity = 0, time = 0.
(M3) step_env, in fp32 and in this order: velocity += (action - 1) * force - cos(3 * position) * gravity; clip the
     velocity to +-max_speed; position += velocity; clip the position to [min_position, max_position];
     velocity *= 1 - (position == min_position) * (velocity < 0); reward = -1; time += 1.
(M4) done = (position >= goal_position and velocity >= goal_velocity) or time >= max_steps_in_episode.
(M5) the observation is [position, velocity] of the new state.

Catch-bsuite (``gymnax.make`` builds 10 rows and 5 columns):

(C1) reset_env: ball_x = randint(key, (), 0, 5), ball_y = 0, paddle_x = 2, paddle_y = 9, prev_done = False, time = 0.
(C2) step_env: paddle_x = clip(paddle_x + action - 1, 0, 4); ball_y += 1; prev_done = ball_y == paddle_y;
     reward = prev_done * (1.0 * caught + -1.0 * (1 - caught)) with caught = paddle_x == ball_x (-0.0 on an earlier
     step where the paddle is not under the ball); time += 1.
(C3) done = ball_y == paddle_y or time >= max_steps_in_episode, so an episode lasts 9 steps.
(C4) the observation is a (10, 5) float board of zeros with 1 set (not added) at (ball_y, ball_x) and at
     (paddle_y, paddle_x).
(C5) max_steps_in_episode defaults to 1000.  It never binds.
(C6) step_env also draws a fresh initial state from its key and selects it where the incoming prev_done is True.
     A state with prev_done = True is always terminal, so ``Environment.step``'s auto-reset replaces it before
     step_env sees it again.  The draw can never matter, and neither this oracle nor the CUDA env makes it.
"""
from __future__ import annotations

import numpy as np

from oracle import gymnax_envs as G
from oracle import jax_prng as jr

F32 = np.float32
I32 = np.int32


class MountainCar:
    name = "MountainCar-v0"
    obs_shape = (2,)
    num_actions = 3
    state_fields = ("position", "velocity", "time")
    min_position = F32(-1.2)
    max_position = F32(0.6)
    max_speed = F32(0.07)
    goal_position = F32(0.5)
    goal_velocity = F32(0.0)
    force = F32(0.001)
    gravity = F32(0.0025)

    def __init__(self, max_steps_in_episode: int = 200):
        self.max_steps_in_episode = int(max_steps_in_episode)

    def get_obs(self, s):
        return np.stack([s["position"], s["velocity"]], axis=-1).astype(F32)                # (M5)

    def reset_env(self, key):
        n = key.shape[0]
        s = dict(position=jr.uniform(key, (), -0.6, -0.4).astype(F32), velocity=np.zeros(n, F32),
                 time=np.zeros(n, I32))                                                    # (M2)
        return self.get_obs(s), s

    def is_terminal(self, s):
        goal = (s["position"] >= self.goal_position) & (s["velocity"] >= self.goal_velocity)
        return goal | (s["time"] >= self.max_steps_in_episode)                              # (M4)

    def step_env(self, key, s, action):
        af = (action.astype(I32) - 1).astype(F32)                                           # (M3)
        cg = (np.cos((F32(3) * s["position"]).astype(F32)).astype(F32) * self.gravity).astype(F32)
        velocity = ((s["velocity"] + (af * self.force).astype(F32)).astype(F32) - cg).astype(F32)
        velocity = np.clip(velocity, -self.max_speed, self.max_speed).astype(F32)
        position = (s["position"] + velocity).astype(F32)
        position = np.clip(position, self.min_position, self.max_position).astype(F32)
        wall = (position == self.min_position) & (velocity < 0)
        velocity = (velocity * (1 - wall.astype(I32)).astype(F32)).astype(F32)
        ns = dict(position=position, velocity=velocity, time=(s["time"] + 1).astype(I32))
        reward = np.full(action.shape[0], -1.0, F32)
        done = self.is_terminal(ns)
        info = {"discount": np.where(done, F32(0.0), F32(1.0)).astype(F32)}
        return self.get_obs(ns), ns, reward, done, info


class Catch:
    name = "Catch-bsuite"
    rows, columns = 10, 5
    obs_shape = (10, 5)
    num_actions = 3
    state_fields = ("ball_x", "ball_y", "paddle_x", "paddle_y", "prev_done", "time")

    def __init__(self, max_steps_in_episode: int = 1000):
        self.max_steps_in_episode = int(max_steps_in_episode)                               # (C5)

    def get_obs(self, s):
        n = s["ball_x"].shape[0]
        idx = np.arange(n)
        board = np.zeros((n, self.rows, self.columns), F32)
        board[idx, s["ball_y"], s["ball_x"]] = 1.0                                         # (C4)
        board[idx, s["paddle_y"], s["paddle_x"]] = 1.0
        return board

    def reset_env(self, key):
        n = key.shape[0]
        s = dict(ball_x=jr.randint(key, (), 0, self.columns).astype(I32), ball_y=np.zeros(n, I32),
                 paddle_x=np.full(n, self.columns // 2, I32), paddle_y=np.full(n, self.rows - 1, I32),
                 prev_done=np.zeros(n, bool), time=np.zeros(n, I32))                        # (C1)
        return self.get_obs(s), s

    def step_env(self, key, s, action):
        assert not s["prev_done"].any(), "(C6): step_env never sees prev_done = True under auto-reset"
        paddle_x = np.clip(s["paddle_x"] + action.astype(I32) - 1, 0, self.columns - 1).astype(I32)   # (C2)
        ball_y = (s["ball_y"] + 1).astype(I32)
        prev_done = ball_y == s["paddle_y"]
        caught = (paddle_x == s["ball_x"]).astype(F32)
        reward = (prev_done.astype(F32) * (F32(1.0) * caught + F32(-1.0) * (F32(1) - caught))).astype(F32)
        ns = dict(ball_x=s["ball_x"].copy(), ball_y=ball_y, paddle_x=paddle_x, paddle_y=s["paddle_y"].copy(),
                  prev_done=prev_done, time=(s["time"] + 1).astype(I32))
        done = prev_done | (ns["time"] >= self.max_steps_in_episode)                        # (C3)
        info = {"discount": np.where(done, F32(0.0), F32(1.0)).astype(F32)}
        return self.get_obs(ns), ns, reward, done, info


CORES = {"MountainCar-v0": MountainCar, "Catch-bsuite": Catch}


def make(env_name: str, flatten: bool = True, log: bool = True, max_steps_in_episode: int | None = None):
    """``LogWrapper([FlattenObservationWrapper(]gymnax.make(env_name)[)])``; ``max_steps_in_episode`` overrides the
    default ``EnvParams`` field."""
    cls = CORES[env_name]
    core = cls() if max_steps_in_episode is None else cls(max_steps_in_episode)
    env = G.Environment(core, flatten=flatten)
    return G.LogWrapper(env) if log else env
