"""NumPy restatement of gymnax==0.0.6 ``environments/misc/gaussian_bandit.py`` (``GaussianBandit``), test
infrastructure for the GaussianBandit-misc env operator (``GaussianBanditEnv`` in ``purejaxql_b200/csrc/env_misc.cuh``).

It plugs into the batched gymnax protocol of ``oracle/gymnax_envs.py`` (``Environment`` auto-reset, ``LogWrapper``),
which it reuses unchanged, and draws its normals from ``tests/jax_normal_oracle.py``.  Reference call sites:
``purejaxql/pqn_gymnax.py:92`` and ``purejaxql/pqn_rnn_gymnax.py:133-139`` (``gymnax.make(config["ENV_NAME"])`` with
default ``EnvParams``).

PARITY UNPINNED: gymnax is not installable here, and every point below rests on recollection of gymnax's code.
``tests/golden/make_gaussian_bandit_golden_from_ref.py`` records real gymnax trajectories and ``EnvParams`` defaults
that check them.  The least certain are the defaults (G1) and the key use (G3, G4).

(G1) EnvParams defaults: mu1 0.0, sigma_p 1.0, sigma_l 1.0, normalize_time True, max_steps_in_episode 100;
     2 actions.
(G2) arm 0 is the deterministic one, paying mu1; arm 1 is the stochastic one, around a mean mu2 drawn per episode.
(G3) reset_env: mu2 = sigma_p * normal(key, ()), drawn from the reset key itself (no split);
     exp_reward_best = max(mu1, mu2); last_action 0, last_reward 0.0, time 0.
(G4) step_env: reward = mu1 where action == 0, else mu2 + sigma_l * normal(key, ()), drawn from the step key itself
     (no split); last_action = action, last_reward = reward, time += 1.
(G5) done = time >= max_steps_in_episode, so every episode lasts 100 steps.
(G6) the observation is [one_hot(last_action, 2), last_reward, time_normalization(time)]: 4 floats, with
     time_normalization as BernoulliBandit's ((T1) of ``tests/misc_envs_oracle.py``).
(G7) the EnvState fields are last_action, last_reward, exp_reward_best, mu2 and time.

fp32: mu2 + sigma_l * n is one fma on a CUDA device ((J4) of ``tests/jax_normal_oracle.py``); at sigma_l = 1 the
product is exact, so the fma and the rounded add agree.  ``log1p`` selects the normal's log1p ((J3)).
"""
from __future__ import annotations

import numpy as np

import jax_normal_oracle as JN
import misc_envs_oracle as M
from oracle import gymnax_envs as G

F32 = np.float32
I32 = np.int32


class GaussianBandit:
    name = "GaussianBandit-misc"
    obs_shape = (4,)
    num_actions = 2
    mu1, sigma_p, sigma_l = F32(0.0), F32(1.0), F32(1.0)                                  # (G1)
    state_fields = ("last_action", "last_reward", "exp_reward_best", "mu2", "time")       # (G7)

    def __init__(self, max_steps_in_episode: int = 100, log1p=JN.log1p_f64):
        self.max_steps_in_episode = int(max_steps_in_episode)
        self.log1p = log1p

    def normal(self, key):
        return JN.normal(key, (), log1p=self.log1p)

    def get_obs(self, s):                                                                   # (G6)
        return np.concatenate([M.one_hot(s["last_action"], 2), s["last_reward"].astype(F32)[:, None],
                               M.time_normalization(s["time"])[:, None]], 1).astype(F32)

    def reset_env(self, key):
        n = key.shape[0]
        mu2 = (self.sigma_p * self.normal(key)).astype(F32)                                 # (G3)
        s = dict(last_action=np.zeros(n, I32), last_reward=np.zeros(n, F32), mu2=mu2,
                 exp_reward_best=np.maximum(self.mu1, mu2).astype(F32), time=np.zeros(n, I32),
                 mu1=np.full(n, self.mu1, F32), sigma_l=np.full(n, self.sigma_l, F32))
        return self.get_obs(s), s

    def step_env(self, key, s, action):
        pull = JN.fma32(s["sigma_l"], self.normal(key), s["mu2"])                           # (G4)
        reward = np.where(action == 0, s["mu1"], pull).astype(F32)                           # (G2)
        ns = dict(s, last_action=action.astype(I32), last_reward=reward, time=(s["time"] + 1).astype(I32))
        ns = {k: v.copy() for k, v in ns.items()}
        done = ns["time"] >= self.max_steps_in_episode                                     # (G5)
        return self.get_obs(ns), ns, reward, done, M._discount(done)


def make(flatten: bool = True, log: bool = True, max_steps_in_episode: int | None = None, log1p=JN.log1p_f64):
    """``LogWrapper([FlattenObservationWrapper(]gymnax.make("GaussianBandit-misc")[)])``; ``log1p`` is the normal's
    log1p ((J3) of ``tests/jax_normal_oracle.py``)."""
    core = GaussianBandit(100 if max_steps_in_episode is None else max_steps_in_episode, log1p)
    env = G.Environment(core, flatten=flatten)
    return G.LogWrapper(env) if log else env
