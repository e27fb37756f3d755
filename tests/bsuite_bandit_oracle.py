"""NumPy restatement of gymnax==0.0.6 ``environments/bsuite/bandit.py`` (``SimpleBandit``), test infrastructure for the
SimpleBandit-bsuite env operator (``purejaxql_b200/csrc/env_bsuite.cuh``).  It plugs into the batched gymnax protocol
of ``oracle/gymnax_envs.py`` (``Environment`` auto-reset, ``LogWrapper``) as ``tests/bsuite_chains_oracle.py`` does.
Reference call sites: ``purejaxql/pqn_gymnax.py:92`` and ``purejaxql/pqn_rnn_gymnax.py:133-139``.

PARITY UNPINNED: gymnax is not installable here, and every point below rests on recollection of gymnax's and jax's
code.  ``tests/golden/make_misc_golden_from_ref.py`` records real gymnax trajectories and ``EnvParams`` defaults that
check them.

SimpleBandit-bsuite (``gymnax.make`` builds num_actions = 11):

(B1) EnvParams defaults: optimal_return 1, max_steps_in_episode 100 (the least certain default: every step is
     terminal, so it only sets TEST_NUM_STEPS); 11 actions.
(B2) reset_env: action_mask = choice(key, arange(11), (11,), replace=False).  Without p, jax's choice without
     replacement is permutation(key, arange(11)), i.e. ``_shuffle``: ceil(3 ln 11 / ln(2**32 - 1)) = 1 round of a
     stable sort of arange(11) by random_bits(sub, 32, (11,)), (key, sub) = split(key)
     (``oracle.jax_prng.permutation_indices``).  rewards = linspace(0, 1, 11)[action_mask], total_regret 0.0, time 0.
(B3) jnp.linspace(0, 1, 11) in jax 0.4.x is start * (1 - step) + stop * step with step = iota(10) / 10 in fp32, then
     the endpoint stop; at start 0 and stop 1 that is the fp32 quotient k / 10 for every k (10 / 10 = 1 included).
     The other reading, start + k * delta with delta = fp32(0.1), differs from it by an ulp at some k
     (``linspace_levels(form="delta")``); the recorded ``rewards`` field tells them apart.
(B4) step_env: reward = rewards[action]; total_regret = total_regret + optimal_return - reward (fp32, left to right);
     time += 1.
(B5) is_terminal returns True ("every step transition is terminal"), so every step auto-resets and redraws the
     mapping from the reset key; the state after a step is always the fresh reset state.
(B6) the observation is ones((1, 1)) fp32, D = 1 once flattened.
"""
from __future__ import annotations

import numpy as np

from oracle import gymnax_envs as G
from oracle import jax_prng as jr

F32 = np.float32
I32 = np.int32


def _discount(done):
    return {"discount": np.where(done, F32(0.0), F32(1.0)).astype(F32)}


def linspace_levels(n=11, form="interp"):
    """fp32 ``jnp.linspace(0, 1, n)`` in either reading of (B3)."""
    k = np.arange(n - 1, dtype=F32)
    div = F32(n - 1)
    if form == "interp":
        step = (k / div).astype(F32)
        out = (F32(0) * (F32(1) - step) + F32(1) * step).astype(F32)
    else:
        out = (F32(0) + k * (F32(1) / div)).astype(F32)
    return np.concatenate([out, np.ones(1, F32)])


class SimpleBandit:
    name = "SimpleBandit-bsuite"
    obs_shape = (1, 1)
    num_actions = 11
    optimal_return = F32(1.0)
    state_fields = ("action_mask", "total_regret", "time")

    def __init__(self, max_steps_in_episode: int = 100):
        self.max_steps_in_episode = int(max_steps_in_episode)                                # (B1)

    def get_obs(self, s):
        return np.ones((s["time"].shape[0], 1, 1), F32)                                     # (B6)

    @staticmethod
    def permutation(key, n):
        """``jr.permutation_indices`` batched over keys [N, 2] for a one-round shuffle (n = 11)."""
        assert int(np.ceil(3 * np.log(n) / np.log(np.iinfo(np.uint32).max))) == 1
        sub = jr.split(key, 2)[:, 1]
        return np.argsort(jr.random_bits(sub, (n,)), axis=1, kind="stable")

    def reset_env(self, key):
        key = np.asarray(key, np.uint32)
        n = key.shape[0]
        mask = self.permutation(key, self.num_actions).astype(I32)                         # (B2)
        s = dict(action_mask=mask, total_regret=np.zeros(n, F32), time=np.zeros(n, I32),
                 optimal_return=np.full(n, self.optimal_return, F32))
        return self.get_obs(s), s

    def rewards(self, s):
        """gymnax's ``EnvState.rewards``: linspace(0, 1, 11)[action_mask], [N, 11] fp32."""
        return linspace_levels(self.num_actions)[s["action_mask"]]                          # (B3)

    def step_env(self, key, s, action):
        n = action.shape[0]
        reward = self.rewards(s)[np.arange(n), action.astype(np.int64)].astype(F32)         # (B4)
        ns = dict(action_mask=s["action_mask"].copy(),
                  total_regret=((s["total_regret"] + s["optimal_return"]).astype(F32) - reward).astype(F32),
                  time=(s["time"] + 1).astype(I32), optimal_return=s["optimal_return"].copy())
        done = np.ones(n, bool)                                                             # (B5)
        return self.get_obs(ns), ns, reward, done, _discount(done)


CORES = {"SimpleBandit-bsuite": SimpleBandit}


def make(env_name: str = "SimpleBandit-bsuite", flatten: bool = True, log: bool = True,
         max_steps_in_episode: int | None = None):
    """``LogWrapper([FlattenObservationWrapper(]gymnax.make(env_name)[)])``."""
    cls = CORES[env_name]
    core = cls() if max_steps_in_episode is None else cls(max_steps_in_episode)
    env = G.Environment(core, flatten=flatten)
    return G.LogWrapper(env) if log else env
