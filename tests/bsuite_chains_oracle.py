"""NumPy restatements of gymnax==0.0.6 ``environments/bsuite/deep_sea.py`` (``DeepSea``), ``umbrella_chain.py``
(``UmbrellaChain``) and ``discounting_chain.py`` (``DiscountingChain``), test infrastructure for the DeepSea-bsuite,
UmbrellaChain-bsuite and DiscountingChain-bsuite env operators (``purejaxql_b200/csrc/env_bsuite.cuh``).

They plug into the batched gymnax protocol of ``oracle/gymnax_envs.py`` (``Environment`` auto-reset, ``LogWrapper``),
which they reuse unchanged, as ``tests/gymnax_extra_oracle.py`` does.  ``oracle.gymnax_envs.make`` does not know these
envs; use :func:`make` below, or register a class in ``oracle.gymnax_envs._REGISTRY`` for the duration of a test.
Reference call sites: ``purejaxql/pqn_gymnax.py:92`` and ``purejaxql/pqn_rnn_gymnax.py:133-139``
(``gymnax.make(config["ENV_NAME"])`` with default ``EnvParams``).

PARITY UNPINNED: gymnax is not installable here, and every point below rests on recollection of gymnax's code.
``tests/golden/make_bsuite_chains_golden_from_ref.py`` records real gymnax trajectories and ``EnvParams`` defaults
that check them.

DeepSea-bsuite (``gymnax.make`` builds size 8):

(S1) EnvParams defaults: deterministic True, sample_action_map False, unscaled_move_cost 0.01, randomize_actions True,
     max_steps_in_episode 2000; 2 actions.
(S2) reset_env: row = column = 0, bad_episode False, total_bad_episodes 0, denoised_return 0, optimal_no_cost 1.0,
     optimal_return = optimal_no_cost - unscaled_move_cost (fp32), time 0; action_mapping = ones((8, 8)) under
     deterministic = True.  (Under the other params it is a bernoulli draw from the reset key; the state keeps the
     whole 8 x 8 map, so either reading fits the layout.)
(S3) step_env: right = action == action_mapping[row, column]; reward = 0.0 + (right & row == 7 & column == 7)
     - right * unscaled_move_cost / 8, in fp32 (0.01 / 8 is exact from fp32 0.01: a power-of-two divisor).
(S4) a left move at row == column sets bad_episode; column = clip(column + 1 if right else column - 1, 0, 7);
     row += 1; total_bad_episodes += bad_episode once row == 8; denoised_return += the treasure; time += 1.
(S5) done = row == 8 or time >= max_steps_in_episode, so an episode lasts 8 steps.
(S6) the observation is the (8, 8) float one-hot of (row, column), all zeros once row == 8.
(S7) step_env's transition uniform is or-ed with deterministic = True, and its normal reward noise is multiplied by
     1 - deterministic = 0.  The noise term is then +-0.0 (the normal is finite), which leaves a reward of
     +0.0 + bool unchanged bit for bit.  Neither draw can reach an output; neither this oracle nor the CUDA env makes
     them.

UmbrellaChain-bsuite (``gymnax.make`` builds n_distractor = 0):

(U1) EnvParams defaults: chain_length 10, max_steps_in_episode 100; 2 actions.
(U2) reset_env: k_need, k_has, k_obs = split(key, 3); need_umbrella = bernoulli(k_need, 0.5, ()),
     has_umbrella = bernoulli(k_has, 0.5, ()), total_regret 0, time 0.
(U3) step_env: k_reward, k_obs = split(key); has_umbrella = action if time == 0; chain_full = time + 1 == chain_length;
     reward = +1 if has_umbrella == need_umbrella else -1 when chain_full, else 2 * bernoulli(k_reward, 0.5, ()) - 1;
     total_regret += 2 when chain_full and they differ; time += 1.
(U4) done = time == chain_length or time >= max_steps_in_episode, so an episode lasts 10 steps.
(U5) the observation is [need_umbrella, has_umbrella, 1 - time / chain_length] (fp32 division) of the new state.

DiscountingChain-bsuite (``gymnax.make`` builds mapping_seed = None):

(D1) EnvParams defaults: reward_timestep [1, 3, 10, 30, 100], max_steps_in_episode 100; 5 actions.
(D2) reset_env: context -1, time 0, rewards = ones(5).at[randint(key, (), 0, 5)].set(1.1) drawn from the reset key.
     (A mapping fixed by mapping_seed at construction fits the same state word, the index of the 1.1.)
(D3) step_env: context = action if time == 0; time += 1; reward = rewards[context] if
     time == reward_timestep[context] else 0.0, so action a is rewarded at step reward_timestep[a] of its episode.
(D4) done = time >= max_steps_in_episode, so every episode lasts 100 steps.
(D5) the observation is [context, time / max_steps_in_episode] (fp32 division) of the new state.
"""
from __future__ import annotations

import numpy as np

from oracle import gymnax_envs as G
from oracle import jax_prng as jr

F32 = np.float32
I32 = np.int32


def _discount(done):
    return {"discount": np.where(done, F32(0.0), F32(1.0)).astype(F32)}


class DeepSea:
    name = "DeepSea-bsuite"
    size = 8
    obs_shape = (8, 8)
    num_actions = 2
    unscaled_move_cost = F32(0.01)
    state_fields = ("row", "column", "bad_episode", "total_bad_episodes", "denoised_return", "optimal_return",
                    "optimal_no_cost", "action_mapping", "time")

    def __init__(self, max_steps_in_episode: int = 2000):
        self.max_steps_in_episode = int(max_steps_in_episode)                                # (S1)

    def get_obs(self, s):
        n = s["row"].shape[0]
        board = np.zeros((n, self.size, self.size), F32)
        on = s["row"] < self.size                                                           # (S6)
        board[np.arange(n)[on], s["row"][on], s["column"][on]] = 1.0
        return board

    def reset_env(self, key):
        n = key.shape[0]
        z = lambda: np.zeros(n, I32)
        no_cost = np.ones(n, F32)
        s = dict(row=z(), column=z(), bad_episode=np.zeros(n, bool), total_bad_episodes=z(), denoised_return=z(),
                 optimal_return=(no_cost - self.unscaled_move_cost).astype(F32), optimal_no_cost=no_cost,
                 action_mapping=np.ones((n, self.size, self.size), F32), time=z())            # (S2)
        return self.get_obs(s), s

    def step_env(self, key, s, action):
        n = action.shape[0]
        idx = np.arange(n)
        right = action.astype(I32) == s["action_mapping"][idx, s["row"], s["column"]]       # (S3)
        treasure = right & (s["row"] == self.size - 1) & (s["column"] == self.size - 1)
        cost = (self.unscaled_move_cost / F32(self.size)).astype(F32)
        reward = ((F32(0.0) + treasure.astype(F32)).astype(F32) - (right.astype(F32) * cost).astype(F32)).astype(F32)
        bad = s["bad_episode"] | (~right & (s["row"] == s["column"]))                       # (S4)
        column = np.clip(np.where(right, s["column"] + 1, s["column"] - 1), 0, self.size - 1).astype(I32)
        row = (s["row"] + 1).astype(I32)
        ns = dict(row=row, column=column, bad_episode=bad,
                  total_bad_episodes=(s["total_bad_episodes"] + ((row == self.size) & bad)).astype(I32),
                  denoised_return=(s["denoised_return"] + treasure).astype(I32),
                  optimal_return=s["optimal_return"].copy(), optimal_no_cost=s["optimal_no_cost"].copy(),
                  action_mapping=s["action_mapping"].copy(), time=(s["time"] + 1).astype(I32))
        done = (row == self.size) | (ns["time"] >= self.max_steps_in_episode)               # (S5)
        return self.get_obs(ns), ns, reward, done, _discount(done)


class UmbrellaChain:
    name = "UmbrellaChain-bsuite"
    chain_length = 10
    obs_shape = (1, 3)
    num_actions = 2
    state_fields = ("need_umbrella", "has_umbrella", "total_regret", "time")

    def __init__(self, max_steps_in_episode: int = 100):
        self.max_steps_in_episode = int(max_steps_in_episode)                                # (U1)

    def get_obs(self, s):
        frac = (s["time"].astype(F32) / F32(self.chain_length)).astype(F32)                 # (U5)
        return np.stack([s["need_umbrella"].astype(F32), s["has_umbrella"].astype(F32),
                         (F32(1.0) - frac).astype(F32)], -1)[:, None, :]

    def reset_env(self, key):
        n = key.shape[0]
        ks = jr.split(key, 3)                                                               # (U2)
        s = dict(need_umbrella=jr.bernoulli(ks[:, 0], 0.5).astype(I32),
                 has_umbrella=jr.bernoulli(ks[:, 1], 0.5).astype(I32),
                 total_regret=np.zeros(n, I32), time=np.zeros(n, I32))
        return self.get_obs(s), s

    def step_env(self, key, s, action):
        k_reward = jr.split(key, 2)[:, 0]                                                   # (U3)
        has = np.where(s["time"] == 0, action.astype(I32), s["has_umbrella"]).astype(I32)
        full = s["time"] + 1 == self.chain_length
        match = has == s["need_umbrella"]
        coin = jr.bernoulli(k_reward, 0.5).astype(I32)
        reward = np.where(full, np.where(match, 1, -1), 2 * coin - 1).astype(F32)
        ns = dict(need_umbrella=s["need_umbrella"].copy(), has_umbrella=has,
                  total_regret=(s["total_regret"] + 2 * (full & ~match)).astype(I32), time=(s["time"] + 1).astype(I32))
        done = (ns["time"] == self.chain_length) | (ns["time"] >= self.max_steps_in_episode)   # (U4)
        return self.get_obs(ns), ns, reward, done, _discount(done)


class DiscountingChain:
    name = "DiscountingChain-bsuite"
    obs_shape = (1, 2)
    num_actions = 5
    reward_timestep = np.array([1, 3, 10, 30, 100], I32)                                     # (D1)
    mapped_reward = F32(1.1)
    state_fields = ("context", "mapped_action", "time")

    def __init__(self, max_steps_in_episode: int = 100):
        self.max_steps_in_episode = int(max_steps_in_episode)

    def get_obs(self, s):
        frac = (s["time"].astype(F32) / F32(self.max_steps_in_episode)).astype(F32)         # (D5)
        return np.stack([s["context"].astype(F32), frac], -1)[:, None, :]

    def reset_env(self, key):
        n = key.shape[0]
        s = dict(context=np.full(n, -1, I32), mapped_action=jr.randint(key, (), 0, self.num_actions).astype(I32),
                 time=np.zeros(n, I32), max_steps_in_episode=np.full(n, self.max_steps_in_episode, I32))   # (D2)
        return self.get_obs(s), s

    def rewards(self, s):
        """gymnax's ``EnvState.rewards``: ones with 1.1 at the mapped action, [N, 5] fp32."""
        r = np.ones((s["mapped_action"].shape[0], self.num_actions), F32)
        r[np.arange(r.shape[0]), s["mapped_action"]] = self.mapped_reward
        return r

    def step_env(self, key, s, action):
        context = np.where(s["time"] == 0, action.astype(I32), s["context"]).astype(I32)   # (D3)
        time = (s["time"] + 1).astype(I32)
        hit = time == self.reward_timestep[np.clip(context, 0, self.num_actions - 1)]
        reward = np.where(hit, self.rewards(s)[np.arange(context.shape[0]), np.clip(context, 0, 4)], F32(0.0))
        ns = dict(context=context, mapped_action=s["mapped_action"].copy(), time=time,
                  max_steps_in_episode=s["max_steps_in_episode"].copy())
        done = time >= self.max_steps_in_episode                                            # (D4)
        return self.get_obs(ns), ns, reward.astype(F32), done, _discount(done)


CORES = {"DeepSea-bsuite": DeepSea, "UmbrellaChain-bsuite": UmbrellaChain, "DiscountingChain-bsuite": DiscountingChain}


def make(env_name: str, flatten: bool = True, log: bool = True, max_steps_in_episode: int | None = None):
    """``LogWrapper([FlattenObservationWrapper(]gymnax.make(env_name)[)])``; ``max_steps_in_episode`` overrides the
    default ``EnvParams`` field."""
    cls = CORES[env_name]
    core = cls() if max_steps_in_episode is None else cls(max_steps_in_episode)
    env = G.Environment(core, flatten=flatten)
    return G.LogWrapper(env) if log else env
