"""NumPy restatement of gymnax==0.0.6 ``environments/bsuite/memory_chain.py`` (``MemoryChain``), test infrastructure
for the MemoryChain-bsuite env operator (``purejaxql_b200/csrc/env_bsuite.cuh``).

It plugs into the batched gymnax protocol of ``oracle/gymnax_envs.py`` (``Environment`` auto-reset,
``LogWrapper``), which it reuses unchanged.  Reference call site: ``purejaxql/pqn_rnn_gymnax.py:134-139``
(``gymnax.make("MemoryChain-bsuite")``, ``EnvParams(memory_length=...)``).

PARITY UNPINNED: gymnax is not installable here.  ``num_bits = 1`` (what ``gymnax.make`` builds), the
``EnvParams`` defaults ``memory_length = 5``, ``max_steps_in_episode = 1000``, the state fields ``context``,
``query``, ``total_perfect``, ``total_regret``, ``time`` and the reset draws ``bernoulli(k_ctx, 0.5, (num_bits,))``,
``randint(k_q, (), 0, num_bits)`` follow bsuite's published task.  These points rest on recollection of gymnax's
code rather than on bsuite's definition; ``tests/golden/make_memory_chain_golden_from_ref.py`` records real gymnax
trajectories that check each of them:

(R1) get_obs[0, 1] = query if time == memory_length - 1, else 0.
(R2) get_obs[0, 2:] = 2 * context - 1 (the +-1 encoding) if time == 0, else 0.
(R3) step_env returns get_obs(state) of the state BEFORE time is incremented.
(R4) done = (time - 1 == memory_length) after the increment, so an episode lasts memory_length + 1 steps.
"""
from __future__ import annotations

import numpy as np

from oracle import gymnax_envs as G
from oracle import jax_prng as jr

F32 = np.float32
I32 = np.int32


class MemoryChain:
    name = "MemoryChain-bsuite"
    num_bits = 1
    obs_shape = (1, num_bits + 2)
    num_actions = 2
    max_steps_in_episode = 1000
    state_fields = ("context", "query", "total_perfect", "total_regret", "time")

    def __init__(self, memory_length: int = 5):
        self.memory_length = int(memory_length)

    def get_obs(self, s):
        n = s["time"].shape[0]
        ml = self.memory_length
        obs = np.zeros((n, 1, self.num_bits + 2), F32)
        obs[:, 0, 0] = F32(1) - s["time"].astype(F32) / F32(ml)                        # fp32 true division
        obs[:, 0, 1] = np.where(s["time"] == ml - 1, s["query"], 0).astype(F32)          # (R1)
        ctx = (2 * s["context"].astype(I32) - 1).astype(F32)
        obs[:, 0, 2:] = np.where((s["time"] == 0)[:, None], ctx, F32(0))                  # (R2)
        return obs

    def reset_env(self, key):
        n = key.shape[0]
        ks = jr.split(key, 2)
        context = jr.bernoulli(ks[:, 0], 0.5, (self.num_bits,))                          # [N, num_bits] bool
        query = jr.randint(ks[:, 1], (), 0, self.num_bits).astype(I32)
        s = dict(context=context, query=query, total_perfect=np.zeros(n, I32), total_regret=np.zeros(n, I32),
                 time=np.zeros(n, I32))
        return self.get_obs(s), s

    def step_env(self, key, s, action):
        obs = self.get_obs(s)                                                             # (R3)
        time = (s["time"] + 1).astype(I32)
        full = ~(time - 1 < self.memory_length)
        correct = action == s["context"][np.arange(action.shape[0]), s["query"]]
        win, lose = full & correct, full & ~correct
        reward = (win.astype(F32) - lose.astype(F32)).astype(F32)
        ns = dict(context=s["context"].copy(), query=s["query"].copy(),
                  total_perfect=(s["total_perfect"] + win).astype(I32),
                  total_regret=(s["total_regret"] + 2 * lose).astype(I32), time=time)
        done = time - 1 == self.memory_length                                            # (R4)
        info = {"discount": (F32(1) - done.astype(F32)).astype(F32)}
        return obs, ns, reward, done, info


def make(memory_length: int = 5, flatten: bool = False, log: bool = True):
    """``LogWrapper([FlattenObservationWrapper(]gymnax.make("MemoryChain-bsuite")[)])`` with
    ``EnvParams(memory_length=memory_length)``."""
    env = G.Environment(MemoryChain(memory_length), flatten=flatten)
    return G.LogWrapper(env) if log else env
