"""Env-sharded rollouts (engine.PQNEngine with ``env_shard``; chosen by DATA_PARALLEL=auto when NUM_SEEDS < world):
each rank runs ``pqn_rollout_act_step`` over its slice [env_offset, env_offset + E) of every seed's envs and must draw
exactly the per-env keys of the unsharded vmap, element env_offset + e of split(key, env_total).  In jax's original
threefry layout that element depends on env_total, so the shard arguments matter for every env.

Checked on one GPU by running the shards one after another: every output of every shard bit for bit against the
matching slice of the unsharded launch, for every env, both threefry layouts, 2 and 3 shards of an env count that
crosses block boundaries, eps in {0, 0.37, 1} and both info modes; the sharded reset keys of the engine; one case per
layout against the oracle's split(key, env_total)[offset + e]; and the refusal of shards outside [0, env_total)."""
import numpy as np
import pytest
import torch

import bsuite_oracle as MC
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from purejaxql_b200.envs import ENV_IDS

pytestmark = pytest.mark.gpu

S, E_TOTAL = 3, 390                  # 390 = 2 x 195 = 3 x 130: no shard boundary falls on a 128-env block boundary
EPS = (0.0, 0.37, 1.0)
PQN_E_INVALID = -1


def dev():
    return torch.device("cuda:0")


def keys_t(k):
    return torch.from_numpy(np.ascontiguousarray(k, np.uint32).view(np.int32)).to(dev())


class Buffers:
    """Outputs of one pqn_rollout_act_step over S seeds x E envs (seed stride E)."""

    def __init__(self, env, E):
        self.E = E
        if env.binary_obs:
            self.obs = torch.zeros((S, E, env.packed_obs_words), dtype=torch.int32, device=dev())
        else:
            self.obs = torch.zeros((S, E, env.obs_dim), dtype=torch.float32, device=dev())
        self.action = torch.zeros((S, E), dtype=torch.int32, device=dev())
        self.reward = torch.zeros((S, E), device=dev())
        self.done = torch.zeros((S, E), dtype=torch.uint8, device=dev())
        self.maxq = torch.zeros((S, E), device=dev())
        self.sums = torch.zeros((S, 5), dtype=torch.float64, device=dev())


def act_step(env, step_keys, q, eps, state, b, done_only, env_total, env_offset, part, rew_scale=0.5):
    from purejaxql_b200 import _lib
    return _lib.lib().pqn_rollout_act_step(
        env.env_id, _lib.p(step_keys), _lib.p(q), _lib.p(eps), _lib.p(state), _lib.p(b.obs), b.E, _lib.p(b.action),
        _lib.p(b.reward), _lib.p(b.done), _lib.p(b.maxq), b.E, _lib.p(b.sums), done_only, S, b.E, env_total,
        env_offset, 0, rew_scale, part, _lib.stream_ptr())


def shard_of(state, lo, hi):
    """Columns of envs [lo, hi) of every seed of a word-major [words, S * E_TOTAL] state block."""
    return state.view(state.shape[0], S, E_TOTAL)[:, :, lo:hi].reshape(state.shape[0], -1).contiguous()


def step_inputs(t, A, gen):
    step_keys = keys_t(jr.split(jr.PRNGKey(1000 + t), 2 * S).reshape(S, 2, 2))
    q = torch.randn((S, E_TOTAL, A), generator=gen).to(dev())
    eps = torch.full((1,), EPS[t % 3], device=dev())
    return step_keys, q, eps, (t // 3) % 2


def sharded_reset(env, kR, lo, E, params, part):
    """engine.PQNEngine.train's reset of env shard [lo, lo + E): split(kR, E_total)[:, lo:lo + E]."""
    from purejaxql_b200 import envs, jaxrandom
    keys = jaxrandom.split(kR, E_TOTAL, part)[:, lo:lo + E].reshape(S * E, 2).contiguous()
    state = torch.empty((env.state_words, S * E), dtype=torch.int32, device=dev())
    obs = torch.empty((S * E, env.obs_dim), dtype=torch.float32, device=dev())
    envs.reset_into(env.env_id, keys, state, obs, S * E, params, part)
    return state, obs.view(S, E, -1)


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("name", sorted(ENV_IDS))
def test_sharded_act_step_equals_unsharded(name, part):
    from purejaxql_b200 import _lib, envs
    env, params = envs.make(name, flatten_obs=True, rng_mode=part)
    params = envs.EnvParams(params.max_steps_in_episode, memory_length=4)   # MemoryChain: episodes of 5 steps
    A, T = env.num_actions, 24
    kR = keys_t(jr.split(jr.PRNGKey(50 + part), S))
    dones = 0
    for W in (2, 3):
        E = E_TOTAL // W
        full_state, _ = sharded_reset(env, kR, 0, E_TOTAL, params, part)
        states = [shard_of(full_state, r * E, (r + 1) * E) for r in range(W)]
        full = Buffers(env, E_TOTAL)
        shards = [Buffers(env, E) for _ in range(W)]
        gen = torch.Generator().manual_seed(W)
        for t in range(T):
            step_keys, q, eps, done_only = step_inputs(t, A, gen)
            full.sums.zero_()
            _lib.check(act_step(env, step_keys, q, eps, full_state, full, done_only, E_TOTAL, 0, part), "full")
            for r, b in enumerate(shards):
                lo = r * E
                b.sums.zero_()
                _lib.check(act_step(env, step_keys, q[:, lo:lo + E].contiguous(), eps, states[r], b, done_only,
                                    E_TOTAL, lo, part), f"shard {r}")
            torch.cuda.synchronize()
            where = (name, part, W, t)
            for r, b in enumerate(shards):
                lo, hi = r * E, (r + 1) * E
                for field in ("action", "reward", "done", "maxq", "obs"):
                    assert torch.equal(getattr(b, field), getattr(full, field)[:, lo:hi]), where + (r, field)
                assert torch.equal(states[r], shard_of(full_state, lo, hi)), where + (r, "state")
            got = sum(b.sums for b in shards).cpu().numpy()
            want = full.sums.cpu().numpy()
            assert np.allclose(got, want, rtol=1e-12, atol=1e-9), where + (got, want)
            dones += int(full.done.sum())
    if name in ("CartPole-v1", "MemoryChain-bsuite", "Catch-bsuite", "DeepSea-bsuite"):
        assert dones > 0, "no episode ended: the auto-reset's keys were never compared"


@pytest.mark.parametrize("part", [0, 1])
def test_sharded_reset_equals_unsharded(part):
    """The engine's reset of a shard, split(kR, E_total)[:, lo:lo + E], against the unsharded reset: every state word
    (parameter words such as MemoryChain's memory_length = 100 and DiscountingChain's max_steps included) and every
    observation row."""
    from purejaxql_b200 import envs
    kR = keys_t(jr.split(jr.PRNGKey(60 + part), S))
    for name in envs.ENV_IDS:
        env, params = envs.make(name, flatten_obs=True, rng_mode=part)
        params = envs.EnvParams(params.max_steps_in_episode, memory_length=100)
        full_state, full_obs = sharded_reset(env, kR, 0, E_TOTAL, params, part)
        if name == "MemoryChain-bsuite":
            assert (envs.state_to_fields(name, full_state.cpu())["memory_length"] == 100).all()
        for W in (2, 3):
            E = E_TOTAL // W
            for r in range(W):
                lo = r * E
                st, obs = sharded_reset(env, kR, lo, E, params, part)
                assert torch.equal(st, shard_of(full_state, lo, lo + E)), (name, part, W, r)
                assert torch.equal(obs, full_obs[:, lo:lo + E]), (name, part, W, r)


@pytest.mark.parametrize("part", [0, 1])
def test_sharded_act_step_matches_oracle(part):
    """MemoryChain (memory_length 4: auto-resets every 5 steps) in 3 shards against the oracle fed
    split(key, E_total)[offset + e]: the kernel compared with itself cannot catch a key bug both launches share."""
    from purejaxql_b200 import _lib, envs
    name, ml, W, T = "MemoryChain-bsuite", 4, 3, 12
    E = E_TOTAL // W
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env, _ = envs.make(name, flatten_obs=True, rng_mode=part)
        oenv = MC.make(ml, flatten=True)
        kR = jr.split(jr.PRNGKey(70 + part), S)
        rk = jr.split(kR, E_TOTAL)                                                   # [S, E_total, 2]
        states, o_st, shards = [], [], []
        for r in range(W):
            lo = r * E
            st, obs = sharded_reset(env, keys_t(kR), lo, E, envs.EnvParams(1000, memory_length=ml), part)
            states.append(st)
            o = [oenv.reset(rk[s, lo:lo + E]) for s in range(S)]
            assert np.array_equal(obs.cpu().numpy(), np.stack([x[0] for x in o])), (part, r)
            o_st.append([x[1] for x in o])
            shards.append(Buffers(env, E))
        gen = torch.Generator().manual_seed(7)
        n_done = 0
        for t in range(T):
            step_keys, q, eps, done_only = step_inputs(t, env.num_actions, gen)
            sk = jr.split(jr.PRNGKey(1000 + t), 2 * S).reshape(S, 2, 2)
            qn = q.cpu().numpy()
            for r, b in enumerate(shards):
                lo = r * E
                _lib.check(act_step(env, step_keys, q[:, lo:lo + E].contiguous(), eps, states[r], b, done_only,
                                    E_TOTAL, lo, part), f"shard {r}")
                torch.cuda.synchronize()
                fields = envs.state_to_fields(name, states[r].cpu())
                for s in range(S):
                    qs = qn[s, lo:lo + E]
                    a = R.eps_greedy(jr.split(sk[s, 0], E_TOTAL)[lo:lo + E], qs, EPS[t % 3])
                    o_obs, o_st[r][s], rew, d, _ = oenv.step(jr.split(sk[s, 1], E_TOTAL)[lo:lo + E], o_st[r][s], a)
                    where = (part, t, r, s)
                    assert np.array_equal(b.action[s].cpu().numpy(), a), where
                    assert np.array_equal(b.reward[s].cpu().numpy(), (np.float32(0.5) * rew).astype(np.float32)), where
                    assert np.array_equal(b.done[s].cpu().numpy().astype(bool), d), where
                    assert np.array_equal(b.maxq[s].cpu().numpy(), qs.max(-1)), where
                    assert np.array_equal(b.obs[s].cpu().numpy(), o_obs), where
                    for k, v in o_st[r][s].items():
                        got = fields[k].numpy()[s * E:(s + 1) * E].astype(v.dtype).reshape(v.shape)
                        assert np.array_equal(got, v), where + (k,)
                    n_done += int(d.sum())
        assert n_done > 0
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def test_refuses_shards_outside_the_env_range():
    from purejaxql_b200 import _lib, envs
    L = _lib.lib()
    env, params = envs.make("CartPole-v1", flatten_obs=True)
    E = 130
    state, _ = sharded_reset(env, keys_t(jr.split(jr.PRNGKey(1), S)), 0, E, params, 0)
    b = Buffers(env, E)
    step_keys, q, eps, _ = step_inputs(0, env.num_actions, torch.Generator().manual_seed(0))
    q = q[:, :E].contiguous()
    for offset in (-1, E_TOTAL - E + 1, E_TOTAL):
        before = state.clone()
        rc = act_step(env, step_keys, q, eps, state, b, 0, E_TOTAL, offset, 0)
        assert rc == PQN_E_INVALID and b"env shard" in L.pqn_last_error(), offset
        assert torch.equal(state, before), offset
    _lib.check(act_step(env, step_keys, q, eps, state, b, 0, E_TOTAL, E_TOTAL - E, 0), "last shard")
