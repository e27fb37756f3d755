"""DeepSea-bsuite, UmbrellaChain-bsuite and DiscountingChain-bsuite without a GPU: the device logic of
csrc/env_bsuite.cuh compiled for the host (tests/host_harness_bsuite_chains.cpp) against the NumPy oracles
(tests/bsuite_chains_oracle.py), self-checks of the oracles' episodes, the state-field conversion of
purejaxql_b200/envs.py, ``pqn_env_info`` and make_train of both scripts."""
import ctypes
import glob
import os
import subprocess

import numpy as np
import pytest
import torch

import bsuite_chains_oracle as B
from oracle import jax_prng as jr
from purejaxql_b200 import envs as E

HERE = os.path.dirname(os.path.abspath(__file__))
SEA, UMB, DISC = "DeepSea-bsuite", "UmbrellaChain-bsuite", "DiscountingChain-bsuite"
PREFIX = {SEA: "deep_sea", UMB: "umbrella", DISC: "discounting"}
EPISODE = {SEA: 8, UMB: 10, DISC: 100}
WORDS = {SEA: 13, UMB: 9, DISC: 9}


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def hlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("harness") / "host_harness_bsuite_chains.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(HERE, "host_harness_bsuite_chains.cpp"), "-o", so])
    return ctypes.CDLL(so)


class HostEnv:
    """Drives the harness like pqn_env_reset / pqn_env_step / pqn_env_obs."""

    def __init__(self, lib, name, part, max_steps=None):
        self.lib, self.part = lib, part
        self.p = PREFIX[name]
        self.words = getattr(lib, f"h_{self.p}_state_words")()
        self.D = getattr(lib, f"h_{self.p}_obs_dim")()
        self.max_steps = max_steps or getattr(lib, f"h_{self.p}_max_steps")()

    def reset(self, keys):
        n = keys.shape[0]
        keys = np.ascontiguousarray(keys, np.uint32)
        state = np.zeros((self.words, n), np.uint32)
        obs = np.zeros((n, self.D), np.float32)
        getattr(self.lib, f"h_{self.p}_reset")(ptr(keys), ptr(state), ptr(obs), ctypes.c_int64(n), self.max_steps,
                                               self.part)
        return obs, state

    def step(self, keys, state, action):
        n = keys.shape[0]
        keys = np.ascontiguousarray(keys, np.uint32)
        action = np.ascontiguousarray(action, np.int32)
        obs = np.zeros((n, self.D), np.float32)
        reward = np.zeros(n, np.float32)
        done = np.zeros(n, np.uint8)
        getattr(self.lib, f"h_{self.p}_step")(ptr(keys), ptr(state), ptr(action), ptr(obs), ptr(reward), ptr(done),
                                              ctypes.c_int64(n), self.max_steps, self.part)
        return obs, state, reward, done.astype(bool)

    def obs(self, state):
        n = state.shape[1]
        obs = np.zeros((n, self.D), np.float32)
        getattr(self.lib, f"h_{self.p}_obs")(ptr(np.ascontiguousarray(state)), ptr(obs), ctypes.c_int64(n))
        return obs


def fields(name, state):
    return {k: v.numpy() for k, v in E.state_to_fields(name, torch.from_numpy(state.view(np.int32))).items()}


def to_state(name, st):
    return E.fields_to_state(name, {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in st.items()}).numpy().view(
        np.uint32).copy()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def random_actions(ka, n, A):
    return jr.randint(jr.split(ka, n), (), 0, A)


# --------------------------------------------------------------------------- #
# pqn_env_info and the env registry
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name,env_id,obs_dim,obs_shape,actions,max_steps",
                         [(SEA, 34, 64, (8, 8), 2, 2000), (UMB, 35, 3, (3,), 2, 100), (DISC, 36, 2, (2,), 5, 100)])
def test_env_info(name, env_id, obs_dim, obs_shape, actions, max_steps):
    """pqn_env_info's table; the observation space is gymnax's shape for DeepSea's board, (64,) once flattened."""
    from purejaxql_b200 import _lib
    info = _lib.EnvInfo()
    _lib.check(_lib.lib().pqn_env_info(env_id, info), "pqn_env_info")
    assert (info.obs_dim, info.num_actions, info.max_steps, info.binary_obs) == (obs_dim, actions, max_steps, 0)
    assert (info.state_words, tuple(info.obs_shape), info.packed_obs_words) == (WORDS[name], (obs_shape + (1, 1))[:3], 0)
    assert E.make(name)[0].observation_space().shape == obs_shape
    env, params = E.make(name, flatten_obs=True)
    assert E.ENV_IDS[name] == env_id and env.env_id == env_id
    assert env.observation_space().shape == (obs_dim,) and env.action_space().n == actions
    assert params.max_steps_in_episode == max_steps and not env.binary_obs


def test_harness_matches_info(hlib):
    from purejaxql_b200 import _lib
    for name, p in PREFIX.items():
        info = _lib.EnvInfo()
        _lib.check(_lib.lib().pqn_env_info(E.ENV_IDS[name], info), "pqn_env_info")
        assert getattr(hlib, f"h_{p}_state_words")() == info.state_words
        assert getattr(hlib, f"h_{p}_obs_dim")() == info.obs_dim
        assert getattr(hlib, f"h_{p}_max_steps")() == info.max_steps


# --------------------------------------------------------------------------- #
# host-compiled device logic against the oracles
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("name", [SEA, UMB, DISC])
def test_host_logic_matches_oracle_bit_exact(hlib, name, part):
    """reset + three episodes and a few steps of random actions (auto-resets included) for a ragged N: obs, reward
    (sign of zero included), done, every state field and the LogWrapper fields equal the oracle bit for bit;
    pqn_env_obs's obs equals the one the step returned."""
    n = 97
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env = B.make(name)
        h = HostEnv(hlib, name, part)
        A = env.num_actions
        key, kr = jr.split(jr.PRNGKey(40 + part), 2)
        rk = jr.split(kr, n)
        o_obs, o_st = env.reset(rk)
        h_obs, h_st = h.reset(rk)
        assert np.array_equal(bits(h_obs), bits(o_obs)) and np.array_equal(bits(h.obs(h_st)), bits(o_obs))
        assert np.array_equal(to_state(name, o_st), h_st)
        dones = 0
        rewards = set()
        for t in range(3 * EPISODE[name] + 3):
            key, ka, ks = jr.split(key, 3)
            act = random_actions(ka, n, A)
            sk = jr.split(ks, n)
            o_obs, o_st, o_r, o_d, _ = env.step(sk, o_st, act)
            h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
            assert np.array_equal(h_d, o_d), t
            assert np.array_equal(bits(h_r), bits(o_r)), t
            assert np.array_equal(bits(h_obs), bits(o_obs)), t
            assert np.array_equal(bits(h.obs(h_st)), bits(o_obs)), t
            assert np.array_equal(to_state(name, o_st), h_st), t
            dones += int(o_d.sum())
            rewards |= set(o_r.tolist())
        assert dones == 3 * n
        assert (o_st["log_returned_episode_lengths"] == EPISODE[name]).all()
        want = {SEA: {0.0, np.float32(-0.00125), np.float32(1 - np.float32(0.00125))}, UMB: {-1.0, 1.0},
                DISC: {0.0, 1.0, np.float32(1.1)}}[name]
        assert rewards <= want and len(rewards) >= 2, rewards
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("part", [0, 1])
def test_reset_draws_cover_their_range(hlib, part):
    """UmbrellaChain draws need and has from two keys of the reset's 3-way split, DiscountingChain the mapped action
    from the reset key: over 97 envs every value appears, and need and has are not the same draw."""
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        rk = jr.split(jr.PRNGKey(9), 97)
        f = fields(UMB, HostEnv(hlib, UMB, part).reset(rk)[1])
        assert set(f["need_umbrella"]) == {0, 1} and set(f["has_umbrella"]) == {0, 1}
        assert not np.array_equal(f["need_umbrella"], f["has_umbrella"])
        f = fields(DISC, HostEnv(hlib, DISC, part).reset(rk)[1])
        assert set(f["mapped_action"]) == set(range(5)) and (f["context"] == -1).all()
        assert np.array_equal(f["mapped_action"], jr.randint(rk, (), 0, 5))
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def test_discounting_chain_observation_follows_max_steps(hlib):
    """The observation divides time by the max_steps_in_episode the env was reset with, and episodes end there."""
    rk = jr.split(jr.PRNGKey(2), 5)
    env = B.make(DISC, max_steps_in_episode=40)
    h = HostEnv(hlib, DISC, 0, max_steps=40)
    o_obs, o_st = env.reset(rk)
    h_obs, h_st = h.reset(rk)
    assert np.array_equal(to_state(DISC, o_st), h_st)
    for t in range(41):
        sk = jr.split(jr.PRNGKey(100 + t), 5)
        act = np.arange(5, dtype=np.int32)
        o_obs, o_st, o_r, o_d, _ = env.step(sk, o_st, act)
        h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
        assert np.array_equal(bits(h_obs), bits(o_obs)) and np.array_equal(h_d, o_d), t
        assert np.array_equal(bits(h_r), bits(o_r)), t
        if t == 38:
            assert np.array_equal(h_obs[:, 1], np.full(5, np.float32(39) / np.float32(40)))
        assert h_d.all() == (t == 39)


# --------------------------------------------------------------------------- #
# the oracles' episodes
# --------------------------------------------------------------------------- #
def _run(name, policy, steps, seed=3, n=64):
    """Steps the oracle ``steps`` times with ``policy(state) -> action``; returns the per-step (reward, done, info)."""
    env = B.make(name)
    key, kr = jr.split(jr.PRNGKey(seed), 2)
    _, st = env.reset(jr.split(kr, n))
    out = []
    for _ in range(steps):
        key, ks = jr.split(key, 2)
        act = policy(st).astype(np.int32)
        _, st, r, d, info = env.step(jr.split(ks, n), st, act)
        out.append((r, d, info))
    return out


def test_deep_sea_oracle_episodes():
    """Always right returns 1 - 8 * (0.01 / 8) in fp32 (7 move costs, then the treasure less one) and always left
    returns 0; every episode lasts 8 steps.  A left move on the diagonal marks the episode bad."""
    n = 64
    c = np.float32(np.float32(0.01) / np.float32(8))
    want = np.float32(0)
    for _ in range(7):
        want = np.float32(want - c)
    want = np.float32(want + np.float32(np.float32(1) - c))
    assert abs(float(want) - 0.99) < 1e-6
    for action, ret in ((1, want), (0, np.float32(0))):
        out = _run(SEA, lambda st: np.full(n, action), 24, n=n)
        for t, (r, d, info) in enumerate(out):
            assert np.array_equal(d, np.full(n, t % 8 == 7)), t
            if action == 0:
                assert (r.view(np.int32) == 0).all()                   # +0.0, never -0.0
        assert (info["returned_episode_returns"] == ret).all() and (info["returned_episode_lengths"] == 8).all()
    core = B.DeepSea()
    _, s = core.reset_env(jr.split(jr.PRNGKey(0), 2))
    obs, s, r, d, _ = core.step_env(None, s, np.array([1, 0], np.int32))
    assert list(s["bad_episode"]) == [False, True] and list(s["column"]) == [1, 0] and list(s["row"]) == [1, 1]
    assert obs[0, 1, 1] == 1 and obs[1, 1, 0] == 1 and (obs.reshape(2, 64).sum(1) == 1).all()
    assert np.float32(s["optimal_return"][0]) == np.float32(np.float32(1) - np.float32(0.01))
    s = dict(s, row=np.full(2, 8, np.int32))
    assert core.get_obs(s).sum() == 0


def test_umbrella_chain_oracle_episodes():
    """Every episode lasts 10 steps; the last reward is +1 exactly when the first action equals need_umbrella, and the
    nine before it are random +-1 (both signs seen)."""
    n = 64
    env = B.make(UMB)
    key, kr = jr.split(jr.PRNGKey(5), 2)
    _, st = env.reset(jr.split(kr, n))
    rng = np.random.default_rng(0)
    mid = set()
    first = None
    need = st["need_umbrella"].copy()
    for t in range(30):
        key, ks = jr.split(key, 2)
        act = rng.integers(0, 2, n).astype(np.int32)
        if t % 10 == 0:
            first, need = act.copy(), st["need_umbrella"].copy()
        obs, st, r, d, info = env.step(jr.split(ks, n), st, act)
        assert np.array_equal(d, np.full(n, t % 10 == 9)), t
        if t % 10 == 9:
            assert np.array_equal(r, np.where(first == need, 1.0, -1.0).astype(np.float32)), t
            assert (info["returned_episode_lengths"] == 10).all()
        else:
            mid |= set(r.tolist())
            assert np.array_equal(obs[:, 1], first.astype(np.float32)), t
            assert np.array_equal(obs[:, 2], np.full(n, np.float32(1) - np.float32(t % 10 + 1) / np.float32(10)))
    assert mid == {-1.0, 1.0}


def test_discounting_chain_oracle_episodes():
    """Action a, taken at the first step, is rewarded exactly once, at step reward_timestep[a] of its episode (1.1 for
    the mapped action, else 1); every episode lasts 100 steps and the context shows -1 only at the reset."""
    n = 5 * 16
    act0 = np.arange(n) % 5
    env = B.make(DISC)
    key, kr = jr.split(jr.PRNGKey(6), 2)
    obs, st = env.reset(jr.split(kr, n))
    assert (obs[:, 0] == -1).all() and (obs[:, 1] == 0).all()
    mapped = st["mapped_action"].copy()
    rng = np.random.default_rng(1)
    for t in range(200):
        key, ks = jr.split(key, 2)
        act = act0 if t % 100 == 0 else rng.integers(0, 5, n)
        if t % 100 == 0:
            mapped = st["mapped_action"].copy()
        obs, st, r, d, info = env.step(jr.split(ks, n), st, act.astype(np.int32))
        step = t % 100 + 1
        hit = B.DiscountingChain.reward_timestep[act0] == step
        want = np.where(hit, np.where(act0 == mapped, np.float32(1.1), np.float32(1.0)), np.float32(0))
        assert np.array_equal(r, want.astype(np.float32)), t
        assert np.array_equal(d, np.full(n, step == 100)), t
        if step < 100:
            assert np.array_equal(obs[:, 0], act0.astype(np.float32))
            assert np.array_equal(obs[:, 1], np.full(n, np.float32(step) / np.float32(100)))
    assert (info["returned_episode_lengths"] == 100).all()
    assert np.array_equal(info["returned_episode_returns"], np.where(act0 == mapped, np.float32(1.1), 1).astype(np.float32))


# --------------------------------------------------------------------------- #
# fields and scripts
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name", [SEA, UMB, DISC])
def test_fields_round_trip(name):
    env = B.make(name)
    key = jr.PRNGKey(11)
    _, st = env.reset(jr.split(key, 50))
    for t in range(6):
        key, ka, ks = jr.split(key, 3)
        _, st, _, _, _ = env.step(jr.split(ks, 50), st, random_actions(ka, 50, env.num_actions))
    f = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in st.items()}
    state = E.fields_to_state(name, f)
    assert state.shape == (WORDS[name], 50)
    back = E.state_to_fields(name, state)
    assert set(back) == set(f)
    for k, v in f.items():
        assert np.array_equal(back[k].numpy().astype(v.numpy().dtype).reshape(v.shape), v.numpy()), k
    assert torch.equal(E.fields_to_state(name, back), state)
    if name == SEA:   # a mapping other than all ones (the other params' reset) survives the round trip
        am = (np.random.default_rng(0).random((50, 8, 8)) < 0.5).astype(np.float32)
        f["action_mapping"] = torch.from_numpy(am)
        assert np.array_equal(E.state_to_fields(name, E.fields_to_state(name, f))["action_mapping"].numpy(), am)


@pytest.mark.parametrize("script", ["pqn_gymnax", "pqn_rnn_gymnax"])
@pytest.mark.parametrize("name,test_steps", [(SEA, 2000), (UMB, 100), (DISC, 100)])
def test_make_train_accepts_env(script, name, test_steps):
    """make_train builds each script's engine for the env with its gymnax defaults; TEST_NUM_STEPS is the env's
    max_steps_in_episode."""
    import importlib
    mod = importlib.import_module(f"purejaxql_b200.{script}")
    cls = "PQNRnnEngine" if script == "pqn_rnn_gymnax" else "PQNEngine"
    seen = {}
    orig = getattr(mod, cls)

    def fake(config, *a, **kw):
        seen["config"], seen["kw"] = config, kw
        raise RuntimeError("stop")
    setattr(mod, cls, fake)
    try:
        cfg = dict(ENV_NAME=name, TOTAL_TIMESTEPS=5e5, TOTAL_TIMESTEPS_DECAY=5e5, NUM_STEPS=64, NUM_ENVS=128,
                   NUM_MINIBATCHES=16, MEMORY_WINDOW=4)
        with pytest.raises(RuntimeError, match="stop"):
            mod.make_train(cfg)
    finally:
        setattr(mod, cls, orig)
    assert seen["config"]["TEST_NUM_STEPS"] == test_steps
    assert seen["config"]["NUM_UPDATES"] == int(5e5 // 64 // 128)
    if script == "pqn_rnn_gymnax":
        assert seen["kw"]["env_params"].max_steps_in_episode == test_steps
    else:
        assert seen["kw"] == {"network": "mlp", "flatten_obs": True}


# --------------------------------------------------------------------------- #
# gymnax's own trajectories, once recorded
# --------------------------------------------------------------------------- #
_REF = sorted(glob.glob(os.path.join(HERE, "golden", "bsuite_chains_*_ref.npz")))
_PARAMS = {SEA: dict(deterministic=True, sample_action_map=False, unscaled_move_cost=0.01, randomize_actions=True,
                     max_steps_in_episode=2000),
           UMB: dict(chain_length=10, max_steps_in_episode=100),
           DISC: dict(max_steps_in_episode=100)}
_SHORT = {"deep_sea": SEA, "umbrella_chain": UMB, "discounting_chain": DISC}


@pytest.mark.skipif(not _REF, reason="no DeepSea / UmbrellaChain / DiscountingChain trajectories recorded from gymnax "
                                     "yet (tests/golden/make_bsuite_chains_golden_from_ref.py)")
@pytest.mark.parametrize("path", _REF or ["none"])
def test_against_reference(path, hlib):
    """Replays a trajectory recorded from gymnax through the oracle and the host-compiled device logic, and checks
    gymnax's default EnvParams and observation shape."""
    g = dict(np.load(path))
    base = os.path.basename(path)
    name = next(v for k, v in _SHORT.items() if f"_{k}_" in base)
    part = "partitionable" in base
    for k, v in _PARAMS[name].items():
        assert np.float32(g[f"param_{k}"]) == np.float32(v), k
    if name == DISC:
        assert np.array_equal(g["param_reward_timestep"], B.DiscountingChain.reward_timestep)
    assert tuple(g["obs_shape"]) == B.CORES[name].obs_shape
    jr.DEFAULT_PARTITIONABLE = part
    try:
        env = B.make(name)
        h = HostEnv(hlib, name, int(part))
        o_obs, o_st = env.reset(g["reset_keys"])
        h_obs, h_st = h.reset(g["reset_keys"])
        assert np.array_equal(o_obs, g["obs0"]) and np.array_equal(h_obs, g["obs0"])
        for t in range(g["action"].shape[0]):
            sk, act = g["step_keys"][t], g["action"][t].astype(np.int32)
            o_obs, o_st, o_r, o_d, o_info = env.step(sk, o_st, act)
            h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
            assert np.array_equal(o_d, g["done"][t]) and np.array_equal(h_d, g["done"][t]), t
            assert np.array_equal(bits(o_r), bits(g["reward"][t].astype(np.float32))), t
            assert np.array_equal(bits(h_r), bits(g["reward"][t].astype(np.float32))), t
            assert np.array_equal(o_obs, g["obs"][t]) and np.array_equal(h_obs, g["obs"][t]), t
            assert np.array_equal(o_info["returned_episode_lengths"], g["len"][t]), t
            assert np.array_equal(o_info["returned_episode_returns"], g["ret"][t]), t
            for k in B.CORES[name].state_fields:
                if k == "mapped_action":
                    assert np.array_equal(env.env.core.rewards(o_st), g["rewards"][t]), t
                else:
                    assert np.array_equal(o_st[k], g[k][t].astype(o_st[k].dtype)), (k, t)
            assert np.array_equal(to_state(name, o_st), h_st), t
    finally:
        jr.DEFAULT_PARTITIONABLE = False
