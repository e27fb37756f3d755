"""MemoryChain-bsuite without a GPU: the device logic of csrc/env_bsuite.cuh compiled for the host
(tests/host_harness_bsuite.cpp) against the NumPy oracle (tests/bsuite_oracle.py) bit for bit, self-checks of the
oracle's episode structure, the state-field conversion of purejaxql_b200/envs.py, the preset and make_train's
argument checks."""
import ctypes
import glob
import os
import subprocess

import numpy as np
import pytest
import torch

import bsuite_oracle as MC
from oracle import jax_prng as jr
from purejaxql_b200 import envs as E

HERE = os.path.dirname(os.path.abspath(__file__))
NAME = "MemoryChain-bsuite"


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def hlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("harness") / "host_harness_bsuite.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(HERE, "host_harness_bsuite.cpp"), "-o", so])
    return ctypes.CDLL(so)


class HostMemoryChain:
    """Drives the harness like pqn_env_reset_params / pqn_env_step / pqn_env_obs."""

    def __init__(self, lib, memory_length, part):
        self.lib, self.ml, self.part = lib, memory_length, part
        self.words = lib.h_mc_state_words()

    def reset(self, keys):
        n = keys.shape[0]
        keys = np.ascontiguousarray(keys, np.uint32)
        state = np.zeros((self.words, n), np.uint32)
        obs = np.zeros((n, 3), np.float32)
        self.lib.h_mc_reset(ptr(keys), ptr(state), ptr(obs), ctypes.c_int64(n), self.ml, self.part)
        return obs, state

    def step(self, keys, state, action):
        n = keys.shape[0]
        keys = np.ascontiguousarray(keys, np.uint32)
        action = np.ascontiguousarray(action, np.int32)
        obs = np.zeros((n, 3), np.float32)
        reward = np.zeros(n, np.float32)
        done = np.zeros(n, np.uint8)
        self.lib.h_mc_step(ptr(keys), ptr(state), ptr(action), ptr(obs), ptr(reward), ptr(done), ctypes.c_int64(n),
                           self.part)
        return obs, state, reward, done.astype(bool)

    def obs(self, state):
        n = state.shape[1]
        obs = np.zeros((n, 3), np.float32)
        self.lib.h_mc_obs(ptr(np.ascontiguousarray(state)), ptr(obs), ctypes.c_int64(n))
        return obs


def _fields(state):
    return E.state_to_fields(NAME, torch.from_numpy(state.view(np.int32)))


def _assert_state_equal(state, o_st, ml, where):
    f = _fields(state)
    for k, v in o_st.items():
        assert np.array_equal(f[k].numpy().astype(v.dtype).reshape(v.shape), v), (where, k)
    assert (f["memory_length"].numpy() == ml).all(), where


def _random_actions(ka, n):
    return jr.randint(jr.split(ka, n), (), 0, 2)


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("ml", [1, 5, 100])
def test_host_logic_matches_oracle_bit_exact(hlib, part, ml):
    """reset + three whole episodes of random actions for a ragged N: obs, reward, done, every state field and the
    LogWrapper fields equal the oracle bit for bit; the obs of pqn_env_obs equals the obs the step returned."""
    n = 97
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env = MC.make(ml, flatten=True)
        h = HostMemoryChain(hlib, ml, part)
        key, kr = jr.split(jr.PRNGKey(7 + ml), 2)
        rkeys = jr.split(kr, n)
        o_obs, o_st = env.reset(rkeys)
        h_obs, h_st = h.reset(rkeys)
        assert np.array_equal(h_obs, o_obs)
        assert np.array_equal(h.obs(h_st), o_obs)
        _assert_state_equal(h_st, o_st, ml, "reset")
        assert set(o_st["context"][:, 0]) == {False, True}
        for t in range(3 * (ml + 1) + 2):
            key, ka, ks = jr.split(key, 3)
            act = _random_actions(ka, n)
            skeys = jr.split(ks, n)
            o_obs, o_st, o_r, o_d, o_info = env.step(skeys, o_st, act)
            h_obs, h_st, h_r, h_d = h.step(skeys, h_st, act)
            assert np.array_equal(h_d, o_d), t
            assert np.array_equal(h_r, o_r), t
            assert np.array_equal(h_obs, o_obs), t
            assert np.array_equal(h.obs(h_st), o_obs), t
            _assert_state_equal(h_st, o_st, ml, t)
        assert (o_st["log_returned_episode_lengths"] == ml + 1).all()
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("ml", [1, 2, 5, 100])
def test_oracle_episode_structure(ml):
    """Episodes last memory_length + 1 steps; the reward is nonzero only on the done step and is +1 iff the action
    equals the context bit; the context is shown only in observations of time-0 states (the reset obs and, through
    the one-step lag, the first step's obs); the query slot is set only for the state at time == memory_length - 1."""
    n = 64
    env = MC.make(ml, flatten=True)
    key, kr = jr.split(jr.PRNGKey(3), 2)
    obs, st = env.reset(jr.split(kr, n))
    assert np.array_equal(obs[:, 2], np.where(st["context"][:, 0], 1.0, -1.0).astype(np.float32))
    assert (obs[:, 0] == 1.0).all() and (obs[:, 1] == 0).all()
    t_in_ep = np.zeros(n, np.int64)
    seen = {1.0: 0, -1.0: 0}
    for t in range(4 * (ml + 1)):
        ctx = st["context"][:, 0].copy()
        time_before = st["time"].copy()
        key, ka, ks = jr.split(key, 3)
        act = _random_actions(ka, n)
        obs, st, r, d, info = env.step(jr.split(ks, n), st, act)
        t_in_ep += 1
        assert np.array_equal(d, t_in_ep == ml + 1), t
        assert np.array_equal(info["discount"], (~d).astype(np.float32))
        assert (r[~d] == 0).all()
        assert np.array_equal(r[d], np.where(act[d] == ctx[d], 1.0, -1.0).astype(np.float32))
        for v in r[d]:
            seen[float(v)] += 1
        # the obs of a step is that of the pre-step state (time_before); after done it is the reset obs (time 0)
        shown_t = np.where(d, 0, time_before)
        assert np.array_equal(obs[:, 2] != 0, shown_t == 0), t
        assert (obs[:, 1] == 0).all()                        # query = 0 with num_bits = 1
        assert np.array_equal(obs[:, 0], (np.float32(1) - shown_t.astype(np.float32) / np.float32(ml)))
        assert np.array_equal(info["returned_episode_lengths"][d], np.full(d.sum(), ml + 1))
        t_in_ep[d] = 0
    assert seen[1.0] > 0 and seen[-1.0] > 0


def test_query_slot_when_query_is_nonzero():
    """The query slot carries `query` at time == memory_length - 1 only (num_bits = 1 makes query 0 in every real
    episode, so this sets it by hand)."""
    core = MC.MemoryChain(6)
    n = 8
    s = dict(context=np.ones((n, 1), bool), query=np.full(n, 3, np.int32), total_perfect=np.zeros(n, np.int32),
             total_regret=np.zeros(n, np.int32), time=np.arange(n, dtype=np.int32))
    o = core.get_obs(s)[:, 0]
    assert np.array_equal(o[:, 1], np.where(np.arange(n) == 5, 3.0, 0.0).astype(np.float32))
    assert np.array_equal(o[:, 2], np.where(np.arange(n) == 0, 1.0, 0.0).astype(np.float32))


def test_fields_round_trip():
    env = MC.make(7, flatten=True)
    key = jr.PRNGKey(11)
    _, st = env.reset(jr.split(key, 50))
    for t in range(5):
        key, ka, ks = jr.split(key, 3)
        _, st, _, _, _ = env.step(jr.split(ks, 50), st, _random_actions(ka, 50))
    f = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in st.items()}
    f["memory_length"] = torch.full((50,), 7, dtype=torch.int32)
    state = E.fields_to_state(NAME, f)
    assert state.shape == (11, 50)
    back = E.state_to_fields(NAME, state)
    for k, v in f.items():
        assert np.array_equal(back[k].numpy().astype(v.numpy().dtype).reshape(v.shape), v.numpy()), k
    assert torch.equal(E.fields_to_state(NAME, back), state)


def test_memory_chain_preset_matches_reference_values():
    from purejaxql_b200 import config_loader
    c = config_loader.compose(["+alg=pqn_rnn_memory_chain"])
    a = c["alg"]
    want = dict(ALG_NAME="pqn_rnn", TOTAL_TIMESTEPS=1e5, TOTAL_TIMESTEPS_DECAY=1e5, NUM_ENVS=32, MEMORY_WINDOW=4,
                NUM_STEPS=128, EPS_START=1.0, EPS_FINISH=0.01, EPS_DECAY=0.1, NUM_MINIBATCHES=16, NUM_EPOCHS=4,
                NORM_INPUT=False, HIDDEN_SIZE=256, NUM_LAYERS=2, NORM_TYPE="layer_norm", LR=0.001, MAX_GRAD_NORM=10,
                LR_LINEAR_DECAY=False, REW_SCALE=1.0, GAMMA=0.99, LAMBDA=0.95, ENV_NAME=NAME,
                ENV_KWARGS={"memory_length": 100}, TEST_DURING_TRAINING=True, TEST_INTERVAL=0.05, TEST_NUM_ENVS=128,
                EPS_TEST=0.0)
    for k, v in want.items():
        assert a[k] == v and type(a[k]) is type(v), (k, a[k], v)
    assert "TEST_NUM_STEPS" not in a
    assert int(a["TOTAL_TIMESTEPS"] // a["NUM_STEPS"] // a["NUM_ENVS"]) == 24
    assert int(24 * a["TEST_INTERVAL"]) == 1


def test_memory_length_defaults_and_checks():
    """make_train's env params: ENV_KWARGS.memory_length, default 10 (pqn_rnn_gymnax.py:134-136); the feed-forward
    script and envs.make use gymnax's default (5).  A memory_length that is not a positive int is refused before any
    device work."""
    from purejaxql_b200 import pqn_rnn_gymnax
    env, params = E.make(NAME, flatten_obs=True)
    assert (params.max_steps_in_episode, params.memory_length) == (1000, 5)
    assert env.num_actions == 2 and env.obs_dim == 3 and env.state_words == 11 and not env.binary_obs
    seen = {}
    orig = pqn_rnn_gymnax.PQNRnnEngine
    try:
        def fake(config, env_params=None):
            seen["params"] = env_params
            seen["config"] = config
            raise RuntimeError("stop")
        pqn_rnn_gymnax.PQNRnnEngine = fake
        for kwargs, want in (({}, 10), ({"memory_length": 3}, 3), (None, 10)):
            cfg = dict(ENV_NAME=NAME, TOTAL_TIMESTEPS=1e5, TOTAL_TIMESTEPS_DECAY=1e5, NUM_STEPS=128, NUM_ENVS=32,
                       NUM_MINIBATCHES=16)
            if kwargs is not None:
                cfg["ENV_KWARGS"] = kwargs
            with pytest.raises(RuntimeError, match="stop"):
                pqn_rnn_gymnax.make_train(cfg)
            assert seen["params"].memory_length == want and seen["params"].max_steps_in_episode == 1000
            assert seen["config"]["TEST_NUM_STEPS"] == 1000 and seen["config"]["NUM_UPDATES"] == 24
    finally:
        pqn_rnn_gymnax.PQNRnnEngine = orig
    for bad in (0, -3, 2.5, "7", True):
        cfg = dict(ENV_NAME=NAME, TOTAL_TIMESTEPS=1e5, TOTAL_TIMESTEPS_DECAY=1e5, NUM_STEPS=128, NUM_ENVS=32,
                   NUM_MINIBATCHES=16, ENV_KWARGS={"memory_length": bad})
        with pytest.raises(ValueError, match="memory_length"):
            pqn_rnn_gymnax.make_train(cfg)


_REF = sorted(glob.glob(os.path.join(HERE, "golden", "memory_chain_L*_ref.npz")))


@pytest.mark.skipif(not _REF, reason="no MemoryChain trajectories recorded from gymnax yet "
                                     "(tests/golden/make_memory_chain_golden_from_ref.py)")
@pytest.mark.parametrize("path", _REF or ["none"])
def test_oracle_against_reference_memory_chain(path, hlib):
    """Replays a trajectory recorded from gymnax through the oracle and the host-compiled device logic."""
    g = dict(np.load(path))
    layout = os.path.basename(path).split("_")[3]
    ml = int(g["memory_length"])
    jr.DEFAULT_PARTITIONABLE = layout == "partitionable"
    try:
        env = MC.make(ml, flatten=True)
        h = HostMemoryChain(hlib, ml, int(layout == "partitionable"))
        o_obs, o_st = env.reset(g["reset_keys"])
        h_obs, h_st = h.reset(g["reset_keys"])
        assert np.array_equal(o_obs, g["obs0"]) and np.array_equal(h_obs, g["obs0"])
        for t in range(g["action"].shape[0]):
            sk, act = g["step_keys"][t], g["action"][t].astype(np.int32)
            o_obs, o_st, o_r, o_d, o_info = env.step(sk, o_st, act)
            h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
            for got in ((o_obs, o_r, o_d), (h_obs, h_r, h_d)):
                assert np.array_equal(got[0], g["obs"][t]), ("obs", t)
                assert np.array_equal(got[1], g["reward"][t].astype(np.float32)), ("reward", t)
                assert np.array_equal(got[2], g["done"][t]), ("done", t)
            assert np.array_equal(o_info["discount"], g["discount"][t].astype(np.float32)), t
            assert np.array_equal(o_info["returned_episode_returns"], g["ret"][t].astype(np.float32)), t
            assert np.array_equal(o_info["returned_episode_lengths"], g["len"][t]), t
            for k in ("context", "query", "total_perfect", "total_regret", "time"):
                assert np.array_equal(o_st[k].reshape(g[k][t].shape), g[k][t].astype(o_st[k].dtype)), (k, t)
            _assert_state_equal(h_st, o_st, ml, t)
    finally:
        jr.DEFAULT_PARTITIONABLE = False
