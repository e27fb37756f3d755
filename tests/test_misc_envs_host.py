"""SimpleBandit-bsuite, BernoulliBandit-misc, FourRooms-misc and MetaMaze-misc without a GPU: the device logic of
csrc/env_bsuite.cuh and csrc/env_misc.cuh compiled for the host (tests/host_harness_misc.cpp) against the NumPy oracles
(tests/bsuite_bandit_oracle.py, tests/misc_envs_oracle.py), self-checks of the oracles' episodes, the state-field
conversion of purejaxql_b200/envs.py, ``pqn_env_info``, make_train of both scripts and the refusal of SimpleBandit's
11 actions at HIDDEN_SIZE 512."""
import ctypes
import glob
import os
import subprocess

import numpy as np
import pytest
import torch

import bsuite_bandit_oracle as BB
import misc_envs_oracle as M
from oracle import jax_prng as jr
from purejaxql_b200 import envs as E

HERE = os.path.dirname(os.path.abspath(__file__))
SB, BERN, ROOMS, MAZE = "SimpleBandit-bsuite", "BernoulliBandit-misc", "FourRooms-misc", "MetaMaze-misc"
NAMES = [SB, BERN, ROOMS, MAZE]
PREFIX = {SB: "simple_bandit", BERN: "bernoulli_bandit", ROOMS: "four_rooms", MAZE: "meta_maze"}
MAX_STEPS = {SB: 100, BERN: 100, ROOMS: 500, MAZE: 200}
WORDS = {SB: 10, BERN: 11, ROOMS: 8, MAZE: 10}


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def hlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("harness") / "host_harness_misc.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(HERE, "host_harness_misc.cpp"), "-o", so])
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
@pytest.mark.parametrize("name,env_id,obs_dim,obs_shape,actions",
                         [(SB, 37, 1, (1, 1), 11), (BERN, 48, 4, (4,), 2), (ROOMS, 49, 4, (4,), 4),
                          (MAZE, 50, 15, (15,), 4)])
def test_env_info(name, env_id, obs_dim, obs_shape, actions):
    """pqn_env_info's table; without flatten_obs the observation space is gymnax's shape, (1, 1) for SimpleBandit."""
    from purejaxql_b200 import _lib
    info = _lib.EnvInfo()
    _lib.check(_lib.lib().pqn_env_info(env_id, info), "pqn_env_info")
    assert (info.obs_dim, info.num_actions, info.max_steps, info.binary_obs) == (obs_dim, actions, MAX_STEPS[name], 0)
    assert (info.state_words, tuple(info.obs_shape), info.packed_obs_words) == (WORDS[name], (obs_shape + (1, 1))[:3], 0)
    assert E.make(name)[0].observation_space().shape == obs_shape == M.CORES[name].obs_shape
    env, params = E.make(name, flatten_obs=True)
    assert E.ENV_IDS[name] == env_id and env.env_id == env_id
    assert env.observation_space().shape == (obs_dim,) and env.action_space().n == actions
    assert params.max_steps_in_episode == MAX_STEPS[name] and not env.binary_obs


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
STEPS = {SB: 40, BERN: 3 * 100 + 3, ROOMS: 2 * 500 + 3, MAZE: 3 * 200 + 3}
REWARDS = {SB: set(BB.linspace_levels().tolist()), BERN: {0.0, 1.0}, ROOMS: {0.0, 1.0}, MAZE: {0.0, 10.0}}


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("name", NAMES)
def test_host_logic_matches_oracle_bit_exact(hlib, name, part):
    """reset + several episodes of random actions (auto-resets included) for a ragged N: obs, reward, done, every
    state field and the LogWrapper fields equal the oracle bit for bit; pqn_env_obs's obs equals the one the step
    returned.  SimpleBandit ends an episode at every step, FourRooms at the goal or after 500 steps."""
    n = 97
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env = M.make(name)
        h = HostEnv(hlib, name, part)
        A = env.num_actions
        key, kr = jr.split(jr.PRNGKey(60 + part), 2)
        rk = jr.split(kr, n)
        o_obs, o_st = env.reset(rk)
        h_obs, h_st = h.reset(rk)
        assert np.array_equal(bits(h_obs), bits(o_obs)) and np.array_equal(bits(h.obs(h_st)), bits(o_obs))
        assert np.array_equal(to_state(name, o_st), h_st)
        dones = 0
        rewards = set()
        for t in range(STEPS[name]):
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
        if name == SB:
            assert dones == STEPS[SB] * n and (o_st["log_returned_episode_lengths"] == 1).all()
            assert len(rewards) == 11
        elif name == ROOMS:
            assert dones >= 2 * n and rewards == {0.0, 1.0}
        else:
            assert dones == 3 * n and (o_st["log_returned_episode_lengths"] == MAX_STEPS[name]).all()
        assert rewards <= REWARDS[name] and len(rewards) >= 2, rewards
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("part", [0, 1])
def test_reset_draws(hlib, part):
    """SimpleBandit's action_mask is permutation_indices of the reset key (a different permutation per env);
    BernoulliBandit's p1 takes both sample_probs; MetaMaze's goal and position are distinct free cells spread over
    the maze; FourRooms starts everywhere at [4, 1] with the goal at [8, 9]."""
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        rk = jr.split(jr.PRNGKey(9), 97)
        f = fields(SB, HostEnv(hlib, SB, part).reset(rk)[1])
        want = np.stack([jr.permutation_indices(rk[i], 11) for i in range(97)])
        assert np.array_equal(f["action_mask"], want)
        assert (np.sort(f["action_mask"], 1) == np.arange(11)).all() and len({tuple(r) for r in want}) == 97
        f = fields(BERN, HostEnv(hlib, BERN, part).reset(rk)[1])
        assert set(f["reward_probs"][:, 0].tolist()) == {np.float32(0.1), np.float32(0.9)}
        assert np.array_equal(f["reward_probs"].sum(1) == 1, np.ones(97, bool))
        f = fields(MAZE, HostEnv(hlib, MAZE, part).reset(rk)[1])
        assert not (f["pos"] == f["goal"]).all(1).any()
        assert len({tuple(g) for g in f["goal"]}) > 20
        assert (M.MetaMaze.env_map[f["pos"][:, 0], f["pos"][:, 1]] == 0).all()
        assert (M.MetaMaze.env_map[f["goal"][:, 0], f["goal"][:, 1]] == 0).all()
        f = fields(ROOMS, HostEnv(hlib, ROOMS, part).reset(rk)[1])
        assert (f["pos"] == [4, 1]).all() and (f["goal"] == [8, 9]).all()
        assert (f["fail_prob"] == np.float32(1.0 / 3)).all()
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def test_four_rooms_without_failures_walks_the_map(hlib):
    """With the fail_prob word set to 0, a scripted 16-step path through the hallways (6, 2) and (10, 6) reaches the
    goal: the host logic and the oracle agree step by step, the reward is 1 only on arrival and the episode ends
    there.  A move into a wall leaves the agent in place."""
    n = 3
    env = M.make(ROOMS)
    h = HostEnv(hlib, ROOMS, 0)
    _, o_st = env.reset(jr.split(jr.PRNGKey(1), n))
    o_st["fail_prob"] = np.zeros(n, np.float32)
    h_st = to_state(ROOMS, o_st)
    path = [1] + [2] * 6 + [1] * 7 + [0] * 2
    for t, a in enumerate(path):
        sk = jr.split(jr.PRNGKey(200 + t), n)
        act = np.full(n, a, np.int32)
        o_obs, o_st, o_r, o_d, _ = env.step(sk, o_st, act)
        h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
        assert np.array_equal(bits(h_obs), bits(o_obs)) and np.array_equal(h_r, o_r) and np.array_equal(h_d, o_d)
        last = t == len(path) - 1
        assert (o_d == last).all() and (o_r == (1.0 if last else 0.0)).all(), t
        if not last:
            o_st["fail_prob"] = np.zeros(n, np.float32)
    assert (o_st["pos"] == [4, 1]).all()                        # the auto-reset after the goal
    s = dict(pos=np.array([[4, 1]], np.int32), goal=np.array([[8, 9]], np.int32), time=np.zeros(1, np.int32),
             fail_prob=np.zeros(1, np.float32))
    _, s2, _, _, _ = M.FourRooms().step_env(jr.split(jr.PRNGKey(0), 1), s, np.array([3], np.int32))
    assert (s2["pos"] == [4, 1]).all()


def test_four_rooms_random_action_rate():
    """fail_prob = 1/3 replaces the action with a uniform one where uniform < 4/9, so pushing into the wall at
    [4, 0] moves the agent in (4/9) * (3/4) = 1/3 of the steps."""
    n = 8192
    core = M.FourRooms()
    _, s = core.reset_env(jr.split(jr.PRNGKey(0), n))
    _, s2, _, _, _ = core.step_env(jr.split(jr.PRNGKey(3), n), s, np.full(n, 3, np.int32))
    moved = (s2["pos"] != s["pos"]).any(1).mean()
    assert abs(moved - 1 / 3) < 0.02, moved
    assert np.float32(np.float32(np.float32(1 / 3) * np.float32(4)) / np.float32(3)) == np.float32(4 / 9)


# --------------------------------------------------------------------------- #
# the oracles' episodes
# --------------------------------------------------------------------------- #
def test_simple_bandit_oracle_episodes():
    """Every step is a whole episode: its return is linspace(0, 1, 11)[action_mask[action]] of the mask drawn at the
    previous reset, the observation is always 1 and the state after a step is the fresh reset state."""
    n = 64
    env = M.make(SB)
    key, kr = jr.split(jr.PRNGKey(4), 2)
    obs, st = env.reset(jr.split(kr, n))
    levels = np.arange(11, dtype=np.float32) / np.float32(10)
    assert np.array_equal(BB.linspace_levels(), levels)
    assert (obs == 1).all() and obs.shape == (n, 1)
    for t in range(12):
        key, ks = jr.split(key, 2)
        act = (np.arange(n) + t) % 11
        mask = st["action_mask"].copy()
        obs, st, r, d, info = env.step(jr.split(ks, n), st, act.astype(np.int32))
        assert np.array_equal(r, levels[mask[np.arange(n), act]]) and d.all()
        assert (obs == 1).all() and (st["time"] == 0).all() and (st["total_regret"] == 0).all()
        assert np.array_equal(info["returned_episode_returns"], r) and (info["returned_episode_lengths"] == 1).all()
    core = BB.SimpleBandit()
    _, s = core.reset_env(jr.split(jr.PRNGKey(0), 2))
    _, s2, r, d, _ = core.step_env(None, s, np.array([0, 1], np.int32))
    assert np.array_equal(s2["total_regret"], (np.float32(1) - r).astype(np.float32)) and (s2["time"] == 1).all()
    assert BB.make(flatten=False).obs_shape == (1, 1)


def test_bernoulli_bandit_oracle_episodes():
    """Pulling arm 0 for 100 steps: the reward rate follows reward_probs[0] (0.1 or 0.9 per env), the observation
    shows the one-hot arm, the last reward and 2 t / 100 - 1; every episode lasts 100 steps."""
    n = 256
    env = M.make(BERN)
    key, kr = jr.split(jr.PRNGKey(7), 2)
    obs, st = env.reset(jr.split(kr, n))
    assert np.array_equal(obs[0], np.array([1, 0, 0, -1], np.float32))
    p0 = st["reward_probs"][:, 0].copy()
    total = np.zeros(n)
    for t in range(100):
        key, ks = jr.split(key, 2)
        obs, st, r, d, info = env.step(jr.split(ks, n), st, np.zeros(n, np.int32))
        total += r
        assert np.array_equal(d, np.full(n, t == 99)), t
        if t < 99:
            assert (obs[:, 0] == 1).all() and np.array_equal(obs[:, 2], r)
            assert (obs[:, 3] == np.float32(np.float32(2 * (t + 1)) / np.float32(100)) - np.float32(1)).all()
    for p in (0.1, 0.9):
        sel = p0 == np.float32(p)
        assert sel.sum() > 50 and abs(total[sel].mean() / 100 - p) < 0.03
    assert (info["returned_episode_lengths"] == 100).all()
    assert np.array_equal(info["returned_episode_returns"], total.astype(np.float32))


def test_meta_maze_oracle_episodes():
    """The map has 41 free cells with a free centre; reaching the goal pays 10 and moves the agent to another free
    cell; the 3 x 3 field, one-hot action, last reward and time sit in the observation; episodes last 200 steps."""
    core = M.MetaMaze()
    assert len(core.coords) == 41 and core.env_map[4, 4] == 0 and core.env_map[2, 2] == 1
    s = dict(last_action=np.zeros(1, np.int32), last_reward=np.zeros(1, np.float32), pos=np.array([[3, 4]], np.int32),
             goal=np.array([[4, 4]], np.int32), time=np.zeros(1, np.int32), reward=np.full(1, 10.0, np.float32))
    obs, s2, r, d, _ = core.step_env(jr.split(jr.PRNGKey(3), 1), s, np.array([2], np.int32))
    assert r[0] == 10 and not (s2["pos"] == [4, 4]).all() and core.env_map[s2["pos"][0, 0], s2["pos"][0, 1]] == 0
    assert np.array_equal(obs[0, 9:13], [0, 0, 1, 0]) and obs[0, 13] == 10
    assert obs[0, 14] == np.float32(np.float32(2) / np.float32(100)) - np.float32(1)
    s3 = dict(s, pos=np.array([[1, 1]], np.int32))
    obs, s4, r, _, _ = core.step_env(jr.split(jr.PRNGKey(3), 1), s3, np.array([0], np.int32))   # into the top wall
    assert (s4["pos"] == [1, 1]).all() and r[0] == 0
    assert np.array_equal(obs[0, :9], [1, 1, 1, 1, 0, 0, 1, 0, 1])
    n = 64
    env = M.make(MAZE)
    key, kr = jr.split(jr.PRNGKey(8), 2)
    _, st = env.reset(jr.split(kr, n))
    for t in range(200):
        key, ka, ks = jr.split(key, 3)
        _, st, r, d, info = env.step(jr.split(ks, n), st, random_actions(ka, n, 4))
        assert np.array_equal(d, np.full(n, t == 199)), t
    assert (info["returned_episode_lengths"] == 200).all() and info["returned_episode_returns"].max() >= 10


# --------------------------------------------------------------------------- #
# fields, scripts and the network limit
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name", NAMES)
def test_fields_round_trip(name):
    env = M.make(name)
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


@pytest.mark.parametrize("script", ["pqn_gymnax", "pqn_rnn_gymnax"])
@pytest.mark.parametrize("name", NAMES)
def test_make_train_accepts_env(script, name):
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
    assert seen["config"]["TEST_NUM_STEPS"] == MAX_STEPS[name]
    assert seen["config"]["NUM_UPDATES"] == int(5e5 // 64 // 128)
    if script == "pqn_rnn_gymnax":
        assert seen["kw"]["env_params"].max_steps_in_episode == MAX_STEPS[name]
    else:
        assert seen["kw"] == {"network": "mlp", "flatten_obs": True}


@pytest.mark.parametrize("H,ok", [(256, True), (512, False)])
def test_simple_bandit_actions_at_hidden_512_are_refused(H, ok):
    """11 actions stay beyond the head backward's shared memory at HIDDEN_SIZE 512 (actions <= 9 there): both
    networks' specs for SimpleBandit are refused with that limit on the host, before anything is allocated, and
    HIDDEN_SIZE 256 is built."""
    from purejaxql_b200 import _lib
    from purejaxql_b200.engine import network_spec
    from purejaxql_b200.networks import NET_RNN, QNetworkSpec
    env, _ = E.make(SB, flatten_obs=True)
    builders = [lambda: network_spec(env, "mlp", {"HIDDEN_SIZE": H, "NUM_LAYERS": 2}),
                lambda: QNetworkSpec(NET_RNN, env.obs_dim, env.num_actions, H, 2)]
    for build in builders:
        if ok:
            build()
        else:
            with pytest.raises(_lib.PqnError) as e:
                build()
            assert "num_actions=11" in str(e.value) and "limit 227 KB" in str(e.value)


# --------------------------------------------------------------------------- #
# gymnax's own trajectories, once recorded
# --------------------------------------------------------------------------- #
_REF = sorted(glob.glob(os.path.join(HERE, "golden", "misc_*_ref.npz")))
_PARAMS = {SB: dict(optimal_return=1, max_steps_in_episode=100),
           BERN: dict(normalize_time=True, max_steps_in_episode=100),
           ROOMS: dict(fail_prob=1.0 / 3, resample_init_pos=False, resample_goal_pos=False, max_steps_in_episode=500),
           MAZE: dict(reward=10.0, normalize_time=True, max_steps_in_episode=200)}
_SHORT = {"simple_bandit": SB, "bernoulli_bandit": BERN, "four_rooms": ROOMS, "meta_maze": MAZE}


@pytest.mark.skipif(not _REF, reason="no SimpleBandit / BernoulliBandit / FourRooms / MetaMaze trajectories recorded "
                                     "from gymnax yet (tests/golden/make_misc_golden_from_ref.py)")
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
    if name == BERN:
        assert np.array_equal(g["param_sample_probs"].astype(np.float32), M.BernoulliBandit.sample_probs)
    assert tuple(g["obs_shape"]) == M.CORES[name].obs_shape
    jr.DEFAULT_PARTITIONABLE = part
    try:
        env = M.make(name)
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
            for k in M.CORES[name].state_fields:
                if k == "action_mask":
                    assert np.array_equal(env.env.core.rewards(o_st), g["rewards"][t]), t
                else:
                    assert np.array_equal(o_st[k], g[k][t].astype(o_st[k].dtype)), (k, t)
            assert np.array_equal(to_state(name, o_st), h_st), t
    finally:
        jr.DEFAULT_PARTITIONABLE = False
