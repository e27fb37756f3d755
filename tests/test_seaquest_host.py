"""Seaquest-MinAtar without a GPU: the device logic of csrc/env_seaquest.cuh compiled for the host
(tests/host_harness_seaquest.cpp) against the NumPy oracle (tests/seaquest_oracle.py) over long random-action runs in
both threefry layouts, oracle episodes that reach every terminal case and surfacing outcome, the state-field
conversion of purejaxql_b200/envs.py, ``pqn_env_info``, make_train of both feed-forward scripts, the recurrent
script's refusal, and the D = 1000 packed-bit MLP descriptor."""
import copy
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import seaquest_oracle as SQ
from oracle import jax_prng as jr
from purejaxql_b200 import envs as E

HERE = os.path.dirname(os.path.abspath(__file__))
NAME = "Seaquest-MinAtar"


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def hlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("harness") / "host_harness_seaquest.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(HERE, "host_harness_seaquest.cpp"), "-o", so])
    return ctypes.CDLL(so)


class HostEnv:
    """Drives the harness like pqn_env_reset / pqn_env_step / pqn_env_obs."""

    def __init__(self, lib, part, max_steps=None):
        self.lib, self.part = lib, part
        self.words = lib.h_sq_state_words()
        self.D = lib.h_sq_obs_dim()
        self.max_steps = max_steps or lib.h_sq_max_steps()

    def reset(self, keys):
        n = keys.shape[0]
        keys = np.ascontiguousarray(keys, np.uint32)
        state = np.zeros((self.words, n), np.uint32)
        obs = np.zeros((n, self.D), np.float32)
        self.lib.h_sq_reset(ptr(keys), ptr(state), ptr(obs), ctypes.c_int64(n), self.max_steps, self.part)
        return obs, state

    def step(self, keys, state, action):
        n = keys.shape[0]
        keys = np.ascontiguousarray(keys, np.uint32)
        action = np.ascontiguousarray(action, np.int32)
        obs = np.zeros((n, self.D), np.float32)
        reward = np.zeros(n, np.float32)
        done = np.zeros(n, np.uint8)
        self.lib.h_sq_step(ptr(keys), ptr(state), ptr(action), ptr(obs), ptr(reward), ptr(done), ctypes.c_int64(n),
                           self.max_steps, self.part)
        return obs, state, reward, done.astype(bool)

    def obs(self, state):
        n = state.shape[1]
        obs = np.zeros((n, self.D), np.float32)
        self.lib.h_sq_obs(ptr(np.ascontiguousarray(state)), ptr(obs), ctypes.c_int64(n))
        return obs


def to_state(st):
    return E.fields_to_state(NAME, {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in st.items()}).numpy().view(
        np.uint32).copy()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def policy_actions(ka, n):
    """uniform actions for even envs; odd envs never press u, so they stay down until oxygen or an enemy ends the
    episode (uniform play mostly ends at the first return to the surface)"""
    a = jr.randint(jr.split(ka, n), (), 0, 6).astype(np.int32)
    a[1::2] = np.where(a[1::2] == 2, 4, a[1::2])
    return a


# --------------------------------------------------------------------------- #
# host-compiled device logic against the oracle
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("part", [0, 1])
def test_host_logic_matches_oracle_bit_exact(hlib, part):
    """reset + 1,200 steps at N = 97 (auto-resets included): obs, reward, done, every state word (lists in order,
    LogWrapper included) equal the oracle bit for bit, and pqn_env_obs's obs equals the step's.  The run reaches
    spawns of both enemy kinds and divers, kills, pickups and oxygen-out and collision terminals."""
    n = 97
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env = SQ.make(flatten=True)
        h = HostEnv(hlib, part)
        key, kr = jr.split(jr.PRNGKey(4), 2)
        rk = jr.split(kr, n)
        o_obs, o_st = env.reset(rk)
        h_obs, h_st = h.reset(rk)
        assert np.array_equal(h_obs, o_obs) and np.array_equal(to_state(o_st), h_st)
        seen = dict(subs=0, fish=0, divers=0, kills=0, dones=0, long=0, bullets=0)
        for t in range(1200):
            key, ka, ks = jr.split(key, 3)
            act = policy_actions(ka, n)
            sk = jr.split(ks, n)
            o_obs, o_st, o_r, o_d, _ = env.step(sk, o_st, act)
            h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
            assert np.array_equal(h_d, o_d), t
            assert np.array_equal(bits(h_r), bits(o_r)), t
            assert np.array_equal(h_obs, o_obs), t
            assert np.array_equal(to_state(o_st), h_st), t
            if t % 50 == 0:
                assert np.array_equal(h.obs(h_st), o_obs), t
            seen["subs"] += int(o_st["n_e_subs"].sum())
            seen["fish"] += int(o_st["n_e_fish"].sum())
            seen["divers"] += int((o_st["diver_count"] > 0).sum())
            seen["bullets"] += int(o_st["n_e_bullets"].sum())
            seen["kills"] += int((o_r > 0).sum())
            seen["dones"] += int(o_d.sum())
            seen["long"] += int((o_d & (o_st["log_returned_episode_lengths"] > 200)).sum())
        assert min(seen.values()) > 0, seen
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def _case(**over):
    """one env: reset state with fields overridden (lists given as Python lists)"""
    _, st = SQ.Seaquest().reset_env(jr.split(jr.PRNGKey(0), 1))
    e = SQ._unpack(st, 0)
    e.update(copy.deepcopy(over))
    return e


CASES = {
    # name: (state overrides, action, expected reward, expected terminal, check on the stepped state)
    "surface_no_diver": (dict(sub_y=1, surface=False), 2, 0, True, None),
    "surface_six_divers": (dict(sub_y=1, surface=False, diver_count=6, oxygen=151), 2, 7, False,
                           lambda e: e["diver_count"] == 0 and e["oxygen"] == 200 and e["ramp_index"] == 1
                           and e["e_spawn_speed"] == 19 and e["move_speed"] == 5),
    "surface_some_divers": (dict(sub_y=1, surface=False, diver_count=3, oxygen=40, ramp_index=1), 2, 0, False,
                            lambda e: e["diver_count"] == 2 and e["oxygen"] == 200 and e["move_speed"] == 4),
    "oxygen_out": (dict(sub_y=4, surface=False, oxygen=-1), 0, 0, True, None),
    "oxygen_last": (dict(sub_y=4, surface=False, oxygen=0), 0, 0, False, lambda e: e["oxygen"] == -1),
    "fish_collision": (dict(sub_y=3, surface=False, e_fish=[[5, 3, 1, 2]]), 0, 0, True, None),
    "fish_moves_onto_sub": (dict(sub_y=3, surface=False, e_fish=[[4, 3, 1, 0]]), 0, 0, True, None),
    "sub_collision": (dict(sub_y=3, surface=False, e_subs=[[6, 3, 0, 0, 4]]), 0, 0, True, None),
    "enemy_bullet": (dict(sub_y=3, surface=False, e_bullets=[[6, 3, 0]]), 0, 0, True, None),
    "shoot_fish": (dict(sub_y=3, surface=False, sub_or=True, e_fish=[[6, 3, 0, 3]]), 5, 1, False,
                   lambda e: not e["e_fish"] and not e["f_bullets"] and e["shot_timer"] == 4),
    "shoot_sub_fish_first": (dict(sub_y=3, surface=False, sub_or=True, e_fish=[[7, 3, 0, 3]],
                                  e_subs=[[7, 3, 0, 3, 5]], f_bullets=[[6, 3, 1]]), 0, 1, False,
                             lambda e: not e["e_fish"] and len(e["e_subs"]) == 1),
    "diver_pickup": (dict(sub_y=3, surface=False, divers=[[5, 3, 1, 2]], diver_count=2), 0, 0, False,
                     lambda e: e["diver_count"] == 3 and not e["divers"]),
    "diver_cap": (dict(sub_y=3, surface=False, divers=[[5, 3, 1, 2]], diver_count=6), 0, 0, False,
                  lambda e: e["diver_count"] == 6 and len(e["divers"]) == 1),
    "sub_fires": (dict(sub_y=3, surface=False, e_subs=[[0, 6, 1, 3, 0]]), 0, 0, False,
                  lambda e: e["e_bullets"] == [[1, 6, 1]] and e["e_subs"][0][4] == 10),
    "sub_leaves_and_fires": (dict(sub_y=3, surface=False, e_subs=[[9, 6, 1, 0, 0]]), 0, 0, False,
                             lambda e: not e["e_subs"] and not e["e_bullets"]),
    "spawn_blocked": (dict(e_spawn_timer=0, e_fish=[[9, y, 0, 4] for y in range(1, 9)]), 0, 0, False, None),
}


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("part", [0, 1])
def test_oracle_cases_and_host(hlib, name, part):
    """each terminal case and each surfacing outcome, reached from a constructed state: the oracle's reward, terminal
    and resulting state as MinAtar's rules give them, and the host-compiled device logic equal to the oracle"""
    over, action, reward, terminal, check = CASES[name]
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        e = _case(**over)
        key = jr.PRNGKey(7)
        r, t = SQ.Seaquest.act(e, action, *(int(d[0]) for d in SQ.Seaquest.draws(key[None])))
        assert (r, t) == (reward, terminal)
        if check is not None:
            assert check(e), e
        if name == "spawn_blocked":   # every row holds a left-moving fish: only a left-moving spawn can happen
            assert len(e["e_subs"]) + len(e["e_fish"]) in (8, 9)
        # the same step through Environment.step (auto-reset) on the oracle and the harness
        env = SQ.make(flatten=True)
        _, st0 = env.reset(jr.split(jr.PRNGKey(0), 1))
        st = dict(st0, **SQ._pack([_case(**over)]))
        sk = jr.split(jr.PRNGKey(9), 1)
        o_obs, o_st, o_r, o_d, _ = env.step(sk, st, np.array([action], np.int32))
        h = HostEnv(hlib, part)
        h_obs, h_st, h_r, h_d = h.step(sk, to_state(st), np.array([action], np.int32))
        assert bool(o_d[0]) == terminal and float(o_r[0]) == reward
        assert np.array_equal(h_d, o_d) and np.array_equal(bits(h_r), bits(o_r)) and np.array_equal(h_obs, o_obs)
        assert np.array_equal(to_state(o_st), h_st)
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def test_oracle_observation_channels():
    """MinAtar's channel order and gauges on one constructed state, including the oxygen gauge at oxygen -1"""
    core = SQ.Seaquest()
    e = _case(sub_x=3, sub_y=2, sub_or=True, oxygen=120, diver_count=2, f_bullets=[[4, 2, 1]], e_bullets=[[7, 5, 0]],
              e_fish=[[0, 6, 1, 1]], e_subs=[[8, 1, 0, 2, 3]], divers=[[5, 8, 1, 0]])
    o = core.get_obs(SQ._pack([e]))[0]
    on = lambda c: sorted(map(tuple, np.argwhere(o[:, :, c] > 0).tolist()))
    assert on(0) == [(2, 3)] and on(1) == [(2, 2)] and on(2) == [(2, 4)] and on(4) == [(5, 7)]
    assert on(5) == [(6, 0)] and on(6) == [(1, 8)] and on(9) == [(8, 5)]
    assert on(3) == [(1, 9), (8, 4)]                      # the fish at column 0 has no trail on the board
    assert on(7) == [(9, x) for x in range(6)] and on(8) == [(9, 7), (9, 8)]
    e["oxygen"] = -1
    assert sorted(np.argwhere(core.get_obs(SQ._pack([e]))[0][:, :, 7] > 0)[:, 1].tolist()) == list(range(9))


# --------------------------------------------------------------------------- #
# registry, fields, scripts
# --------------------------------------------------------------------------- #
def test_env_info(hlib):
    """pqn_env_info's table and the harness agree; Seaquest is registered, and not among gymnax's MinAtar games"""
    from purejaxql_b200 import _lib
    info = _lib.EnvInfo()
    _lib.check(_lib.lib().pqn_env_info(4, info), "pqn_env_info")
    assert (info.obs_dim, info.num_actions, info.max_steps, info.binary_obs) == (1000, 6, 1000, 1)
    assert (info.state_words, tuple(info.obs_shape), info.packed_obs_words) == (24, (10, 10, 10), 32)
    assert (hlib.h_sq_state_words(), hlib.h_sq_obs_dim(), hlib.h_sq_max_steps()) == (24, 1000, 1000)
    env, params = E.make(NAME)
    assert E.ENV_IDS[NAME] == 4 and env.binary_obs and env.observation_space().shape == (10, 10, 10)
    assert E.make(NAME, flatten_obs=True)[0].observation_space().shape == (1000,)
    assert NAME in E.MINATAR_UNREGISTERED and NAME not in E.MINATAR_GAMES and len(E.MINATAR_GAMES) == 4


def test_fields_round_trip():
    env = SQ.make()
    key = jr.PRNGKey(11)
    _, st = env.reset(jr.split(key, 40))
    for t in range(120):
        key, ka, ks = jr.split(key, 3)
        _, st, _, _, _ = env.step(jr.split(ks, 40), st, policy_actions(ka, 40))
    assert st["n_e_fish"].sum() + st["n_e_subs"].sum() > 0
    f = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in st.items()}
    state = E.fields_to_state(NAME, f)
    assert state.shape == (24, 40)
    back = E.state_to_fields(NAME, state)
    assert set(back) == set(f)
    for k, v in f.items():
        assert np.array_equal(back[k].numpy().astype(v.numpy().dtype).reshape(v.shape), v.numpy()), k
    assert torch.equal(E.fields_to_state(NAME, back), state)


@pytest.mark.parametrize("script,network", [("pqn_minatar", "cnn"), ("pqn_gymnax", "mlp")])
def test_make_train_accepts_seaquest(script, network):
    """make_train builds each feed-forward script's engine for Seaquest: the CNN for pqn_minatar, the MLP on the
    flattened observation for pqn_gymnax"""
    import importlib
    mod = importlib.import_module(f"purejaxql_b200.{script}")
    seen = {}
    orig = mod.PQNEngine

    def fake(config, *a, **kw):
        seen["config"], seen["kw"] = config, kw
        raise RuntimeError("stop")
    mod.PQNEngine = fake
    try:
        cfg = dict(ENV_NAME=NAME, TOTAL_TIMESTEPS=5e5, TOTAL_TIMESTEPS_DECAY=5e5, NUM_STEPS=32, NUM_ENVS=128,
                   NUM_MINIBATCHES=16)
        with pytest.raises(RuntimeError, match="stop"):
            mod.make_train(cfg)
    finally:
        mod.PQNEngine = orig
    assert seen["config"]["ENV_NAME"] == NAME
    assert seen["kw"].get("network", "cnn") == network


def test_recurrent_script_refuses_seaquest():
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = dict(ENV_NAME=NAME, TOTAL_TIMESTEPS=5e5, TOTAL_TIMESTEPS_DECAY=5e5, NUM_STEPS=64, NUM_ENVS=128,
               NUM_MINIBATCHES=16, MEMORY_WINDOW=4)
    with pytest.raises(NotImplementedError) as e:
        pqn_rnn_gymnax.make_train(cfg)
    with pytest.raises(NotImplementedError) as e_breakout:
        pqn_rnn_gymnax.make_train(dict(cfg, ENV_NAME="Breakout-MinAtar"))
    assert str(e.value).replace(NAME, "<env>") == str(e_breakout.value).replace("Breakout-MinAtar", "<env>")


def test_bits_descriptor_and_layout_at_1000():
    """the packed-bit MLP is built for D = 1000 (Seaquest's 10 x 10 x 10) and lays out its parameters as the MLP on
    1000 float inputs; widths that are not 100 * C of a built game stay refused"""
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_MLP, NET_MLP_BITS, QNetworkSpec
    lib = _lib.lib()
    for H in (64, 128, 256, 512):
        for layers in (1, 2, 4):
            for nt in ("layer_norm", "batch_norm", "none"):
                for ni in (False, True):
                    b = QNetworkSpec(NET_MLP_BITS, 1000, 6, H, layers, norm_type=nt, norm_input=ni)
                    m = QNetworkSpec(NET_MLP, 1000, 6, H, layers, norm_type=nt, norm_input=ni)
                    assert b.total == m.total and b.entries == m.entries
                    assert lib.pqn_net_workspace_bytes(b.desc, 2, 1000) > 0
    for D in (900, 1100, 1024):
        with pytest.raises(Exception, match="1000 for Seaquest"):
            QNetworkSpec(NET_MLP_BITS, D, 6, 128, 1)
