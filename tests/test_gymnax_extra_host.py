"""MountainCar-v0 and Catch-bsuite without a GPU: the device logic of csrc/env_classic.cuh and csrc/env_bsuite.cuh
compiled for the host (tests/host_harness_gymnax_extra.cpp) against the NumPy oracles (tests/gymnax_extra_oracle.py),
self-checks of the oracles' episodes, the state-field conversion of purejaxql_b200/envs.py, ``pqn_env_info``,
make_train of both scripts, and the network workspace sizes of the shapes built before these envs."""
import ctypes
import glob
import os
import subprocess

import numpy as np
import pytest
import torch

import gymnax_extra_oracle as X
from oracle import jax_prng as jr
from purejaxql_b200 import envs as E

HERE = os.path.dirname(os.path.abspath(__file__))
MCAR, CATCH = "MountainCar-v0", "Catch-bsuite"
PREFIX = {MCAR: "mcar", CATCH: "catch"}


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def hlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("harness") / "host_harness_gymnax_extra.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(HERE, "host_harness_gymnax_extra.cpp"), "-o", so])
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


def ulps(got, want, floor):
    """|got - want| in fp32 ulps of max(|want|, floor)."""
    scale = np.maximum(np.abs(want.astype(np.float64)), floor)
    return np.abs(got.astype(np.float64) - want.astype(np.float64)) / np.spacing(scale.astype(np.float32)).astype(np.float64)


def assert_mcar_close(got_state, o_st, prev, where, tol=2.0):
    """position and velocity within ``tol`` fp32 ulps of the largest magnitude their step adds: the previous value,
    max_speed (0.07) for the position and the gravity term (0.0025) for the velocity."""
    f = fields(MCAR, got_state)
    for k, floor in (("position", 0.07), ("velocity", 0.0025)):
        u = ulps(f[k], o_st[k], np.maximum(np.abs(prev[k]), floor))
        assert u.max() <= tol, (where, k, float(u.max()))
    assert np.array_equal(f["time"], o_st["time"]), where
    return float(ulps(f["velocity"], o_st["velocity"], np.maximum(np.abs(prev["velocity"]), 0.0025)).max())


def random_actions(ka, n):
    return jr.randint(jr.split(ka, n), (), 0, 3)


# --------------------------------------------------------------------------- #
# pqn_env_info and the env registry
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name,env_id,obs_dim,obs_shape,actions,max_steps,words",
                         [(MCAR, 18, 2, (2,), 3, 200, 8), (CATCH, 33, 50, (10, 5), 3, 1000, 7)])
def test_env_info(name, env_id, obs_dim, obs_shape, actions, max_steps, words):
    """pqn_env_info's table; the observation space is gymnax's shape, (50,) for Catch once flattened."""
    from purejaxql_b200 import _lib
    info = _lib.EnvInfo()
    _lib.check(_lib.lib().pqn_env_info(env_id, info), "pqn_env_info")
    assert (info.obs_dim, info.num_actions, info.max_steps, info.binary_obs) == (obs_dim, actions, max_steps, 0)
    assert (info.state_words, tuple(info.obs_shape), info.packed_obs_words) == (words, (obs_shape + (1, 1))[:3], 0)
    assert E.make(name)[0].observation_space().shape == obs_shape
    env, params = E.make(name, flatten_obs=True)
    assert E.ENV_IDS[name] == env_id and env.env_id == env_id
    assert env.observation_space().shape == (obs_dim,) and env.action_space().n == actions
    assert params.max_steps_in_episode == max_steps and not env.binary_obs


def test_unknown_env_lists_new_names():
    with pytest.raises(KeyError) as e:
        E.make("Pendulum-v1")
    assert MCAR in str(e.value) and CATCH in str(e.value)


# --------------------------------------------------------------------------- #
# host-compiled device logic against the oracles
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("part", [0, 1])
def test_catch_host_logic_matches_oracle_bit_exact(hlib, part):
    """reset + five episodes of random actions (auto-resets included) for a ragged N: obs, reward (sign of zero
    included), done, every state field and the LogWrapper fields equal the oracle bit for bit; pqn_env_obs's obs
    equals the one the step returned."""
    n = 97
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env = X.make(CATCH)
        h = HostEnv(hlib, CATCH, part)
        key, kr = jr.split(jr.PRNGKey(21), 2)
        rk = jr.split(kr, n)
        o_obs, o_st = env.reset(rk)
        h_obs, h_st = h.reset(rk)
        assert np.array_equal(bits(h_obs), bits(o_obs)) and np.array_equal(h.obs(h_st), o_obs)
        assert np.array_equal(to_state(CATCH, o_st), h_st)
        assert set(o_st["ball_x"]) == set(range(5))
        for t in range(5 * 9 + 4):
            key, ka, ks = jr.split(key, 3)
            act = random_actions(ka, n)
            sk = jr.split(ks, n)
            o_obs, o_st, o_r, o_d, _ = env.step(sk, o_st, act)
            h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
            assert np.array_equal(h_d, o_d), t
            assert np.array_equal(bits(h_r), bits(o_r)), t
            assert np.array_equal(bits(h_obs), bits(o_obs)), t
            assert np.array_equal(bits(h.obs(h_st)), bits(o_obs)), t
            assert np.array_equal(to_state(CATCH, o_st), h_st), t
        assert (o_st["log_returned_episode_lengths"] == 9).all()
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("part", [0, 1])
def test_mountain_car_host_logic_teacher_forced(hlib, part):
    """The reset is bit-exact.  Then 230 steps of random actions (every episode truncates at 200), each started from
    the oracle's state: position and velocity within 2 ulps, reward, done, time and the LogWrapper fields exact, and
    the obs equals [position, velocity] of the state."""
    n = 97
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env = X.make(MCAR)
        h = HostEnv(hlib, MCAR, part)
        key, kr = jr.split(jr.PRNGKey(5), 2)
        rk = jr.split(kr, n)
        o_obs, o_st = env.reset(rk)
        h_obs, h_st = h.reset(rk)
        assert np.array_equal(bits(h_obs), bits(o_obs))
        assert np.array_equal(to_state(MCAR, o_st), h_st)
        worst = 0.0
        for t in range(230):
            key, ka, ks = jr.split(key, 3)
            act = random_actions(ka, n)
            sk = jr.split(ks, n)
            h_st, prev = to_state(MCAR, o_st), o_st
            o_obs, o_st, o_r, o_d, o_info = env.step(sk, o_st, act)
            h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
            assert np.array_equal(h_d, o_d), t
            assert np.array_equal(h_r, o_r), t
            worst = max(worst, assert_mcar_close(h_st, o_st, prev, t))
            f = fields(MCAR, h_st)
            assert np.array_equal(h_obs, np.stack([f["position"], f["velocity"]], 1)), t
            assert np.array_equal(h.obs(h_st), h_obs), t
            for k in ("log_episode_lengths", "log_returned_episode_lengths", "log_timestep", "log_episode_returns",
                      "log_returned_episode_returns"):
                assert np.array_equal(f[k], o_st[k]), (t, k)
            if t == 199:
                assert o_d.all() and (o_info["returned_episode_lengths"] == 200).all()
        print(f"MountainCar host vs oracle: worst velocity error {worst:.2f} ulps")
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def test_mountain_car_host_wall_and_goal(hlib):
    """Hand-set states: at the left wall with negative velocity the velocity comes back 0 and the position clamped to
    -1.2; a car just below the goal with positive velocity crosses it (done, reward -1, auto-reset); the same car
    with negative velocity at the goal is not done."""
    n = 4
    st = dict(position=np.array([-1.199, -1.2, 0.4995, 0.5], np.float32),
              velocity=np.array([-0.05, -0.01, 0.02, -0.001], np.float32), time=np.array([3, 7, 50, 8], np.int32))
    for k in X.G.LogWrapper.LOG:
        st[k] = np.zeros(n, np.float32 if "returns" in k else np.int32)
    core = X.MountainCar()
    act = np.array([0, 1, 2, 1], np.int32)
    keys = jr.split(jr.PRNGKey(0), n)
    o_obs, o_st, o_r, o_d, _ = core.step_env(jr.split(keys, 2)[:, 0], st, act)
    assert np.array_equal(o_st["position"][:2], np.full(2, -1.2, np.float32))
    assert (o_st["velocity"][:2] == 0).all() and np.signbit(o_st["velocity"][:2]).all()     # -0.0, as gymnax gives
    assert np.array_equal(o_d, [False, False, True, False]) and (o_r == -1).all()
    h = HostEnv(hlib, MCAR, 0)
    h_obs, h_st, h_r, h_d = h.step(keys, to_state(MCAR, st), act)
    assert np.array_equal(h_d, o_d) and (h_r == -1).all()
    f = fields(MCAR, h_st)
    assert np.array_equal(bits(f["velocity"][:2]), bits(o_st["velocity"][:2]))
    assert np.array_equal(f["position"][:2], o_st["position"][:2])
    assert f["time"][2] == 0 and -0.6 <= f["position"][2] <= -0.4 and f["velocity"][2] == 0    # auto-reset
    assert f["log_returned_episode_lengths"][2] == 1 and f["log_returned_episode_returns"][2] == -1


# --------------------------------------------------------------------------- #
# the oracles' episodes
# --------------------------------------------------------------------------- #
def test_catch_oracle_episodes():
    """Every episode lasts 9 steps, only its last step is rewarded, with +1 exactly when the paddle ends under the
    ball; the board shows the ball and the paddle (a single 1 once the ball is caught)."""
    n = 200
    env = X.make(CATCH)
    key, kr = jr.split(jr.PRNGKey(3), 2)
    obs, st = env.reset(jr.split(kr, n))
    assert (obs.sum(1) == 2).all() and (obs.reshape(n, 10, 5)[:, 9, 2] == 1).all()
    seen = {1.0: 0, -1.0: 0}
    for t in range(4 * 9):
        key, ka, ks = jr.split(key, 3)
        act = random_actions(ka, n)
        before = {k: v.copy() for k, v in st.items()}
        obs, st, r, d, info = env.step(jr.split(ks, n), st, act)
        assert np.array_equal(d, np.full(n, t % 9 == 8)), t
        assert (r[~d] == 0).all()
        px = np.clip(before["paddle_x"] + act - 1, 0, 4)
        assert np.array_equal(r[d], np.where(px[d] == before["ball_x"][d], 1.0, -1.0).astype(np.float32))
        for v in r[d]:
            seen[float(v)] += 1
        if not d.any():
            board = obs.reshape(n, 10, 5)
            idx = np.arange(n)
            assert (board[idx, st["ball_y"], st["ball_x"]] == 1).all() and (obs.sum(1) == 2).all()
        assert (info["returned_episode_lengths"][d] == 9).all()
    assert seen[1.0] > 0 and seen[-1.0] > 0
    core = X.Catch()
    s = dict(ball_x=np.array([2]), ball_y=np.array([9]), paddle_x=np.array([2]), paddle_y=np.array([9]))
    assert core.get_obs(s).sum() == 1


def test_mountain_car_oracle_episodes():
    """Random actions truncate at 200 steps; pushing along the velocity reaches the goal in fewer than 200 steps."""
    n = 64
    env = X.make(MCAR)
    key, kr = jr.split(jr.PRNGKey(8), 2)
    _, st = env.reset(jr.split(kr, n))
    for t in range(200):
        key, ka, ks = jr.split(key, 3)
        _, st, r, d, info = env.step(jr.split(ks, n), st, random_actions(ka, n))
        assert (r == -1).all()
        assert np.array_equal(d, np.full(n, t == 199)), t
    assert (info["returned_episode_lengths"] == 200).all() and (info["returned_episode_returns"] == -200).all()
    _, st = env.reset(jr.split(kr, n))
    done_at = np.zeros(n, np.int64)
    for t in range(200):
        act = np.where(st["velocity"] >= 0, 2, 0).astype(np.int32)
        key, ks = jr.split(key, 2)
        _, st, r, d, info = env.step(jr.split(ks, n), st, act)
        done_at = np.where(d & (done_at == 0), t + 1, done_at)
    assert (done_at > 0).all() and (done_at < 200).all(), done_at
    print(f"push-along-velocity episodes: {done_at.min()}-{done_at.max()} steps")


def test_mountain_car_oracle_left_wall():
    core = X.MountainCar()
    s = dict(position=np.array([-1.19, -1.2], np.float32), velocity=np.array([-0.07, -0.01], np.float32),
             time=np.zeros(2, np.int32))
    _, ns, _, d, _ = core.step_env(None, s, np.zeros(2, np.int32))
    assert (ns["position"] == np.float32(-1.2)).all() and (ns["velocity"] == 0).all() and not d.any()


# --------------------------------------------------------------------------- #
# fields, scripts, workspaces
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name", [MCAR, CATCH])
def test_fields_round_trip(name):
    env = X.make(name)
    key = jr.PRNGKey(11)
    _, st = env.reset(jr.split(key, 50))
    for t in range(6):
        key, ka, ks = jr.split(key, 3)
        _, st, _, _, _ = env.step(jr.split(ks, 50), st, random_actions(ka, 50))
    f = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in st.items()}
    state = E.fields_to_state(name, f)
    assert state.shape == ({MCAR: 8, CATCH: 7}[name], 50)
    back = E.state_to_fields(name, state)
    assert set(back) == set(f)
    for k, v in f.items():
        assert np.array_equal(back[k].numpy().astype(v.numpy().dtype).reshape(v.shape), v.numpy()), k
    assert torch.equal(E.fields_to_state(name, back), state)
    if name == CATCH:   # prev_done is a field of the word even though a stored state never has it set
        f["prev_done"] = torch.ones(50, dtype=torch.bool)
        assert E.state_to_fields(name, E.fields_to_state(name, f))["prev_done"].all()


@pytest.mark.parametrize("script", ["pqn_gymnax", "pqn_rnn_gymnax"])
@pytest.mark.parametrize("name,test_steps", [(MCAR, 200), (CATCH, 1000)])
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



# pqn_net_workspace_bytes(desc, S=2, rows=1000) of the GRU at the widths built before MountainCar and Catch, per
# (in_c, NORM_TYPE, NORM_INPUT), over HIDDEN_SIZE 64, 128, 256, 512 x NUM_LAYERS 1, 2, 4
RNN_WORKSPACE = {
    (3, 'layer_norm', False): [51256320, 51256320, 53320704, 66663424, 66663424, 70775808,
        98200064, 98200064, 106408448, 163764736, 163764736, 180165120],
    (3, 'layer_norm', True): [51364864, 51368960, 53441536, 66771968, 66776064, 70896640,
        98308608, 98312704, 106529280, 163885568, 163893760, 180310528],
    (3, 'batch_norm', False): [51364864, 51368960, 53441536, 66771968, 66776064, 70896640,
        98308608, 98312704, 106529280, 163885568, 163893760, 180310528],
    (3, 'batch_norm', True): [51364864, 51368960, 53441536, 66771968, 66776064, 70896640,
        98308608, 98312704, 106529280, 163885568, 163893760, 180310528],
    (3, 'none', False): [51364864, 51368960, 53441536, 66771968, 66776064, 70896640,
        98308608, 98312704, 106529280, 163885568, 163893760, 180310528],
    (3, 'none', True): [51364864, 51368960, 53441536, 66771968, 66776064, 70896640,
        98308608, 98312704, 106529280, 163885568, 163893760, 180310528],
    (4, 'layer_norm', False): [51256320, 51256320, 53320704, 66663424, 66663424, 70775808,
        98200064, 98200064, 106408448, 163764736, 163764736, 180165120],
    (4, 'layer_norm', True): [51396608, 51400704, 53473280, 66803712, 66807808, 70928384,
        98340352, 98344448, 106561024, 163917312, 163925504, 180342272],
    (4, 'batch_norm', False): [51396608, 51400704, 53473280, 66803712, 66807808, 70928384,
        98340352, 98344448, 106561024, 163917312, 163925504, 180342272],
    (4, 'batch_norm', True): [51396608, 51400704, 53473280, 66803712, 66807808, 70928384,
        98340352, 98344448, 106561024, 163917312, 163925504, 180342272],
    (4, 'none', False): [51396608, 51400704, 53473280, 66803712, 66807808, 70928384,
        98340352, 98344448, 106561024, 163917312, 163925504, 180342272],
    (4, 'none', True): [51396608, 51400704, 53473280, 66803712, 66807808, 70928384,
        98340352, 98344448, 106561024, 163917312, 163925504, 180342272],
    (6, 'layer_norm', False): [51256320, 51256320, 53320704, 66663424, 66663424, 70775808,
        98200064, 98200064, 106408448, 163764736, 163764736, 180165120],
    (6, 'layer_norm', True): [51461120, 51465216, 53537792, 66868224, 66872320, 70992896,
        98404864, 98408960, 106625536, 163981824, 163990016, 180406784],
    (6, 'batch_norm', False): [51461120, 51465216, 53537792, 66868224, 66872320, 70992896,
        98404864, 98408960, 106625536, 163981824, 163990016, 180406784],
    (6, 'batch_norm', True): [51461120, 51465216, 53537792, 66868224, 66872320, 70992896,
        98404864, 98408960, 106625536, 163981824, 163990016, 180406784],
    (6, 'none', False): [51461120, 51465216, 53537792, 66868224, 66872320, 70992896,
        98404864, 98408960, 106625536, 163981824, 163990016, 180406784],
    (6, 'none', True): [51461120, 51465216, 53537792, 66868224, 66872320, 70992896,
        98404864, 98408960, 106625536, 163981824, 163990016, 180406784],
}
# sha256 of the JSON of every row of the same grid for the GRU, the MLP (in_c 3, 4, 6), the packed-bits MLP
# (in_c 400, 600, 700; 6 actions) and the CNN (C 4, 6, 7, 10; 6 actions), keyed "kind,in_c,NORM_TYPE,NORM_INPUT"
ALL_WORKSPACE_SHA256 = "71d449c37019249e757e81252a113a0725f6bc5ccd041d9955c650b9d03c96e6"


def _workspace_grid():
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_CNN, NET_MLP, NET_MLP_BITS, NET_RNN, QNetworkSpec
    lib = _lib.lib()
    grid = {}
    norms = [(nt, ni) for nt in ("layer_norm", "batch_norm", "none") for ni in (False, True)]
    for kind, ds, A in ((NET_RNN, (3, 4, 6), 3), (NET_MLP, (3, 4, 6), 3), (NET_MLP_BITS, (400, 600, 700), 6)):
        for D in ds:
            for nt, ni in norms:
                grid[f"{kind},{D},{nt},{int(ni)}"] = [
                    int(lib.pqn_net_workspace_bytes(QNetworkSpec(kind, D, A, H, layers, norm_type=nt, norm_input=ni).desc,
                                                    2, 1000))
                    for H in (64, 128, 256, 512) for layers in (1, 2, 4)]
    for C in (4, 6, 7, 10):
        for nt in ("layer_norm", "batch_norm", "none"):
            grid[f"{NET_CNN},{C},{nt},0"] = [int(lib.pqn_net_workspace_bytes(QNetworkSpec(NET_CNN, C, 6, norm_type=nt).desc,
                                                                             2, 1000))]
    return grid


def test_workspace_of_existing_shapes_unchanged():
    """The GRU's per-channel tables now grow with the input width beyond 256; every shape built before keeps its
    workspace size to the byte."""
    import hashlib
    import json
    grid = _workspace_grid()
    for (D, nt, ni), want in RNN_WORKSPACE.items():
        assert grid[f"2,{D},{nt},{int(ni)}"] == want, (D, nt, ni)
    assert hashlib.sha256(json.dumps(grid, sort_keys=True).encode()).hexdigest() == ALL_WORKSPACE_SHA256


def test_rnn_workspace_grows_with_wide_inputs():
    """From D = 257 the GRU's per-channel tables hold 2 x D floats per seed, and its reduction partials 64 of those:
    going from D = 256 to 1024 adds at least those tables on top of the four row buffers of D floats per row."""
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_RNN, QNetworkSpec
    S, rows = 2, 1000
    ws = lambda D: int(_lib.lib().pqn_net_workspace_bytes(
        QNetworkSpec(NET_RNN, D, 3, 64, 2, norm_type="batch_norm", norm_input=True).desc, S, rows))
    row_buffers = 4 * S * rows * (1024 - 256) * 4
    partials = S * 64 * 2 * (1024 - 256) * 4
    assert ws(1024) - ws(256) >= row_buffers + partials


_REF = sorted(glob.glob(os.path.join(HERE, "golden", "gymnax_extra_*_ref.npz")))
_PARAMS = {MCAR: dict(min_position=-1.2, max_position=0.6, max_speed=0.07, goal_position=0.5, goal_velocity=0.0,
                      force=0.001, gravity=0.0025, max_steps_in_episode=200),
           CATCH: dict(max_steps_in_episode=1000)}


@pytest.mark.skipif(not _REF, reason="no MountainCar / Catch trajectories recorded from gymnax yet "
                                     "(tests/golden/make_gymnax_extra_golden_from_ref.py)")
@pytest.mark.parametrize("path", _REF or ["none"])
def test_against_reference(path, hlib):
    """Replays a trajectory recorded from gymnax through the oracle and the host-compiled device logic (MountainCar
    teacher-forced), and checks gymnax's default EnvParams."""
    g = dict(np.load(path))
    base = os.path.basename(path)
    name = MCAR if "mountain_car" in base else CATCH
    part = "partitionable" in base
    for k, v in _PARAMS[name].items():
        assert np.float32(g[f"param_{k}"]) == np.float32(v), k
    jr.DEFAULT_PARTITIONABLE = part
    try:
        env = X.make(name)
        h = HostEnv(hlib, name, int(part))
        o_obs, o_st = env.reset(g["reset_keys"])
        h_obs, h_st = h.reset(g["reset_keys"])
        assert np.array_equal(o_obs, g["obs0"]) and np.array_equal(h_obs, g["obs0"])
        for t in range(g["action"].shape[0]):
            sk, act = g["step_keys"][t], g["action"][t].astype(np.int32)
            prev = o_st
            if name == MCAR:
                h_st = to_state(MCAR, o_st)
            o_obs, o_st, o_r, o_d, o_info = env.step(sk, o_st, act)
            h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
            assert np.array_equal(o_d, g["done"][t]) and np.array_equal(h_d, g["done"][t]), t
            assert np.array_equal(o_r, g["reward"][t].astype(np.float32)), t
            assert np.array_equal(h_r, g["reward"][t].astype(np.float32)), t
            assert np.array_equal(o_info["returned_episode_lengths"], g["len"][t]), t
            if name == CATCH:
                assert np.array_equal(o_obs, g["obs"][t]) and np.array_equal(h_obs, g["obs"][t]), t
                for k in X.Catch.state_fields:
                    assert np.array_equal(o_st[k], g[k][t].astype(o_st[k].dtype)), (k, t)
                assert np.array_equal(to_state(CATCH, o_st), h_st), t
            else:
                want = {"position": g["position"][t].astype(np.float32), "velocity": g["velocity"][t].astype(np.float32),
                        "time": g["time"][t].astype(np.int32)}
                assert_mcar_close(h_st, want, prev, t)
                o_st = dict(o_st, **want)          # teacher-force the oracle with gymnax's state
    finally:
        jr.DEFAULT_PARTITIONABLE = False
