"""jax.random.normal and GaussianBandit-misc without a GPU: the device logic of csrc/threefry.cuh and csrc/env_misc.cuh
compiled for the host (tests/host_harness_gaussian_bandit.cpp) against the NumPy oracles (tests/jax_normal_oracle.py,
tests/gaussian_bandit_oracle.py), the normal against scipy's fp64 erfinv, self-checks of the oracle's episodes, the
state-field conversion of purejaxql_b200/envs.py, ``pqn_env_info`` and make_train of both scripts.

The normal has 2^23 possible values, one per value of bits >> 9, and the tests below cover all of them.  The host
build calls the C library's log1pf where the device calls libdevice's; everything else is exact fp32 arithmetic, so
the tests that check bits hand the oracle the log1p of the build under test."""
import ctypes
import glob
import os
import subprocess

import numpy as np
import pytest
import torch

import gaussian_bandit_oracle as GB
import jax_normal_oracle as JN
from oracle import jax_prng as jr
from purejaxql_b200 import envs as E

HERE = os.path.dirname(os.path.abspath(__file__))
NAME = "GaussianBandit-misc"
F32 = np.float32


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def hlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("harness") / "host_harness_gaussian_bandit.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(HERE, "host_harness_gaussian_bandit.cpp"), "-o", so])
    return ctypes.CDLL(so)


def host_call(lib, fn, *arrays):
    """fn(in..., out, n) over float32 / uint32 arrays of one length."""
    n = arrays[0].shape[0]
    ins = [np.ascontiguousarray(a) for a in arrays]
    out = np.empty(n, F32)
    getattr(lib, fn)(*[ptr(a) for a in ins], ptr(out), ctypes.c_int64(n))
    return out


def host_log1p(lib):
    return lambda x: host_call(lib, "h_log1pf", np.asarray(x, F32))


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.int32)


@pytest.fixture(scope="module")
def exhaustive(hlib):
    """The 2^23 inputs, their uniforms, the host build's normals and w, and the oracle's w."""
    b = JN.all_bits()
    u = JN.uniform_from_bits(b)
    return dict(bits=b, u=u, host=host_call(hlib, "h_normal_from_bits", b),
                w_host=JN.erf_inv_w(u, host_log1p(hlib)), w_oracle=JN.erf_inv_w(u))


# --------------------------------------------------------------------------- #
# jax.random.normal
# --------------------------------------------------------------------------- #
def test_uniform_is_exact_and_covers_both_branches(exhaustive):
    """u = 2 f - (1 - 2^-24) exactly, for f = k * 2^-23: strictly inside (-1, 1), never 0, symmetric under
    k -> 2^23 - 1 - k up to the 2^-23 offset; the lower clamp is not active; both branches of erf_inv occur."""
    u, k = exhaustive["u"], np.arange(1 << 23, dtype=np.float64)
    assert np.array_equal(u.astype(np.float64), 2 * k * 2.0 ** -23 - (1 - 2.0 ** -24))
    assert u[0] == JN.LO and u.min() == JN.LO and u.max() == F32(1 - 2.0 ** -22 + 2.0 ** -24)
    assert (u != 0).all() and (np.abs(u) < 1).all()
    w = exhaustive["w_oracle"]
    assert (w < 5).sum() > 0 and (w >= 5).sum() > 0
    assert np.abs(u[w >= 5]).min() > F32(0.996)


def test_host_normal_matches_oracle_bit_exact_given_log1p(hlib, exhaustive):
    """With the same w, the C++ polynomial (fmaf Horner steps, sqrt, the final products) equals the NumPy restatement
    bit for bit at all 2^23 inputs; so does the whole host normal_from_bits against the oracle on the host's log1pf."""
    u, w = exhaustive["u"], exhaustive["w_host"]
    assert np.array_equal(bits(host_call(hlib, "h_erf_inv_from_w", u, w)), bits(JN.erf_inv_from_w(u, w)))
    want = (JN.SQRT2 * JN.erf_inv_from_w(u, w)).astype(F32)
    assert np.array_equal(bits(exhaustive["host"]), bits(want))


def test_host_normal_against_default_oracle(exhaustive):
    """Against the oracle's own log1p (fp64 log1p rounded to fp32): the host normal differs only where the C library's
    log1pf gives another w, that w is 1 ulp away, and the normal is then at most NORMAL_ULP_BOUND ulps away.  The
    differing values stay a small fraction of the 2^23."""
    h, o = exhaustive["host"], JN.normal_from_bits(exhaustive["bits"])
    dw = JN.ulp_distance(exhaustive["w_host"], exhaustive["w_oracle"])
    assert dw.max() <= 1
    differ = bits(h) != bits(o)
    assert not (differ & (dw == 0)).any()
    assert JN.ulp_distance(h, o).max() <= JN.NORMAL_ULP_BOUND
    assert differ.sum() < 0.02 * (1 << 23), differ.sum()


def test_normal_ulp_bound_of_a_one_ulp_log1p(exhaustive):
    """NORMAL_ULP_BOUND: moving w by one ulp either way moves the normal by at most 3 ulps, at every input; and 3 is
    reached."""
    u, w = exhaustive["u"], exhaustive["w_oracle"]
    base = (JN.SQRT2 * JN.erf_inv_from_w(u, w)).astype(F32)
    worst = 0
    for d in (np.inf, -np.inf):
        r = (JN.SQRT2 * JN.erf_inv_from_w(u, np.nextafter(w, F32(d)).astype(F32))).astype(F32)
        worst = max(worst, int(JN.ulp_distance(base, r).max()))
    assert worst == JN.NORMAL_ULP_BOUND == 3


def test_normal_against_scipy_erfinv(exhaustive):
    """Against sqrt(2) * erfinv(u) in fp64 at all 2^23 inputs.  Giles' approximation itself, evaluated in fp64 on
    the exact w, is within 1.3e-7 relative (his single-precision target).  In fp32 the normal is within 4e-7 relative
    (4 ulps) for |u| < 0.99.  Closer to +-1 the rounding of u * u to fp32 costs 1 - u^2 its low bits before log1p sees
    it, as in jax's fp32 formula, and the error grows to 6e-6 relative (about 91 ulps at |u| = 0.99983)."""
    from scipy.special import erfinv
    u = exhaustive["u"]
    u64 = u.astype(np.float64)
    exact = np.sqrt(2.0) * erfinv(u64)
    w = -np.log1p(-u64 * u64)
    lt = w < 5
    t = np.where(lt, w - 2.5, np.sqrt(w) - 3)
    p = np.where(lt, JN.CENTRAL[0], JN.TAIL[0]).astype(np.float64)
    for i in range(1, 9):
        p = p * t + np.where(lt, JN.CENTRAL[i], JN.TAIL[i]).astype(np.float64)
    assert (np.abs(np.sqrt(2.0) * p * u64 - exact) / np.abs(exact)).max() < 1.3e-7
    h = exhaustive["host"].astype(np.float64)
    rel = np.abs(h - exact) / np.abs(exact)
    inner = np.abs(u) < 0.99
    assert rel[inner].max() < 4e-7 and JN.ulp_distance(exhaustive["host"][inner], exact[inner].astype(F32)).max() <= 4
    assert rel.max() < 6e-6, rel.max()
    assert np.array_equal(np.sign(h), np.sign(u))
    assert abs(h.mean()) < 1e-6 and abs(h.std() - 1) < 1e-3


def test_contraction_changes_bits():
    """(J4) matters: without fma contraction (jax on the CPU) the Horner steps round differently at some inputs, by
    at most 3 ulps."""
    b = JN.all_bits()[::7]
    fused, plain = JN.normal_from_bits(b), JN.normal_from_bits(b, fma=False)
    differ = bits(fused) != bits(plain)
    assert differ.any() and JN.ulp_distance(fused, plain).max() <= 3


def test_fma32_is_correctly_rounded():
    """The oracle's fp32 fma against exact rational arithmetic: random operands, sums with heavy cancellation and
    exact ties of the fp32 rounding (round half to even)."""
    from fractions import Fraction
    rng = np.random.default_rng(0)
    n = 3000
    a, b, c = (rng.standard_normal(n).astype(F32) for _ in range(3))
    c[1::3] = (-(a[1::3].astype(np.float64) * b[1::3])).astype(F32)               # heavy cancellation
    a[2::3], b[2::3] = F32(1 + 2.0 ** -12), F32(1 + 2.0 ** -12)                     # a * b = 1 + 2^-11 + 2^-24
    c[2::3] = F32(0)
    got = JN.fma32(a, b, c)
    for i in range(n):
        want = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        g = got[i]
        err = abs(Fraction(float(g)) - want)
        for nb in (np.nextafter(g, F32(-np.inf)), np.nextafter(g, F32(np.inf))):
            e2 = abs(Fraction(float(nb)) - want)
            assert err < e2 or (err == e2 and (int(np.asarray(g).view(np.int32)) & 1) == 0), i
    assert got[2] == F32(1 + 2.0 ** -11)                                           # the tie, rounded to even


@pytest.mark.parametrize("part", [0, 1])
def test_normal_scalar_matches_oracle_at_keys(hlib, part):
    """normal(key, ()) of 4099 split keys, bit for bit against the oracle on the host's log1pf, in both layouts; the
    oracle's normal(key, (n,)) uses random_bits(key, (n,))."""
    keys = jr.split(jr.PRNGKey(31 + part), 4099, bool(part))
    out = np.empty(4099, F32)
    hlib.h_normal_scalar(ptr(np.ascontiguousarray(keys)), ptr(out), ctypes.c_int64(4099), part)
    want = JN.normal(keys, (), bool(part), log1p=host_log1p(hlib))
    assert np.array_equal(bits(out), bits(want))
    vec = JN.normal(keys[0], (6,), bool(part))
    assert np.array_equal(bits(vec), bits(JN.normal_from_bits(jr.random_bits(keys[0], (6,), bool(part)))))


# --------------------------------------------------------------------------- #
# the env: pqn_env_info, host logic against the oracle
# --------------------------------------------------------------------------- #
def test_env_info(hlib):
    from purejaxql_b200 import _lib
    info = _lib.EnvInfo()
    _lib.check(_lib.lib().pqn_env_info(51, info), "pqn_env_info")
    assert (info.obs_dim, info.num_actions, info.max_steps, info.binary_obs) == (4, 2, 100, 0)
    assert (info.state_words, tuple(info.obs_shape), info.packed_obs_words) == (12, (4, 1, 1), 0)
    assert E.ENV_IDS[NAME] == 51
    env, params = E.make(NAME)
    assert env.env_id == 51 and env.observation_space().shape == (4,) == GB.GaussianBandit.obs_shape
    assert env.action_space().n == 2 and params.max_steps_in_episode == 100 and not env.binary_obs
    assert hlib.h_gaussian_bandit_state_words() == info.state_words
    assert hlib.h_gaussian_bandit_obs_dim() == info.obs_dim and hlib.h_gaussian_bandit_max_steps() == 100


class HostEnv:
    """Drives the harness like pqn_env_reset / pqn_env_step / pqn_env_obs."""

    def __init__(self, lib, part):
        self.lib, self.part = lib, part

    def reset(self, keys):
        n = keys.shape[0]
        state, obs = np.zeros((12, n), np.uint32), np.zeros((n, 4), F32)
        self.lib.h_gaussian_bandit_reset(ptr(np.ascontiguousarray(keys, np.uint32)), ptr(state), ptr(obs),
                                         ctypes.c_int64(n), 100, self.part)
        return obs, state

    def step(self, keys, state, action):
        n = keys.shape[0]
        obs, reward, done = np.zeros((n, 4), F32), np.zeros(n, F32), np.zeros(n, np.uint8)
        self.lib.h_gaussian_bandit_step(ptr(np.ascontiguousarray(keys, np.uint32)), ptr(state),
                                        ptr(np.ascontiguousarray(action, np.int32)), ptr(obs), ptr(reward), ptr(done),
                                        ctypes.c_int64(n), 100, self.part)
        return obs, state, reward, done.astype(bool)

    def obs(self, state):
        n = state.shape[1]
        obs = np.zeros((n, 4), F32)
        self.lib.h_gaussian_bandit_obs(ptr(np.ascontiguousarray(state)), ptr(obs), ctypes.c_int64(n))
        return obs


def to_state(st):
    return E.fields_to_state(NAME, {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in st.items()}).numpy().view(
        np.uint32).copy()


def fields(state):
    return {k: v.numpy() for k, v in E.state_to_fields(NAME, torch.from_numpy(state.view(np.int32))).items()}


@pytest.mark.parametrize("part", [0, 1])
def test_host_logic_matches_oracle_bit_exact(hlib, part):
    """reset + 3 episodes and 3 steps of random actions (auto-resets included) at N = 97: obs, reward, done, every state
    field and the LogWrapper fields equal the oracle on the host's log1pf bit for bit; pqn_env_obs's obs equals the
    step's.  Against the oracle's own log1p, rewards and mu2 stay within the normal's ulp bound."""
    n = 97
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env = GB.make(log1p=host_log1p(hlib))
        ref = GB.make()
        h = HostEnv(hlib, part)
        key, kr = jr.split(jr.PRNGKey(70 + part), 2)
        rk = jr.split(kr, n)
        o_obs, o_st = env.reset(rk)
        _, r_st = ref.reset(rk)
        h_obs, h_st = h.reset(rk)
        assert np.array_equal(bits(h_obs), bits(o_obs)) and np.array_equal(bits(h.obs(h_st)), bits(o_obs))
        assert np.array_equal(to_state(o_st), h_st)
        assert JN.ulp_distance(r_st["mu2"], o_st["mu2"]).max() <= JN.NORMAL_ULP_BOUND
        dones, pulls = 0, 0
        for t in range(3 * 100 + 3):
            key, ka, ks = jr.split(key, 3)
            act = jr.randint(jr.split(ka, n), (), 0, 2)
            sk = jr.split(ks, n)
            o_obs, o_st, o_r, o_d, _ = env.step(sk, o_st, act)
            h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
            assert np.array_equal(h_d, o_d), t
            assert np.array_equal(bits(h_r), bits(o_r)), t
            assert np.array_equal(bits(h_obs), bits(o_obs)), t
            assert np.array_equal(bits(h.obs(h_st)), bits(o_obs)), t
            assert np.array_equal(to_state(o_st), h_st), t
            assert (o_r[act == 0] == 0).all()
            dones += int(o_d.sum())
            pulls += int((act == 1).sum())
        assert dones == 3 * n and (o_st["log_returned_episode_lengths"] == 100).all()
        assert pulls > 100 * n
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def test_reset_and_pull_draws(hlib):
    """mu2 is normal(reset key) and exp_reward_best = max(0, mu2); a pull of arm 1 pays mu2 + normal(step key), one
    of arm 0 pays mu1 = 0."""
    n = 64
    rk = jr.split(jr.PRNGKey(3), n)
    f = fields(HostEnv(hlib, 0).reset(rk)[1])
    lp = host_log1p(hlib)
    assert np.array_equal(bits(f["mu2"]), bits(JN.normal(rk, (), log1p=lp)))
    assert np.array_equal(f["exp_reward_best"], np.maximum(F32(0), f["mu2"]))
    assert (f["mu1"] == 0).all() and (f["sigma_l"] == 1).all() and (f["time"] == 0).all()
    core = GB.GaussianBandit(log1p=lp)
    _, s = core.reset_env(rk)
    sk = jr.split(jr.PRNGKey(4), n)
    _, s2, r, d, _ = core.step_env(sk, s, np.ones(n, np.int32))
    assert np.array_equal(bits(r), bits((s["mu2"] + JN.normal(sk, (), log1p=lp)).astype(F32)))
    assert np.array_equal(s2["last_reward"], r) and (s2["last_action"] == 1).all() and not d.any()
    _, _, r0, _, _ = core.step_env(sk, s, np.zeros(n, np.int32))
    assert (r0 == 0).all()


def test_oracle_episodes():
    """Pulling arm 1 for a whole episode: the rewards scatter around each env's mu2 with unit spread, the observation
    shows the one-hot arm, the last reward and 2 t / 100 - 1, and every episode lasts 100 steps."""
    n = 512
    env = GB.make()
    key, kr = jr.split(jr.PRNGKey(9), 2)
    obs, st = env.reset(jr.split(kr, n))
    assert np.array_equal(obs[0], np.array([1, 0, 0, -1], F32))
    mu2 = st["mu2"].copy()
    assert abs(mu2.mean()) < 0.15 and abs(mu2.std() - 1) < 0.1
    rs = []
    for t in range(100):
        key, ks = jr.split(key, 2)
        obs, st, r, d, info = env.step(jr.split(ks, n), st, np.ones(n, np.int32))
        rs.append(r)
        assert np.array_equal(d, np.full(n, t == 99)), t
        if t < 99:
            assert (obs[:, 1] == 1).all() and np.array_equal(obs[:, 2], r)
            assert (obs[:, 3] == F32(F32(2 * (t + 1)) / F32(100)) - F32(1)).all()
    noise = np.stack(rs) - mu2[None]
    assert abs(noise.mean()) < 0.02 and abs(noise.std() - 1) < 0.02
    assert (info["returned_episode_lengths"] == 100).all()


def test_fields_round_trip():
    env = GB.make()
    key = jr.PRNGKey(11)
    _, st = env.reset(jr.split(key, 50))
    for t in range(6):
        key, ka, ks = jr.split(key, 3)
        _, st, _, _, _ = env.step(jr.split(ks, 50), st, jr.randint(jr.split(ka, 50), (), 0, 2))
    f = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in st.items()}
    state = E.fields_to_state(NAME, f)
    assert state.shape == (12, 50)
    back = E.state_to_fields(NAME, state)
    assert set(back) == set(f)
    for k, v in f.items():
        assert np.array_equal(back[k].numpy().astype(v.numpy().dtype).reshape(v.shape), v.numpy()), k
    assert torch.equal(E.fields_to_state(NAME, back), state)


@pytest.mark.parametrize("script", ["pqn_gymnax", "pqn_rnn_gymnax"])
def test_make_train_accepts_env(script):
    """make_train builds each script's engine with the env's gymnax defaults; TEST_NUM_STEPS is max_steps_in_episode."""
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
        cfg = dict(ENV_NAME=NAME, TOTAL_TIMESTEPS=5e5, TOTAL_TIMESTEPS_DECAY=5e5, NUM_STEPS=64, NUM_ENVS=128,
                   NUM_MINIBATCHES=16, MEMORY_WINDOW=4)
        with pytest.raises(RuntimeError, match="stop"):
            mod.make_train(cfg)
    finally:
        setattr(mod, cls, orig)
    assert seen["config"]["TEST_NUM_STEPS"] == 100
    assert seen["config"]["NUM_UPDATES"] == int(5e5 // 64 // 128)
    if script == "pqn_rnn_gymnax":
        assert seen["kw"]["env_params"].max_steps_in_episode == 100
    else:
        assert seen["kw"] == {"network": "mlp", "flatten_obs": True}


# --------------------------------------------------------------------------- #
# jax's and gymnax's own values, once recorded
# --------------------------------------------------------------------------- #
_NORMAL_REF = os.path.join(HERE, "golden", "gaussian_bandit_normal_ref.npz")
_TRAJ_REF = sorted(glob.glob(os.path.join(HERE, "golden", "gaussian_bandit_*_traj_ref.npz")))
# |mu2|, |normal| < 5.5 < 8, so an ulp of either is at most 2^-21: 3 ulps of each plus the rounding of the sum
REWARD_ATOL = 7 * 2.0 ** -21


@pytest.mark.skipif(not os.path.exists(_NORMAL_REF),
                    reason="no jax.random.normal values recorded yet (tests/golden/make_gaussian_bandit_golden_from_ref.py)")
def test_normal_against_reference(hlib):
    """jax's normal at the recorded inputs: the oracle's formula within NORMAL_ULP_BOUND ulps on every device (CPU
    without contraction, CUDA with it), and jax.random.normal(key, (n,)) is the normal of random_bits(key, (n,))."""
    g = dict(np.load(_NORMAL_REF))
    for dev, fma in (("cpu", False), ("cuda", True)):
        if f"normal_{dev}" not in g:
            continue
        want = g[f"normal_{dev}"]
        assert JN.ulp_distance(JN.normal_from_bits(g["bits"], fma=fma), want).max() <= JN.NORMAL_ULP_BOUND, dev
        for part in (0, 1):
            keys = g[f"keys_{part}"]
            got = np.stack([JN.normal(k, (g[f"key_normal_{dev}_{part}"].shape[1],), bool(part), fma=fma) for k in keys])
            assert JN.ulp_distance(got, g[f"key_normal_{dev}_{part}"]).max() <= JN.NORMAL_ULP_BOUND, (dev, part)


@pytest.mark.skipif(not _TRAJ_REF, reason="no GaussianBandit-misc trajectories recorded from gymnax yet "
                                          "(tests/golden/make_gaussian_bandit_golden_from_ref.py)")
@pytest.mark.parametrize("path", _TRAJ_REF or ["none"])
def test_against_reference(path, hlib):
    """Replays a trajectory recorded from gymnax through the oracle and the host-compiled device logic: dones,
    actions and times exactly, rewards, mu2 and the observations within the normal's bound; and checks gymnax's
    default EnvParams, EnvState fields and observation shape."""
    g = dict(np.load(path))
    part = "partitionable" in os.path.basename(path)
    for k, v in dict(mu1=0.0, sigma_p=1.0, sigma_l=1.0, normalize_time=True, max_steps_in_episode=100).items():
        assert np.float32(g[f"param_{k}"]) == np.float32(v), k
    assert tuple(g["obs_shape"]) == GB.GaussianBandit.obs_shape
    assert sorted(k[6:] for k in g if k.startswith("state_")) == sorted(GB.GaussianBandit.state_fields)
    jr.DEFAULT_PARTITIONABLE = part
    try:
        env = GB.make()
        h = HostEnv(hlib, int(part))
        o_obs, o_st = env.reset(g["reset_keys"])
        h_obs, h_st = h.reset(g["reset_keys"])
        assert np.abs(o_obs - g["obs0"]).max() <= REWARD_ATOL and np.abs(h_obs - g["obs0"]).max() <= REWARD_ATOL
        for t in range(g["action"].shape[0]):
            sk, act = g["step_keys"][t], g["action"][t].astype(np.int32)
            o_obs, o_st, o_r, o_d, _ = env.step(sk, o_st, act)
            h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
            assert np.array_equal(o_d, g["done"][t]) and np.array_equal(h_d, g["done"][t]), t
            for r in (o_r, h_r):
                assert np.abs(r - g["reward"][t]).max() <= REWARD_ATOL, t
            for ob in (o_obs, h_obs):
                assert np.abs(ob - g["obs"][t]).max() <= REWARD_ATOL, t
            assert np.array_equal(o_st["time"], g["state_time"][t]) and np.array_equal(o_st["last_action"],
                                                                                      g["state_last_action"][t])
            for k in ("mu2", "exp_reward_best", "last_reward"):
                assert np.abs(o_st[k] - g[f"state_{k}"][t]).max() <= REWARD_ATOL, (k, t)
    finally:
        jr.DEFAULT_PARTITIONABLE = False
