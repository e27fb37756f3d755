"""jax.random.normal and GaussianBandit-misc on the GPU, against the host build of the same code
(tests/host_harness_gaussian_bandit.cpp) and the NumPy oracles (tests/jax_normal_oracle.py,
tests/gaussian_bandit_oracle.py).

The device's normal calls libdevice's log1pf.  torch's CUDA log1p on fp32 is that same function, so the oracle run on
torch's log1p restates the device bit for bit; against the oracle's own log1p the normal stays within
NORMAL_ULP_BOUND ulps.

- ``pqn_normal_from_bits`` over all 2^23 distinct inputs and ``pqn_random_normal`` at real keys, in both layouts.
- The env operator at N = 100,003 and the fused ``pqn_rollout_act_step`` at 3 x 33,335 envs with done_only 0 and 1,
  both layouts: every word bit for bit.
- Two whole updates of each script against an oracle replay, CUDA-graph replay of the GRU against the eager run,
  bit-identical repeats, and a save-and-evaluate run per script."""
import ctypes
import os

import numpy as np
import pytest
import torch

import gaussian_bandit_oracle as GB
import jax_normal_oracle as JN
import test_gpu_gymnax_extra as GX
import test_gpu_misc_envs as MT
import test_gpu_net_shapes as NS
from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from test_gaussian_bandit_host import fields, host_call

pytestmark = pytest.mark.gpu
NAME = "GaussianBandit-misc"
N_BIG = 100_003
dev, t_, keys_t, np_state, to_dev_state = GX.dev, GX.t_, GX.keys_t, GX.np_state, GX.to_dev_state
HERE = os.path.dirname(os.path.abspath(__file__))


def cuda_log1p(x):
    """libdevice's log1pf, through torch's CUDA log1p."""
    return torch.log1p(torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dev())).cpu().numpy()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def device_normal_from_bits(b):
    from purejaxql_b200 import _lib
    bd = torch.from_numpy(b.view(np.int32)).to(dev())
    out = torch.empty(b.shape[0], dtype=torch.float32, device=dev())
    _lib.check(_lib.lib().pqn_normal_from_bits(_lib.p(bd), _lib.p(out), b.shape[0], _lib.stream_ptr()),
               "pqn_normal_from_bits")
    return out.cpu().numpy()


@pytest.fixture(scope="module")
def hlib(tmp_path_factory):
    import subprocess
    so = str(tmp_path_factory.mktemp("harness") / "host_harness_gaussian_bandit.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(HERE, "host_harness_gaussian_bandit.cpp"), "-o", so])
    return ctypes.CDLL(so)


class CudaGaussianBandit(GB.GaussianBandit):
    """The oracle on libdevice's log1pf."""

    def __init__(self, max_steps_in_episode: int = 100):
        super().__init__(max_steps_in_episode, cuda_log1p)


def oracle_env():
    return GB.make(log1p=cuda_log1p)


# --------------------------------------------------------------------------- #
# jax.random.normal
# --------------------------------------------------------------------------- #
def test_normal_from_bits_all_inputs(hlib):
    """All 2^23 inputs: the device equals the host build's polynomial on libdevice's w and the oracle on libdevice's
    log1p, bit for bit; against the host build as it stands (the C library's log1pf) it differs only where the two
    log1pf differ, by at most NORMAL_ULP_BOUND ulps; against the oracle's own log1p by at most that too.  The low 9
    bits of the input do not matter."""
    b = JN.all_bits()
    d = device_normal_from_bits(b)
    u = JN.uniform_from_bits(b)
    w_dev = JN.erf_inv_w(u, cuda_log1p)
    poly = host_call(hlib, "h_erf_inv_from_w", u, w_dev)
    assert np.array_equal(bits(d), bits((JN.SQRT2 * poly).astype(np.float32)))
    assert np.array_equal(bits(d), bits(JN.normal_from_bits(b, log1p=cuda_log1p)))
    h = host_call(hlib, "h_normal_from_bits", b)
    w_host = JN.erf_inv_w(u, lambda x: host_call(hlib, "h_log1pf", np.asarray(x, np.float32)))
    differ = bits(d) != bits(h)
    assert not (differ & (bits(w_dev) == bits(w_host))).any()
    assert JN.ulp_distance(d, h).max() <= JN.NORMAL_ULP_BOUND
    assert JN.ulp_distance(w_dev, JN.erf_inv_w(u)).max() <= 1
    assert JN.ulp_distance(d, JN.normal_from_bits(b)).max() <= JN.NORMAL_ULP_BOUND
    print(f"device vs host build: {int(differ.sum())} of {b.size} values differ")
    low = (b | np.uint32(0x1FF))[::4099]
    assert np.array_equal(bits(device_normal_from_bits(low)), bits(d[::4099]))


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("n", [1, 6, 100_003])
def test_random_normal_at_keys(part, n):
    """jaxrandom.normal(key, n) == jax.random.normal(key, (n,)) of the oracle on libdevice's log1p, bit for bit, for
    even and odd n (the original layout pads odd counts), in both layouts."""
    from purejaxql_b200 import _lib, jaxrandom
    for seed in (0, 17):
        key = jr.split(jr.PRNGKey(seed), 2, bool(part))[1]
        got = jaxrandom.normal(jaxrandom.as_key_tensor(key, dev()), n, rng_mode=part).cpu().numpy()
        want = JN.normal(key, (n,), bool(part), log1p=cuda_log1p)
        assert got.shape == (n,) and np.array_equal(bits(got), bits(want)), seed
    with pytest.raises(ValueError):
        jaxrandom.normal(torch.zeros((2, 2), dtype=torch.int32, device=dev()), 4)
    out = torch.empty(1, device=dev())
    key = torch.zeros(2, dtype=torch.int32, device=dev())
    assert _lib.lib().pqn_random_normal(_lib.p(key), _lib.p(out), 1 << 31, part, _lib.stream_ptr()) != 0


# --------------------------------------------------------------------------- #
# env operator and fused rollout step
# --------------------------------------------------------------------------- #
def assert_state(st, o_st, where):
    f = fields(np_state(st))
    for k, v in o_st.items():
        assert np.array_equal(np.ascontiguousarray(f[k].astype(v.dtype).reshape(v.shape)).view(np.uint8),
                              np.ascontiguousarray(v).view(np.uint8)), (where, k)


@pytest.mark.parametrize("part", [0, 1])
def test_env_operator_bit_exact(part):
    """reset / step / obs at N = 100,003 over 24 steps of random actions from 1-23 steps before the time limit
    (auto-resets included): obs, reward, done, info and every state word bit for bit; pqn_env_obs returns the step's
    obs."""
    from purejaxql_b200 import _lib, envs
    n, L = N_BIG, _lib.lib()
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env, params = envs.make(NAME, flatten_obs=True, rng_mode=part)
        oenv = oracle_env()
        key, kr = jr.split(jr.PRNGKey(13), 2)
        rk = jr.split(kr, n)
        obs, st = env.reset(keys_t(rk), params)
        o_obs, o_st = oenv.reset(rk)
        assert np.array_equal(bits(obs.cpu().numpy()), bits(o_obs))
        assert_state(st, o_st, "reset")
        o_st["time"] = np.random.default_rng(7).integers(100 - 23, 100, n).astype(np.int32)
        st = to_dev_state(NAME, o_st)
        rng = np.random.default_rng(part)
        dones = np.zeros(n, np.int64)
        for t in range(24):
            key, ks = jr.split(key, 2)
            sk = jr.split(ks, n)
            act = rng.integers(0, 2, n).astype(np.int32)
            obs, st, r, d, info = env.step(keys_t(sk), st, t_(act), params)
            o_obs, o_st, o_r, o_d, o_info = oenv.step(sk, o_st, act)
            assert np.array_equal(d.cpu().numpy(), o_d), t
            assert np.array_equal(bits(r.cpu().numpy()), bits(o_r)), t
            assert np.array_equal(bits(obs.cpu().numpy()), bits(o_obs)), t
            for k in ("discount", "returned_episode_returns", "returned_episode_lengths", "timestep"):
                assert np.array_equal(info[k].cpu().numpy(), o_info[k]), (t, k)
            assert_state(st, o_st, t)
            ob2 = torch.empty((n, 4), device=dev())
            _lib.check(L.pqn_env_obs(env.env_id, _lib.p(st), _lib.p(ob2), n, _lib.stream_ptr()), "pqn_env_obs")
            assert torch.equal(ob2, obs), t
            dones += o_d
        assert (dones >= 1).all()
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("done_only", [0, 1])
def test_rollout_act_step_matches_oracle(done_only, part):
    """The fused eps-greedy + step + LogWrapper launch over 3 seeds x 33,335 envs, starting 1-10 steps before the time
    limit: actions, rewards, dones, max q, obs rows, every state word and the info sums, bit for bit."""
    from purejaxql_b200 import _lib, envs
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        L = _lib.lib()
        S, E, eps, rew_scale, T, D, A = 3, 33_335, 0.4, 0.5, 12, 4, 2
        env, _ = envs.make(NAME, flatten_obs=True, rng_mode=part)
        oenv = oracle_env()
        seeds = jr.split(jr.PRNGKey(79), S)
        rk = np.stack([jr.split(seeds[s], E) for s in range(S)])
        o = [oenv.reset(rk[s]) for s in range(S)]
        o_obs, o_st = [x[0] for x in o], [x[1] for x in o]
        for s in range(S):
            o_st[s]["time"] = np.random.default_rng(s).integers(90, 100, E).astype(np.int32)
        state = torch.cat([to_dev_state(NAME, o_st[s]) for s in range(S)], 1).contiguous()
        obs_buf = torch.zeros((S, T + 1, E, D), device=dev())
        act = torch.zeros((S, T, E), dtype=torch.int32, device=dev())
        rew = torch.zeros((S, T, E), device=dev())
        done = torch.zeros((S, T, E), dtype=torch.uint8, device=dev())
        maxq = torch.zeros((S, T, E), device=dev())
        sums = torch.zeros((S, 5), dtype=torch.float64, device=dev())
        o_sums = np.zeros((S, 5))
        eps_d = torch.full((1,), eps, device=dev())
        rng = np.random.default_rng(6)
        for t in range(T):
            q = rng.standard_normal((S * E, A)).astype(np.float32)
            step_keys = np.stack([np.stack(jr.split(jr.PRNGKey(1000 * t + s), 2)) for s in range(S)])
            keys_d, q_d = keys_t(step_keys), t_(q)
            _lib.check(L.pqn_rollout_act_step(env.env_id, _lib.p(keys_d), _lib.p(q_d), _lib.p(eps_d), _lib.p(state),
                                              _lib.raw(obs_buf[:, t + 1]), (T + 1) * E, _lib.raw(act[:, t]),
                                              _lib.raw(rew[:, t]), _lib.raw(done[:, t]), _lib.raw(maxq[:, t]), T * E,
                                              _lib.p(sums), done_only, S, E, 0, 0, 0, rew_scale, part,
                                              _lib.stream_ptr()), "pqn_rollout_act_step")
            for s in range(S):
                qs = q.reshape(S, E, A)[s]
                a = R.eps_greedy(jr.split(step_keys[s, 0], E), qs, eps)
                o_obs[s], o_st[s], r, d, info = oenv.step(jr.split(step_keys[s, 1], E), o_st[s], a)
                assert np.array_equal(act[s, t].cpu().numpy(), a), (t, s)
                assert np.array_equal(bits(rew[s, t].cpu().numpy()), bits((np.float32(rew_scale) * r).astype(np.float32)))
                assert np.array_equal(done[s, t].cpu().numpy().astype(bool), d), (t, s)
                assert np.array_equal(maxq[s, t].cpu().numpy(), qs.max(-1)), (t, s)
                assert np.array_equal(bits(obs_buf[s, t + 1].cpu().numpy()), bits(o_obs[s])), (t, s)
                assert_state(state[:, s * E:(s + 1) * E], o_st[s], (t, s))
                m = d if done_only else np.ones(E, bool)
                o_sums[s] += [info["returned_episode_returns"][m].astype(np.float64).sum(),
                              info["returned_episode_lengths"][m].sum(), info["timestep"][m].sum(), d.sum(),
                              info["discount"][m].sum()]
        assert np.array_equal(sums.cpu().numpy(), o_sums)
        assert o_sums[:, 3].min() >= E
    finally:
        jr.DEFAULT_PARTITIONABLE = False


# --------------------------------------------------------------------------- #
# whole runs
# --------------------------------------------------------------------------- #
def test_mlp_two_updates_match_oracle(monkeypatch):
    """Two whole updates of pqn_gymnax (eps = 1) against the oracle's update_step."""
    import test_gpu_train as TT
    from purejaxql_b200 import pqn_gymnax
    monkeypatch.setitem(G._REGISTRY, NAME, CudaGaussianBandit)
    cfg = TT._cfg(NAME, HIDDEN_SIZE=128, NUM_LAYERS=2, REW_SCALE=1.0, LAMBDA=0.95, NUM_ENVS=32, NUM_STEPS=16)
    TT._run_updates_against_oracle(pqn_gymnax, NAME, "mlp", True, cfg, nupd=2)


def test_rnn_two_updates_match_oracle():
    """Two whole updates of pqn_rnn_gymnax (eps = 1) against the oracle replay of test_gpu_memory_chain."""
    import test_gpu_memory_chain as MCT
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = MCT._rnn_cfg(ENV_NAME=NAME)
    del cfg["ENV_KWARGS"]
    nupd = 2
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_rnn_gymnax.make_train(cfg)
    eng = train.engine
    assert (eng.D, eng.A) == (4, 2)
    rngs = jr.split(jr.PRNGKey(33), 2)
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    out = train(rngs)
    MCT._replay_rnn_updates(cfg, out, eng.spec.unflatten(cap["flat"]), eng.spec, rngs, nupd, oracle_env)


@pytest.mark.parametrize("norm_type,norm_input", [("layer_norm", False), ("batch_norm", True)])
def test_rnn_cuda_graph_replay_equals_eager_and_repeats(norm_type, norm_input):
    eager, graph, again = (MT._rnn_run(NAME, False, norm_type, norm_input), MT._rnn_run(NAME, True, norm_type, norm_input),
                           MT._rnn_run(NAME, True, norm_type, norm_input))
    for a, b, c in zip(eager, graph, again):
        assert np.array_equal(a, b, equal_nan=True) and np.array_equal(b, c, equal_nan=True)
    assert np.isfinite(eager[1]).all()


def test_mlp_is_bit_reproducible():
    from purejaxql_b200 import pqn_gymnax
    outs = []
    for _ in range(2):
        cfg = NS._mlp_cfg(256, 2)
        cfg.update(ENV_NAME=NAME, NORM_INPUT=True)
        out = pqn_gymnax.make_train(cfg)(jr.split(jr.PRNGKey(11), 2))
        outs.append((out["runner_state"][0].params_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy()))
    assert np.isfinite(outs[0][1]).all()
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("script,preset", [("pqn_gymnax", "pqn_cartpole"), ("pqn_rnn_gymnax", "pqn_rnn_cartpole")])
def test_smoke_with_eval_and_save(script, preset, tmp_path):
    """The command lines of the README: both scripts train, evaluate greedy 100-step episodes and save safetensors
    with the flax names."""
    import importlib
    from purejaxql_b200 import config_loader
    from purejaxql_b200.utils.save_load import load_params
    mod = importlib.import_module(f"purejaxql_b200.{script}")
    c = config_loader.compose([f"+alg={preset}", f"alg.ENV_NAME={NAME}", "NUM_SEEDS=2", f"SAVE_PATH={tmp_path}",
                               "alg.TOTAL_TIMESTEPS=2e4", "alg.TOTAL_TIMESTEPS_DECAY=2e4", "alg.TEST_NUM_ENVS=16",
                               "alg.TEST_INTERVAL=0.5"])
    out = mod.single_run(c)
    m = out["metrics"]
    assert torch.isfinite(m["td_loss"]).all() and "test/returned_episode_returns" in m
    assert (m["test/returned_episode_lengths"] == 100).all()
    assert torch.isfinite(torch.as_tensor(m["test/returned_episode_returns"])).all()
    files = sorted(tmp_path.rglob("*.safetensors"))
    assert len(files) == 2, files
    tree = load_params(str(files[0]))
    assert tree["Dense_0"]["kernel"].shape[0] == 4


# --------------------------------------------------------------------------- #
# jax's own values on a CUDA device, once recorded
# --------------------------------------------------------------------------- #
_NORMAL_REF = os.path.join(HERE, "golden", "gaussian_bandit_normal_ref.npz")


@pytest.mark.skipif(not os.path.exists(_NORMAL_REF),
                    reason="no jax.random.normal values recorded yet (tests/golden/make_gaussian_bandit_golden_from_ref.py)")
def test_device_normal_against_reference():
    """The device normal against jax's on a CUDA device at the recorded inputs: equal bit for bit when (J3) and (J4)
    of tests/jax_normal_oracle.py hold; the number of differing values says how far they do not."""
    g = dict(np.load(_NORMAL_REF))
    if "normal_cuda" not in g:
        pytest.skip("the recording has no CUDA values")
    d = device_normal_from_bits(g["bits"])
    differ = bits(d) != bits(g["normal_cuda"])
    assert not differ.any(), (int(differ.sum()), int(JN.ulp_distance(d, g["normal_cuda"]).max()))
