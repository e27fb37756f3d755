"""MemoryChain-bsuite on the GPU against the NumPy oracle (tests/bsuite_oracle.py): the env operator through
pqn_env_reset_params / pqn_env_step / pqn_env_obs and the fused pqn_rollout_act_step bit for bit, two whole recurrent
updates against an oracle replay, CUDA-graph replay against the eager run, and smoke runs of both training scripts."""
import numpy as np
import pytest
import torch

import bsuite_oracle as MC
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_rnn_ref as RR

pytestmark = pytest.mark.gpu
NAME = "MemoryChain-bsuite"


def dev():
    return torch.device("cuda:0")


def t_(a, dt=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev())
    return t if dt is None else t.to(dt)


def keys_t(k):
    return t_(np.ascontiguousarray(k, np.uint32).view(np.int32))


def _assert_state_equal(state, o_st, ml, where):
    from purejaxql_b200 import envs
    f = envs.state_to_fields(NAME, state.cpu())
    for k, v in o_st.items():
        assert np.array_equal(f[k].numpy().astype(v.dtype).reshape(v.shape), v), (where, k)
    assert (f["memory_length"].numpy() == ml).all(), where


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("ml", [1, 5, 100])
def test_env_operator_matches_oracle_bit_exact(part, ml):
    """reset_params / step / obs for N = 100,003 envs over more than one episode (so every env auto-resets and
    must carry memory_length over): obs, reward, done, info and every state field bit for bit."""
    from purejaxql_b200 import _lib, envs
    n = 100_003
    L = _lib.lib()
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env, _ = envs.make(NAME, flatten_obs=True, rng_mode=part)
        params = envs.EnvParams(1000, memory_length=ml)
        oenv = MC.make(ml, flatten=True)
        key, kr = jr.split(jr.PRNGKey(40 + ml), 2)
        rk = jr.split(kr, n)
        obs, st = env.reset(keys_t(rk), params)
        o_obs, o_st = oenv.reset(rk)
        assert np.array_equal(obs.cpu().numpy(), o_obs)
        _assert_state_equal(st, o_st, ml, "reset")
        rng = np.random.default_rng(ml + 10 * part)
        for t in range(min(3 * (ml + 1), ml + 4)):
            key, ks = jr.split(key, 2)
            sk = jr.split(ks, n)
            act = rng.integers(0, 2, n).astype(np.int32)
            obs, st, r, d, info = env.step(keys_t(sk), st, t_(act), params)
            o_obs, o_st, o_r, o_d, o_info = oenv.step(sk, o_st, act)
            assert np.array_equal(d.cpu().numpy(), o_d), t
            assert np.array_equal(r.cpu().numpy(), o_r), t
            assert np.array_equal(obs.cpu().numpy(), o_obs), t
            for k in ("discount", "returned_episode_returns", "returned_episode_lengths", "timestep"):
                assert np.array_equal(info[k].cpu().numpy(), o_info[k]), (t, k)
            _assert_state_equal(st, o_st, ml, t)
            ob2 = torch.empty((n, 3), device=dev())
            _lib.check(L.pqn_env_obs(env.env_id, _lib.p(st), _lib.p(ob2), n, _lib.stream_ptr()), "pqn_env_obs")
            assert np.array_equal(ob2.cpu().numpy(), o_obs), t
        assert (o_st["log_returned_episode_lengths"] == ml + 1).all()
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def test_reset_params_defaults_and_rejects_bad_memory_length():
    from purejaxql_b200 import _lib, envs
    L = _lib.lib()
    n = 1000
    env, params = envs.make(NAME, flatten_obs=True)
    k = keys_t(jr.split(jr.PRNGKey(1), n))
    st = torch.empty((env.state_words, n), dtype=torch.int32, device=dev())
    obs = torch.empty((n, 3), device=dev())
    for ml in (0, -1):
        rc = L.pqn_env_reset_params(env.env_id, _lib.p(k), _lib.p(st), _lib.p(obs), n, _lib.EnvParams(0, ml), 0,
                                    _lib.stream_ptr())
        assert rc == -1 and b"memory_length" in L.pqn_last_error()
    # pqn_env_reset and a NULL params pointer give gymnax's default memory_length = 5
    for call in (lambda: L.pqn_env_reset(env.env_id, _lib.p(k), _lib.p(st), _lib.p(obs), n, 0, 0, _lib.stream_ptr()),
                 lambda: L.pqn_env_reset_params(env.env_id, _lib.p(k), _lib.p(st), _lib.p(obs), n, None, 0,
                                                _lib.stream_ptr())):
        st.fill_(-7)
        _lib.check(call(), "reset")
        f = envs.state_to_fields(NAME, st.cpu())
        assert (f["memory_length"] == 5).all() and (f["time"] == 0).all()
    o_obs, _ = MC.make(5, flatten=True).reset(jr.split(jr.PRNGKey(1), n))
    assert np.array_equal(obs.cpu().numpy(), o_obs)
    # other envs ignore memory_length: CartPole through reset_params with memory_length = 0 equals pqn_env_reset
    cp, _ = envs.make("CartPole-v1", flatten_obs=True)
    a = torch.empty((cp.state_words, n), dtype=torch.int32, device=dev())
    b = torch.empty_like(a)
    _lib.check(L.pqn_env_reset(cp.env_id, _lib.p(k), _lib.p(a), None, n, 0, 0, _lib.stream_ptr()), "reset")
    _lib.check(L.pqn_env_reset_params(cp.env_id, _lib.p(k), _lib.p(b), None, n, _lib.EnvParams(0, 0), 0,
                                      _lib.stream_ptr()), "reset_params")
    assert torch.equal(a, b)


@pytest.mark.parametrize("done_only", [0, 1])
def test_rollout_act_step_matches_oracle(done_only):
    """The fused eps-greedy + step + LogWrapper launch: transition rows, float obs rows, info sums."""
    from purejaxql_b200 import _lib, envs
    L = _lib.lib()
    S, E, T, ml, eps, rew_scale = 3, 257, 14, 4, 0.4, 0.5
    env, _ = envs.make(NAME, flatten_obs=True)
    oenv = MC.make(ml, flatten=True)
    seeds = jr.split(jr.PRNGKey(77), S)
    rk = np.stack([jr.split(seeds[s], E) for s in range(S)])               # [S, E, 2]
    obs, state = env.reset(keys_t(rk.reshape(S * E, 2)), envs.EnvParams(1000, memory_length=ml))
    o = [oenv.reset(rk[s]) for s in range(S)]
    o_obs, o_st = [x[0] for x in o], [x[1] for x in o]
    obs_buf = torch.zeros((S, T + 1, E, 3), device=dev())
    obs_buf[:, 0] = obs.view(S, E, 3)
    act = torch.zeros((S, T, E), dtype=torch.int32, device=dev())
    rew = torch.zeros((S, T, E), device=dev())
    done = torch.zeros((S, T, E), dtype=torch.uint8, device=dev())
    maxq = torch.zeros((S, T, E), device=dev())
    sums = torch.zeros((S, 5), dtype=torch.float64, device=dev())
    o_sums = np.zeros((S, 5))
    eps_d = torch.full((1,), eps, device=dev())
    rng = np.random.default_rng(5)
    for t in range(T):
        q = rng.standard_normal((S * E, 2)).astype(np.float32)
        step_keys = np.stack([np.stack(jr.split(jr.PRNGKey(1000 * t + s), 2)) for s in range(S)])   # [S, 2, 2]
        _lib.check(L.pqn_rollout_act_step(env.env_id, _lib.p(keys_t(step_keys)), _lib.p(t_(q)), _lib.p(eps_d),
                                          _lib.p(state), _lib.raw(obs_buf[:, t + 1]), (T + 1) * E, _lib.raw(act[:, t]),
                                          _lib.raw(rew[:, t]), _lib.raw(done[:, t]), _lib.raw(maxq[:, t]), T * E,
                                          _lib.p(sums), done_only, S, E, 0, 0, 0, rew_scale, 0, _lib.stream_ptr()),
                   "pqn_rollout_act_step")
        for s in range(S):
            qs = q.reshape(S, E, 2)[s]
            a = R.eps_greedy(jr.split(step_keys[s, 0], E), qs, eps)
            o_obs[s], o_st[s], r, d, info = oenv.step(jr.split(step_keys[s, 1], E), o_st[s], a)
            assert np.array_equal(act[s, t].cpu().numpy(), a), (t, s)
            assert np.array_equal(rew[s, t].cpu().numpy(), (np.float32(rew_scale) * r).astype(np.float32)), (t, s)
            assert np.array_equal(done[s, t].cpu().numpy().astype(bool), d), (t, s)
            assert np.array_equal(maxq[s, t].cpu().numpy(), qs.max(-1)), (t, s)
            assert np.array_equal(obs_buf[s, t + 1].cpu().numpy(), o_obs[s]), (t, s)
            m = d if done_only else np.ones(E, bool)
            o_sums[s] += [info["returned_episode_returns"][m].astype(np.float64).sum(),
                          info["returned_episode_lengths"][m].sum(), info["timestep"][m].sum(), d.sum(),
                          info["discount"][m].sum()]
    for s in range(S):
        _assert_state_equal(state[:, s * E:(s + 1) * E], o_st[s], ml, s)
    assert np.array_equal(sums.cpu().numpy(), o_sums)
    assert o_sums[:, 3].min() > 0


def _rnn_cfg(**kw):
    c = dict(ENV_NAME=NAME, ENV_KWARGS={"memory_length": 4}, NUM_ENVS=8, NUM_STEPS=12, MEMORY_WINDOW=3,
             NUM_MINIBATCHES=4, NUM_EPOCHS=2, EPS_START=1.0, EPS_FINISH=1.0, EPS_DECAY=0.2, LR=1e-4, MAX_GRAD_NORM=10,
             GAMMA=0.99, LAMBDA=0.95, NORM_TYPE="layer_norm", NORM_INPUT=False, HIDDEN_SIZE=128, NUM_LAYERS=2,
             LR_LINEAR_DECAY=True, REW_SCALE=1.0, WANDB_MODE="disabled", TEST_DURING_TRAINING=False)
    c.update(kw)
    return c


def _oracle_step(env, p, hs, obs, ld, la, st, rng, eps, rew_scale, E):
    """_step_env / _random_step (pqn_rnn_gymnax.py:192-236, :514-529) for one seed."""
    ks = jr.split(rng, 3)
    rng, rng_a, rng_s = ks[0], ks[1], ks[2]
    new_hs, q = RR.rnn_forward(p, hs, obs[None], ld[None], la[None])
    act = R.eps_greedy(jr.split(rng_a, E), q[0], eps)
    new_obs, st, reward, done, info = env.step(jr.split(rng_s, E), st, act)
    tr = dict(last_hs=hs, obs=obs, action=act, reward=(np.float32(rew_scale) * reward).astype(np.float32), done=done,
              last_done=ld, last_action=la)
    return (new_hs.astype(np.float32), new_obs, done, act, st, rng), tr


def _replay_rnn_updates(cfg, out, tree0, spec, rngs, nupd, make_env):
    """Oracle replay of whole recurrent updates at eps = 1 (memory warm-up, key chain, env-axis minibatches, in-loss
    Q(lambda), RAdam): per-update td_loss, final parameters and final rng of every seed."""
    T, E, W, nmb, H = cfg["NUM_STEPS"], cfg["NUM_ENVS"], cfg["MEMORY_WINDOW"], cfg["NUM_MINIBATCHES"], cfg["HIDDEN_SIZE"]
    Bm = E // nmb
    ts = out["runner_state"][0]
    dones = 0
    for s in range(rngs.shape[0]):
        def leaf(tree, path):
            d = tree
            for k in path:
                d = d[k]
            return d[s].cpu().numpy()
        params = {"/".join(p): leaf(tree0, p).astype(np.float32) for p, *_ in spec.entries}
        env = make_env()
        k = jr.split(rngs[s], 2); rng = k[0]                               # :255
        k = jr.split(rng, 2); rng = k[0]                                   # :505
        k = jr.split(rng, 2); rng, kR = k[0], k[1]                         # :508
        obs, st = env.reset(jr.split(kR, E))
        hs = np.zeros((E, H), np.float32); ld = np.zeros(E, bool); la = np.zeros(E, np.int32)
        k = jr.split(rng, 2); carry = k[1]                                 # :531
        mem = []
        for _ in range(W + T):
            (hs, obs, ld, la, st, carry), tr = _oracle_step(env, params, hs, obs, ld, la, st, carry, 1.0,
                                                            cfg["REW_SCALE"], E)
            mem.append(tr)
        rng = carry
        k = jr.split(rng, 2); rng = k[1]                                   # :541
        opt = R.opt_init(params)
        total = cfg["NUM_UPDATES_DECAY"] * nmb * cfg["NUM_EPOCHS"]
        lr_fn = lambda i: R.linear_schedule(cfg["LR"], 1e-20, total, i)
        for u in range(nupd):
            k = jr.split(rng, 2); carry = k[1]                             # :222
            new = []
            for _ in range(T):
                (hs, obs, ld, la, st, carry), tr = _oracle_step(env, params, hs, obs, ld, la, st, carry, 1.0,
                                                                cfg["REW_SCALE"], E)
                new.append(tr)
            rng = carry
            mem = mem[T:] + new                                            # :239-243
            stack = {kk: np.stack([m[kk] for m in mem]) for kk in mem[0]}
            dones += int(stack["done"].sum())
            k = jr.split(rng, 2); r = k[0]                                 # :381
            losses = []
            for _ in range(cfg["NUM_EPOCHS"]):
                k = jr.split(r, 2); r, kperm = k[0], k[1]                  # :368
                perm = jr.permutation_indices(kperm, E)
                r = jr.split(r, 2)[0]                                      # :375
                for mb in range(nmb):
                    idx = perm[mb * Bm:(mb + 1) * Bm]
                    loss, _, g = RR.rnn_loss_and_grads(
                        params, stack["last_hs"][0][idx], stack["obs"][:, idx], stack["last_done"][:, idx],
                        stack["last_action"][:, idx], stack["action"][:, idx], stack["reward"][:, idx],
                        stack["done"][:, idx], cfg["GAMMA"], cfg["LAMBDA"])
                    params, opt, _ = R.radam_clip_step(params, g, opt, lr_fn(opt["count"]), cfg["MAX_GRAD_NORM"])
                    losses.append(loss)
            rng = r
            got = float(out["metrics"]["td_loss"][s, u])
            assert abs(got - np.mean(losses)) < 2e-3 * max(1.0, abs(np.mean(losses))), (u, got, np.mean(losses))
        for p, *_ in spec.entries:
            d = np.abs(leaf(ts.params, p) - params["/".join(p)])
            assert np.quantile(d, 0.99) < 1e-4 and d.max() < 1e-3, (p, d.max())
        assert np.array_equal(out["runner_state"][4][s].cpu().numpy().view(np.uint32), rng)
    return dones


def test_rnn_memory_chain_update_steps_match_oracle():
    """Two whole updates of pqn_rnn_gymnax.make_train/train on MemoryChain (memory_length 4: episodes of 5 steps end
    inside the 15-step windows) with eps = 1 against the oracle replay."""
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = _rnn_cfg()
    nupd = 2
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_rnn_gymnax.make_train(cfg)
    eng = train.engine
    assert eng.env_params.memory_length == 4 and eng.D == 3
    rngs = jr.split(jr.PRNGKey(31), 2)
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    out = train(rngs)
    dones = _replay_rnn_updates(cfg, out, eng.spec.unflatten(cap["flat"]), eng.spec, rngs, nupd,
                                lambda: MC.make(4, flatten=True))
    assert dones > 0
    m = out["metrics"]
    assert (m["returned_episode_lengths"][:, -1] > 0).all()


def test_rnn_memory_chain_cuda_graph_replay_equals_eager():
    from purejaxql_b200 import pqn_rnn_gymnax
    outs = []
    for graph in (False, True):
        cfg = _rnn_cfg(EPS_FINISH=0.1, EPS_DECAY=0.5, TEST_DURING_TRAINING=True, TEST_INTERVAL=0.4, TEST_NUM_ENVS=8,
                       TEST_NUM_STEPS=20, EPS_TEST=0.0, CUDA_GRAPH=graph)
        cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(5 * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
        train = pqn_rnn_gymnax.make_train(cfg)
        out = train(jr.split(jr.PRNGKey(5), 2))
        assert train.engine.graph_captured == graph
        outs.append((out["runner_state"][0].params_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy(),
                     out["metrics"]["returned_episode_returns"].cpu().numpy(),
                     out["metrics"]["test/returned_episode_lengths"].cpu().numpy(),
                     out["runner_state"][2][4].cpu().numpy(), out["runner_state"][4].cpu().numpy()))
    for a, b in zip(*outs):
        assert np.array_equal(a, b, equal_nan=True)
    assert (outs[0][3] == 5).all()


def test_rnn_memory_chain_preset_smoke_with_eval():
    from purejaxql_b200 import config_loader, pqn_rnn_gymnax
    c = config_loader.compose(["+alg=pqn_rnn_memory_chain", "NUM_SEEDS=2", "SAVE_PATH=null",
                               "alg.TOTAL_TIMESTEPS=8192", "alg.TEST_NUM_ENVS=16", "alg.TEST_INTERVAL=0.5"])
    cfg = {**c, **c["alg"]}
    out = pqn_rnn_gymnax.make_train(cfg)(jr.split(jr.PRNGKey(0), 2))
    assert cfg["TEST_NUM_STEPS"] == 1000 and cfg["NUM_UPDATES"] == 2
    m = out["metrics"]
    assert m["td_loss"].shape == (2, 2) and torch.isfinite(m["td_loss"]).all()
    assert (m["test/returned_episode_lengths"] == 101).all()
    r = m["test/returned_episode_returns"]
    assert ((r >= -1) & (r <= 1)).all()
    assert m["env_step"][0, -1].item() == 8192


def test_mlp_memory_chain_smoke_with_eval():
    """pqn_gymnax with alg.ENV_NAME=MemoryChain-bsuite: gymnax's default params (memory_length 5, episodes of 6
    steps), as pqn_gymnax.py:92 builds them."""
    from purejaxql_b200 import config_loader, pqn_gymnax
    c = config_loader.compose(["+alg=pqn_cartpole", f"alg.ENV_NAME={NAME}", "NUM_SEEDS=2", "SAVE_PATH=null",
                               "alg.TOTAL_TIMESTEPS=8192", "alg.TEST_NUM_ENVS=16", "alg.TEST_INTERVAL=0.25"])
    cfg = {**c, **c["alg"]}
    train = pqn_gymnax.make_train(cfg)
    assert train.engine.env_params.memory_length == 5 and cfg["TEST_NUM_STEPS"] == 1000
    out = train(jr.split(jr.PRNGKey(0), 2))
    m = out["metrics"]
    assert m["td_loss"].shape == (2, 4) and torch.isfinite(m["td_loss"]).all()
    assert (m["test/returned_episode_lengths"] == 6).all()
    assert (m["returned_episode_lengths"][:, 1:] == 6).all()      # from the second update on, every env has ended one
    r = m["test/returned_episode_returns"]
    assert ((r >= -1) & (r <= 1)).all()
