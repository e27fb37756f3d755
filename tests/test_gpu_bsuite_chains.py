"""DeepSea-bsuite, UmbrellaChain-bsuite and DiscountingChain-bsuite on the GPU, against the NumPy oracles of
tests/bsuite_chains_oracle.py.

- The env operator (reset, step, obs, auto-reset, LogWrapper words) at N = 100,003 and the fused
  ``pqn_rollout_act_step`` at 3 x 33,335 envs, with both threefry layouts: bit for bit.
- The MLP and GRU Q-networks at DeepSea's input width, D = 64, for HIDDEN_SIZE 64 to 512 on tensor-core paths 2 and
  0, against the fp64 oracles with the bars of tests/test_gpu_gymnax_extra.py, and every NORM_TYPE x NORM_INPUT with
  batch_stats at D = 64.
- Two whole updates through make_train on DeepSea and on UmbrellaChain (whose rewards come from the step keys) against
  an oracle replay for both scripts, CUDA-graph replay of the GRU against the eager run, bit-identical repeated runs,
  and a save-and-evaluate smoke run per script and env."""
import numpy as np
import pytest
import torch

import bsuite_chains_oracle as B
import test_gpu_gymnax_extra as GX
import test_gpu_net_shapes as NS
from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_ref_norm as RN
from test_bsuite_chains_host import EPISODE, fields

pytestmark = pytest.mark.gpu
SEA, UMB, DISC = "DeepSea-bsuite", "UmbrellaChain-bsuite", "DiscountingChain-bsuite"
N_BIG = 100_003
dev, t_, keys_t, np_state, to_dev_state = GX.dev, GX.t_, GX.keys_t, GX.np_state, GX.to_dev_state


def assert_state(name, st, o_st, where):
    f = fields(name, np_state(st))
    for k, v in o_st.items():
        assert np.array_equal(f[k].astype(v.dtype).reshape(v.shape), v), (where, k)


@pytest.fixture(params=[2, 0], ids=["tc_path2", "ffma_path0"])
def tc_path(request):
    from purejaxql_b200 import _lib
    _lib.check(_lib.lib().pqn_set_tensor_core_path(request.param))
    yield request.param
    _lib.lib().pqn_set_tensor_core_path(2)


# --------------------------------------------------------------------------- #
# env operator
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("name", [SEA, UMB, DISC])
def test_env_operator_bit_exact(name, part):
    """reset / step / obs at N = 100,003 over more than two episodes of random actions: obs, reward (sign of zero
    included), done, info and every state field bit for bit; pqn_env_obs returns the obs the step returned."""
    from purejaxql_b200 import _lib, envs
    n, L = N_BIG, _lib.lib()
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env, params = envs.make(name, flatten_obs=True, rng_mode=part)
        oenv = B.make(name)
        D, A = env.obs_dim, env.num_actions
        key, kr = jr.split(jr.PRNGKey(12), 2)
        rk = jr.split(kr, n)
        obs, st = env.reset(keys_t(rk), params)
        o_obs, o_st = oenv.reset(rk)
        assert np.array_equal(obs.cpu().numpy().view(np.int32), o_obs.view(np.int32))
        assert_state(name, st, o_st, "reset")
        if name == SEA:   # unflattened: gymnax's (8, 8) board
            board, _ = envs.make(SEA, rng_mode=part)[0].reset(keys_t(rk), params)
            assert board.shape == (n, 8, 8) and np.array_equal(board.cpu().numpy().reshape(n, 64), o_obs)
        rng = np.random.default_rng(part)
        steps = 2 * EPISODE[name] + 3
        dones = 0
        for t in range(steps):
            key, ks = jr.split(key, 2)
            sk = jr.split(ks, n)
            act = rng.integers(0, A, n).astype(np.int32)
            obs, st, r, d, info = env.step(keys_t(sk), st, t_(act), params)
            o_obs, o_st, o_r, o_d, o_info = oenv.step(sk, o_st, act)
            assert np.array_equal(d.cpu().numpy(), o_d), t
            assert np.array_equal(r.cpu().numpy().view(np.int32), o_r.view(np.int32)), t
            assert np.array_equal(obs.cpu().numpy().view(np.int32), o_obs.view(np.int32)), t
            for k in ("discount", "returned_episode_returns", "returned_episode_lengths", "timestep"):
                assert np.array_equal(info[k].cpu().numpy(), o_info[k]), (t, k)
            assert_state(name, st, o_st, t)
            ob2 = torch.empty((n, D), device=dev())
            _lib.check(L.pqn_env_obs(env.env_id, _lib.p(st), _lib.p(ob2), n, _lib.stream_ptr()), "pqn_env_obs")
            assert torch.equal(ob2, obs), t
            dones += int(o_d.sum())
        assert dones == 2 * n
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("name", [SEA, UMB, DISC])
@pytest.mark.parametrize("done_only", [0, 1])
def test_rollout_act_step_matches_oracle(name, done_only, part):
    """The fused eps-greedy + step + LogWrapper launch over 3 seeds x 33,335 envs (100,005 in all; not a multiple of
    the block), in both threefry layouts: actions, rewards, dones, max q, the obs rows, every state field and the
    info sums, bit for bit.  DeepSea and UmbrellaChain run past two episodes; DiscountingChain starts at times 90-99
    so that its episodes end inside the window."""
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        _rollout_act_step_against_oracle(name, done_only, part)
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def _rollout_act_step_against_oracle(name, done_only, part):
    from purejaxql_b200 import _lib, envs
    L = _lib.lib()
    S, E, eps, rew_scale = 3, 33_335, 0.4, 0.5
    T = 12 if name == DISC else 2 * EPISODE[name] + 2
    env, _ = envs.make(name, flatten_obs=True, rng_mode=part)
    oenv = B.make(name)
    D, A = env.obs_dim, env.num_actions
    seeds = jr.split(jr.PRNGKey(78), S)
    rk = np.stack([jr.split(seeds[s], E) for s in range(S)])
    o = [oenv.reset(rk[s]) for s in range(S)]
    o_obs, o_st = [x[0] for x in o], [x[1] for x in o]
    if name == DISC:
        for s in range(S):
            o_st[s]["time"] = np.random.default_rng(s).integers(90, 100, E).astype(np.int32)
            o_st[s]["context"] = np.random.default_rng(10 + s).integers(0, 5, E).astype(np.int32)
    state = torch.cat([to_dev_state(name, o_st[s]) for s in range(S)], 1).contiguous()
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
        _lib.check(L.pqn_rollout_act_step(env.env_id, _lib.p(keys_d), _lib.p(q_d), _lib.p(eps_d),
                                          _lib.p(state), _lib.raw(obs_buf[:, t + 1]), (T + 1) * E, _lib.raw(act[:, t]),
                                          _lib.raw(rew[:, t]), _lib.raw(done[:, t]), _lib.raw(maxq[:, t]), T * E,
                                          _lib.p(sums), done_only, S, E, 0, 0, 0, rew_scale, part, _lib.stream_ptr()),
                   "pqn_rollout_act_step")
        for s in range(S):
            qs = q.reshape(S, E, A)[s]
            a = R.eps_greedy(jr.split(step_keys[s, 0], E), qs, eps)
            o_obs[s], o_st[s], r, d, info = oenv.step(jr.split(step_keys[s, 1], E), o_st[s], a)
            assert np.array_equal(act[s, t].cpu().numpy(), a), (t, s)
            assert np.array_equal(rew[s, t].cpu().numpy().view(np.int32),
                                  (np.float32(rew_scale) * r).astype(np.float32).view(np.int32)), (t, s)
            assert np.array_equal(done[s, t].cpu().numpy().astype(bool), d), (t, s)
            assert np.array_equal(maxq[s, t].cpu().numpy(), qs.max(-1)), (t, s)
            assert np.array_equal(obs_buf[s, t + 1].cpu().numpy().view(np.int32), o_obs[s].view(np.int32)), (t, s)
            assert_state(name, state[:, s * E:(s + 1) * E], o_st[s], (t, s))
            m = d if done_only else np.ones(E, bool)
            o_sums[s] += [info["returned_episode_returns"][m].astype(np.float64).sum(),
                          info["returned_episode_lengths"][m].sum(), info["timestep"][m].sum(), d.sum(),
                          info["discount"][m].sum()]
    assert np.array_equal(sums.cpu().numpy(), o_sums)
    assert o_sums[:, 3].min() > 0


# --------------------------------------------------------------------------- #
# networks at D = 64
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("H", [64, 128, 256, 512])
def test_mlp_forward_and_loss_grad_at_d64(H, tc_path):
    GX.test_mlp_forward_and_loss_grad_at_new_widths(64, H, tc_path)


@pytest.mark.parametrize("H", [64, 128, 256, 512])
def test_rnn_step_and_window_loss_grad_at_d64(H, tc_path):
    GX.test_rnn_step_and_window_loss_grad_at_new_widths(64, H, tc_path)


@pytest.mark.parametrize("norm_type,norm_input", GX.NORMS6)
def test_rnn_norm_variants_at_d64(norm_type, norm_input, tc_path):
    GX.test_rnn_norm_variants_at_wide_inputs(norm_type, norm_input, 64, tc_path)


@pytest.mark.parametrize("norm_type,norm_input", GX.NORMS6)
def test_mlp_norm_variants_at_d64(norm_type, norm_input, tc_path):
    """Eval forward, loss / gradients and the updated batch_stats (hidden in place, input through bn_sums) at D = 64
    on one-hot rows, as DeepSea feeds them."""
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_MLP, QNetworkSpec
    D, A, H, Ls, S, total, rows = 64, 2, 256, 2, 2, 300, 256
    spec = QNetworkSpec(NET_MLP, D, A, H, Ls, norm_type=norm_type, norm_input=norm_input)
    ps = [R.random_params(RN.mlp_param_shapes(D, A, H, Ls, norm_type), 30 + s) for s in range(S)]
    if norm_type == "batch_norm":
        for p in ps:
            for layer in range(Ls):
                p[f"Dense_{layer}/bias"] = np.zeros_like(p[f"Dense_{layer}/bias"])
    sts = [NS._rand_stats(RN.mlp_batch_stats(D, H, Ls, norm_type), 50 + s) for s in range(S)]
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    stf = torch.cat([spec.flatten_stats(st, 1, dev()) for st in sts], 0).contiguous()
    rng = np.random.default_rng(4)
    obs = np.zeros((S, total, D), np.float32)
    hot = rng.integers(0, D + 8, (S, total))                 # some rows all zeros, as once row == 8
    for s in range(S):
        on = hot[s] < D
        obs[s, np.nonzero(on)[0], hot[s][on]] = 1.0
    dev_obs = t_(obs, torch.float32)
    L_ = _lib.lib()
    q = torch.zeros((S * total, A), device=dev())
    ws_f, ws_l = NS._ws(spec, S, total), NS._ws(spec, S, rows)
    _lib.check(L_.pqn_qnet_forward(spec.desc, _lib.p(flat), _lib.p(stf), _lib.p(dev_obs), None, total, _lib.p(q), S,
                                   total, _lib.p(ws_f), _lib.stream_ptr()), "pqn_qnet_forward")
    torch.cuda.synchronize()
    qn = q.cpu().numpy().reshape(S, total, A)
    for s in range(S):
        ref, _ = RN.mlp_forward(ps[s], sts[s], obs[s], False, norm_type, norm_input)
        assert np.abs(qn[s] - ref).max() < 1e-5 * max(1.0, np.abs(ref).max()), (s, np.abs(qn[s] - ref).max())
    gather = np.stack([rng.permutation(total)[:rows] for _ in range(S)]).astype(np.int32)
    act = rng.integers(0, A, (S, total)).astype(np.int32)
    tgt = rng.standard_normal((S, total)).astype(np.float32)
    grads = torch.zeros_like(flat)
    ls, qs, bn = torch.zeros(S, device=dev()), torch.zeros(S, device=dev()), torch.zeros((S, 2 * D), device=dev())
    st_dev = stf.clone()
    tg_, ta_, tt_ = t_(gather, torch.int32), t_(act, torch.int32), t_(tgt, torch.float32)
    _lib.check(L_.pqn_qnet_loss_grad(spec.desc, _lib.p(flat), _lib.p(st_dev), _lib.p(dev_obs), _lib.p(tg_), total,
                                     _lib.p(ta_), _lib.p(tt_), total, _lib.p(grads), _lib.p(ls), _lib.p(qs), _lib.p(bn), S,
                                     rows, _lib.p(ws_l), _lib.stream_ptr()), "pqn_qnet_loss_grad")
    _lib.check(L_.pqn_bn_stats_update(_lib.p(st_dev), _lib.p(bn), S, D, spec.stats_total, float(rows), 0.99,
                                      _lib.stream_ptr()))
    torch.cuda.synchronize()
    gtree, sttree = spec.unflatten(grads), spec.unflatten_stats(st_dev)
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        st64 = {k: {kk: vv.astype(np.float64) for kk, vv in v.items()} for k, v in sts[s].items()}
        loss, q_sa, g, new_stats = RN.mlp_loss_and_grads(p64, st64, obs[s][gather[s]].astype(np.float64),
                                                         act[s][gather[s]], tgt[s][gather[s]].astype(np.float64),
                                                         norm_type, norm_input)
        assert abs(float(ls[s]) - loss) < 5e-5 * max(1.0, abs(loss)), (float(ls[s]), loss)
        assert abs(float(qs[s]) - q_sa.mean()) < 5e-5 * max(1.0, abs(q_sa.mean()))
        scale = max(np.abs(v).max() for v in g.values())
        errs = {}
        for path, *_ in spec.entries:
            name = "/".join(path)
            tol = 2e-5
            if norm_type == "batch_norm":
                tol = 5e-2 if name.startswith("Dense_") and name.endswith("/bias") and name != f"Dense_{Ls}/bias" else 2e-4
            errs[name] = (float(np.abs(NS._leaf(gtree, path, s) - g[name]).max() / scale), tol)
        bad = {k: v for k, v in errs.items() if not v[0] < v[1]}
        assert not bad, (bad, errs)
        for path, off, n in spec.stats_entries():
            d = sttree
            for k in path:
                d = d[k]
            want = new_stats["/".join(path)]
            assert np.allclose(d["mean"][s].cpu().numpy(), want["mean"], atol=2e-6), path
            assert np.allclose(d["var"][s].cpu().numpy(), want["var"], atol=2e-6), path


# --------------------------------------------------------------------------- #
# whole runs
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name", [SEA, UMB])
def test_mlp_two_updates_match_oracle(name, monkeypatch):
    """Two whole updates of pqn_gymnax (eps = 1) against the oracle's update_step."""
    import test_gpu_train as TT
    from purejaxql_b200 import pqn_gymnax
    monkeypatch.setitem(G._REGISTRY, name, B.CORES[name])
    cfg = TT._cfg(name, HIDDEN_SIZE=128, NUM_LAYERS=2, REW_SCALE=1.0, LAMBDA=0.95, NUM_ENVS=32, NUM_STEPS=16)
    TT._run_updates_against_oracle(pqn_gymnax, name, "mlp", True, cfg, nupd=2)


@pytest.mark.parametrize("name", [SEA, UMB])
def test_rnn_two_updates_match_oracle(name):
    """Two whole updates of pqn_rnn_gymnax (eps = 1; 8- and 10-step episodes end inside the 15-step windows) against
    the oracle replay of test_gpu_memory_chain."""
    import test_gpu_memory_chain as MCT
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = MCT._rnn_cfg(ENV_NAME=name)
    del cfg["ENV_KWARGS"]
    nupd = 2
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_rnn_gymnax.make_train(cfg)
    eng = train.engine
    assert eng.D == {SEA: 64, UMB: 3}[name]
    rngs = jr.split(jr.PRNGKey(32), 2)
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    out = train(rngs)
    dones = MCT._replay_rnn_updates(cfg, out, eng.spec.unflatten(cap["flat"]), eng.spec, rngs, nupd,
                                    lambda: B.make(name))
    assert dones > 0


def _rnn_run(name, graph, norm_type="layer_norm", norm_input=False):
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = NS._rnn_cfg(128, 2, env=name, nupd=5, graph=graph)
    cfg.update(NORM_TYPE=norm_type, NORM_INPUT=norm_input, TEST_NUM_STEPS=30)
    train = pqn_rnn_gymnax.make_train(cfg)
    out = train(jr.split(jr.PRNGKey(5), 2))
    assert train.engine.graph_captured == graph
    return (out["runner_state"][0].params_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy(),
            out["metrics"]["returned_episode_returns"].cpu().numpy(),
            out["metrics"]["test/returned_episode_lengths"].cpu().numpy(), out["runner_state"][4].cpu().numpy())


@pytest.mark.parametrize("name", [SEA, UMB])
@pytest.mark.parametrize("norm_type,norm_input", [("layer_norm", False), ("batch_norm", True)])
def test_rnn_cuda_graph_replay_equals_eager_and_repeats(name, norm_type, norm_input):
    eager, graph, again = (_rnn_run(name, False, norm_type, norm_input), _rnn_run(name, True, norm_type, norm_input),
                           _rnn_run(name, True, norm_type, norm_input))
    for a, b, c in zip(eager, graph, again):
        assert np.array_equal(a, b, equal_nan=True) and np.array_equal(b, c, equal_nan=True)
    assert np.isfinite(eager[1]).all() and (eager[3] == EPISODE[name]).all()


@pytest.mark.parametrize("name", [SEA, UMB, DISC])
def test_mlp_is_bit_reproducible(name):
    from purejaxql_b200 import pqn_gymnax
    outs = []
    for _ in range(2):
        cfg = NS._mlp_cfg(256, 2)
        cfg.update(ENV_NAME=name, NORM_INPUT=True)
        out = pqn_gymnax.make_train(cfg)(jr.split(jr.PRNGKey(11), 2))
        outs.append((out["runner_state"][0].params_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy()))
    assert np.isfinite(outs[0][1]).all()
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


RETURN_RANGE = {SEA: (-8 * 0.00125, 0.99), UMB: (-10.0, 10.0), DISC: (1.0, 1.1)}


@pytest.mark.parametrize("script,preset", [("pqn_gymnax", "pqn_cartpole"), ("pqn_rnn_gymnax", "pqn_rnn_cartpole")])
@pytest.mark.parametrize("name", [SEA, UMB, DISC])
def test_smoke_with_eval_and_save(script, preset, name, tmp_path):
    import importlib
    from purejaxql_b200 import config_loader
    from purejaxql_b200.utils.save_load import load_params
    mod = importlib.import_module(f"purejaxql_b200.{script}")
    c = config_loader.compose([f"+alg={preset}", f"alg.ENV_NAME={name}", "NUM_SEEDS=2", f"SAVE_PATH={tmp_path}",
                               "alg.TOTAL_TIMESTEPS=2e4", "alg.TOTAL_TIMESTEPS_DECAY=2e4", "alg.TEST_NUM_ENVS=16",
                               "alg.TEST_INTERVAL=0.5"])
    out = mod.single_run(c)
    m = out["metrics"]
    assert torch.isfinite(m["td_loss"]).all() and "test/returned_episode_returns" in m
    assert (m["test/returned_episode_lengths"] == EPISODE[name]).all()
    lo, hi = RETURN_RANGE[name]
    r = m["test/returned_episode_returns"]
    assert ((r >= lo - 1e-6) & (r <= hi + 1e-6)).all(), r
    files = [p for p in tmp_path.rglob("*.safetensors")]
    assert len(files) == 2, files
    tree = load_params(str(sorted(files)[0]))
    assert tree["Dense_0"]["kernel"].shape[0] == {SEA: 64, UMB: 3, DISC: 2}[name]
