"""GPU parity of the MLP and GRU Q-networks at the widths and depths beyond 128/256 x 1/2: HIDDEN_SIZE 64 (hidden
layers on the FFMA kernels with 64-wide tiles) and 512 (raw product + LayerNorm row kernel; wgmma hidden layers), and
up to four stacked hidden layers (the fp16-split pre-scaling of dz through every tensor-core layer).  Same tolerances
as the existing parity tests: forward 1e-5, loss / gradients 2e-5 of the gradient's scale against fp64 (BatchNorm
variants: the existing test_gpu_norm bounds)."""
import numpy as np
import pytest
import torch

from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_ref_norm as RN
from oracle import pqn_rnn_ref as RR

pytestmark = pytest.mark.gpu

MLP_SHAPES = [(4, 64, 2, 2), (6, 64, 3, 3), (4, 512, 1, 2), (6, 512, 4, 3), (4, 128, 3, 2), (3, 256, 4, 2)]


def dev():
    return torch.device("cuda:0")


def t_(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


def _ws(spec, S, rows):
    from purejaxql_b200 import _lib
    return torch.empty(int(_lib.lib().pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())


def _leaf(tree, path, s):
    d = tree
    for k in path:
        d = d[k]
    return d[s].cpu().numpy()


@pytest.fixture(params=[2, 0], ids=["hidden_layers_wgmma_f16split", "ffma"])
def mlp_path(request):
    from purejaxql_b200 import _lib
    _lib.check(_lib.lib().pqn_set_tensor_core_path(request.param))
    yield request.param
    _lib.lib().pqn_set_tensor_core_path(2)


def _mlp_setup(D, H, L, A, S, seed):
    from purejaxql_b200.networks import NET_MLP, QNetworkSpec
    spec = QNetworkSpec(NET_MLP, D, A, H, L)
    ps = [R.random_params(R.mlp_param_shapes(D, A, H, L), seed + s) for s in range(S)]
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    return spec, ps, flat


@pytest.mark.parametrize("D,H,L,A", MLP_SHAPES)
def test_mlp_forward_matches_oracle(D, H, L, A, mlp_path):
    from purejaxql_b200 import _lib
    S, rows = 3, 515
    spec, ps, flat = _mlp_setup(D, H, L, A, S, 20)
    obs = np.random.default_rng(2).standard_normal((S, rows, D)).astype(np.float32)
    q = torch.zeros((S * rows, A), device=dev())
    to_, ws = t_(obs, torch.float32), _ws(spec, S, rows)
    _lib.check(_lib.lib().pqn_qnet_forward(spec.desc, _lib.p(flat), None, _lib.p(to_), None, rows, _lib.p(q), S, rows,
                                           _lib.p(ws), _lib.stream_ptr()), "pqn_qnet_forward")
    q = q.cpu().numpy().reshape(S, rows, A)
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        err = np.abs(q[s] - R.mlp_forward(p64, obs[s].astype(np.float64))).max()
        assert err < 1e-5, (s, err)


@pytest.mark.parametrize("D,H,L,A", MLP_SHAPES)
def test_mlp_loss_grad_matches_fp64_oracle(D, H, L, A, mlp_path):
    from purejaxql_b200 import _lib
    rng = np.random.default_rng(7)
    S, total, rows = 3, 1400, 515
    spec, ps, flat = _mlp_setup(D, H, L, A, S, 30)
    obs = rng.standard_normal((S, total, D)).astype(np.float32)
    gather = np.stack([rng.permutation(total)[:rows] for _ in range(S)]).astype(np.int32)
    act = rng.integers(0, A, (S, total)).astype(np.int32)
    tgt = rng.standard_normal((S, total)).astype(np.float32)
    grads = torch.zeros_like(flat)
    ls, qs, bn = torch.zeros(S, device=dev()), torch.zeros(S, device=dev()), torch.zeros((S, 2 * D), device=dev())
    to_, tg_, ta_, tt_, ws = t_(obs, torch.float32), t_(gather, torch.int32), t_(act, torch.int32), t_(tgt, torch.float32), \
        _ws(spec, S, rows)
    _lib.check(_lib.lib().pqn_qnet_loss_grad(spec.desc, _lib.p(flat), None, _lib.p(to_), _lib.p(tg_), total, _lib.p(ta_),
                                             _lib.p(tt_), total, _lib.p(grads), _lib.p(ls), _lib.p(qs), _lib.p(bn), S, rows,
                                             _lib.p(ws), _lib.stream_ptr()), "pqn_qnet_loss_grad")
    torch.cuda.synchronize()
    gtree = spec.unflatten(grads)
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        o = obs[s][gather[s]].astype(np.float64)
        loss, q_sa, g = R.mlp_loss_and_grads(p64, o, act[s][gather[s]], tgt[s][gather[s]].astype(np.float64))
        assert abs(float(ls[s]) - loss) < 1e-5 * max(1, abs(loss)) and abs(float(qs[s]) - q_sa.mean()) < 1e-5
        for path, *_ in spec.entries:
            ref = g["/".join(path)]
            scale = max(np.abs(ref).max(), 1e-3)
            err = np.abs(_leaf(gtree, path, s) - ref).max()
            assert err < 2e-5 * scale + 1e-7, (path, err, scale)


def _rand_stats(stats, seed):
    rng = np.random.default_rng(seed)
    return {k: {"mean": (0.1 * rng.standard_normal(v["mean"].shape)).astype(np.float32),
                "var": (0.5 + rng.random(v["var"].shape)).astype(np.float32)} for k, v in stats.items()}


NORM_VARIANTS = [("batch_norm", False), ("none", False), ("layer_norm", True), ("batch_norm", True)]


@pytest.mark.parametrize("H,L", [(64, 3), (512, 3)])
@pytest.mark.parametrize("norm_type,norm_input", NORM_VARIANTS)
def test_mlp_norm_variants_match_oracle(H, L, norm_type, norm_input):
    """Eval forward, loss / gradients and the updated batch_stats of the modular NORM_TYPE / NORM_INPUT path at three
    hidden layers: the hidden BatchNorms' statistics and the input BatchNorm's must not share a table."""
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_MLP, QNetworkSpec
    D, A, S, total, rows = 4, 2, 2, 300, 256
    spec = QNetworkSpec(NET_MLP, D, A, H, L, norm_type=norm_type, norm_input=norm_input)
    ps = [R.random_params(RN.mlp_param_shapes(D, A, H, L, norm_type), 30 + s) for s in range(S)]
    if norm_type == "batch_norm":   # a bias in front of a BatchNorm is a no-op (see test_gpu_norm)
        for p in ps:
            for layer in range(L):
                p[f"Dense_{layer}/bias"] = np.zeros_like(p[f"Dense_{layer}/bias"])
    sts = [_rand_stats(RN.mlp_batch_stats(D, H, L, norm_type), 50 + s) for s in range(S)]
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    stf = torch.cat([spec.flatten_stats(st, 1, dev()) for st in sts], 0).contiguous()
    obs = np.random.default_rng(4).standard_normal((S, total, D)).astype(np.float32) * np.array([1, 2, .2, 3], np.float32)
    dev_obs = t_(obs, torch.float32)
    L_ = _lib.lib()
    # eval forward on the running statistics
    q = torch.zeros((S * total, A), device=dev())
    ws = _ws(spec, S, total)
    _lib.check(L_.pqn_qnet_forward(spec.desc, _lib.p(flat), _lib.p(stf), _lib.p(dev_obs), None, total, _lib.p(q), S, total,
                                   _lib.p(ws), _lib.stream_ptr()), "pqn_qnet_forward")
    torch.cuda.synchronize()
    qn = q.cpu().numpy().reshape(S, total, A)
    for s in range(S):
        ref, _ = RN.mlp_forward(ps[s], sts[s], obs[s], False, norm_type, norm_input)
        assert np.abs(qn[s] - ref).max() < 1e-5 * max(1.0, np.abs(ref).max()), (s, np.abs(qn[s] - ref).max())
    # training loss / gradients, batch_stats updated in place (hidden) and through bn_sums (input)
    rng = np.random.default_rng(7)
    gather = np.stack([rng.permutation(total)[:rows] for _ in range(S)]).astype(np.int32)
    act = rng.integers(0, A, (S, total)).astype(np.int32)
    tgt = rng.standard_normal((S, total)).astype(np.float32)
    grads = torch.zeros_like(flat)
    ls, qs, bn = torch.zeros(S, device=dev()), torch.zeros(S, device=dev()), torch.zeros((S, 2 * D), device=dev())
    st_dev = stf.clone()
    tg_, ta_, tt_, ws = t_(gather, torch.int32), t_(act, torch.int32), t_(tgt, torch.float32), _ws(spec, S, rows)
    _lib.check(L_.pqn_qnet_loss_grad(spec.desc, _lib.p(flat), _lib.p(st_dev), _lib.p(dev_obs), _lib.p(tg_), total,
                                     _lib.p(ta_), _lib.p(tt_), total, _lib.p(grads), _lib.p(ls), _lib.p(qs), _lib.p(bn), S,
                                     rows, _lib.p(ws), _lib.stream_ptr()), "pqn_qnet_loss_grad")
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
            if norm_type == "batch_norm":   # fp32 batch statistics; dead biases in front of a BatchNorm
                tol = 5e-2 if name.startswith("Dense_") and name.endswith("/bias") and name != f"Dense_{L}/bias" else 2e-4
            errs[name] = (float(np.abs(_leaf(gtree, path, s) - g[name]).max() / scale), tol)
        bad = {k: v for k, v in errs.items() if not v[0] < v[1]}
        assert not bad, (bad, errs)
        for path, off, n in spec.stats_entries():
            d = sttree
            for k in path:
                d = d[k]
            want = new_stats["/".join(path)]
            assert np.allclose(d["mean"][s].cpu().numpy(), want["mean"], atol=2e-6), path
            assert np.allclose(d["var"][s].cpu().numpy(), want["var"], atol=2e-6), path


def _rnn_setup(S, D, A, H, L):
    from purejaxql_b200.networks import NET_RNN, QNetworkSpec
    spec = QNetworkSpec(NET_RNN, D, A, H, L)
    ps = [R.random_params(RR.rnn_param_shapes(D, A, H, L), 70 + s) for s in range(S)]
    for p in ps:   # recurrent kernels at an orthogonal-like scale (spectral norm ~ 1)
        for gate in ("hr", "hz", "hn"):
            p[RR.G + gate + "/kernel"] = (p[RR.G + gate + "/kernel"] * 0.5 * np.sqrt(128.0 / H)).astype(np.float32)
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    return spec, ps, flat


RNN_SHAPES = [(H, L) for H in (64, 512) for L in (1, 3, 4)]


@pytest.mark.parametrize("H,L", RNN_SHAPES)
def test_rnn_step_matches_oracle(H, L):
    from purejaxql_b200 import _lib
    S, E, D, A = 2, 37, 4, 2
    spec, ps, flat = _rnn_setup(S, D, A, H, L)
    rng = np.random.default_rng(0)
    hs = rng.standard_normal((S, E, H)).astype(np.float32) * 0.5
    obs = rng.standard_normal((S, E, D)).astype(np.float32)
    ld = rng.random((S, E)) < 0.3
    la = rng.integers(0, A, (S, E)).astype(np.int32)
    hs_d, obs_d, ld_d, la_d = t_(hs, torch.float32), t_(obs, torch.float32), t_(ld.astype(np.uint8), torch.uint8), t_(la, torch.int32)
    q = torch.zeros((S * E, A), device=dev())
    ws = _ws(spec, S, E)
    _lib.check(_lib.lib().pqn_rnn_step(spec.desc, _lib.p(flat), _lib.p(hs_d), _lib.p(obs_d), E, _lib.p(ld_d), _lib.p(la_d),
                                       _lib.p(q), S, E, _lib.p(ws), _lib.stream_ptr()), "pqn_rnn_step")
    torch.cuda.synchronize()
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        new_h, qq = RR.rnn_forward(p64, hs[s].astype(np.float64), obs[s][None].astype(np.float64), ld[s][None], la[s][None])
        assert np.abs(q.cpu().numpy().reshape(S, E, A)[s] - qq[0]).max() < 1e-5
        assert np.abs(hs_d.cpu().numpy()[s] - new_h).max() < 1e-5


@pytest.mark.parametrize("H,L", RNN_SHAPES)
def test_rnn_loss_grad_matches_fp64_oracle(H, L):
    from purejaxql_b200 import _lib
    S, D, A, T, B = 2, 4, 2, 9, 5
    spec, ps, flat = _rnn_setup(S, D, A, H, L)
    rng = np.random.default_rng(1)
    hs0 = rng.standard_normal((S, B, H)).astype(np.float32) * 0.5
    obs = rng.standard_normal((S, T, B, D)).astype(np.float32)
    ld = rng.random((S, T, B)) < 0.15
    la = rng.integers(0, A, (S, T, B)).astype(np.int32)
    ac = rng.integers(0, A, (S, T, B)).astype(np.int32)
    rw = (rng.random((S, T, B)) * 0.1).astype(np.float32)
    dn = rng.random((S, T, B)) < 0.15
    bufs = [t_(hs0, torch.float32), t_(obs, torch.float32), t_(ld.astype(np.uint8), torch.uint8), t_(la, torch.int32),
            t_(ac, torch.int32), t_(rw, torch.float32), t_(dn.astype(np.uint8), torch.uint8)]
    grads = torch.zeros_like(flat)
    ls, qs = torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
    ws = _ws(spec, S, T * B)
    _lib.check(_lib.lib().pqn_rnn_loss_grad(spec.desc, _lib.p(flat), *[_lib.p(b) for b in bufs], _lib.p(grads), _lib.p(ls),
                                            _lib.p(qs), S, T, B, 0.99, 0.95, _lib.p(ws), _lib.stream_ptr()),
               "pqn_rnn_loss_grad")
    torch.cuda.synchronize()
    gtree = spec.unflatten(grads)
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        loss, chosen, g = RR.rnn_loss_and_grads(p64, hs0[s].astype(np.float64), obs[s].astype(np.float64), ld[s], la[s],
                                                ac[s], rw[s].astype(np.float64), dn[s], 0.99, 0.95)
        assert abs(float(ls[s]) - loss) < 1e-5 * max(1.0, abs(loss)), (float(ls[s]), loss)
        assert abs(float(qs[s]) - chosen.mean()) < 1e-5 * max(1.0, abs(chosen.mean()))
        scale = max(np.abs(v).max() for v in g.values())
        for path, *_ in spec.entries:
            err = np.abs(_leaf(gtree, path, s) - g["/".join(path)]).max()
            assert err < 2e-5 * scale, (path, err, scale)


# ---- whole runs through train() ------------------------------------------------------------------------------------
def _mlp_cfg(H, L, nupd=2):
    cfg = dict(ENV_NAME="CartPole-v1", NUM_ENVS=64, NUM_STEPS=8, NUM_MINIBATCHES=4, NUM_EPOCHS=2, EPS_START=1.0,
               EPS_FINISH=0.05, EPS_DECAY=0.5, LR=1e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65, NORM_TYPE="layer_norm",
               NORM_INPUT=False, HIDDEN_SIZE=H, NUM_LAYERS=L, LR_LINEAR_DECAY=True, REW_SCALE=0.1, WANDB_MODE="disabled",
               TEST_DURING_TRAINING=False)
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    return cfg


def _rnn_cfg(H, L, env="CartPole-v1", nupd=2, graph=None):
    cfg = dict(ENV_NAME=env, NUM_ENVS=8, NUM_STEPS=12, MEMORY_WINDOW=3, NUM_MINIBATCHES=4, NUM_EPOCHS=2, EPS_START=1.0,
               EPS_FINISH=0.1, EPS_DECAY=0.5, LR=1e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.95, NORM_TYPE="layer_norm",
               NORM_INPUT=False, HIDDEN_SIZE=H, NUM_LAYERS=L, LR_LINEAR_DECAY=True, REW_SCALE=0.1, WANDB_MODE="disabled",
               TEST_DURING_TRAINING=True, TEST_INTERVAL=0.4, TEST_NUM_ENVS=8, EPS_TEST=0.0)
    if graph is not None:
        cfg["CUDA_GRAPH"] = graph
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    return cfg


def test_mlp_train_two_updates_match_oracle_512x4():
    """Two whole updates of pqn_gymnax CartPole at 512 x 4 (eps = 1) against the oracle's update_step, through the
    engine parity helper of test_gpu_train: episode metrics, td_loss, mean q and the key chain of every seed."""
    import test_gpu_train as TT
    from purejaxql_b200 import pqn_gymnax
    cfg = TT._cfg("CartPole-v1", HIDDEN_SIZE=512, NUM_LAYERS=4, REW_SCALE=0.1, LAMBDA=0.95, NUM_ENVS=32, NUM_STEPS=16)
    TT._run_updates_against_oracle(pqn_gymnax, "CartPole-v1", "mlp", True, cfg, nupd=2)


@pytest.mark.parametrize("kind", ["mlp", "rnn"])
def test_train_is_bit_reproducible_512x4(kind):
    from purejaxql_b200 import pqn_gymnax, pqn_rnn_gymnax
    outs = []
    for _ in range(2):
        if kind == "mlp":
            out = pqn_gymnax.make_train(_mlp_cfg(512, 4))(jr.split(jr.PRNGKey(11), 2))
        else:
            out = pqn_rnn_gymnax.make_train(_rnn_cfg(512, 4))(jr.split(jr.PRNGKey(11), 2))
        outs.append((out["runner_state"][0].params_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy()))
    assert np.isfinite(outs[0][1]).all()
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_rnn_cuda_graph_replay_equals_eager_512x4():
    from purejaxql_b200 import pqn_rnn_gymnax
    outs = []
    for graph in (False, True):
        train = pqn_rnn_gymnax.make_train(_rnn_cfg(512, 4, nupd=4, graph=graph))
        out = train(jr.split(jr.PRNGKey(5), 2))
        assert train.engine.graph_captured == graph
        outs.append((out["runner_state"][0].params_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy(),
                     out["metrics"]["test/returned_episode_returns"].cpu().numpy(), out["runner_state"][4].cpu().numpy()))
    for a, b in zip(*outs):
        assert np.array_equal(a, b, equal_nan=True)


def test_rnn_memory_chain_update_steps_match_oracle_64x3():
    """Two whole updates of pqn_rnn_gymnax MemoryChain at 64 x 3 (eps = 1) against the oracle replay of
    test_gpu_memory_chain: per-update td_loss, final parameters and final key of every seed."""
    import bsuite_oracle as MC
    import test_gpu_memory_chain as TM
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = TM._rnn_cfg(HIDDEN_SIZE=64, NUM_LAYERS=3)
    nupd = 2
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_rnn_gymnax.make_train(cfg)
    eng = train.engine
    rngs = jr.split(jr.PRNGKey(31), 2)
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    out = train(rngs)
    dones = TM._replay_rnn_updates(cfg, out, eng.spec.unflatten(cap["flat"]), eng.spec, rngs, nupd,
                                   lambda: MC.make(4, flatten=True))
    assert dones > 0


def test_memory_chain_preset_at_the_reference_network_defaults():
    """+alg=pqn_rnn_memory_chain with RNNQNetwork's own defaults (hidden_size 512, num_layers 4), with evaluation."""
    from purejaxql_b200 import config_loader, pqn_rnn_gymnax
    c = config_loader.compose(["+alg=pqn_rnn_memory_chain", "NUM_SEEDS=1", "SAVE_PATH=null", "alg.HIDDEN_SIZE=512",
                               "alg.NUM_LAYERS=4"])
    cfg = {**c, **c["alg"]}
    per_update = cfg["NUM_STEPS"] * cfg["NUM_ENVS"]
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = 3 * per_update
    out = pqn_rnn_gymnax.make_train(cfg)(jr.split(jr.PRNGKey(0), 1))
    m = out["metrics"]
    assert m["td_loss"].shape[-1] == 3 and torch.isfinite(m["td_loss"]).all()
    assert "test/returned_episode_returns" in m and torch.isfinite(m["test/returned_episode_returns"]).all()
