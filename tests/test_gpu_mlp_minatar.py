"""GPU parity of the MLP Q-network on packed MinAtar observations (PQN_NET_MLP_BITS: pqn_gymnax.py's QNetwork behind
FlattenObservationWrapper) against the fp64 oracles fed the unpacked rows as floats: forward to 1e-5, loss / gradients to
2e-5 of the gradient's scale (BatchNorm variants: the test_gpu_norm bounds), the batch_stats side effects, whole updates
through pqn_gymnax.make_train (eager and CUDA-graph replay), determinism and a smoke run per game.  Every comparison is
made on tensor-core path 2 (Dense_0 on mma.sync from the bits) and on path 0 (expanded fp32 rows, FFMA kernels)."""
import functools

import numpy as np
import pytest
import torch

from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_ref_norm as RN

pytestmark = pytest.mark.gpu

GAMES = {"Breakout-MinAtar": 4, "Asterix-MinAtar": 4, "SpaceInvaders-MinAtar": 6, "Freeway-MinAtar": 7}


def dev():
    return torch.device("cuda:0")


def t_(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


def _pack(bits):
    """{0,1} rows [n, D] -> int32 [n, packed words] (bit f of a row = element f; rows padded to 16 bytes)."""
    n, nb = bits.shape
    pw = ((nb + 31) // 32 + 3) // 4 * 4
    padded = np.zeros((n, pw * 32), np.uint8)
    padded[:, :nb] = bits
    return np.ascontiguousarray(np.packbits(padded, axis=-1, bitorder="little")).view("<u4").view(np.int32)


@functools.lru_cache(maxsize=None)
def _env_bits(game, n, seed):
    """Real observations (sparse: a few % ones) after 25 random steps, flattened: [n, 100 * C] uint8."""
    env = G.make(game, log=False)
    obs, st = env.reset(jr.split(jr.PRNGKey(seed), n))
    rng = np.random.default_rng(seed)
    for t in range(25):
        obs, st, *_ = env.step(jr.split(jr.PRNGKey(seed * 1000 + t), n), st,
                               rng.integers(0, env.num_actions, n).astype(np.int32))
    return (np.asarray(obs).reshape(n, -1) != 0).astype(np.uint8)


def _rows(game, S, total, seed):
    """Per seed: half real env observations, half dense random bits (p = 0.5), shuffled."""
    D = 100 * GAMES[game]
    rng = np.random.default_rng(seed)
    out = []
    for s in range(S):
        real = _env_bits(game, total // 2, seed + s)
        dense = (rng.random((total - total // 2, D)) < 0.5).astype(np.uint8)
        x = np.concatenate([real, dense])
        out.append(x[rng.permutation(total)])
    return np.stack(out)


@pytest.fixture
def path():
    from purejaxql_b200 import _lib
    yield lambda p: _lib.check(_lib.lib().pqn_set_tensor_core_path(p))
    _lib.lib().pqn_set_tensor_core_path(2)


def _ws(spec, S, rows):
    from purejaxql_b200 import _lib
    return torch.empty(int(_lib.lib().pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())


def _leaf(tree, path_, s):
    d = tree
    for k in path_:
        d = d[k]
    return d[s].cpu().numpy()


def _spec(game, H, L, A=None, norm_type="layer_norm", norm_input=False):
    from purejaxql_b200.networks import NET_MLP_BITS, QNetworkSpec
    D = 100 * GAMES[game]
    return QNetworkSpec(NET_MLP_BITS, D, A or 3, H, L, norm_type=norm_type, norm_input=norm_input)


@pytest.mark.parametrize("L", [1, 2, 4])
@pytest.mark.parametrize("H", [64, 128, 256, 512])
@pytest.mark.parametrize("game", sorted(GAMES))
def test_forward_matches_oracle(game, H, L, path):
    from purejaxql_b200 import _lib
    S, total, rows, A = 2, 402, 333, 5
    spec = _spec(game, H, L, A)
    D = spec.in_c
    ps = [R.random_params(R.mlp_param_shapes(D, A, H, L), 20 + s) for s in range(S)]
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    x = _rows(game, S, total, 3)
    gather = np.stack([np.random.default_rng(s).permutation(total)[:rows] for s in range(S)]).astype(np.int32)
    obs, tg = t_(np.stack([_pack(x[s]) for s in range(S)]), torch.int32), t_(gather, torch.int32)
    for p in (2, 0):
        path(p)
        for g, n in ((tg, rows), (None, total)):
            q = torch.zeros((S * n, A), device=dev())
            ws = _ws(spec, S, n)
            _lib.check(_lib.lib().pqn_qnet_forward(spec.desc, _lib.p(flat), None, _lib.p(obs), _lib.p(g), total, _lib.p(q),
                                                   S, n, _lib.p(ws), _lib.stream_ptr()), "pqn_qnet_forward")
            qn = q.cpu().numpy().reshape(S, n, A)
            for s in range(S):
                xs = x[s][gather[s]] if g is not None else x[s]
                ref = R.mlp_forward({k: v.astype(np.float64) for k, v in ps[s].items()}, xs.astype(np.float64))
                err = np.abs(qn[s] - ref).max()
                assert err < 1e-5, (p, g is not None, s, err)


@pytest.mark.parametrize("game,H,L,S,total,rows", [
    ("Breakout-MinAtar", 256, 2, 1, 70000, 65536),
    ("Freeway-MinAtar", 512, 1, 1, 65536, 65536),
    ("SpaceInvaders-MinAtar", 64, 3, 2, 5000, 4001),
    ("Asterix-MinAtar", 128, 4, 3, 1500, 999),
])
def test_loss_grad_matches_fp64_oracle(game, H, L, S, total, rows, path):
    from purejaxql_b200 import _lib
    A = 4
    spec = _spec(game, H, L, A)
    D = spec.in_c
    rng = np.random.default_rng(7)
    ps = [R.random_params(R.mlp_param_shapes(D, A, H, L), 30 + s) for s in range(S)]
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    x = _rows(game, S, total, 11)
    x[:, :, 3:11] = 0          # feature columns that are all 0 ...
    x[:, :, 40:47] = 1         # ... and all 1
    gather = np.stack([rng.permutation(total)[:rows] for _ in range(S)]).astype(np.int32)
    act = rng.integers(0, A, (S, total)).astype(np.int32)
    tgt = rng.standard_normal((S, total)).astype(np.float32)
    obs, tg, ta, tt = (t_(np.stack([_pack(x[s]) for s in range(S)]), torch.int32), t_(gather, torch.int32),
                       t_(act, torch.int32), t_(tgt, torch.float32))
    refs = []
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        refs.append(R.mlp_loss_and_grads(p64, x[s][gather[s]].astype(np.float64), act[s][gather[s]],
                                         tgt[s][gather[s]].astype(np.float64)))
    out = {}
    for p in (2, 0):
        path(p)
        grads = torch.zeros_like(flat)
        ls, qs, bn = torch.zeros(S, device=dev()), torch.zeros(S, device=dev()), torch.zeros((S, 2 * D), device=dev())
        ws = _ws(spec, S, rows)
        _lib.check(_lib.lib().pqn_qnet_loss_grad(spec.desc, _lib.p(flat), None, _lib.p(obs), _lib.p(tg), total, _lib.p(ta),
                                                 _lib.p(tt), total, _lib.p(grads), _lib.p(ls), _lib.p(qs), _lib.p(bn), S,
                                                 rows, _lib.p(ws), _lib.stream_ptr()), "pqn_qnet_loss_grad")
        torch.cuda.synchronize()
        gtree = spec.unflatten(grads)
        out[p] = grads.cpu().numpy()
        for s in range(S):
            loss, q_sa, g = refs[s]
            assert abs(float(ls[s]) - loss) < 1e-5 * max(1, abs(loss)) and abs(float(qs[s]) - q_sa.mean()) < 1e-5
            scale = max(np.abs(v).max() for v in g.values())     # the gradient's scale (as test_gpu_norm)
            for path_, *_ in spec.entries:
                err = np.abs(_leaf(gtree, path_, s) - g["/".join(path_)]).max()
                assert err < 2e-5 * scale, (p, path_, err, scale)
            # BatchNorm_0 statistics of the minibatch: per-feature popcounts
            cnt = x[s][gather[s]].sum(0).astype(np.float32)
            assert np.array_equal(bn[s].cpu().numpy(), np.concatenate([cnt, cnt])), p
        lay = spec.layout
        w0 = out[p].reshape(S, -1)[:, lay.d0_w:lay.d0_w + D * H].reshape(S, D, H)
        assert not w0[:, 3:11].any(), p       # all-0 feature columns have an exactly zero kernel gradient


def _rand_stats(stats, seed):
    rng = np.random.default_rng(seed)
    return {k: {"mean": (0.1 * rng.standard_normal(v["mean"].shape)).astype(np.float32),
                "var": (0.5 + rng.random(v["var"].shape)).astype(np.float32)} for k, v in stats.items()}


VARIANTS = [("layer_norm", False), ("layer_norm", True), ("batch_norm", False), ("batch_norm", True), ("none", False),
            ("none", True)]


@pytest.mark.parametrize("norm_type,norm_input", VARIANTS)
def test_norm_variants_match_oracle(norm_type, norm_input, path):
    """Eval forward (running statistics), training loss / gradients and the batch_stats after the update, BatchNorm_0's
    running statistics included (also under the default network, whose BatchNorm_0 output is discarded)."""
    from purejaxql_b200 import _lib
    game, H, L, A, S, total, rows = "Breakout-MinAtar", 128, 2, 3, 2, 300, 256
    spec = _spec(game, H, L, A, norm_type, norm_input)
    D = spec.in_c
    ps = [R.random_params(RN.mlp_param_shapes(D, A, H, L, norm_type), 30 + s) for s in range(S)]
    if norm_type == "batch_norm":   # a bias in front of a BatchNorm is a no-op (see test_gpu_norm)
        for p in ps:
            for layer in range(L):
                p[f"Dense_{layer}/bias"] = np.zeros_like(p[f"Dense_{layer}/bias"])
    sts = [_rand_stats(RN.mlp_batch_stats(D, H, L, norm_type), 50 + s) for s in range(S)]
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    stf = torch.cat([spec.flatten_stats(st, 1, dev()) for st in sts], 0).contiguous()
    x = _rows(game, S, total, 5)
    x[:, :, 7:12] = 0
    x[:, :, 20:23] = 1
    obs = t_(np.stack([_pack(x[s]) for s in range(S)]), torch.int32)
    rng = np.random.default_rng(7)
    gather = np.stack([rng.permutation(total)[:rows] for _ in range(S)]).astype(np.int32)
    act = rng.integers(0, A, (S, total)).astype(np.int32)
    tgt = rng.standard_normal((S, total)).astype(np.float32)
    tg, ta, tt = t_(gather, torch.int32), t_(act, torch.int32), t_(tgt, torch.float32)
    L_ = _lib.lib()
    for p in (2, 0):
        path(p)
        q = torch.zeros((S * total, A), device=dev())
        ws = _ws(spec, S, total)
        _lib.check(L_.pqn_qnet_forward(spec.desc, _lib.p(flat), _lib.p(stf), _lib.p(obs), None, total, _lib.p(q), S, total,
                                       _lib.p(ws), _lib.stream_ptr()), "pqn_qnet_forward")
        qn = q.cpu().numpy().reshape(S, total, A)
        for s in range(S):
            ref, _ = RN.mlp_forward(ps[s], sts[s], x[s].astype(np.float32), False, norm_type, norm_input)
            assert np.abs(qn[s] - ref).max() < 1e-5 * max(1.0, np.abs(ref).max()), (p, s, np.abs(qn[s] - ref).max())
        grads = torch.zeros_like(flat)
        ls, qs, bn = torch.zeros(S, device=dev()), torch.zeros(S, device=dev()), torch.zeros((S, 2 * D), device=dev())
        st_dev = stf.clone()
        ws = _ws(spec, S, rows)
        _lib.check(L_.pqn_qnet_loss_grad(spec.desc, _lib.p(flat), _lib.p(st_dev), _lib.p(obs), _lib.p(tg), total,
                                         _lib.p(ta), _lib.p(tt), total, _lib.p(grads), _lib.p(ls), _lib.p(qs), _lib.p(bn), S,
                                         rows, _lib.p(ws), _lib.stream_ptr()), "pqn_qnet_loss_grad")
        _lib.check(L_.pqn_bn_stats_update(_lib.p(st_dev), _lib.p(bn), S, D, spec.stats_total, float(rows), 0.99,
                                          _lib.stream_ptr()))
        torch.cuda.synchronize()
        gtree, sttree = spec.unflatten(grads), spec.unflatten_stats(st_dev)
        for s in range(S):
            p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
            st64 = {k: {kk: vv.astype(np.float64) for kk, vv in v.items()} for k, v in sts[s].items()}
            loss, q_sa, g, new_stats = RN.mlp_loss_and_grads(p64, st64, x[s][gather[s]].astype(np.float64),
                                                             act[s][gather[s]], tgt[s][gather[s]].astype(np.float64),
                                                             norm_type, norm_input)
            assert abs(float(ls[s]) - loss) < 5e-5 * max(1.0, abs(loss)), (p, float(ls[s]), loss)
            assert abs(float(qs[s]) - q_sa.mean()) < 5e-5 * max(1.0, abs(q_sa.mean()))
            scale = max(np.abs(v).max() for v in g.values())
            errs = {}
            for path_, *_ in spec.entries:
                name = "/".join(path_)
                tol = 2e-5
                if norm_type == "batch_norm":   # fp32 batch statistics; dead biases in front of a BatchNorm
                    tol = 5e-2 if name.startswith("Dense_") and name.endswith("/bias") and name != f"Dense_{L}/bias" else 2e-4
                errs[name] = (float(np.abs(_leaf(gtree, path_, s) - g[name]).max() / scale), tol)
            bad = {k: v for k, v in errs.items() if not v[0] < v[1]}
            assert not bad, (p, bad, errs)
            for path_, off, n in spec.stats_entries():
                d = sttree
                for k in path_:
                    d = d[k]
                want = new_stats["/".join(path_)]
                assert np.allclose(d["mean"][s].cpu().numpy(), want["mean"], atol=2e-6), (p, path_)
                assert np.allclose(d["var"][s].cpu().numpy(), want["var"], atol=2e-6), (p, path_)


def _cfg(env, **kw):
    c = dict(ENV_NAME=env, NUM_ENVS=64, NUM_STEPS=8, NUM_MINIBATCHES=4, NUM_EPOCHS=2, EPS_START=1.0, EPS_FINISH=1.0,
             EPS_DECAY=0.1, LR=5e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.95, REW_SCALE=0.1, NORM_TYPE="layer_norm",
             LR_LINEAR_DECAY=True, WANDB_MODE="disabled", TEST_DURING_TRAINING=False, HIDDEN_SIZE=128, NUM_LAYERS=2)
    c.update(kw)
    return c


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda_graph"])
@pytest.mark.parametrize("game", ["Breakout-MinAtar", "Freeway-MinAtar"])
def test_update_steps_match_oracle(game, graph):
    """Whole `_update_step`s through pqn_gymnax.make_train against the oracle's update_step(kind="mlp") on the flattened
    observations (eps = 1: integer-exact rollouts): metrics of every update, the key chain, the parameters and the
    BatchNorm_0 running statistics after the last one."""
    from purejaxql_b200 import pqn_gymnax
    nupd = 4 if graph else 2
    cfg = _cfg(game, CUDA_GRAPH=graph)
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_gymnax.make_train(cfg)
    eng = train.engine
    S = 2
    rngs = jr.split(jr.PRNGKey(3), S)
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    out = train(rngs)
    assert eng.graph_captured == graph
    ts = out["runner_state"][0]
    tree0 = eng.spec.unflatten(cap["flat"])
    E = cfg["NUM_ENVS"]
    assert "env_frame" not in out["metrics"]
    for s in range(S):
        params = {"/".join(p): _leaf(tree0, p, s).astype(np.float32) for p, *_ in eng.spec.entries}
        K1 = jr.split(rngs[s], 2)[0]
        K2 = jr.split(K1, 2)[0]
        k = jr.split(K2, 2); K3, kR = k[0], k[1]
        env = G.make(game, flatten=True)
        obs, st = env.reset(jr.split(kR, E))
        rng = jr.split(K3, 2)[1]
        opt = R.opt_init(params)
        D = eng.spec.in_c
        bs = {"mean": np.zeros(D, np.float32), "var": np.ones(D, np.float32)}
        total = cfg["NUM_UPDATES_DECAY"] * cfg["NUM_MINIBATCHES"] * cfg["NUM_EPOCHS"]
        lr_fn = lambda i: R.linear_schedule(cfg["LR"], 1e-20, total, i)
        for u in range(nupd):
            params, opt, bs, obs, st, rng, m, tr, tg = R.update_step(env, "mlp", params, opt, bs, obs, st, rng, dict(cfg), u,
                                                                     lr_fn)
            got = {kk: float(v[s, u]) for kk, v in out["metrics"].items()}
            for kk in ("returned_episode_returns", "returned_episode_lengths", "timestep", "returned_episode", "discount"):
                assert abs(got[kk] - m[kk]) < 1e-6 * max(1, abs(m[kk])), (u, kk, got[kk], m[kk])
            assert abs(got["td_loss"] - m["td_loss"]) < 1e-4 * max(1.0, abs(m["td_loss"])), (u, got["td_loss"], m["td_loss"])
            assert abs(got["qvals"] - m["qvals"]) < 1e-4 * max(1.0, abs(m["qvals"])), u
        for p, *_ in eng.spec.entries:
            assert np.abs(_leaf(ts.params, p, s) - params["/".join(p)]).max() < 1e-4, p
        bn0 = ts.batch_stats["BatchNorm_0"]
        assert np.allclose(bn0["mean"][s].cpu().numpy(), bs["mean"], atol=1e-6)
        assert np.allclose(bn0["var"][s].cpu().numpy(), bs["var"], atol=1e-6)
        assert np.array_equal(out["runner_state"][3][s].cpu().numpy().view(np.uint32), rng)


def test_training_is_deterministic():
    from purejaxql_b200 import pqn_gymnax
    outs = []
    for _ in range(2):
        cfg = _cfg("Breakout-MinAtar", NUM_ENVS=4096, NUM_STEPS=8, NUM_MINIBATCHES=2, EPS_FINISH=0.1, HIDDEN_SIZE=256,
                   CUDA_GRAPH=False)
        cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(2 * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
        out = pqn_gymnax.make_train(cfg)(jr.split(jr.PRNGKey(9), 2))
        ts = out["runner_state"][0]
        outs.append((ts.params_flat.cpu().numpy().copy(), ts.batch_stats_flat.cpu().numpy().copy()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])


def test_path2_runs_the_bits_kernels():
    from purejaxql_b200 import _lib, pqn_gymnax
    cfg = _cfg("SpaceInvaders-MinAtar", CUDA_GRAPH=False)
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_gymnax.make_train(cfg)
    _lib.lib().pqn_profile_enable(1)
    try:
        _lib.profile_read(reset=True)
        train(jr.split(jr.PRNGKey(1), 1))
        torch.cuda.synchronize()
        names = _lib.profile_read(reset=True)
    finally:
        _lib.lib().pqn_profile_enable(0)
    assert names["bits_dense_fwd"][1] > 0 and names["bits_wgrad"][1] > 0
    assert "dense_fwd" not in names and "wgrad" not in names   # H = 128: every other layer is on wgmma


@pytest.mark.parametrize("game", sorted(GAMES))
def test_smoke_with_eval_and_save(game, tmp_path):
    from purejaxql_b200 import config_loader, pqn_gymnax
    from purejaxql_b200.utils.save_load import load_params
    c = config_loader.compose(["+alg=pqn_cartpole", f"alg.ENV_NAME={game}", "NUM_SEEDS=2", f"SAVE_PATH={tmp_path}",
                               "alg.TOTAL_TIMESTEPS=2e4", "alg.TOTAL_TIMESTEPS_DECAY=2e4", "alg.NUM_ENVS=64",
                               "alg.TEST_NUM_ENVS=16", "alg.TEST_NUM_STEPS=64", "alg.TEST_INTERVAL=0.5"])
    out = pqn_gymnax.single_run(c)
    m = out["metrics"]
    assert torch.isfinite(m["td_loss"]).all() and "test/returned_episode_returns" in m and "env_frame" not in m
    d = tmp_path / game
    files = sorted(p.name for p in d.iterdir())
    assert f"pqn_{game}_seed0_vmap1.safetensors" in files and f"pqn_{game}_seed0_config.yaml" in files
    tree = load_params(str(d / f"pqn_{game}_seed0_vmap0.safetensors"))
    D, H = 100 * GAMES[game], 256
    assert tuple(tree["Dense_0"]["kernel"].shape) == (D, H)
    assert tuple(tree["BatchNorm_0"]["scale"].shape) == (D,)
    assert tuple(tree["Dense_1"]["kernel"].shape) == (H, H) and tree["Dense_2"]["kernel"].shape[0] == H
