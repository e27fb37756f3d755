"""GPU parity of the recurrent network's NORM_TYPE x NORM_INPUT variants (purejaxql/pqn_rnn_gymnax.py:57-94) against
the oracle of tests/rnn_norm_oracle.py: one eval-mode step and a window loss + BPTT gradients + running statistics
through pqn_rnn_step_stats / pqn_rnn_loss_grad_stats, the default network through the same entries, the refusals,
and whole updates, CUDA-graph replay and the MemoryChain preset through pqn_rnn_gymnax.make_train/train."""
import numpy as np
import pytest
import torch

import bsuite_oracle as MC
import rnn_norm_oracle as RO
from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_rnn_ref as RR

pytestmark = pytest.mark.gpu

VARIANTS = [("batch_norm", False), ("batch_norm", True), ("none", False), ("none", True), ("layer_norm", True)]
PQN_E_INVALID, PQN_E_UNSUPPORTED = -1, -3


def dev():
    return torch.device("cuda:0")


def t_(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


def _setup(S, D, A, H, Ls, norm_type, norm_input):
    from purejaxql_b200.networks import NET_RNN, QNetworkSpec
    spec = QNetworkSpec(NET_RNN, D, A, H, Ls, norm_type=norm_type, norm_input=norm_input)
    rng = np.random.default_rng(H + Ls)
    ps, sts = [], []
    for s in range(S):
        p = R.random_params(RO.rnn_param_shapes(D, A, H, Ls, norm_type), 70 + s)
        for g in ("hr", "hz", "hn"):
            p[RR.G + g + "/kernel"] = (p[RR.G + g + "/kernel"] * 0.5).astype(np.float32)
        for k in p:   # norm scales / biases away from (1, 0)
            if k.startswith(("BatchNorm_", "LayerNorm_")):
                p[k] = (p[k] + rng.standard_normal(p[k].shape) * 0.2).astype(np.float32)
        st = RO.rnn_init_stats(D, H, Ls, norm_type)
        for v in st.values():   # non-trivial running statistics
            v["mean"] = (rng.standard_normal(v["mean"].shape) * 0.3).astype(np.float32)
            v["var"] = rng.uniform(0.5, 2.0, v["var"].shape).astype(np.float32)
        ps.append(p)
        sts.append(st)
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    stats = torch.cat([spec.flatten_stats(st, 1, dev()) for st in sts], 0).contiguous()
    return spec, ps, sts, flat, stats


def _ws(spec, S, rows):
    from purejaxql_b200 import _lib
    return torch.empty(int(_lib.lib().pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())


def _f64(p):
    return {k: v.astype(np.float64) for k, v in p.items()}


def _st64(st):
    return {k: {kk: vv.astype(np.float64) for kk, vv in v.items()} for k, v in st.items()}


def _leaf(tree, path, s):
    d = tree
    for k in path:
        d = d[k]
    return d[s].cpu().numpy()


def _step(spec, flat, stats, hs_d, obs_d, orps, ld_d, la_d, q, S, E, ws, fn="pqn_rnn_step_stats"):
    from purejaxql_b200 import _lib
    L = _lib.lib()
    if fn == "pqn_rnn_step":
        return L.pqn_rnn_step(spec.desc, _lib.p(flat), _lib.p(hs_d), _lib.p(obs_d), orps, _lib.p(ld_d), _lib.p(la_d),
                              _lib.p(q), S, E, _lib.p(ws), _lib.stream_ptr())
    return L.pqn_rnn_step_stats(spec.desc, _lib.p(flat), _lib.p(stats) if stats is not None else None, _lib.p(hs_d),
                                _lib.p(obs_d), orps, _lib.p(ld_d), _lib.p(la_d), _lib.p(q), S, E, _lib.p(ws),
                                _lib.stream_ptr())


def _loss(spec, flat, stats, bufs, grads, ls, qs, S, T, B, ws, fn="pqn_rnn_loss_grad_stats"):
    from purejaxql_b200 import _lib
    L = _lib.lib()
    if fn == "pqn_rnn_loss_grad":
        return L.pqn_rnn_loss_grad(spec.desc, _lib.p(flat), *[_lib.p(b) for b in bufs], _lib.p(grads), _lib.p(ls),
                                   _lib.p(qs), S, T, B, 0.99, 0.95, _lib.p(ws), _lib.stream_ptr())
    return L.pqn_rnn_loss_grad_stats(spec.desc, _lib.p(flat), _lib.p(stats) if stats is not None else None,
                                     *[_lib.p(b) for b in bufs], _lib.p(grads), _lib.p(ls), _lib.p(qs), S, T, B, 0.99,
                                     0.95, _lib.p(ws), _lib.stream_ptr())


def _step_inputs(S, E, D, A, H, pad=0, seed=0):
    rng = np.random.default_rng(seed)
    hs = rng.standard_normal((S, E, H)).astype(np.float32) * 0.5
    obs = (rng.standard_normal((S, E + pad, D)) * 1.5 + 0.3).astype(np.float32)
    ld = rng.random((S, E)) < 0.3
    la = rng.integers(0, A, (S, E)).astype(np.int32)
    return hs, obs, ld, la


@pytest.mark.parametrize("H,Ls", [(64, 3), (512, 1)])
@pytest.mark.parametrize("norm_type,norm_input", VARIANTS)
def test_rnn_step_stats_matches_oracle(norm_type, norm_input, H, Ls):
    """Eval mode: the running statistics normalise.  The obs rows are strided (obs_rows_per_seed = E + 5)."""
    from purejaxql_b200 import _lib
    S, E, D, A, pad = 2, 37, 3, 2, 5
    spec, ps, sts, flat, stats = _setup(S, D, A, H, Ls, norm_type, norm_input)
    hs, obs, ld, la = _step_inputs(S, E, D, A, H, pad)
    hs_d = t_(hs, torch.float32)
    q = torch.zeros((S * E, A), device=dev())
    stats0 = stats.clone()
    _lib.check(_step(spec, flat, stats, hs_d, t_(obs, torch.float32), E + pad, t_(ld.astype(np.uint8), torch.uint8),
                     t_(la, torch.int32), q, S, E, _ws(spec, S, E)), "pqn_rnn_step_stats")
    torch.cuda.synchronize()
    assert torch.equal(stats, stats0)                                       # train=False: read only
    for s in range(S):
        new_h, qq = RO.rnn_forward(_f64(ps[s]), hs[s].astype(np.float64), obs[s][None, :E].astype(np.float64),
                                   ld[s][None], la[s][None], norm_type=norm_type, norm_input=norm_input,
                                   batch_stats=_st64(sts[s]), train=False)
        assert np.abs(q.cpu().numpy().reshape(S, E, A)[s] - qq[0]).max() < 1e-5
        assert np.abs(hs_d.cpu().numpy()[s] - new_h).max() < 1e-5


def _window(S, T, B, D, A, H, seed=1):
    rng = np.random.default_rng(seed)
    w = dict(hs0=rng.standard_normal((S, B, H)).astype(np.float32) * 0.5,
             obs=(rng.standard_normal((S, T, B, D)) * 1.5 + 0.3).astype(np.float32),
             ld=rng.random((S, T, B)) < 0.15, la=rng.integers(0, A, (S, T, B)).astype(np.int32),
             ac=rng.integers(0, A, (S, T, B)).astype(np.int32), rw=(rng.random((S, T, B)) * 0.5).astype(np.float32),
             dn=rng.random((S, T, B)) < 0.15)
    bufs = [t_(w["hs0"], torch.float32), t_(w["obs"], torch.float32), t_(w["ld"].astype(np.uint8), torch.uint8),
            t_(w["la"], torch.int32), t_(w["ac"], torch.int32), t_(w["rw"], torch.float32),
            t_(w["dn"].astype(np.uint8), torch.uint8)]
    return w, bufs


@pytest.mark.parametrize("H,Ls,T,B", [(64, 3, 9, 3), (512, 1, 8, 4), (128, 2, 10, 5)])
@pytest.mark.parametrize("norm_type,norm_input", VARIANTS)
def test_rnn_loss_grad_stats_matches_fp64_oracle(norm_type, norm_input, H, Ls, T, B):
    from purejaxql_b200 import _lib
    S, D, A = 2, 3, 2
    spec, ps, sts, flat, stats = _setup(S, D, A, H, Ls, norm_type, norm_input)
    w, bufs = _window(S, T, B, D, A, H)
    grads = torch.zeros_like(flat)
    ls, qs = torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
    _lib.check(_loss(spec, flat, stats, bufs, grads, ls, qs, S, T, B, _ws(spec, S, T * B)), "pqn_rnn_loss_grad_stats")
    torch.cuda.synchronize()
    gtree, sttree = spec.unflatten(grads), spec.unflatten_stats(stats)
    dead = {f"Dense_{l}/bias" for l in range(Ls)} if norm_type == "batch_norm" else set()
    for s in range(S):
        loss, chosen, g, new_stats = RO.rnn_loss_and_grads(
            _f64(ps[s]), w["hs0"][s].astype(np.float64), w["obs"][s].astype(np.float64), w["ld"][s], w["la"][s],
            w["ac"][s], w["rw"][s].astype(np.float64), w["dn"][s], 0.99, 0.95, norm_type, norm_input, _st64(sts[s]))
        assert abs(float(ls[s]) - loss) < 5e-5 * max(1.0, abs(loss)), (float(ls[s]), loss)
        assert abs(float(qs[s]) - chosen.mean()) < 5e-5 * max(1.0, abs(chosen.mean()))
        scale = max(np.abs(v).max() for v in g.values())
        errs = {}
        for path, *_ in spec.entries:
            name = "/".join(path)
            tol = 2e-5
            if norm_type == "batch_norm":
                # fp32 batch statistics, as in tests/test_gpu_norm.py: 2e-4 of the scale, and 5e-2 on a bias in front
                # of a BatchNorm, whose exact gradient is zero (the sum of a batch-normalised gradient)
                tol = 5e-2 if name in dead else 2e-4
            errs[name] = (float(np.abs(_leaf(gtree, path, s) - g[name]).max() / scale), tol)
        bad = {k: v for k, v in errs.items() if not v[0] < v[1]}
        assert not bad, (bad, errs)
        for path, off, n in spec.stats_entries():
            want = new_stats["/".join(path)]
            d = sttree
            for k in path:
                d = d[k]
            assert np.abs(d["mean"][s].cpu().numpy() - want["mean"]).max() < 2e-6, path
            assert np.abs(d["var"][s].cpu().numpy() - want["var"]).max() < 2e-6, path


@pytest.mark.parametrize("H,Ls", [(128, 2), (64, 3)])
def test_default_network_through_the_stats_entries(H, Ls):
    """With batch_stats = NULL the new entries give exactly what pqn_rnn_step / pqn_rnn_loss_grad give.  With a
    batch_stats block, the loss also moves BatchNorm_0's running statistics (its output stays discarded) and
    everything else is still bit-identical."""
    from purejaxql_b200 import _lib
    S, E, D, A, T, B = 2, 29, 4, 2, 9, 3
    spec, ps, sts, flat, stats = _setup(S, D, A, H, Ls, "layer_norm", False)
    hs, obs, ld, la = _step_inputs(S, E, D, A, H)
    outs = []
    for fn, st in (("pqn_rnn_step", None), ("pqn_rnn_step_stats", None), ("pqn_rnn_step_stats", stats)):
        hs_d = t_(hs, torch.float32)
        q = torch.zeros((S * E, A), device=dev())
        _lib.check(_step(spec, flat, st, hs_d, t_(obs, torch.float32), E, t_(ld.astype(np.uint8), torch.uint8),
                         t_(la, torch.int32), q, S, E, _ws(spec, S, E), fn), fn)
        outs.append((q.cpu(), hs_d.cpu()))
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(outs[0], o))
    w, bufs = _window(S, T, B, D, A, H)
    outs = []
    stats0 = stats.clone()
    for fn, st in (("pqn_rnn_loss_grad", None), ("pqn_rnn_loss_grad_stats", None), ("pqn_rnn_loss_grad_stats", stats)):
        grads = torch.full_like(flat, 7.0)
        ls, qs = torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
        _lib.check(_loss(spec, flat, st, bufs, grads, ls, qs, S, T, B, _ws(spec, S, T * B), fn), fn)
        outs.append((grads.cpu(), ls.cpu(), qs.cpu()))
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(outs[0], o))
    torch.cuda.synchronize()
    assert spec.stats_total == 2 * D
    for s in range(S):
        want = RO.rnn_batch_stats(_f64(ps[s]), _st64(sts[s]), w["hs0"][s].astype(np.float64),
                                  w["obs"][s].astype(np.float64), w["ld"][s], w["la"][s])
        got = spec.unflatten_stats(stats)["BatchNorm_0"]
        assert np.abs(got["mean"][s].cpu().numpy() - want["BatchNorm_0"]["mean"]).max() < 2e-6
        assert np.abs(got["var"][s].cpu().numpy() - want["BatchNorm_0"]["var"]).max() < 2e-6
    assert not torch.equal(stats, stats0)
    # the default network's workspace is what it was: the modular trunk's buffers are not carved for it
    from purejaxql_b200 import _lib as lb
    from purejaxql_b200.networks import NET_RNN, QNetworkSpec
    bn = QNetworkSpec(NET_RNN, D, A, H, Ls, norm_type="batch_norm")
    assert lb.lib().pqn_net_workspace_bytes(bn.desc, S, T * B) > lb.lib().pqn_net_workspace_bytes(spec.desc, S, T * B)


@pytest.mark.parametrize("norm_type,norm_input", VARIANTS)
def test_refusals(norm_type, norm_input):
    """A NULL batch_stats is refused for every non-default descriptor; the entries without batch_stats still refuse
    these descriptors."""
    from purejaxql_b200 import _lib
    S, E, D, A, H, T, B = 1, 8, 3, 2, 64, 4, 2
    spec, _, _, flat, stats = _setup(S, D, A, H, 1, norm_type, norm_input)
    hs, obs, ld, la = _step_inputs(S, E, D, A, H)
    q = torch.zeros((S * E, A), device=dev())
    args = (t_(hs, torch.float32), t_(obs, torch.float32), E, t_(ld.astype(np.uint8), torch.uint8), t_(la, torch.int32),
            q, S, E, _ws(spec, S, E))
    assert _step(spec, flat, None, *args) == PQN_E_INVALID
    assert _step(spec, flat, None, *args, fn="pqn_rnn_step") == PQN_E_UNSUPPORTED
    _, bufs = _window(S, T, B, D, A, H)
    grads, ls, qs = torch.zeros_like(flat), torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
    ws = _ws(spec, S, T * B)
    assert _loss(spec, flat, None, bufs, grads, ls, qs, S, T, B, ws) == PQN_E_INVALID
    assert _loss(spec, flat, stats, bufs, grads, ls, qs, S, T, B, ws, fn="pqn_rnn_loss_grad") == PQN_E_UNSUPPORTED
    torch.cuda.synchronize()
    assert not grads.any() and not ls.any()


# --------------------------------------------------------------------------------------------------------------------
# whole updates through make_train / train
# --------------------------------------------------------------------------------------------------------------------
def _cfg(env_name, norm_type, norm_input, **kw):
    c = dict(ENV_NAME=env_name, NUM_ENVS=8, NUM_STEPS=12, MEMORY_WINDOW=3, NUM_MINIBATCHES=4, NUM_EPOCHS=2,
             EPS_START=1.0, EPS_FINISH=1.0, EPS_DECAY=0.2, LR=1e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.95,
             NORM_TYPE=norm_type, NORM_INPUT=norm_input, HIDDEN_SIZE=128, NUM_LAYERS=2, LR_LINEAR_DECAY=True,
             REW_SCALE=0.1, WANDB_MODE="disabled", TEST_DURING_TRAINING=False)
    if env_name == "MemoryChain-bsuite":
        c.update(ENV_KWARGS={"memory_length": 4}, REW_SCALE=1.0)
    c.update(kw)
    return c


def _oracle_step(env, p, stats, nt, ni, hs, obs, ld, la, st, rng, eps, rew_scale, E):
    """_step_env / _random_step (:192-236, :514-529) for one seed: eval mode, running statistics read."""
    ks = jr.split(rng, 3)
    rng, rng_a, rng_s = ks[0], ks[1], ks[2]
    new_hs, q = RO.rnn_forward(p, hs, obs[None], ld[None], la[None], norm_type=nt, norm_input=ni, batch_stats=stats)
    act = R.eps_greedy(jr.split(rng_a, E), q[0], eps)
    new_obs, st, reward, done, info = env.step(jr.split(rng_s, E), st, act)
    tr = dict(last_hs=hs, obs=obs, action=act, reward=(np.float32(rew_scale) * reward).astype(np.float32), done=done,
              last_done=ld, last_action=la)
    return (new_hs.astype(np.float32), new_obs, done, act, st, rng), tr


@pytest.mark.parametrize("env_name,norm_type,norm_input", [("CartPole-v1", "batch_norm", False),
                                                           ("CartPole-v1", "none", True),
                                                           ("MemoryChain-bsuite", "batch_norm", True)])
def test_rnn_norm_update_steps_match_oracle(env_name, norm_type, norm_input):
    """Two whole updates with eps = 1 (the rollouts do not depend on the network) against an oracle replay: per-update
    td_loss, the final parameters and the final batch_stats."""
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = _cfg(env_name, norm_type, norm_input)
    nupd = 2
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_rnn_gymnax.make_train(cfg)
    eng = train.engine
    spec = eng.spec
    assert eng.with_stats
    rngs = jr.split(jr.PRNGKey(31), 2)
    cap = {}
    orig = spec.init
    spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    out = train(rngs)
    ts = out["runner_state"][0]
    tree0 = spec.unflatten(cap["flat"])
    T, E, W, nmb, H = cfg["NUM_STEPS"], cfg["NUM_ENVS"], cfg["MEMORY_WINDOW"], cfg["NUM_MINIBATCHES"], cfg["HIDDEN_SIZE"]
    Bm = E // nmb
    stol = 5e-4 if norm_type == "batch_norm" else 1e-5
    for s in range(rngs.shape[0]):
        params = {"/".join(p): _leaf(tree0, p, s).astype(np.float32) for p, *_ in spec.entries}
        stats = RO.rnn_init_stats(eng.D, H, cfg["NUM_LAYERS"], norm_type)
        env = MC.make(4, flatten=True) if env_name == "MemoryChain-bsuite" else G.make(env_name, flatten=True)
        k = jr.split(rngs[s], 2); rng = k[0]                               # :255
        k = jr.split(rng, 2); rng = k[0]                                   # :505
        k = jr.split(rng, 2); rng, kR = k[0], k[1]                         # :508
        obs, st = env.reset(jr.split(kR, E))
        hs = np.zeros((E, H), np.float32); ld = np.zeros(E, bool); la = np.zeros(E, np.int32)
        k = jr.split(rng, 2); carry = k[1]                                 # :531
        mem = []
        for _ in range(W + T):
            (hs, obs, ld, la, st, carry), tr = _oracle_step(env, params, stats, norm_type, norm_input, hs, obs, ld, la,
                                                            st, carry, 1.0, cfg["REW_SCALE"], E)
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
                (hs, obs, ld, la, st, carry), tr = _oracle_step(env, params, stats, norm_type, norm_input, hs, obs, ld,
                                                                la, st, carry, 1.0, cfg["REW_SCALE"], E)
                new.append(tr)
            rng = carry
            mem = mem[T:] + new                                            # :239-243
            stack = {kk: np.stack([m[kk] for m in mem]) for kk in mem[0]}
            k = jr.split(rng, 2); r = k[0]                                 # :381
            losses = []
            for _ in range(cfg["NUM_EPOCHS"]):
                k = jr.split(r, 2); r, kperm = k[0], k[1]                  # :368
                perm = jr.permutation_indices(kperm, E)
                r = jr.split(r, 2)[0]                                      # :375
                for mb in range(nmb):
                    idx = perm[mb * Bm:(mb + 1) * Bm]
                    loss, _, g, stats = RO.rnn_loss_and_grads(
                        params, stack["last_hs"][0][idx], stack["obs"][:, idx], stack["last_done"][:, idx],
                        stack["last_action"][:, idx], stack["action"][:, idx], stack["reward"][:, idx],
                        stack["done"][:, idx], cfg["GAMMA"], cfg["LAMBDA"], norm_type, norm_input, stats)
                    params, opt, _ = R.radam_clip_step(params, g, opt, lr_fn(opt["count"]), cfg["MAX_GRAD_NORM"])
                    losses.append(loss)
            rng = r
            got = float(out["metrics"]["td_loss"][s, u])
            assert abs(got - np.mean(losses)) < 2e-3 * max(1.0, abs(np.mean(losses))), (u, got, np.mean(losses))
        for p, *_ in spec.entries:
            d = np.abs(_leaf(ts.params, p, s) - params["/".join(p)])
            assert np.quantile(d, 0.99) < 1e-4 and d.max() < 1e-3, (p, d.max())
        for path, off, n in spec.stats_entries():
            want = stats["/".join(path)]
            d = ts.batch_stats
            for kk in path:
                d = d[kk]
            assert np.abs(d["mean"][s].cpu().numpy() - want["mean"]).max() < stol, path
            assert np.abs(d["var"][s].cpu().numpy() - want["var"]).max() < stol, path
        assert np.array_equal(out["runner_state"][4][s].cpu().numpy().view(np.uint32), rng)


def _graph_run(graph, seed=5):
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = _cfg("CartPole-v1", "batch_norm", False, EPS_FINISH=0.1, EPS_DECAY=0.5, TEST_DURING_TRAINING=True,
               TEST_INTERVAL=0.4, TEST_NUM_ENVS=8, EPS_TEST=0.0, CUDA_GRAPH=graph)
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(5 * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_rnn_gymnax.make_train(cfg)
    out = train(jr.split(jr.PRNGKey(seed), 2))
    assert train.engine.graph_captured == graph
    ts = out["runner_state"][0]
    return (ts.params_flat.cpu().numpy(), ts.batch_stats_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy(),
            out["metrics"]["test/returned_episode_returns"].cpu().numpy(), out["runner_state"][4].cpu().numpy(),
            train.engine.spec.init_stats(2, "cpu").numpy())


def test_rnn_batch_norm_cuda_graph_replay_equals_eager_and_is_deterministic():
    eager, graph, again = _graph_run(False), _graph_run(True), _graph_run(True)
    for a, b, c in zip(eager, graph, again):
        assert np.array_equal(a, b, equal_nan=True) and np.array_equal(b, c, equal_nan=True)
    assert not np.array_equal(eager[1], eager[5])                         # the running statistics moved


def test_rnn_memory_chain_batch_norm_preset_smoke_with_eval():
    from purejaxql_b200 import config_loader, pqn_rnn_gymnax
    c = config_loader.compose(["+alg=pqn_rnn_memory_chain", "alg.NORM_TYPE=batch_norm", "alg.NORM_INPUT=True",
                               "NUM_SEEDS=2", "SAVE_PATH=null", "alg.TOTAL_TIMESTEPS=8192", "alg.TEST_NUM_ENVS=16",
                               "alg.TEST_INTERVAL=0.5"])
    cfg = {**c, **c["alg"]}
    out = pqn_rnn_gymnax.make_train(cfg)(jr.split(jr.PRNGKey(0), 2))
    m = out["metrics"]
    assert m["td_loss"].shape == (2, 2) and torch.isfinite(m["td_loss"]).all()
    assert all(torch.isfinite(m[k]).all() for k in m if k.startswith("test/"))
    ts = out["runner_state"][0]
    L = cfg["NUM_LAYERS"]
    assert set(ts.batch_stats) == {"BatchNorm_0"} | {f"BatchNorm_{l + 1}" for l in range(L)}
    assert set(ts.params) >= {"BatchNorm_0", *[f"BatchNorm_{l + 1}" for l in range(L)], "ScannedRNN_0"}
    assert not any(k.startswith("LayerNorm_") for k in ts.params)
    for v in ts.batch_stats.values():
        assert torch.isfinite(v["mean"]).all() and (v["var"] >= 0).all()
    assert not torch.equal(ts.batch_stats["BatchNorm_1"]["var"], torch.ones_like(ts.batch_stats["BatchNorm_1"]["var"]))
