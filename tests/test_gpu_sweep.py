"""Hyperparameter grids trained as one batched run (sweep.Grid), on the GPU.

1. Slice identity: for every grid point g, seeds g*n .. g*n+n-1 of the sweep are bit-identical to a standalone train of
   point g's scalar config given the same tiled key array (same S, so split counts and reduction orders match):
   per-update metrics, final parameters, RAdam moments, running statistics and final keys; eagerly and under CUDA-graph
   replay, for pqn_minatar, pqn_gymnax (MLP and packed-bit MLP) and pqn_rnn_gymnax (default and batch_norm network).
2. The *_seeds entry points: with broadcast values bit-identical to the scalar entries; with distinct per-seed values
   seed s equals the scalar entry called on the same S seeds with seed s's scalars.
3. A 2-point LR x LAMBDA sweep of pqn_rnn_gymnax against the oracle replay of tests/test_gpu_rnn_eval.py.
4. Two gloo ranks on one GPU, seed-sharded and env-sharded, and single_run's checkpoints of a sweep."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_rnn_ref as RR
from purejaxql_b200 import _lib, engine, envs, sweep
from purejaxql_b200.networks import NET_RNN, QNetworkSpec

pytestmark = pytest.mark.gpu
N, NUPD = 2, 3                      # seeds per grid point; 3 updates so that the graph captures and replays

_RUN = dict(NUM_EPOCHS=2, LR_LINEAR_DECAY=True, WANDB_MODE="disabled", TEST_DURING_TRAINING=False, NUM_SEEDS=N)
CASES = {
    "minatar_breakout_cnn": ("pqn_minatar", dict(
        ENV_NAME="Breakout-MinAtar", NUM_ENVS=64, NUM_STEPS=8, NUM_MINIBATCHES=4, EPS_START=1.0, EPS_FINISH=0.05,
        EPS_DECAY=0.5, LR=[5e-4, 1e-4], MAX_GRAD_NORM=10, GAMMA=[0.99, 0.9], LAMBDA=0.65, NORM_TYPE="layer_norm")),
    "gymnax_cartpole_mlp": ("pqn_gymnax", dict(
        ENV_NAME="CartPole-v1", NUM_ENVS=32, NUM_STEPS=16, NUM_MINIBATCHES=4, EPS_START=[1.0, 0.5], EPS_FINISH=0.2,
        EPS_DECAY=0.5, LR=1e-4, MAX_GRAD_NORM=[10, 0.5], GAMMA=0.99, LAMBDA=[0.95, 0.5], REW_SCALE=[0.1, 1.0],
        HIDDEN_SIZE=128, NUM_LAYERS=2, NORM_TYPE="layer_norm")),
    "gymnax_breakout_bits": ("pqn_gymnax", dict(
        ENV_NAME="Breakout-MinAtar", NUM_ENVS=64, NUM_STEPS=8, NUM_MINIBATCHES=4, EPS_START=1.0,
        EPS_FINISH=[0.05, 0.5], EPS_DECAY=0.5, LR=[5e-4, 1e-4], MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65,
        HIDDEN_SIZE=128, NUM_LAYERS=2, NORM_TYPE="layer_norm")),
    "rnn_cartpole": ("pqn_rnn_gymnax", dict(
        ENV_NAME="CartPole-v1", NUM_ENVS=16, NUM_STEPS=12, MEMORY_WINDOW=3, NUM_MINIBATCHES=4, EPS_START=0.6,
        EPS_FINISH=0.1, EPS_DECAY=1.0, LR=[1e-3, 1e-4], MAX_GRAD_NORM=10, GAMMA=[0.99, 0.9], LAMBDA=0.95,
        REW_SCALE=0.1, HIDDEN_SIZE=128, NUM_LAYERS=2, NORM_TYPE="layer_norm", NORM_INPUT=False)),
    "rnn_memory_chain_batch_norm": ("pqn_rnn_gymnax", dict(
        ENV_NAME="MemoryChain-bsuite", ENV_KWARGS={"memory_length": 4}, NUM_ENVS=16, NUM_STEPS=12, MEMORY_WINDOW=3,
        NUM_MINIBATCHES=4, EPS_START=0.6, EPS_FINISH=0.1, EPS_DECAY=[1.0, 0.2], LR=[1e-3, 1e-4],
        MAX_GRAD_NORM=[10, 1], GAMMA=0.99, LAMBDA=[0.95, 0.5], REW_SCALE=1.0, HIDDEN_SIZE=128, NUM_LAYERS=2,
        NORM_TYPE="batch_norm", NORM_INPUT=False)),
}


def dev():
    return torch.device("cuda:0")


def _cfg(case, **kw):
    module, c = CASES[case]
    c = {**c, **_RUN, **kw}
    c["TOTAL_TIMESTEPS"] = c["TOTAL_TIMESTEPS_DECAY"] = float(NUPD * c["NUM_STEPS"] * c["NUM_ENVS"])
    return module, c


def _run(module, cfg, rngs, graph, seed_lo=0, shard=None):
    """Everything a train() returns that the slice identity compares, on the host."""
    mod = importlib.import_module(f"purejaxql_b200.{module}")
    train = mod.make_train(dict(cfg, CUDA_GRAPH=graph))
    train.engine.seed_lo = seed_lo
    if shard is not None:
        train.engine.env_shard = shard
    out = train(rngs)
    assert train.engine.graph_captured == graph
    ts = out["runner_state"][0]
    res = {"params": ts.params_flat, "mu": ts.opt_state.mu, "nu": ts.opt_state.nu, "stats": ts.batch_stats_flat,
           "rng": out["runner_state"][-1]}
    res.update({f"metric:{k}": v for k, v in out["metrics"].items()})
    return {k: v.cpu().numpy() for k, v in res.items()}, out["sweep"]


def _same(a, b, where):
    for k, v in a.items():
        assert v.shape == b[k].shape and np.array_equal(v, b[k], equal_nan=v.dtype.kind == "f"), where + (k,)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda_graph"])
@pytest.mark.parametrize("case", list(CASES))
def test_sweep_slice_equals_standalone_run(case, graph):
    module, cfg = _cfg(case)
    grid = sweep.Grid(cfg)
    assert len(grid.axes) >= 2 and grid.G >= 4
    rngs = grid.tile(jr.split(jr.PRNGKey(7), N))
    got, table = _run(module, cfg, rngs, graph)
    assert table == grid.table(0, grid.total_seeds)
    for g in range(grid.G):
        want, _ = _run(module, grid.config(g), rngs, graph)
        sl = slice(g * N, (g + 1) * N)
        _same({k: v[sl] for k, v in got.items()}, {k: v[sl] for k, v in want.items()}, (case, graph, g))
    for g in range(1, grid.G):                       # the points train differently from the same keys
        assert not np.array_equal(got["params"][:N], got["params"][g * N:(g + 1) * N]), g


# --------------------------------------------------------------------------- #
# entry points
# --------------------------------------------------------------------------- #
def _f(x):
    return torch.as_tensor(np.asarray(x, np.float32), device=dev()).contiguous()


def test_radam_clip_step_seeds_entry():
    L, S, P, steps = _lib.lib(), 6, 4 * 2500, 4
    gen = torch.Generator(device="cpu").manual_seed(0)
    params0 = torch.randn(S, P, generator=gen).to(dev())
    grads = [(torch.randn(S, P, generator=gen) * torch.linspace(0.01, 0.4, S)[:, None]).to(dev()) for _ in range(steps)]
    lrs = [5e-4, 1e-4, 1e-3, 5e-5, 2e-4, 1e-4]
    norms = [10.0, 1.0, 5.0, 0.5, 10.0, 2.0]                  # the gradient norms run from ~0.5 to ~20: some clip
    tab = {lr: engine.radam_schedule_table(steps, lambda i, lr=lr: engine.linear_schedule(lr, 1e-20, 8, i))
           for lr in set(lrs)}

    def run(call):
        p, mu, nu = params0.clone(), torch.zeros_like(params0), torch.zeros_like(params0)
        step, gn = torch.zeros(1, dtype=torch.int32, device=dev()), torch.zeros(S * 64, device=dev())
        for g in grads:
            _lib.check(call(p, g, mu, nu, step, gn))
        torch.cuda.synchronize()
        return {"p": p.cpu().numpy(), "mu": mu.cpu().numpy(), "nu": nu.cpu().numpy(), "step": step.cpu().numpy()}

    def scalar(sched, mn):
        s = _f(sched)
        return run(lambda p, g, mu, nu, st, gn: L.pqn_radam_clip_step(
            _lib.p(p), _lib.p(g), _lib.p(mu), _lib.p(nu), _lib.p(s), _lib.p(st), _lib.p(gn), S, P, mn, 0.9, 0.999,
            1e-8, _lib.stream_ptr()))

    def seeds(sched, stride, mn):
        s, m = _f(sched), _f(mn)
        return run(lambda p, g, mu, nu, st, gn: L.pqn_radam_clip_step_seeds(
            _lib.p(p), _lib.p(g), _lib.p(mu), _lib.p(nu), _lib.p(s), stride, _lib.p(st), _lib.p(gn), S, P, _lib.p(m),
            0.9, 0.999, 1e-8, _lib.stream_ptr()))
    _same(seeds(tab[5e-4], 0, [1.0] * S), scalar(tab[5e-4], 1.0), ("broadcast",))
    got = seeds(np.stack([tab[lr] for lr in lrs]), 4 * steps, norms)
    for s in range(S):
        want = scalar(tab[lrs[s]], norms[s])
        _same({k: v[s] for k, v in got.items() if k != "step"}, {k: v[s] for k, v in want.items() if k != "step"},
              ("per-seed", s))
    assert got["step"][0] == steps


def test_qlambda_seeds_entry():
    L, T, S, E, A = _lib.lib(), 9, 5, 37, 4
    rng = np.random.default_rng(1)
    reward, maxq = _f(rng.normal(size=(S, T, E))), _f(rng.normal(size=(S, T, E)))
    done = torch.from_numpy((rng.random((S, T, E)) < 0.2).astype(np.uint8)).to(dev())
    q_last = _f(rng.normal(size=(S * E, A)))
    gammas, lams = [0.99, 0.9, 0.5, 0.99, 0.0], [0.95, 0.65, 0.0, 1.0, 0.5]

    def scalar(gm, lm):
        t = torch.zeros(S, T, E, device=dev())
        _lib.check(L.pqn_qlambda(_lib.p(reward), _lib.p(done), _lib.p(maxq), _lib.p(q_last), _lib.p(t), T, S, E, A, gm,
                                 lm, _lib.stream_ptr()))
        return t.cpu().numpy()

    def seeds(gm, lm):
        t, g, l_ = torch.zeros(S, T, E, device=dev()), _f(gm), _f(lm)
        _lib.check(L.pqn_qlambda_seeds(_lib.p(reward), _lib.p(done), _lib.p(maxq), _lib.p(q_last), _lib.p(t), T, S, E,
                                       A, _lib.p(g), _lib.p(l_), _lib.stream_ptr()))
        return t.cpu().numpy()
    assert np.array_equal(seeds([0.99] * S, [0.65] * S), scalar(0.99, 0.65))
    got = seeds(gammas, lams)
    for s in range(S):
        assert np.array_equal(got[s], scalar(gammas[s], lams[s])[s]), s


@pytest.mark.parametrize("env_name", ["CartPole-v1", "Breakout-MinAtar"])
def test_rollout_act_step_seeds_entry(env_name):
    L, S, E = _lib.lib(), 4, 300
    env, params = envs.make(env_name)
    A = env.num_actions
    W, dt = (env.packed_obs_words, torch.int32) if env.binary_obs else (env.obs_dim, torch.float32)
    state0 = torch.empty((env.state_words, S * E), dtype=torch.int32, device=dev())
    envs.reset_into(env.env_id, jr_keys(jr.split(jr.PRNGKey(3), S * E)), state0, None, S * E, params, 0)
    rng = np.random.default_rng(2)
    q = _f(rng.normal(size=(S * E, A)))
    step_keys = jr_keys(jr.split(jr.PRNGKey(4), S * 2)).reshape(S, 2, 2).contiguous()
    eps_s, rew_s = [0.0, 0.3, 0.9, 1.0], [0.1, 1.0, 0.5, 2.0]

    def run(call):
        st = state0.clone()
        obs = torch.zeros((S, E, W), dtype=dt, device=dev())
        a, r = torch.zeros((S, E), dtype=torch.int32, device=dev()), torch.zeros((S, E), device=dev())
        d, mq = torch.zeros((S, E), dtype=torch.uint8, device=dev()), torch.zeros((S, E), device=dev())
        sums = torch.zeros((S, 5), dtype=torch.float64, device=dev())
        for _ in range(3):                                   # a few steps, so that some envs finish (CartPole)
            _lib.check(call(st, obs, a, r, d, mq, sums))
        torch.cuda.synchronize()
        return {"state": st.view(-1, S, E).transpose(0, 1).cpu().numpy(), "obs": obs.cpu().numpy(),
                "a": a.cpu().numpy(), "r": r.cpu().numpy(), "d": d.cpu().numpy(), "mq": mq.cpu().numpy(),
                "sums": sums.cpu().numpy()}

    def scalar(eps, rs):
        e = _f([eps])
        return run(lambda st, obs, a, r, d, mq, sums: L.pqn_rollout_act_step(
            env.env_id, _lib.p(step_keys), _lib.p(q), _lib.p(e), _lib.p(st), _lib.p(obs), E, _lib.p(a), _lib.p(r),
            _lib.p(d), _lib.p(mq), E, _lib.p(sums), 0, S, E, 0, 0, 0, rs, 0, _lib.stream_ptr()))

    def seeds(eps, rs):
        e, k = _f(eps), _f(rs)
        return run(lambda st, obs, a, r, d, mq, sums: L.pqn_rollout_act_step_seeds(
            env.env_id, _lib.p(step_keys), _lib.p(q), _lib.p(e), _lib.p(st), _lib.p(obs), E, _lib.p(a), _lib.p(r),
            _lib.p(d), _lib.p(mq), E, _lib.p(sums), 0, S, E, 0, 0, 0, _lib.p(k), 0, _lib.stream_ptr()))
    _same(seeds([0.4] * S, [0.5] * S), scalar(0.4, 0.5), ("broadcast",))
    got = seeds(eps_s, rew_s)
    for s in range(S):
        want = scalar(eps_s[s], rew_s[s])
        _same({k: v[s] for k, v in got.items()}, {k: v[s] for k, v in want.items()}, ("per-seed", s))


def jr_keys(k):
    return torch.from_numpy(np.ascontiguousarray(k, np.uint32).view(np.int32)).to(dev())


@pytest.mark.parametrize("norm_type", ["layer_norm", "batch_norm"])
def test_rnn_loss_grad_seeds_entry(norm_type):
    L, S, T, B, D, A, H = _lib.lib(), 4, 6, 8, 4, 2, 128
    spec = QNetworkSpec(NET_RNN, D, A, H, 2, norm_type=norm_type, norm_input=False)
    with_stats = norm_type != "layer_norm"
    params = spec.init(jr_keys(jr.split(jr.PRNGKey(5), S)), dev())
    stats0 = spec.init_stats(S, dev()) if with_stats else None
    rng = np.random.default_rng(3)
    hs0, obs = _f(rng.normal(size=(S, B, H)) * 0.3), _f(rng.normal(size=(S, T, B, D)))
    u8 = lambda p: torch.from_numpy((rng.random((S, T, B)) < p).astype(np.uint8)).to(dev())
    i32 = lambda: torch.from_numpy(rng.integers(0, A, (S, T, B)).astype(np.int32)).to(dev())
    ld, la, ac, rw, dn = u8(0.1), i32(), i32(), _f(rng.normal(size=(S, T, B))), u8(0.1)
    ws = torch.empty(int(L.pqn_net_workspace_bytes(spec.desc, S, T * B)), dtype=torch.uint8, device=dev())
    gammas, lams = [0.99, 0.9, 0.5, 0.0], [0.95, 0.0, 0.65, 1.0]

    def run(call):
        g, ls, qs = torch.zeros_like(params), torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
        st = stats0.clone() if with_stats else None
        _lib.check(call(g, ls, qs, st))
        torch.cuda.synchronize()
        out = {"g": g.cpu().numpy(), "loss": ls.cpu().numpy(), "qsa": qs.cpu().numpy()}
        if with_stats:
            out["stats"] = st.cpu().numpy()
        return out
    args = lambda: (_lib.p(hs0), _lib.p(obs), _lib.p(ld), _lib.p(la), _lib.p(ac), _lib.p(rw), _lib.p(dn))

    def scalar(gm, lm):
        if with_stats:
            return run(lambda g, ls, qs, st: L.pqn_rnn_loss_grad_stats(
                spec.desc, _lib.p(params), _lib.p(st), *args(), _lib.p(g), _lib.p(ls), _lib.p(qs), S, T, B, gm, lm,
                _lib.p(ws), _lib.stream_ptr()))
        return run(lambda g, ls, qs, st: L.pqn_rnn_loss_grad(
            spec.desc, _lib.p(params), *args(), _lib.p(g), _lib.p(ls), _lib.p(qs), S, T, B, gm, lm, _lib.p(ws),
            _lib.stream_ptr()))

    def seeds(gm, lm):
        gt, lt = _f(gm), _f(lm)
        return run(lambda g, ls, qs, st: L.pqn_rnn_loss_grad_seeds(
            spec.desc, _lib.p(params), _lib.p(st), *args(), _lib.p(g), _lib.p(ls), _lib.p(qs), S, T, B, _lib.p(gt),
            _lib.p(lt), _lib.p(ws), _lib.stream_ptr()))
    _same(seeds([0.99] * S, [0.95] * S), scalar(0.99, 0.95), ("broadcast", norm_type))
    got = seeds(gammas, lams)
    for s in range(S):
        want = scalar(gammas[s], lams[s])
        _same({k: v[s] for k, v in got.items()}, {k: v[s] for k, v in want.items()}, ("per-seed", norm_type, s))


# --------------------------------------------------------------------------- #
# oracle
# --------------------------------------------------------------------------- #
def test_rnn_lr_lambda_sweep_matches_oracle():
    """A 2 x 2 LR x LAMBDA sweep of pqn_rnn_gymnax (CartPole, eps 0.6 -> 0.1, 3 updates) replayed seed by seed with
    each seed's own LR schedule and LAMBDA, to the tolerances of test_rnn_train_with_eps_schedule_matches_oracle."""
    from test_gpu_rnn_eval import _leaf, _oracle_step, report
    from purejaxql_b200 import pqn_rnn_gymnax
    _, cfg = _cfg("rnn_cartpole", GAMMA=0.99, LR=[1e-3, 1e-4], LAMBDA=[0.95, 0.5], NUM_SEEDS=1)
    grid = sweep.Grid(cfg)
    assert [k for k, _ in grid.axes] == ["LR", "LAMBDA"] and grid.G == 4
    train = pqn_rnn_gymnax.make_train(dict(cfg, CUDA_GRAPH=True))
    eng = train.engine
    T, E, W, nmb, H = cfg["NUM_STEPS"], cfg["NUM_ENVS"], cfg["MEMORY_WINDOW"], cfg["NUM_MINIBATCHES"], cfg["HIDDEN_SIZE"]
    Bm, S = E // nmb, grid.total_seeds
    rngs = grid.tile(jr.split(jr.PRNGKey(41), 1))
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    snaps = []
    eng.on_update_end = lambda n, b: snaps.append(b["mem"].action[:, W:W + T].clone())
    out = train(rngs)
    assert eng.graph_captured and len(snaps) == NUPD
    m, ts = out["metrics"], out["runner_state"][0]
    nud = eng.cfg["NUM_UPDATES_DECAY"]
    tree0 = eng.spec.unflatten(cap["flat"])
    ties = []
    for s in range(S):
        c = grid.config(s)
        params = {"/".join(p): _leaf(tree0, p, s).astype(np.float32) for p, *_ in eng.spec.entries}
        env = G.make("CartPole-v1", flatten=True)
        rng = jr.split(rngs[s], 2)[0]
        rng = jr.split(rng, 2)[0]
        k = jr.split(rng, 2); rng, kR = k[0], k[1]
        obs, st = env.reset(jr.split(kR, E))
        hs = np.zeros((E, H), np.float32); ld = np.zeros(E, bool); la = np.zeros(E, np.int32)
        carry = jr.split(rng, 2)[1]
        mem = []
        for _ in range(W + T):
            (hs, obs, ld, la, st, carry), tr, _ = _oracle_step(env, params, hs, obs, ld, la, st, carry, 1.0,
                                                               c["REW_SCALE"], E)
            mem.append(tr)
        rng = jr.split(carry, 2)[1]
        opt = R.opt_init(params)
        total = nud * nmb * c["NUM_EPOCHS"]
        lr_fn = lambda i: R.linear_schedule(c["LR"], 1e-20, total, i)
        for u in range(NUPD):
            eps = R.linear_schedule(c["EPS_START"], c["EPS_FINISH"], c["EPS_DECAY"] * nud, u)
            engine_actions = snaps[u][s].cpu().numpy()
            carry = jr.split(rng, 2)[1]
            new, infos = [], []
            for t in range(T):
                (hs, obs, ld, la, st, carry), tr, info = _oracle_step(
                    env, params, hs, obs, ld, la, st, carry, eps, c["REW_SCALE"], E, engine_actions[t], ties,
                    ("sweep", s, u, t))
                new.append(tr)
                infos.append(info)
            rng = carry
            mem = mem[T:] + new
            stack = {kk: np.stack([x[kk] for x in mem]) for kk in mem[0]}
            r = jr.split(rng, 2)[0]
            losses, qvals = [], []
            for _ in range(c["NUM_EPOCHS"]):
                k = jr.split(r, 2); r, kperm = k[0], k[1]
                perm = jr.permutation_indices(kperm, E)
                r = jr.split(r, 2)[0]
                for mb in range(nmb):
                    idx = perm[mb * Bm:(mb + 1) * Bm]
                    loss, chosen, g = RR.rnn_loss_and_grads(
                        params, stack["last_hs"][0][idx], stack["obs"][:, idx], stack["last_done"][:, idx],
                        stack["last_action"][:, idx], stack["action"][:, idx], stack["reward"][:, idx],
                        stack["done"][:, idx], c["GAMMA"], c["LAMBDA"])
                    params, opt, _ = R.radam_clip_step(params, g, opt, lr_fn(opt["count"]), c["MAX_GRAD_NORM"])
                    losses.append(loss)
                    qvals.append(chosen.mean())
            rng = r
            for name, want in (("td_loss", np.mean(losses)), ("qvals", np.mean(qvals))):
                got = float(m[name][s, u])
                assert abs(got - want) < 2e-3 * max(1.0, abs(want)), (s, u, name, got, want)
            for kk in R.INFO_KEYS:
                want = float(np.mean([x[kk].astype(np.float64).mean() for x in infos]))
                assert abs(float(m[kk][s, u]) - want) <= 1e-5 * max(1.0, abs(want)), (s, u, kk)
        for p, *_ in eng.spec.entries:
            d = np.abs(_leaf(ts.params, p, s) - params["/".join(p)])
            assert np.quantile(d, 0.99) < 1e-4 and d.max() < 1e-3, (s, p, d.max())
        assert np.array_equal(out["runner_state"][4][s].cpu().numpy().view(np.uint32), rng)
    report("recurrent LR x LAMBDA sweep", ties, S * NUPD * T * E)


# --------------------------------------------------------------------------- #
# ranks and checkpoints
# --------------------------------------------------------------------------- #
def _rank_worker(rank, world, mode, out_dir):
    from test_gpu_env_shard_train import _init_group
    from purejaxql_b200._runner import seed_slice
    dist, _ = _init_group(rank, world, out_dir)
    try:
        module, cfg = _cfg("gymnax_cartpole_mlp")
        grid = sweep.Grid(cfg)
        rngs = grid.tile(jr.split(jr.PRNGKey(7), N))
        res = {}
        if mode == "seeds":
            lo, hi = seed_slice(grid.total_seeds, rank, world)
            got, table = _run(module, cfg, rngs[lo:hi], False, seed_lo=lo)
            assert table == grid.table(lo, hi - lo)
            res.update({f"sweep:{k}": v for k, v in got.items()})
        else:
            got, _ = _run(module, cfg, rngs, False, shard=(rank, world))
            res.update({f"sweep:{k}": v for k, v in got.items()})
            for g in range(grid.G):
                want, _ = _run(module, grid.config(g), rngs, False, shard=(rank, world))
                res.update({f"point{g}:{k}": v for k, v in want.items()})
        np.savez(os.path.join(out_dir, f"{mode}{rank}.npz"), **res)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode", ["seeds", "envs"])
def test_two_ranks_train_the_sweep(mode, tmp_path):
    """seeds: the two ranks' slices, concatenated, are the single-process sweep bit for bit.  envs: every rank holds
    every seed; the ranks agree, and each point's seeds equal the env-sharded standalone run of that point (an
    env-sharded run draws its own minibatch permutation per rank, so it is compared with env-sharded runs)."""
    from test_gpu_env_shard_train import _spawn
    _spawn(_rank_worker, 2, (mode,), tmp_path)
    ranks = [dict(np.load(tmp_path / f"{mode}{r}.npz")) for r in range(2)]
    module, cfg = _cfg("gymnax_cartpole_mlp")
    grid = sweep.Grid(cfg)
    if mode == "seeds":
        rngs = grid.tile(jr.split(jr.PRNGKey(7), N))
        single, _ = _run(module, cfg, rngs, False)
        _same({k: np.concatenate([ranks[0][f"sweep:{k}"], ranks[1][f"sweep:{k}"]]) for k in single}, single,
              ("seeds",))
        return
    for k, v in ranks[0].items():
        assert np.array_equal(ranks[1][k], v, equal_nan=v.dtype.kind == "f"), k
    for g in range(grid.G):
        sl = slice(g * N, (g + 1) * N)
        for k in [k[len("sweep:"):] for k in ranks[0] if k.startswith("sweep:")]:
            a, b = ranks[0][f"sweep:{k}"][sl], ranks[0][f"point{g}:{k}"][sl]
            assert np.array_equal(a, b, equal_nan=a.dtype.kind == "f"), (g, k)


def test_single_run_saves_one_checkpoint_per_point_and_seed(tmp_path):
    from purejaxql_b200 import config_loader, pqn_gymnax
    from purejaxql_b200.utils.save_load import load_params
    c = config_loader.compose(["+alg=pqn_cartpole", "NUM_SEEDS=2", f"SAVE_PATH={tmp_path}", "alg.TOTAL_TIMESTEPS=4096",
                               "alg.TOTAL_TIMESTEPS_DECAY=4096", "alg.TEST_DURING_TRAINING=False",
                               "alg.LR=[0.001,0.0001]", "alg.GAMMA=[0.99,0.9]"])
    out = pqn_gymnax.single_run(c)
    d = tmp_path / "CartPole-v1"
    names = sorted(p.name for p in d.iterdir())
    assert names == sorted(["pqn_CartPole-v1_seed0_config.yaml", "pqn_CartPole-v1_seed0_sweep.yaml"] +
                           [f"pqn_CartPole-v1_seed0_g{g}_vmap{i}.safetensors" for g in range(4) for i in range(2)])
    import yaml
    table = yaml.safe_load((d / "pqn_CartPole-v1_seed0_sweep.yaml").read_text())
    assert table["axes"] == {"LR": [0.001, 0.0001], "GAMMA": [0.99, 0.9]} and table["num_seeds"] == 2
    assert table["seeds"] == out["sweep"] and out["sweep"]["GAMMA"][2:4] == [0.9, 0.9]
    from test_gpu_env_shard_train import _leaves
    saved = dict(_leaves(load_params(str(d / "pqn_CartPole-v1_seed0_g2_vmap1.safetensors"))))
    trained = dict(_leaves(out["runner_state"][0].params))
    assert saved and sorted(saved) == sorted(trained)
    for k, v in saved.items():                       # point 2, seed 1 = seed index 5 of the run
        assert np.array_equal(v.numpy(), trained[k][5].cpu().numpy()), k
