"""Population-based training on the GPU (purejaxql_b200/pbt.py).

1. pqn_pbt_event against the NumPy oracle (tests/pbt_oracle.py) on random rows, S from 2 to 65,535, both counter
   layouts, two chained events: fitness, order, parents, row copies, tables and the event key exactly.
2. pqn_radam_clip_step_pbt: bit-identical to pqn_radam_clip_step_seeds with sched_src = s (or a shared table) and
   lr_mult = 1, and with a permuted source and multipliers equal to the seeds entry on the scaled tables.
3. Each script (CNN on Breakout, packed-bit MLP with batch_norm, GRU on CartPole): PBT_INTERVAL >= NUM_UPDATES is the
   run without PBT bit for bit; a run with events matches it up to the first event, a seed never replaced matches it to
   the end, and at each event the children hold their parents' pre-event rows and hyperparameters as the oracle
   prescribes; graph and eager runs are bit-identical; a run resumed after an event ends like the uninterrupted run.
4. A two-point grid over a two-env list, two env-sharded ranks over gloo, and single_run's lineage yaml."""
import ctypes
import importlib
import os

import numpy as np
import pytest
import torch

import pbt_oracle as O
from oracle import jax_prng as jr
from purejaxql_b200 import _lib, engine, pbt, sweep

pytestmark = pytest.mark.gpu
NUPD, K = 5, 2                        # events after updates 2 and 4
ALL_KEYS = ["LAMBDA", "LR", "REW_SCALE", "GAMMA", "MAX_GRAD_NORM"]
_RUN = dict(NUM_EPOCHS=2, LR_LINEAR_DECAY=True, WANDB_MODE="disabled", TEST_DURING_TRAINING=False, NUM_SEEDS=4,
            SEED=0, PBT_PERTURB=ALL_KEYS, PBT_FACTORS=[0.8, 1.25], PBT_SEED=3, EPS_START=1.0, EPS_FINISH=0.05,
            EPS_DECAY=0.5, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65, REW_SCALE=1.0, LR=[5e-4, 1e-4])
CASES = {
    "minatar_cnn": ("pqn_minatar", dict(ENV_NAME="Breakout-MinAtar", NUM_ENVS=32, NUM_STEPS=8, NUM_MINIBATCHES=4,
                                        NORM_TYPE="layer_norm")),
    "gymnax_bits_batch_norm": ("pqn_gymnax", dict(ENV_NAME="Breakout-MinAtar", NUM_ENVS=32, NUM_STEPS=8,
                                                  NUM_MINIBATCHES=4, HIDDEN_SIZE=128, NUM_LAYERS=2,
                                                  NORM_TYPE="batch_norm")),
    "rnn_cartpole": ("pqn_rnn_gymnax", dict(ENV_NAME="CartPole-v1", NUM_ENVS=16, NUM_STEPS=12, MEMORY_WINDOW=3,
                                            NUM_MINIBATCHES=4, HIDDEN_SIZE=128, NUM_LAYERS=2, NORM_TYPE="layer_norm")),
}


def dev():
    return torch.device("cuda:0")


def _cfg(case, **kw):
    module, c = CASES[case]
    c = {**_RUN, **c, **kw}
    c["TOTAL_TIMESTEPS"] = c["TOTAL_TIMESTEPS_DECAY"] = float(NUPD * c["NUM_STEPS"] * c["NUM_ENVS"])
    return module, c


def _host(out):
    ts = out["runner_state"][0]
    res = {"params": ts.params_flat, "mu": ts.opt_state.mu, "nu": ts.opt_state.nu, "stats": ts.batch_stats_flat,
           "rng": out["runner_state"][-1]}
    res.update({f"metric:{k}": v for k, v in out["metrics"].items()})
    res = {k: v.cpu().numpy() for k, v in res.items()}
    if "pbt" in out:
        p = out["pbt"]
        res.update({"pbt:fitness": p["fitness"], "pbt:parent": p["parent"],
                    **{f"pbt:{k}": v for k, v in p["values"].items()}})
    return res


def _train(module, cfg, rngs, graph=True, hook=None):
    mod = importlib.import_module(f"purejaxql_b200.{module}")
    train = mod.make_train(dict(cfg, CUDA_GRAPH=graph))
    if hook:
        hook(train.engine)
    out = train(rngs)
    assert train.engine.graph_captured == graph
    return _host(out), out, train.engine


def _same(a, b, where, keys=None):
    for k in keys or a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), where + (k,)


# --------------------------------------------------------------------------- #
# 1. the event entry point against the oracle
# --------------------------------------------------------------------------- #
def _event_args(S, m, fit, cols, kp, part, perturb, factors, t, order, parent, fitness, ws):
    a = _lib.PbtEvent()
    a.S, a.m, a.fit, a.fit_stride, a.fit_cols = S, m, fit.data_ptr(), fit.stride(0), cols
    a.rng_mode, a.key = part, kp.data_ptr()
    a.n_perturb = len(perturb)
    for i, k in enumerate(perturb):
        a.perturb[i] = pbt.PERTURB_CODES[k]
    a.factors[0], a.factors[1] = factors
    a.params, a.mu, a.nu, a.P = t["params"].data_ptr(), t["mu"].data_ptr(), t["nu"].data_ptr(), t["params"].shape[1]
    a.batch_stats, a.stats_floats = t["stats"].data_ptr(), t["stats"].shape[1]
    a.eps, a.eps_rows, a.eps_from = t["eps"].data_ptr(), t["eps"].shape[0], 3
    for f, k in (("sched_src", "sched_src"), ("lr_mult", "lr_mult"), ("gamma", "gamma"), ("lambda_", "lam"),
                 ("max_norm", "max_norm"), ("rew_scale", "rew_scale")):
        setattr(a, f, t[k].data_ptr())
    a.fitness, a.order, a.parent, a.workspace = fitness.data_ptr(), order.data_ptr(), parent.data_ptr(), ws.data_ptr()
    return a


@pytest.mark.parametrize("part", [0, 1], ids=["original", "partitionable"])
@pytest.mark.parametrize("S", [2, 9, 1000, 65535])
def test_event_matches_the_oracle(S, part):
    L, rng = _lib.lib(), np.random.default_rng(S + part)
    m, cols, P, F, rows = max(1, S // 4), 3, 12, 6, 7
    perturb, factors = ["GAMMA", "LR", "LAMBDA", "REW_SCALE", "MAX_GRAD_NORM"], (0.8, 1.25)
    host = dict(params=rng.normal(size=(S, P)).astype(np.float32), mu=rng.normal(size=(S, P)).astype(np.float32),
                nu=rng.random((S, P)).astype(np.float32), stats=rng.normal(size=(S, F)).astype(np.float32),
                eps=rng.random((rows, S)).astype(np.float32), sched_src=np.arange(S, dtype=np.int32),
                lr_mult=np.ones(S, np.float32), gamma=rng.choice([0.99, 0.9, 0.1], S).astype(np.float32),
                lam=rng.choice([0.95, 0.65, 0.0], S).astype(np.float32),
                max_norm=rng.choice([10.0, 0.5], S).astype(np.float32),
                rew_scale=rng.choice([1.0, 0.1], S).astype(np.float32))
    t = {k: torch.from_numpy(v).to(dev()) for k, v in host.items()}
    kp_host = jr.PRNGKey(5)
    kp = torch.from_numpy(kp_host.view(np.int32).copy()).to(dev())
    ws = torch.empty(int(L.pqn_pbt_workspace_bytes(S, m)), dtype=torch.uint8, device=dev())
    for ev in range(2):
        fit_h = np.round(rng.normal(size=(S, cols + 2)), 1)          # ties, and NaN rows
        fit_h[rng.random(S) < 0.1, 1] = np.nan
        fit = torch.from_numpy(fit_h).to(dev())
        order = torch.zeros(S, dtype=torch.int32, device=dev())
        parent = torch.zeros(S, dtype=torch.int32, device=dev())
        fitness = torch.zeros(S, dtype=torch.float64, device=dev())
        _lib.check(L.pqn_pbt_event(ctypes.byref(_event_args(S, m, fit[:, 1:], cols, kp, part, perturb, factors, t,
                                                            order, parent, fitness, ws)), _lib.stream_ptr()))
        torch.cuda.synchronize()
        f = O.fitness(fit_h[:, 1:1 + cols])
        kp_host, o, par, children, parents, phi = O.plan(f, m, kp_host, len(perturb), factors, bool(part))
        assert np.array_equal(fitness.cpu().numpy(), f, equal_nan=True), ev
        assert np.array_equal(order.cpu().numpy(), o), ev
        assert np.array_equal(parent.cpu().numpy(), par), ev
        assert np.array_equal(kp.cpu().numpy().view(np.uint32), kp_host), ev
        for k in ("params", "mu", "nu", "stats"):
            want = host[k].copy()
            want[children] = host[k][parents]
            host[k] = want
        tabs, host["eps"] = O.apply({k: host[k] for k in ("sched_src", "lr_mult", "gamma", "lam", "max_norm",
                                                          "rew_scale")}, children, parents, phi, perturb, host["eps"], 3)
        host.update(tabs)
        for k, v in host.items():
            assert np.array_equal(t[k].cpu().numpy(), v), (ev, k)


def test_radam_clip_step_pbt_entry():
    L, S, P, steps = _lib.lib(), 6, 4 * 700, 4
    gen = torch.Generator(device="cpu").manual_seed(0)
    params0 = torch.randn(S, P, generator=gen).to(dev())
    grads = [(torch.randn(S, P, generator=gen) * torch.linspace(0.01, 0.4, S)[:, None]).to(dev()) for _ in range(steps)]
    lrs = [5e-4, 1e-4, 1e-3, 5e-5, 2e-4, 1e-4]
    tabs = np.stack([engine.radam_schedule_table(steps, lambda i, lr=lr: engine.linear_schedule(lr, 1e-20, 8, i))
                     for lr in lrs])
    mn = torch.tensor([10.0, 1.0, 5.0, 0.5, 10.0, 2.0], device=dev())

    def run(call, sched):
        s = torch.from_numpy(np.ascontiguousarray(sched)).to(dev())
        p, mu, nu = params0.clone(), torch.zeros_like(params0), torch.zeros_like(params0)
        st, gn = torch.zeros(1, dtype=torch.int32, device=dev()), torch.zeros(S * 64, device=dev())
        for g in grads:
            _lib.check(call(p, g, mu, nu, s, st, gn))
        torch.cuda.synchronize()
        return {"p": p.cpu().numpy(), "mu": mu.cpu().numpy(), "nu": nu.cpu().numpy()}

    def seeds(stride):
        return lambda p, g, mu, nu, s, st, gn: L.pqn_radam_clip_step_seeds(
            _lib.p(p), _lib.p(g), _lib.p(mu), _lib.p(nu), _lib.p(s), stride, _lib.p(st), _lib.p(gn), S, P, _lib.p(mn),
            0.9, 0.999, 1e-8, _lib.stream_ptr())

    def pbt_(stride, src, mult):
        src_t = torch.tensor(src, dtype=torch.int32, device=dev())
        mult_t = torch.tensor(mult, dtype=torch.float32, device=dev())
        return lambda p, g, mu, nu, s, st, gn: L.pqn_radam_clip_step_pbt(
            _lib.p(p), _lib.p(g), _lib.p(mu), _lib.p(nu), _lib.p(s), stride, _lib.p(src_t), _lib.p(mult_t),
            _lib.p(st), _lib.p(gn), S, P, _lib.p(mn), 0.9, 0.999, 1e-8, _lib.stream_ptr())
    ident, ones = list(range(S)), [1.0] * S
    _same(run(pbt_(4 * steps, ident, ones), tabs), run(seeds(4 * steps), tabs), ("per-seed tables",))
    _same(run(pbt_(0, [0] * S, ones), tabs[1]), run(seeds(0), tabs[1]), ("shared table",))
    src, mult = [3, 0, 0, 5, 1, 2], np.array([1.25, 0.8, 1.0, 1.5625, 0.64, 1.25], np.float32)
    scaled = tabs[src].copy()
    scaled[:, :, 0] = scaled[:, :, 0] * mult[:, None]
    _same(run(pbt_(4 * steps, src, mult.tolist()), tabs), run(seeds(4 * steps), scaled), ("source and multiplier",))


# --------------------------------------------------------------------------- #
# 3. the scripts
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("case", list(CASES))
def test_interval_at_or_past_the_end_is_the_run_without_pbt(case):
    module, cfg = _cfg(case, PBT_INTERVAL=0)
    S = sweep.Grid(cfg).total_seeds
    rngs = sweep.Grid(cfg).tile(jr.split(jr.PRNGKey(7), 4))
    base, _, _ = _train(module, cfg, rngs)
    got, out, eng = _train(module, dict(cfg, PBT_INTERVAL=NUPD), rngs)
    assert eng.population is not None and out["pbt"]["events"] == [] and S == 8
    _same(base, got, (case,), keys=list(base))
    assert np.array_equal(out["pbt"]["values"]["LR"][0], [5e-4] * 4 + [1e-4] * 4)


def _capture(caps):
    """Wrap each engine's Population.event: the buffers it reads before and after every event."""
    def hook(eng):
        orig = pbt.Population.event

        def snap(pop, params, mu, nu, stats):
            d = {"params": params, "mu": mu, "nu": nu, "eps": pop.hp["eps"], "sched_src": pop.sched_src,
                 "lr_mult": pop.lr_mult, "gamma": pop.hp["gamma"], "lam": pop.hp["lam"],
                 "max_norm": pop.hp["max_norm"], "rew_scale": pop.hp["rew_scale"], "kp": pop.kp}
            if stats is not None:
                d["stats"] = stats
            torch.cuda.synchronize()
            return {k: v.cpu().numpy().copy() for k, v in d.items()}

        def event(pop, n_done, fit, c0, cols, params, mu, nu, stats):
            torch.cuda.synchronize()
            pre = snap(pop, params, mu, nu, stats)
            pre["fit"] = fit.cpu().numpy()[:, c0:c0 + cols].copy()
            orig(pop, n_done, fit, c0, cols, params, mu, nu, stats)
            caps.append((n_done, pre, snap(pop, params, mu, nu, stats)))
        eng_pop = eng._population

        def population(*a, **kw):
            p = eng_pop(*a, **kw)
            p.event = event.__get__(p)
            return p
        eng._population = population
    return hook


@pytest.mark.parametrize("case", list(CASES))
def test_events_exploit_and_explore_as_the_oracle_prescribes(case):
    module, cfg = _cfg(case, PBT_INTERVAL=0)
    rngs = sweep.Grid(cfg).tile(jr.split(jr.PRNGKey(7), 4))
    base, _, _ = _train(module, cfg, rngs)
    caps = []
    got, out, eng = _train(module, dict(cfg, PBT_INTERVAL=K), rngs, hook=_capture(caps))
    res = out["pbt"]
    assert res["events"] == [2, 4] and [c[0] for c in caps] == [2, 4]
    S, m = 8, 2
    metric_keys = [k for k in base if k.startswith("metric:")]
    for k in metric_keys:                                 # updates 1 and 2 come before the first event
        assert np.array_equal(got[k][:, :K], base[k][:, :K], equal_nan=True), k
    replaced = set()
    kp = jr.PRNGKey(3)
    for e, (n, pre, post) in enumerate(caps):
        f = O.fitness(pre["fit"])
        assert np.array_equal(res["fitness"][e], f, equal_nan=True)
        kp, o, par, children, parents, phi = O.plan(f, m, kp, len(ALL_KEYS), (0.8, 1.25))
        assert np.array_equal(res["parent"][e], par) and np.array_equal(post["kp"].view(np.uint32), kp)
        replaced |= set(children.tolist())
        for k in ("params", "mu", "nu", "stats"):
            if k in pre:
                want = pre[k].copy()
                want[children] = pre[k][parents]
                assert np.array_equal(post[k], want), (e, k)
        tabs, eps = O.apply({k: pre[k] for k in ("sched_src", "lr_mult", "gamma", "lam", "max_norm", "rew_scale")},
                            children, parents, phi, ALL_KEYS, pre["eps"], n)
        for k, v in tabs.items():
            assert np.array_equal(post[k], v), (e, k)
        assert np.array_equal(post["eps"], eps)
        for key, row in (("GAMMA", "gamma"), ("LAMBDA", "lam"), ("MAX_GRAD_NORM", "max_norm"),
                         ("REW_SCALE", "rew_scale")):
            assert np.array_equal(res["values"][key][e + 1], post[row].astype(np.float64)), key
        lr_pt = np.array([5e-4, 1e-4])[sweep.Grid(cfg).point_of(0, S)[post["sched_src"]]]
        assert np.array_equal(res["values"]["LR"][e + 1], lr_pt * post["lr_mult"].astype(np.float64))
    kept = [s for s in range(S) if s not in replaced]
    assert kept and len(replaced) >= m
    for k in base:
        assert np.array_equal(got[k][kept], base[k][kept], equal_nan=True), k
    assert not np.array_equal(got["params"][sorted(replaced)], base["params"][sorted(replaced)])
    # graph and eager runs take the same decisions and end in the same bits
    eager, out_e, _ = _train(module, dict(cfg, PBT_INTERVAL=K), rngs, graph=False)
    _same(eager, got, (case, "eager"))


@pytest.mark.parametrize("case", list(CASES))
def test_resume_after_an_event_ends_like_the_uninterrupted_run(case, tmp_path):
    module, cfg = _cfg(case, PBT_INTERVAL=K, STATE_SAVE_INTERVAL=4, SAVE_PATH=str(tmp_path), ALG_NAME="pqn")
    rngs = sweep.Grid(cfg).tile(jr.split(jr.PRNGKey(7), 4))
    full, _, _ = _train(module, cfg, rngs)
    from purejaxql_b200 import state
    path = state.state_file(dict(cfg))
    assert os.path.exists(path)                           # written after update 4, after its event
    resumed, _, eng = _train(module, dict(cfg, RESUME_FROM=path, STATE_SAVE_INTERVAL=0), rngs, graph=False)
    assert eng.resume["meta"]["n_done"] == 4
    _same(resumed, full, (case, "resumed"))


# --------------------------------------------------------------------------- #
# 4. composition
# --------------------------------------------------------------------------- #
def test_grid_and_env_list_compose():
    from purejaxql_b200 import pqn_gymnax
    c = dict(_RUN, ENV_NAME=["CartPole-v1", "Acrobot-v1"], NUM_ENVS=32, NUM_STEPS=8, NUM_MINIBATCHES=4, NUM_SEEDS=2,
             HIDDEN_SIZE=128, NUM_LAYERS=2, NORM_TYPE="layer_norm", PBT_INTERVAL=1, PBT_FRACTION=0.5)
    c["TOTAL_TIMESTEPS"] = c["TOTAL_TIMESTEPS_DECAY"] = float(NUPD * 8 * 32)
    rngs = sweep.Grid(c).tile(jr.split(jr.PRNGKey(7), 2))
    outs = pqn_gymnax.make_train(dict(c))(rngs)
    for name in c["ENV_NAME"]:
        alone, out, _ = _train("pqn_gymnax", dict(c, ENV_NAME=name), rngs)
        assert out["pbt"]["events"] == [1, 2, 3, 4]
        _same(_host(outs[name]), alone, (name,))


def _rank_worker(rank, world, out_dir):
    from test_gpu_env_shard_train import _init_group
    dist, _ = _init_group(rank, world, out_dir)
    try:
        from purejaxql_b200 import pqn_gymnax
        _, cfg = _cfg("gymnax_bits_batch_norm", ENV_NAME="CartPole-v1", NORM_TYPE="layer_norm", PBT_INTERVAL=1)
        train = pqn_gymnax.make_train(dict(cfg, CUDA_GRAPH=False))
        train.engine.env_shard = (rank, world)
        out = train(sweep.Grid(cfg).tile(jr.split(jr.PRNGKey(7), 4)))
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **_host(out))
    finally:
        dist.destroy_process_group()


def test_two_env_sharded_ranks_take_the_same_decisions(tmp_path):
    from test_gpu_env_shard_train import _spawn
    _spawn(_rank_worker, 2, (), tmp_path)
    ranks = [dict(np.load(tmp_path / f"rank{r}.npz")) for r in range(2)]
    assert ranks[0]["pbt:parent"].shape == (NUPD - 1, 8)
    assert (ranks[0]["pbt:parent"] != np.arange(8)).any()
    for k, v in ranks[0].items():
        if k == "rng" or k.startswith("metric:"):
            continue
        assert np.array_equal(ranks[1][k], v, equal_nan=v.dtype.kind == "f"), k


def test_single_run_writes_the_lineage(tmp_path):
    import yaml
    from purejaxql_b200 import config_loader, pqn_minatar
    c = config_loader.compose(["+alg=pqn_minatar", "NUM_SEEDS=8", "alg.LR=[0.001,0.0005,0.0001,0.00005]",
                               "PBT_INTERVAL=20", f"SAVE_PATH={tmp_path}", "alg.TOTAL_TIMESTEPS=90112",
                               "alg.TOTAL_TIMESTEPS_DECAY=1e7", "alg.TEST_DURING_TRAINING=False"])
    out = pqn_minatar.single_run(c)
    d = tmp_path / "Asterix-MinAtar"
    lin = yaml.safe_load((d / "pqn_Asterix-MinAtar_seed0_pbt.yaml").read_text())
    assert lin["events"] == [20] == out["pbt"]["events"] and len(lin["parent"][0]) == 32
    assert lin["settings"]["interval"] == 20 and sorted(lin["values"]) == sorted(sweep.SWEEP_KEYS)
    assert sum(p != s for s, p in enumerate(lin["parent"][0])) == 8
