"""Env-sharded training (engine.PQNEngine with ``env_shard``, what DATA_PARALLEL=auto picks when NUM_SEEDS < world)
against the NumPy replay of tests/env_shard_oracle.py, on one GPU.

W processes share cuda:0 and join a gloo process group through a FileStore (no TCP port); the engine's
``dist.all_reduce`` calls on CUDA tensors go through gloo.  Each rank trains its env shard of every seed and saves
what it ends with; the parent process replays the sharded algorithm for the union of the shards in NumPy and checks:

* across ranks, bit for bit: parameters, RAdam moments, running statistics, final key and every metric;
* the concatenated rank rollouts (action, reward, done) against the oracle's unsharded rollout;
* per update: td_loss, qvals and the five episode metrics (union means over T * E_total), env_step and grad_steps;
* after the last update: parameters, the BatchNorm_0 running statistics of the union minibatches (whose count is
  mb * world, times 100 pixels for the CNN), the final key, and each rank's env state against its slice;
* with eps < 1, the engine's actions against the oracle's eps-greedy ones (a flip only on a numerical Q tie), and
  the evaluation metrics, which every rank computes on the full parameters, against ``get_test_metrics``.

The refusal of batch statistics in this mode and ``single_run`` under a 2-rank launch are checked as well.
The checks are of the algorithm, not of NCCL: in-stream collectives and collectives inside a CUDA graph are left to
tests/test_gpu_multi.py on a machine with two GPUs."""
import importlib
import json
import multiprocessing
import os
from datetime import timedelta

import numpy as np
import pytest
import torch

import env_shard_oracle as SO
from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R

pytestmark = pytest.mark.gpu

S, NUPD = 2, 3                      # 3 updates x 2 epochs x 4 minibatches: the first five RAdam steps are unrectified
INTEGER_ENVS = ("Breakout-MinAtar",)


def _cfg(env, **kw):
    c = dict(ENV_NAME=env, NUM_ENVS=128, NUM_STEPS=8, NUM_MINIBATCHES=4, NUM_EPOCHS=2, EPS_START=1.0, EPS_FINISH=1.0,
             EPS_DECAY=0.1, LR=5e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65, NORM_TYPE="layer_norm",
             LR_LINEAR_DECAY=True, WANDB_MODE="disabled", TEST_DURING_TRAINING=False, CUDA_GRAPH=False)
    c.update(kw)
    c["TOTAL_TIMESTEPS"] = c["TOTAL_TIMESTEPS_DECAY"] = float(NUPD * c["NUM_STEPS"] * c["NUM_ENVS"])
    return c


def _leaves(tree, prefix=""):
    for k, v in tree.items():
        if isinstance(v, dict):
            yield from _leaves(v, f"{prefix}{k}/")
        else:
            yield f"{prefix}{k}", v


def _init_group(rank, world, out_dir):
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method=f"file://{out_dir}/pg", rank=rank, world_size=world,
                            timeout=timedelta(seconds=120))
    calls = [0]
    all_reduce = dist.all_reduce

    def counted(*a, **kw):                          # the engine looks dist.all_reduce up at every call
        calls[0] += 1
        return all_reduce(*a, **kw)
    dist.all_reduce = counted
    return dist, calls


def _train_worker(rank, world, case, out_dir):
    dist, calls = _init_group(rank, world, out_dir)
    try:
        mod = importlib.import_module(f"purejaxql_b200.{case['module']}")
        cfg = dict(case["cfg"])
        train = mod.make_train(cfg)
        eng = train.engine
        eng.env_shard = (rank, world)
        cap = {}
        orig = eng.spec.init
        eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
        bufs = {k: [] for k in ("action", "reward", "done")}
        eng.on_update_end = lambda n, b: [v.append(b[k].cpu().numpy()) for k, v in bufs.items()]
        rngs = case["rngs"]                                                          # uint32 [S, 2]
        if case.get("refused"):
            try:
                train(rngs)
            except NotImplementedError as e:
                with open(os.path.join(out_dir, f"refused{rank}.json"), "w") as f:
                    json.dump({"message": str(e), "collectives": calls[0]}, f)
                return
            raise AssertionError("env-sharded training with batch statistics was not refused")
        out = train(rngs)
        ts = out["runner_state"][0]
        save = {"params_flat": ts.params_flat, "mu": ts.opt_state.mu, "nu": ts.opt_state.nu,
                "batch_stats_flat": ts.batch_stats_flat, "rng": out["runner_state"][3],
                "env_state": out["runner_state"][1][1]}
        save.update({f"metric:{k}": v for k, v in out["metrics"].items()})
        save.update({f"init:{k}": v for k, v in _leaves(eng.spec.unflatten(cap["flat"]))})
        save.update({f"params:{k}": v for k, v in _leaves(ts.params)})
        save.update({f"stats:{k}": v for k, v in _leaves(ts.batch_stats)})
        arrays = {k: v.cpu().numpy() for k, v in save.items()}
        arrays.update({f"buf:{k}": np.stack(v) for k, v in bufs.items()})          # [NUPD, S, T, E / world]
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **arrays)
        with open(os.path.join(out_dir, f"cfg{rank}.json"), "w") as f:
            json.dump({"NUM_UPDATES_DECAY": cfg["NUM_UPDATES_DECAY"], "TEST_NUM_STEPS": cfg["TEST_NUM_STEPS"],
                       "collectives": calls[0]}, f)
    finally:
        dist.destroy_process_group()


def _spawn(fn, world, args, tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(fn, args=(world,) + args + (str(tmp_path),), nprocs=world, join=True)
    assert not multiprocessing.active_children()


def _fields(env_name, state):
    from purejaxql_b200 import envs
    return {k: v.numpy() for k, v in envs.state_to_fields(env_name, torch.from_numpy(state)).items()}


def _check_against_oracle(case, world, tmp_path):
    cfg, name, kind = case["cfg"], case["cfg"]["ENV_NAME"], case["kind"]
    T, E, nmb, epochs = cfg["NUM_STEPS"], cfg["NUM_ENVS"], cfg["NUM_MINIBATCHES"], cfg["NUM_EPOCHS"]
    E_l = E // world
    ranks = [dict(np.load(tmp_path / f"rank{r}.npz")) for r in range(world)]
    used = json.loads((tmp_path / "cfg0.json").read_text())
    # ---- every rank ends with the same replicated state
    for k, v in ranks[0].items():
        if k.startswith(("buf:", "env_state")):
            continue
        for r in range(1, world):
            assert np.array_equal(ranks[r][k], v, equal_nan=v.dtype.kind == "f"), (k, r)
    # 2 all-reduces per minibatch step (gradient, input statistics) and 3 per update (loss, qvals, info sums)
    assert used["collectives"] == NUPD * (2 * nmb * epochs + 3), used
    cfg = dict(cfg, NUM_UPDATES_DECAY=used["NUM_UPDATES_DECAY"])
    eps_lt_1 = cfg["EPS_START"] < 1.0
    integer = name in INTEGER_ENVS
    itol, ltol = (1e-6, 2e-4 if eps_lt_1 else 1e-4) if integer else (2e-2, 2e-2)
    m0 = {k[len("metric:"):]: v for k, v in ranks[0].items() if k.startswith("metric:")}
    fwd = R.cnn_forward if kind == "cnn" else R.mlp_forward
    total = cfg["NUM_UPDATES_DECAY"] * nmb * epochs
    lr_fn = lambda i: R.linear_schedule(cfg["LR"], 1e-20, total, i)
    test = cfg["TEST_DURING_TRAINING"]
    ties, done_flips, compared_eval = [], 0, 0
    for s in range(S):
        params = {k[len("init:"):]: v[s].astype(np.float32) for k, v in ranks[0].items() if k.startswith("init:")}
        K1 = jr.split(case["rngs"][s], 2)[0]
        K2 = jr.split(K1, 2)[0]
        k = jr.split(K2, 2); K3, kR = k[0], k[1]
        env = G.make(name, flatten=case["flatten"])
        obs, st = env.reset(jr.split(kR, E))
        rng = jr.split(K3, 2)[1]
        opt = R.opt_init(params)
        F = ranks[0]["stats:BatchNorm_0/mean"].shape[1]
        bs = {"mean": np.zeros(F, np.float32), "var": np.ones(F, np.float32)}
        if test:
            def evaluate(p, key):
                return R.get_test_metrics(G.make(name, flatten=case["flatten"]), fwd, p, key, cfg["TEST_NUM_ENVS"],
                                          used["TEST_NUM_STEPS"], cfg["EPS_TEST"])
            test_every = int(NUPD * cfg["TEST_INTERVAL"])
            evals = evaluate(params, jr.split(K1, 2)[1])
        bad_envs = set()
        for u in range(NUPD):
            got = {kk: float(v[s, u]) for kk, v in m0.items()}
            union = {kk: np.concatenate([rk[f"buf:{kk}"][u, s] for rk in ranks], axis=1) for kk in ("action", "reward",
                                                                                                 "done")}
            log = []
            params, opt, bs, obs, st, rng, m, tr, tg = SO.update_step_sharded(
                env, kind, params, opt, bs, obs, st, rng, cfg, u, lr_fn, world,
                forced_actions=union["action"] if eps_lt_1 else None, tie_log=log)
            where = (name, world, s, u)
            for (t, e, a_own, a_forced, gap) in log:
                assert gap < 1e-4, where + (t, e, a_own, a_forced, gap)
            ties += [where + x for x in log]
            assert np.array_equal(union["action"], tr["action"]), where
            if integer:
                assert np.array_equal(union["reward"], tr["reward"]), where
                assert np.array_equal(union["done"].astype(bool), tr["done"].astype(bool)), where
            else:                              # fp32 physics: a termination may flip where a pole is at its limit
                flip = union["done"].astype(bool) != tr["done"].astype(bool)
                done_flips += int(flip.sum())
                bad_envs |= set(np.nonzero(flip.any(0))[0].tolist())
                assert np.abs(union["reward"] - tr["reward"]).max() < 1e-6, where
            for kk in R.INFO_KEYS:
                assert abs(got[kk] - m[kk]) < itol * max(1, abs(m[kk])), where + (kk, got[kk], m[kk])
            assert abs(got["td_loss"] - m["td_loss"]) < ltol * max(1.0, abs(m["td_loss"])), where + (got["td_loss"],
                                                                                                   m["td_loss"])
            assert abs(got["qvals"] - m["qvals"]) < ltol * max(1.0, abs(m["qvals"])), where + (got["qvals"], m["qvals"])
            assert int(got["env_step"]) == (u + 1) * T * E, where
            assert int(got["grad_steps"]) == (u + 1) * nmb * epochs, where
            if test:
                k = jr.split(rng, 2); rng, kT = k[0], k[1]
                if (u + 1) % test_every == 0:
                    evals = evaluate(params, kT)
                for kk in R.INFO_KEYS:
                    g, w = got[f"test/{kk}"], evals[kk]
                    if np.isnan(w):
                        assert np.isnan(g), where + (kk, g)
                    else:
                        compared_eval += 1
                        assert abs(g - w) <= 1e-6 * max(1.0, abs(w)), where + (kk, g, w)
        if kind == "cnn" or integer:
            ptol = 5e-5 if kind == "cnn" else 1e-4
            for p, want in params.items():
                d = np.abs(ranks[0][f"params:{p}"][s] - want).max()
                assert d < ptol, (name, world, s, p, d)
        for j in ("mean", "var"):
            d = np.abs(ranks[0][f"stats:BatchNorm_0/{j}"][s] - bs[j]).max()
            assert d < (1e-6 if integer else 1e-5), (name, world, s, j, d)
        assert np.array_equal(ranks[0]["rng"][s].view(np.uint32), rng), (name, world, s)
        for r in range(world):
            lo = r * E_l
            f = _fields(name, ranks[r]["env_state"][:, s * E_l:(s + 1) * E_l])
            keep = np.array([lo + e not in bad_envs for e in range(E_l)])
            for kk, v in st.items():
                g = f[kk].astype(v.dtype).reshape(v[lo:lo + E_l].shape)[keep]
                w = v[lo:lo + E_l][keep]
                if integer or v.dtype.kind != "f":
                    assert np.array_equal(g, w), (name, world, s, r, kk)
                else:
                    assert np.allclose(g, w, rtol=1e-4, atol=1e-4), (name, world, s, r, kk)
    if eps_lt_1:
        print(f"\n[env-shard eps<1] {name} world {world}: {len(ties)} argmax flips on Q ties out of "
              f"{S * NUPD * T * E} actions", ties[:5])
        assert len(ties) <= 2e-3 * S * NUPD * T * E
    if test:
        assert compared_eval > 0, "no evaluation episode ended: the test metrics were never compared"
    if not integer:
        print(f"\n[env-shard] {name} world {world}: {done_flips} termination flips out of {S * NUPD * T * E} steps "
              f"(an env with a flip is left out of the state check of its seed)")
        assert done_flips <= 1e-3 * S * NUPD * T * E


CASES = {
    # MinAtar CNN; mb = 390 (world 2) and 260 (world 3) rows: ragged tiles, shard bounds off the 128-env blocks
    "cnn_breakout_e390": dict(module="pqn_minatar", kind="cnn", flatten=False, cfg=_cfg("Breakout-MinAtar", NUM_ENVS=390)),
    "mlp_cartpole": dict(module="pqn_gymnax", kind="mlp", flatten=True,
                         cfg=_cfg("CartPole-v1", NUM_ENVS=64, NUM_STEPS=16, HIDDEN_SIZE=128, NUM_LAYERS=2,
                                  REW_SCALE=0.1, LAMBDA=0.95)),
    "mlp_cartpole_partitionable": dict(module="pqn_gymnax", kind="mlp", flatten=True, partitionable=True,
                                       cfg=_cfg("CartPole-v1", NUM_ENVS=64, NUM_STEPS=16, HIDDEN_SIZE=128,
                                                NUM_LAYERS=2, REW_SCALE=0.1, LAMBDA=0.95,
                                                JAX_THREEFRY_PARTITIONABLE=1)),
    # packed-bit MLP on MinAtar: its input statistics count mb * world rows, not pixels
    "mlp_bits_breakout": dict(module="pqn_gymnax", kind="mlp", flatten=True,
                              cfg=_cfg("Breakout-MinAtar", HIDDEN_SIZE=128, NUM_LAYERS=2, REW_SCALE=0.1, LAMBDA=0.95)),
    # greedy actions and the evaluation rollout on every rank
    "cnn_breakout_eps_eval": dict(module="pqn_minatar", kind="cnn", flatten=False,
                                  cfg=_cfg("Breakout-MinAtar", EPS_START=0.6, EPS_FINISH=0.1, EPS_DECAY=1.0,
                                           TEST_DURING_TRAINING=True, TEST_INTERVAL=0.67, TEST_NUM_ENVS=8,
                                           EPS_TEST=0.0)),
}


@pytest.mark.parametrize("case_name,world", [("cnn_breakout_e390", 2), ("cnn_breakout_e390", 3), ("mlp_cartpole", 2),
                                             ("mlp_cartpole_partitionable", 2), ("mlp_bits_breakout", 2),
                                             ("cnn_breakout_eps_eval", 2)])
def test_env_sharded_training_matches_oracle(case_name, world, tmp_path):
    case = dict(CASES[case_name])
    part = bool(case.get("partitionable", False))
    jr.DEFAULT_PARTITIONABLE = part
    try:
        case["rngs"] = jr.split(jr.PRNGKey(7), S)
        _spawn(_train_worker, world, (case,), tmp_path)
        _check_against_oracle(case, world, tmp_path)
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("module,env_name,extra", [
    ("pqn_minatar", "Breakout-MinAtar", dict(NORM_TYPE="batch_norm")),
    ("pqn_gymnax", "CartPole-v1", dict(NORM_INPUT=True, HIDDEN_SIZE=128, NUM_LAYERS=2)),
], ids=["batch_norm", "norm_input"])
def test_batch_statistics_are_refused_before_any_collective(module, env_name, extra, tmp_path):
    case = dict(module=module, refused=True, rngs=jr.split(jr.PRNGKey(3), S), cfg=_cfg(env_name, **extra))
    _spawn(_train_worker, 2, (case,), tmp_path)
    for r in range(2):
        got = json.loads((tmp_path / f"refused{r}.json").read_text())
        assert "DATA_PARALLEL=seeds" in got["message"] and got["collectives"] == 0, (r, got)


def _single_run_worker(rank, world, out_dir):
    os.environ.update(WORLD_SIZE=str(world), LOCAL_RANK="0", RANK=str(rank))
    dist, calls = _init_group(rank, world, out_dir)
    try:
        from purejaxql_b200 import config_loader, pqn_minatar
        engines = []
        make_train = pqn_minatar.make_train

        def recording_make_train(config):
            train = make_train(config)
            engines.append(train.engine)
            return train
        pqn_minatar.make_train = recording_make_train
        c = config_loader.compose(["+alg=pqn_minatar", "alg.ENV_NAME=Breakout-MinAtar", "NUM_SEEDS=1",
                                   f"SAVE_PATH={out_dir}/save{rank}", "alg.TOTAL_TIMESTEPS=8192",
                                   "alg.TOTAL_TIMESTEPS_DECAY=8192", "alg.TEST_DURING_TRAINING=False"])
        out = pqn_minatar.single_run(c)
        assert dist.get_backend() == "gloo" and len(engines) == 1
        arrays = {f"params:{k}": v.cpu().numpy() for k, v in _leaves(out["runner_state"][0].params)}
        arrays["env_step"] = out["metrics"]["env_step"].cpu().numpy()
        np.savez(os.path.join(out_dir, f"single{rank}.npz"), **arrays)
        with open(os.path.join(out_dir, f"single{rank}.json"), "w") as f:
            json.dump({"env_shard": list(engines[0].env_shard), "collectives": calls[0]}, f)
    finally:
        dist.destroy_process_group()


def test_single_run_shards_envs_and_saves_on_rank_zero(tmp_path):
    """NUM_SEEDS=1 under a 2-rank launch: ``auto`` picks env sharding, the ranks end with the same parameters and
    rank 0 alone writes the checkpoint, which holds the returned parameters."""
    from purejaxql_b200.utils.save_load import load_params
    _spawn(_single_run_worker, 2, (), tmp_path)
    outs = [dict(np.load(tmp_path / f"single{r}.npz")) for r in range(2)]
    for r in range(2):
        info = json.loads((tmp_path / f"single{r}.json").read_text())
        assert info["env_shard"] == [r, 2] and info["collectives"] > 0, (r, info)
    for k, v in outs[0].items():
        assert np.array_equal(outs[1][k], v), k
    assert outs[0]["env_step"][0, -1] == 8192                      # counted over both shards' 2 x 64 envs
    assert not (tmp_path / "save1").exists(), "rank 1 wrote a checkpoint"
    d = tmp_path / "save0" / "Breakout-MinAtar"
    assert sorted(p.name for p in d.iterdir()) == ["pqn_Breakout-MinAtar_seed0_config.yaml",
                                                   "pqn_Breakout-MinAtar_seed0_vmap0.safetensors"]
    tree = load_params(str(d / "pqn_Breakout-MinAtar_seed0_vmap0.safetensors"))
    saved = dict(_leaves(tree))
    assert sorted(saved) == sorted(k[len("params:"):] for k in outs[0] if k.startswith("params:"))
    for k, v in saved.items():
        assert np.array_equal(v.numpy(), outs[0][f"params:{k}"][0]), k
