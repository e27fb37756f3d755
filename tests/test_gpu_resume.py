"""Resuming a run from its training state (STATE_SAVE_INTERVAL / RESUME_FROM) gives the bits of the uninterrupted run.

Run A trains 5 updates with STATE_SAVE_INTERVAL=2 and keeps a copy of the state written after update 2.  Run B is a
new make_train with RESUME_FROM set to that copy: it runs updates 3..5 only (no initialiser, reset or warm-up) and
must return what A returned, bit for bit: parameters, running statistics, RAdam moments, every metric column, the
test history and last evaluation, the runner key, the env state, the last observations and, for the GRU, its memory
and hidden state.  The state B writes after update 4 must equal A's.  Two gloo ranks on one GPU (FileStore, as in
tests/test_gpu_env_shard_train.py) resume their own files, seed-sharded and env-sharded."""
import hashlib
import importlib
import json
import multiprocessing
import os
import shutil
from datetime import timedelta

import numpy as np
import pytest
import torch

from oracle import jax_prng as jr

pytestmark = pytest.mark.gpu

NUPD = 5


def _cfg(env, **kw):
    c = dict(ENV_NAME=env, ALG_NAME="pqn", NUM_ENVS=64, NUM_STEPS=8, NUM_MINIBATCHES=4, NUM_EPOCHS=2, EPS_START=1.0,
             EPS_FINISH=0.05, EPS_DECAY=0.5, LR=5e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65,
             NORM_TYPE="layer_norm", LR_LINEAR_DECAY=True, WANDB_MODE="disabled", TEST_DURING_TRAINING=False,
             SEED=0, NUM_SEEDS=2, HIDDEN_SIZE=128, NUM_LAYERS=2, REW_SCALE=1.0)
    c.update(kw)
    c["TOTAL_TIMESTEPS"] = c["TOTAL_TIMESTEPS_DECAY"] = float(NUPD * c["NUM_STEPS"] * c["NUM_ENVS"])
    return c


def _rnn_cfg(**kw):
    return _cfg("CartPole-v1", ALG_NAME="pqn_rnn", NUM_ENVS=32, NUM_STEPS=16, NUM_MINIBATCHES=4, NUM_EPOCHS=2,
                MEMORY_WINDOW=4, LAMBDA=0.95, **kw)


_EVAL = dict(TEST_DURING_TRAINING=True, TEST_INTERVAL=0.4, TEST_NUM_ENVS=8, TEST_NUM_STEPS=60, EPS_TEST=0.0)
CASES = {
    "cnn_breakout": ("pqn_minatar", _cfg("Breakout-MinAtar", NUM_ENVS=128)),
    "cnn_breakout_eval": ("pqn_minatar", _cfg("Breakout-MinAtar", NUM_ENVS=128, **_EVAL)),
    "mlp_cartpole": ("pqn_gymnax", _cfg("CartPole-v1")),
    "mlp_cartpole_partitionable": ("pqn_gymnax", _cfg("CartPole-v1", JAX_THREEFRY_PARTITIONABLE=1)),
    "mlp_cartpole_lr_grid": ("pqn_gymnax", _cfg("CartPole-v1", LR=[5e-4, 1e-3])),
    "mlp_cartpole_eval": ("pqn_gymnax", _cfg("CartPole-v1", **_EVAL)),
    "mlp_bits_breakout": ("pqn_gymnax", _cfg("Breakout-MinAtar")),
    "rnn_cartpole": ("pqn_rnn_gymnax", _rnn_cfg()),
    "rnn_cartpole_batch_norm": ("pqn_rnn_gymnax", _rnn_cfg(NORM_TYPE="batch_norm")),
    "rnn_cartpole_eval": ("pqn_rnn_gymnax", _rnn_cfg(**_EVAL)),
    "rnn_cartpole_partitionable": ("pqn_rnn_gymnax", _rnn_cfg(JAX_THREEFRY_PARTITIONABLE=1)),
}


def _collect(out):
    """Everything train() returned, as host arrays."""
    ts, tail = out["runner_state"][0], out["runner_state"][1:]
    d = {"params": ts.params_flat, "batch_stats": ts.batch_stats_flat, "mu": ts.opt_state.mu, "nu": ts.opt_state.nu}
    d.update({f"metric/{k}": v for k, v in out["metrics"].items()})
    if len(tail) == 3:                                             # feed-forward: ((obs, env_state), test, rng)
        (obs, st), tm, rng = tail
        d.update(last_obs=obs, env_state=st, rng=rng)
    else:                                                          # GRU: (mem, (hs, obs, done, action, env_state), ...)
        mem, (hs, lo, ld, la, st), tm, rng = tail
        d.update({f"mem/{k}": v for k, v in vars(mem).items()})
        d.update(hs=hs, last_obs=lo, last_done=ld, last_action=la, env_state=st, rng=rng)
    if tm is not None:
        d.update({f"test_metrics/{k}": v for k, v in tm.items()})
    return {k: np.ascontiguousarray(v.detach().cpu().numpy()) for k, v in d.items()}


def _assert_same_bits(a, b, where):
    assert sorted(a) == sorted(b), where
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, (where, k)
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), (where, k)


def _train(module, cfg, rngs, keep=None, **engine_attrs):
    """make_train + train; returns (host outputs, sweep table, engine, columns it ran, whether it initialised).  With
    `keep`, the state file written after update 2 is copied there."""
    mod = importlib.import_module(f"purejaxql_b200.{module}")
    train = mod.make_train(dict(cfg))
    eng = train.engine
    for k, v in engine_attrs.items():
        setattr(eng, k, v)
    ran, inits = [], []
    orig = eng.spec.init
    eng.spec.init = lambda *a: inits.append(1) or orig(*a)

    def begin(col):
        ran.append(col)
        if keep and col == 2:                                      # the state written after update 2
            shutil.copyfile(eng_state_path(eng), keep)
    eng.on_update_begin = begin
    out = train(rngs)
    return _collect(out), out["sweep"], eng, ran, bool(inits)


def eng_state_path(eng):
    from purejaxql_b200 import state
    return state.state_file(eng.cfg, *eng._placement()[1:])


def _a_then_b(module, cfg, rngs, tmp, tag=""):
    """Run A (5 updates, state after every 2nd) and B (resumed from A's state after update 2); returns both."""
    keep = os.path.join(tmp, f"after2{tag}.safetensors")
    cfg_a = dict(cfg, SAVE_PATH=os.path.join(tmp, f"a{tag}"), STATE_SAVE_INTERVAL=2)
    a, sweep_a, eng_a, ran_a, init_a = _train(module, cfg_a, rngs, keep)
    assert ran_a == list(range(NUPD)) and init_a
    cfg_b = dict(cfg, SAVE_PATH=os.path.join(tmp, f"b{tag}"), STATE_SAVE_INTERVAL=2, RESUME_FROM=keep)
    b, sweep_b, eng_b, ran_b, init_b = _train(module, cfg_b, rngs)
    assert ran_b == [2, 3, 4] and not init_b, (ran_b, init_b)
    assert sweep_a == sweep_b
    from purejaxql_b200.utils.save_load import load_state
    sa, sb = load_state(eng_state_path(eng_a)), load_state(eng_state_path(eng_b))
    assert sa["meta"] == sb["meta"] and sa["meta"]["n_done"] == 4
    _assert_same_bits({k: v.numpy() for k, v in sa["tensors"].items()},
                      {k: v.numpy() for k, v in sb["tensors"].items()}, "state after update 4")
    return a, b, eng_a, eng_b


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_resumed_run_matches_the_uninterrupted_one(case, graph, tmp_path):
    module, cfg = CASES[case]
    cfg = dict(cfg, CUDA_GRAPH=graph)
    rngs = jr.split(jr.PRNGKey(7), cfg["NUM_SEEDS"])
    if isinstance(cfg["LR"], list):
        rngs = np.tile(rngs, (len(cfg["LR"]), 1))
    a, b, eng_a, eng_b = _a_then_b(module, cfg, rngs, str(tmp_path))
    _assert_same_bits(a, b, case)
    assert eng_a.graph_captured == graph and eng_b.graph_captured == graph
    if cfg.get("TEST_DURING_TRAINING"):                            # evaluations at updates 2 and 4: one on each side
        assert "test_metrics/returned_episode_returns" in a and "metric/test/returned_episode_returns" in a


def test_default_keys_write_no_state_and_change_nothing(tmp_path):
    module, cfg = CASES["mlp_cartpole"]
    rngs = jr.split(jr.PRNGKey(7), cfg["NUM_SEEDS"])
    plain, _, _, ran, _ = _train(module, dict(cfg, SAVE_PATH=str(tmp_path / "plain")), rngs)
    assert ran == list(range(NUPD))
    assert not (tmp_path / "plain").exists(), "a run with STATE_SAVE_INTERVAL=0 wrote a file"
    saving, _, _, _, _ = _train(module, dict(cfg, SAVE_PATH=str(tmp_path / "s"), STATE_SAVE_INTERVAL=1), rngs)
    _assert_same_bits(plain, saving, "writing the state does not change the run")


def test_resume_refuses_other_keys(tmp_path):
    module, cfg = CASES["mlp_cartpole"]
    rngs = jr.split(jr.PRNGKey(7), cfg["NUM_SEEDS"])
    keep = str(tmp_path / "after2.safetensors")
    _train(module, dict(cfg, SAVE_PATH=str(tmp_path / "a"), STATE_SAVE_INTERVAL=2), rngs, keep)
    mod = importlib.import_module(f"purejaxql_b200.{module}")
    train = mod.make_train(dict(cfg, RESUME_FROM=keep))
    with pytest.raises(ValueError, match="keys differ"):
        train(jr.split(jr.PRNGKey(8), cfg["NUM_SEEDS"]))


# ---------------------------------------------------------------- two gloo ranks on one GPU
def _rank_worker(rank, world, mode, out_dir):
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method=f"file://{out_dir}/pg", rank=rank, world_size=world,
                            timeout=timedelta(seconds=120))
    try:
        if mode == "seeds":                                        # each rank trains its slice of 4 seeds
            cfg = _cfg("Breakout-MinAtar", NUM_SEEDS=4, CUDA_GRAPH=False)
            rngs = jr.split(jr.PRNGKey(7), 4)[2 * rank:2 * rank + 2]
            attrs = dict(seed_lo=2 * rank)
        else:                                                      # each rank trains its half of the envs of 2 seeds
            cfg = _cfg("Breakout-MinAtar", NUM_ENVS=128, CUDA_GRAPH=False)
            rngs = jr.split(jr.PRNGKey(7), 2)
            attrs = dict(env_shard=(rank, world))
        # every rank keeps its own copy of the state after update 2: {rank} in RESUME_FROM picks it
        keep_dir = os.path.join(out_dir, "keep")
        os.makedirs(keep_dir, exist_ok=True)
        cfg_a = dict(cfg, SAVE_PATH=os.path.join(out_dir, "a"), STATE_SAVE_INTERVAL=2)
        a, _, eng_a, _, _ = _train("pqn_minatar", cfg_a, rngs, os.path.join(keep_dir, f"after2_rank{rank}.safetensors"),
                                   **attrs)
        assert eng_state_path(eng_a).endswith(f"_rank{rank}_state.safetensors")
        cfg_b = dict(cfg, SAVE_PATH=os.path.join(out_dir, "b"),
                     RESUME_FROM=os.path.join(keep_dir, "after2_rank{rank}.safetensors"))
        b, _, eng_b, ran_b, init_b = _train("pqn_minatar", cfg_b, rngs, **attrs)
        assert ran_b == [2, 3, 4] and not init_b
        _assert_same_bits(a, b, (mode, rank))
        with open(os.path.join(out_dir, f"ok{rank}.json"), "w") as f:
            json.dump({"params": hashlib.sha256(a["params"].tobytes()).hexdigest(),
                       "env_state": hashlib.sha256(a["env_state"].tobytes()).hexdigest()}, f)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode", ["seeds", "envs"])
def test_two_ranks_resume_their_own_files(mode, tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_rank_worker, args=(2, mode, str(tmp_path)), nprocs=2, join=True)
    assert not multiprocessing.active_children()
    got = [json.loads((tmp_path / f"ok{r}.json").read_text()) for r in range(2)]
    if mode == "envs":          # replicated parameters, different env shards
        assert got[0]["params"] == got[1]["params"] and got[0]["env_state"] != got[1]["env_state"]
    else:                       # different seeds
        assert got[0]["params"] != got[1]["params"]
