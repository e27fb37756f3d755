"""The training-state file (utils.save_load.save_state / load_state) and the checks RESUME_FROM runs before anything is
built (purejaxql_b200.state), on the host: a stub stands in for the engine, so a refusal that reaches it would be
one that came too late."""
import os

import pytest
import torch

from purejaxql_b200 import config_loader, pqn_gymnax, pqn_minatar, pqn_rnn_gymnax, state
from purejaxql_b200.utils import save_load

SCRIPTS = {"pqn_gymnax": (pqn_gymnax, "PQNEngine"), "pqn_minatar": (pqn_minatar, "PQNEngine"),
           "pqn_rnn_gymnax": (pqn_rnn_gymnax, "PQNRnnEngine")}


class StubEngine:
    """Stands in for the CUDA engine: records that make_train got as far as building one."""
    built = []

    def __init__(self, config, *a, **kw):
        StubEngine.built.append(config)


def _cfg(script, **kw):
    c = dict(ENV_NAME="Breakout-MinAtar" if script == "pqn_minatar" else "CartPole-v1", NUM_ENVS=64, NUM_STEPS=8,
             NUM_MINIBATCHES=4, NUM_EPOCHS=2, EPS_START=1.0, EPS_FINISH=0.05, EPS_DECAY=0.1, LR=5e-4,
             MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65, LR_LINEAR_DECAY=True, TOTAL_TIMESTEPS=2560.0,
             TOTAL_TIMESTEPS_DECAY=2560.0, SEED=0, NUM_SEEDS=2, TEST_DURING_TRAINING=False, WANDB_MODE="disabled",
             ALG_NAME="pqn_rnn" if script == "pqn_rnn_gymnax" else "pqn", SAVE_PATH=None)
    if script == "pqn_rnn_gymnax":
        c.update(MEMORY_WINDOW=4, HIDDEN_SIZE=128, NUM_LAYERS=2)
    c.update(kw)
    return c


@pytest.fixture
def stub(monkeypatch):
    StubEngine.built = []
    for mod, cls in SCRIPTS.values():
        monkeypatch.setattr(mod, cls, StubEngine)
    return StubEngine


def _write_state(path, script, cfg, n_done=2, rank=0, world=1, fmt=state.FORMAT_VERSION):
    """A state file whose metadata describes `cfg` (prepared the way make_train prepares it) after n_done updates."""
    c = dict(cfg)
    SCRIPTS[script][0].make_train(c)                                # the stub engine: no device work
    meta = dict(format=fmt, script=script, env=c["ENV_NAME"], n_done=n_done, num_updates=int(c["NUM_UPDATES"]),
                rank=rank, world=world, seed_lo=0, num_seeds_local=c["NUM_SEEDS"], data_parallel="seeds",
                config=state.run_keys(c))
    save_load.save_state(path, {"tensors": {"keys": torch.zeros((c["NUM_SEEDS"], 2), dtype=torch.int32)},
                                "meta": meta})
    return meta


def test_state_file_round_trips(tmp_path):
    t = {"params": torch.randn(3, 17), "idx": torch.tensor([5], dtype=torch.int64),
         "env_state": torch.randint(-2 ** 31, 2 ** 31 - 1, (6, 12), dtype=torch.int32),
         "mem/done": torch.randint(0, 2, (2, 4, 3), dtype=torch.uint8),
         "metrics/td_loss": torch.randn(3, 4, dtype=torch.float64),
         "last_obs": torch.randn(2, 9, 4)[:, :, 1]}                  # a strided view is saved as its values
    meta = {"format": 1, "n_done": 4, "sweep": {"LR": [0.001, 0.0005]}, "network": {"kind": "cnn", "D": 4}}
    p = tmp_path / "run_state.safetensors"
    save_load.save_state(p, {"tensors": t, "meta": meta})
    got = save_load.load_state(p)
    assert got["meta"] == meta and save_load.read_state_meta(p) == meta
    assert sorted(got["tensors"]) == sorted(t)
    for k, v in t.items():
        assert got["tensors"][k].dtype == v.dtype and torch.equal(got["tensors"][k], v), k
    assert [f.name for f in tmp_path.iterdir()] == [p.name]


def test_interrupted_write_keeps_the_previous_state(tmp_path, monkeypatch):
    p = tmp_path / "run_state.safetensors"
    save_load.save_state(p, {"tensors": {"x": torch.arange(4.0)}, "meta": {"n_done": 2}})

    def killed(src, dst):
        raise KeyboardInterrupt("killed before the rename")
    monkeypatch.setattr(save_load.os, "replace", killed)
    with pytest.raises(KeyboardInterrupt):
        save_load.save_state(p, {"tensors": {"x": torch.arange(8.0)}, "meta": {"n_done": 4}})
    monkeypatch.undo()
    got = save_load.load_state(p)
    assert got["meta"] == {"n_done": 2} and torch.equal(got["tensors"]["x"], torch.arange(4.0))
    assert [f.name for f in tmp_path.iterdir()] == [p.name], "the temporary file was left behind"


def test_a_params_checkpoint_is_not_a_state_file(tmp_path):
    p = tmp_path / "vmap0.safetensors"
    save_load.save_params({"Dense_0": {"kernel": torch.zeros(2, 2)}}, p)
    with pytest.raises(ValueError, match="not a training-state file"):
        save_load.load_state(p)


# a value other than the saved run's for every key that shapes a run
MISMATCHES = [
    ("ENV_NAME", "Acrobot-v1"), ("ENV_KWARGS", {"memory_length": 3}), ("HIDDEN_SIZE", 256), ("NUM_LAYERS", 3),
    ("NORM_TYPE", "batch_norm"), ("NORM_INPUT", True), ("NUM_ENVS", 128), ("NUM_STEPS", 4), ("NUM_MINIBATCHES", 2),
    ("NUM_EPOCHS", 1), ("MEMORY_WINDOW", 2), ("TOTAL_TIMESTEPS", 5120.0), ("TOTAL_TIMESTEPS_DECAY", 1e6),
    ("LR", 1e-3), ("LR", [5e-4, 1e-3]), ("MAX_GRAD_NORM", 1.0), ("GAMMA", 0.9), ("LAMBDA", 0.9), ("REW_SCALE", 0.1),
    ("EPS_START", 0.5), ("EPS_FINISH", 0.1), ("EPS_DECAY", 0.2), ("SEED", 1), ("NUM_SEEDS", 4),
    ("JAX_THREEFRY_PARTITIONABLE", 1), ("TEST_DURING_TRAINING", True), ("TEST_INTERVAL", 0.5), ("TEST_NUM_ENVS", 8),
    ("TEST_NUM_STEPS", 50), ("EPS_TEST", 0.1), ("LR_LINEAR_DECAY", False), ("DATA_PARALLEL", "envs"),
    ("ALG_NAME", "other"),
]


@pytest.mark.parametrize("key,value", MISMATCHES, ids=[f"{k}={v}" for k, v in MISMATCHES])
def test_each_mismatched_key_is_refused_before_the_engine(key, value, tmp_path, stub):
    base = _cfg("pqn_gymnax", TEST_INTERVAL=0.25, TEST_NUM_ENVS=4, TEST_NUM_STEPS=20, EPS_TEST=0.0)
    p = str(tmp_path / "s.safetensors")
    _write_state(p, "pqn_gymnax", base)
    stub.built.clear()
    with pytest.raises(ValueError, match=f"RESUME_FROM: {key}="):
        pqn_gymnax.make_train(dict(base, RESUME_FROM=p, **{key: value}))
    assert not stub.built


@pytest.mark.parametrize("script", sorted(SCRIPTS))
def test_the_same_run_reaches_the_engine_with_the_state(script, tmp_path, stub):
    """Keys that do not shape the run may differ; the engine receives the loaded state."""
    base = _cfg(script)
    p = str(tmp_path / "s.safetensors")
    meta = _write_state(p, script, base)
    stub.built.clear()
    train = SCRIPTS[script][0].make_train(dict(base, RESUME_FROM=p, CUDA_GRAPH=True, WANDB_MODE="online",
                                               SAVE_PATH=str(tmp_path / "elsewhere"), STATE_SAVE_INTERVAL=3))
    assert len(stub.built) == 1
    assert train.engine.resume["meta"] == meta and train.engine.resume["path"] == p
    assert train.engine.resume["tensors"]["keys"].shape == (2, 2)


@pytest.mark.parametrize("script,other", [("pqn_gymnax", "pqn_minatar"), ("pqn_minatar", "pqn_gymnax"),
                                          ("pqn_rnn_gymnax", "pqn_gymnax")])
def test_a_file_from_another_script_is_refused(script, other, tmp_path, stub):
    p = str(tmp_path / "s.safetensors")
    _write_state(p, script, _cfg(script))
    stub.built.clear()
    with pytest.raises(ValueError, match=f"written by '{script}', not '{other}'"):
        SCRIPTS[other][0].make_train(dict(_cfg(other), RESUME_FROM=p))
    assert not stub.built


def test_a_file_from_another_rank_format_or_a_finished_run_is_refused(tmp_path, stub, monkeypatch):
    base = _cfg("pqn_gymnax")
    cases = {"rank1": (dict(rank=1, world=2), "holds rank 1 of 2; this process is rank 0 of 2"),
             "world2": (dict(rank=0, world=2), "holds rank 0 of 2; this process is rank 0 of 1"),
             "format": (dict(fmt=99), "state format 99"),
             "finished": (dict(n_done=5), "the saved run is finished \\(5 of 5 updates\\)")}
    for name, (kw, msg) in cases.items():
        p = str(tmp_path / f"{name}.safetensors")
        _write_state(p, "pqn_gymnax", base, **kw)
        stub.built.clear()
        if name == "rank1":
            monkeypatch.setattr(state, "dist_placement", lambda: (0, 2))
        with pytest.raises(ValueError, match=msg):
            pqn_gymnax.make_train(dict(base, RESUME_FROM=p))
        monkeypatch.undo()
        for mod, cls in SCRIPTS.values():
            monkeypatch.setattr(mod, cls, StubEngine)
        assert not stub.built, name


def test_rank_placeholder_picks_this_ranks_file(tmp_path, stub, monkeypatch):
    base = _cfg("pqn_gymnax")
    for r in range(2):
        _write_state(str(tmp_path / f"s_rank{r}.safetensors"), "pqn_gymnax", base, rank=r, world=2)
    monkeypatch.setattr(state, "dist_placement", lambda: (1, 2))
    train = pqn_gymnax.make_train(dict(base, RESUME_FROM=str(tmp_path / "s_rank{rank}.safetensors")))
    assert train.engine.resume["meta"]["rank"] == 1 and train.engine.resume["path"].endswith("s_rank1.safetensors")


def test_placement_and_save_interval_checks():
    meta = dict(data_parallel="seeds", seed_lo=4, num_seeds_local=4)
    state.check_placement(meta, "seeds", 4, 4)
    for got in (("envs", 4, 4), ("seeds", 0, 4), ("seeds", 4, 2)):
        with pytest.raises(ValueError, match="this rank trains"):
            state.check_placement(meta, *got)
    with pytest.raises(ValueError, match="needs SAVE_PATH"):
        state.save_interval({"STATE_SAVE_INTERVAL": 2, "SAVE_PATH": None})
    with pytest.raises(ValueError, match="non-negative int"):
        state.save_interval({"STATE_SAVE_INTERVAL": -1, "SAVE_PATH": "m"})
    assert state.save_interval({"STATE_SAVE_INTERVAL": 5, "SAVE_PATH": "m"}) == 5
    assert state.state_file({"SAVE_PATH": "m", "ENV_NAME": "CartPole-v1", "SEED": 3}) == os.path.join(
        "m", "CartPole-v1", "pqn_CartPole-v1_seed3_state.safetensors")
    assert state.state_file({"SAVE_PATH": "m", "ENV_NAME": "E", "SEED": 0, "ALG_NAME": "pqn_rnn"}, 1, 2).endswith(
        "pqn_rnn_E_seed0_rank1_state.safetensors")


def test_a_save_interval_without_save_path_is_refused_before_the_engine(stub):
    with pytest.raises(ValueError, match="needs SAVE_PATH"):
        pqn_gymnax.make_train(_cfg("pqn_gymnax", STATE_SAVE_INTERVAL=2))
    assert not stub.built


@pytest.mark.parametrize("alg", ["pqn_minatar", "pqn_cartpole", "pqn_rnn_cartpole", "pqn_rnn_memory_chain"])
def test_default_configs_write_no_state(alg):
    c = config_loader.compose([f"+alg={alg}"])
    c = {**c, **c["alg"]}
    assert c["STATE_SAVE_INTERVAL"] == 0 and c["RESUME_FROM"] is None
    assert state.save_interval(c) == 0
