"""Which data-parallel mode single_run picks under a two-rank launch (CPU: init_distributed is stubbed to (0, 2), no
process group).  The recurrent script has no env-sharded engine, so it must shard seeds, and refuse an explicit
DATA_PARALLEL=envs before anything is built; the feed-forward script keeps choosing env sharding for one seed."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import jax_prng as oracle_jr
from purejaxql_b200 import _runner, config_loader, pqn_gymnax, pqn_rnn_gymnax


def _run(monkeypatch, module, preset, built, *overrides):
    """module.single_run under a stubbed rank 0 of 2, with a make_train that records the engine it hands out."""
    def make_train(config):
        engine = SimpleNamespace()
        built.append(engine)

        def train(rngs):
            engine.num_seeds = rngs.shape[0]
            return {"runner_state": (None,)}
        train.engine = engine
        return train
    monkeypatch.setattr(_runner, "init_distributed", lambda: (0, 2))
    monkeypatch.setattr(module, "make_train", make_train)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
    # the seed keys on the host (the library's split runs on the device)
    monkeypatch.setattr(_runner, "jr", SimpleNamespace(
        PRNGKey=oracle_jr.PRNGKey,
        split=lambda k, n, mode=0: torch.from_numpy(oracle_jr.split(k, n, bool(mode)).view(np.int32).copy())))
    module.single_run(config_loader.compose([f"+alg={preset}", "NUM_SEEDS=1", "SAVE_PATH=null", *overrides]))


@pytest.mark.parametrize("preset", ["pqn_rnn_cartpole", "pqn_rnn_memory_chain"])
@pytest.mark.parametrize("overrides", [(), ("DATA_PARALLEL=auto",), ("DATA_PARALLEL=seeds",)])
def test_recurrent_script_shards_seeds(monkeypatch, preset, overrides):
    built = []
    _run(monkeypatch, pqn_rnn_gymnax, preset, built, *overrides)
    assert len(built) == 1
    assert getattr(built[0], "env_shard", None) is None
    assert built[0].num_seeds == 1


def test_recurrent_script_refuses_env_sharding_before_building(monkeypatch):
    built = []
    with pytest.raises(ValueError, match="DATA_PARALLEL=seeds"):
        _run(monkeypatch, pqn_rnn_gymnax, "pqn_rnn_cartpole", built, "DATA_PARALLEL=envs")
    assert built == []


def test_feed_forward_script_still_shards_envs(monkeypatch):
    built = []
    _run(monkeypatch, pqn_gymnax, "pqn_cartpole", built)
    assert built[0].env_shard == (0, 2) and built[0].num_seeds == 1
