"""A list-valued ENV_NAME on the GPU: every env of a list run is bit-identical to a standalone make_train of that env
on the same keys, while the engines run concurrently, each on its own CUDA stream.

Compared with np.array_equal (NaN where no episode ended counts as equal): parameters, running statistics, RAdam
moments, every metric column (test/* included), the last evaluation, the runner key, the env state words, the last
observation rows and, for the GRU, its memory and hidden state.  Eager and under CUDA-graph replay, with evaluation
after every update; one case trains a two-point LR grid and two run the batch_norm network."""
import importlib

import numpy as np
import pytest
import torch

from oracle import jax_prng as jr
from purejaxql_b200 import sweep

pytestmark = pytest.mark.gpu
N, NUPD = 2, 3                      # seeds; 3 updates so that the graph captures and replays

_RUN = dict(NUM_EPOCHS=2, LR_LINEAR_DECAY=True, WANDB_MODE="disabled", NUM_SEEDS=N, TEST_DURING_TRAINING=True,
            TEST_INTERVAL=0.4, TEST_NUM_ENVS=16, EPS_TEST=0.0)
_MINATAR = dict(NUM_ENVS=64, NUM_STEPS=8, NUM_MINIBATCHES=4, EPS_START=1.0, EPS_FINISH=0.05, EPS_DECAY=0.5, LR=5e-4,
                MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65, NORM_TYPE="layer_norm")
_GYMNAX = dict(NUM_ENVS=32, NUM_STEPS=16, NUM_MINIBATCHES=4, EPS_START=1.0, EPS_FINISH=0.2, EPS_DECAY=0.5, LR=1e-4,
               MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.95, REW_SCALE=0.1, HIDDEN_SIZE=128, NUM_LAYERS=2,
               NORM_TYPE="layer_norm")
_RNN = dict(NUM_ENVS=16, NUM_STEPS=12, MEMORY_WINDOW=3, NUM_MINIBATCHES=4, EPS_START=0.6, EPS_FINISH=0.1,
            EPS_DECAY=1.0, LR=1e-3, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.95, REW_SCALE=0.1, HIDDEN_SIZE=128,
            NUM_LAYERS=2, NORM_TYPE="layer_norm", NORM_INPUT=False, ENV_KWARGS={"memory_length": 4})
CASES = {
    "minatar_cnn": ("pqn_minatar", ["Breakout-MinAtar", "Freeway-MinAtar"], _MINATAR),               # C = 4 and 7
    "gymnax_mlp_and_bits": ("pqn_gymnax", ["CartPole-v1", "Catch-bsuite", "Breakout-MinAtar"], _GYMNAX),
    "rnn_gru": ("pqn_rnn_gymnax", ["CartPole-v1", "MemoryChain-bsuite"], _RNN),
    "gymnax_lr_grid": ("pqn_gymnax", ["CartPole-v1", "Catch-bsuite"], dict(_GYMNAX, LR=[1e-3, 1e-4])),
    "minatar_batch_norm": ("pqn_minatar", ["Breakout-MinAtar", "Freeway-MinAtar"],
                           dict(_MINATAR, NORM_TYPE="batch_norm")),
    "rnn_batch_norm": ("pqn_rnn_gymnax", ["CartPole-v1", "MemoryChain-bsuite"], dict(_RNN, NORM_TYPE="batch_norm")),
}


def _cfg(case, env_name, graph):
    module, _, c = CASES[case]
    c = {**c, **_RUN, "ENV_NAME": env_name, "CUDA_GRAPH": graph}
    c["TOTAL_TIMESTEPS"] = c["TOTAL_TIMESTEPS_DECAY"] = float(NUPD * c["NUM_STEPS"] * c["NUM_ENVS"])
    return importlib.import_module(f"purejaxql_b200.{module}"), c


def _collect(out):
    """Everything a train() returns that the parity compares, on the host."""
    ts = out["runner_state"][0]
    res = {"params": ts.params_flat, "batch_stats": ts.batch_stats_flat, "mu": ts.opt_state.mu, "nu": ts.opt_state.nu,
           "rng": out["runner_state"][-1]}
    res.update({f"metric:{k}": v for k, v in out["metrics"].items()})
    tail = out["runner_state"][1:-1]
    if len(tail) == 2:                                   # PQNEngine: ((obs, env_state), test_metrics)
        (obs, state), test_metrics = tail
        res.update(last_obs=obs, env_state=state)
    else:                                                # PQNRnnEngine: (memory, expl_state, test_metrics)
        mem, (hs, last_obs, last_done, last_action, state), test_metrics = tail
        res.update(hs=hs, last_obs=last_obs, last_done=last_done, last_action=last_action, env_state=state)
        res.update({f"mem/{k}": v for k, v in vars(mem).items()})
    res.update({f"test_metrics:{k}": v for k, v in test_metrics.items()})
    return {k: v.cpu().numpy() for k, v in res.items()}


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda_graph"])
@pytest.mark.parametrize("case", list(CASES))
def test_env_list_equals_standalone_runs(case, graph):
    _, names, _ = CASES[case]
    mod, cfg = _cfg(case, names, graph)
    grid = sweep.Grid(cfg)
    rngs = grid.tile(jr.split(jr.PRNGKey(11), N))
    train = mod.make_train(cfg)
    assert list(train.engines) == names and cfg["NUM_UPDATES"] == NUPD
    streams = {}
    for name, eng in train.engines.items():
        eng.on_update_begin = lambda n, name=name: streams.setdefault(name, []).append(torch.cuda.current_stream())
    outs = train(rngs)
    assert list(outs) == names
    # every engine ran each update on one stream of its own, not the caller's
    default = torch.cuda.current_stream()
    for name in names:
        assert len(streams[name]) == NUPD and all(s == streams[name][0] for s in streams[name]), name
        assert streams[name][0] != default, name
    assert len({streams[name][0].cuda_stream for name in names}) == len(names)
    for name, eng in train.engines.items():
        assert eng.graph_captured == graph, name
        assert eng.cfg["ENV_NAME"] == name
    got = {name: _collect(outs[name]) for name in names}
    for name in names:
        mod, one_cfg = _cfg(case, name, graph)
        one = mod.make_train(one_cfg)
        want = _collect(one(rngs))
        assert one.engine.graph_captured == graph
        assert one_cfg["TEST_NUM_STEPS"] == train.engines[name].cfg["TEST_NUM_STEPS"], name
        assert sorted(got[name]) == sorted(want) and any(k.startswith("metric:test/") for k in want)
        for k, v in want.items():
            g = got[name][k]
            assert g.shape == v.shape and np.array_equal(g, v, equal_nan=v.dtype.kind == "f"), (case, graph, name, k)
