"""A list of envs trained as one run: one engine per env, each on its own CUDA stream.

    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole NUM_SEEDS=4 "alg.ENV_NAME=[CartPole-v1,Acrobot-v1,Catch-bsuite]"

Different envs cannot share launches: observation width, channel count, action count, network layout and the kernels
all differ.  They can share the GPU.  Each env of the list gets the engine a standalone run of that env builds (its own
env params, ``TEST_NUM_STEPS``, network, workspace, buffers, CUDA graph and evaluation) on a config copy whose
``ENV_NAME`` is that env, and its own CUDA stream.  One host thread steps the engines in lockstep, one update of each in
turn (``EngineBase.train_steps``), so the device overlaps their launches and graph replays, while a graph capture never
overlaps another engine's CUDA calls.

Each env trains bit for bit what the standalone run trains on the same keys: the library keeps no device state shared
between calls, and every launch shape depends only on the seeds, rows, network shape and the SM count.

Refused before any env is built: env-sharded data parallelism, the training state (``STATE_SAVE_INTERVAL``,
``RESUME_FROM``) and ``HYP_TUNE``.
"""
from __future__ import annotations

import torch

from . import _runner, state, sweep


def refuse(config: dict, world: int, env_sharding: bool = True):
    """Refuse what a list of envs cannot train with, before anything is built."""
    names = sweep.env_names(config)
    if config.get("HYP_TUNE", False):
        raise ValueError(f"HYP_TUNE=True with ENV_NAME={names}: the wandb LR sweep tunes one env; give one ENV_NAME")
    if config.get("STATE_SAVE_INTERVAL") or config.get("RESUME_FROM") is not None:
        raise ValueError(f"ENV_NAME={names}: STATE_SAVE_INTERVAL and RESUME_FROM save and resume one env's run; "
                         f"train each env on its own to save its state")
    dp = config.get("DATA_PARALLEL", "auto")
    if dp == "envs" or (env_sharding and world > 1 and _runner.pick_data_parallel(config, world) == "envs"):
        raise ValueError(f"ENV_NAME={names}: a list of envs shards seeds over the GPUs, not envs "
                         f"(DATA_PARALLEL={dp} picks env sharding here); use DATA_PARALLEL=seeds with at least as "
                         f"many seeds as GPUs")


def make_train(config: dict, make_one, check_env, env_sharding: bool = True):
    """``make_train`` of a list-valued ENV_NAME.  ``make_one(config)`` is the script's make_train of one env and
    ``check_env(name)`` its refusal of an env it cannot train (raised for every name before any env is built).

    The caller's config gets NUM_UPDATES and NUM_UPDATES_DECAY; each engine's config copy holds its own TEST_NUM_STEPS.
    ``train(rngs)`` returns {env: what a standalone train(rngs) returns} in list order; ``train.engines`` maps every
    env to its engine."""
    names = sweep.env_names(config)
    refuse(config, state.dist_placement()[1], env_sharding)
    for name in names:
        check_env(name)
    base = dict(config)
    engines, streams = {}, {}
    for name in names:
        one = {**base, "ENV_NAME": name}
        streams[name] = torch.cuda.Stream()
        with torch.cuda.stream(streams[name]):
            engines[name] = make_one(one).engine
        engines[name].log_prefix = f"{name}/"
    config["NUM_UPDATES"], config["NUM_UPDATES_DECAY"] = one["NUM_UPDATES"], one["NUM_UPDATES_DECAY"]

    def train(rngs):
        return train_all(engines, streams, rngs)

    train.engines = engines
    return train


def train_all(engines: dict, streams: dict, rngs) -> dict:
    """Every engine's train(rngs), each on its stream, one update of each engine in turn.  The streams first wait for
    the caller's stream, which queued the keys and may still read the tensors an earlier train returned; the device
    is synchronised only once every engine's last update is queued."""
    caller = torch.cuda.current_stream()
    runs = []
    for name, eng in engines.items():
        streams[name].wait_stream(caller)
        runs.append((name, eng.train_steps(rngs)))
    out = {}
    while runs:
        left = []
        for name, steps in runs:
            with torch.cuda.stream(streams[name]):
                try:
                    next(steps)
                    left.append((name, steps))
                except StopIteration as done:
                    out[name] = done.value
        runs = left
    torch.cuda.synchronize()
    return {name: out[name] for name in engines}
