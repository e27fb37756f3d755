"""Training state of a run between two updates: what ``STATE_SAVE_INTERVAL`` writes and ``RESUME_FROM`` continues from.

Every update reads and writes only static device buffers, and the whole key chain lives on the device, so those
buffers (parameters, running statistics, RAdam moments and step counter, runner key, update index, env state, the
engine's carried rollout buffers) plus the metric columns written so far describe a run completely.  A run resumed from
them computes the bits of the uninterrupted run.

The file is safetensors (``utils.save_load.save_state``) whose metadata records what produced it.  ``check_meta``
compares it with the resuming config before anything is allocated and refuses any difference in a key that shapes the
run (``RUN_KEYS``); the engine then checks its seed slice, data-parallel mode and keys (``check_placement``).
"""
from __future__ import annotations

import json
import os

from . import pbt, sweep

FORMAT_VERSION = 1
# the config keys that shape a run, with the value an absent key stands for; a resumed run must match each one
RUN_KEYS = {
    "ALG_NAME": "pqn", "ENV_NAME": None, "ENV_KWARGS": None,
    "HIDDEN_SIZE": 128, "NUM_LAYERS": 2, "NORM_TYPE": "layer_norm", "NORM_INPUT": False,
    "NUM_ENVS": None, "NUM_STEPS": None, "NUM_MINIBATCHES": None, "NUM_EPOCHS": None, "MEMORY_WINDOW": 0,
    "TOTAL_TIMESTEPS": None, "TOTAL_TIMESTEPS_DECAY": None,
    **{k: sweep._DEFAULTS.get(k) for k in sweep.SWEEP_KEYS},
    "SEED": 0, "NUM_SEEDS": 1, "JAX_THREEFRY_PARTITIONABLE": 0,
    "TEST_DURING_TRAINING": False, "TEST_INTERVAL": None, "TEST_NUM_ENVS": None, "TEST_NUM_STEPS": None,
    "EPS_TEST": None, "LR_LINEAR_DECAY": False, "DATA_PARALLEL": "auto",
    **pbt.DEFAULTS,       # a state file written before PBT existed lacks these keys: it resumes a run without PBT
}


def _jsonable(v):
    return json.loads(json.dumps(v, default=lambda o: o.item() if hasattr(o, "item") else str(o)))


def run_keys(config: dict) -> dict:
    """RUN_KEYS of a config (after make_train's prepare_config), as they are stored in a state file."""
    return {k: _jsonable(d if config.get(k) is None else config[k]) for k, d in RUN_KEYS.items()}


def save_interval(config: dict) -> int:
    """STATE_SAVE_INTERVAL: write the state after every k-th update (0: never)."""
    k = config.get("STATE_SAVE_INTERVAL") or 0
    if isinstance(k, bool) or not isinstance(k, int) or k < 0:
        raise ValueError(f"STATE_SAVE_INTERVAL={k!r}: expected a non-negative int (0 writes no state)")
    if k and config.get("SAVE_PATH") is None:
        raise ValueError(f"STATE_SAVE_INTERVAL={k} needs SAVE_PATH: the state file goes next to the checkpoints")
    return k


def state_file(config: dict, rank: int = 0, world: int = 1) -> str:
    """<SAVE_PATH>/<ENV_NAME>/<ALG_NAME>_<ENV_NAME>_seed<SEED>[_rank<r>]_state.safetensors"""
    alg, env = config.get("ALG_NAME", "pqn"), config["ENV_NAME"]
    rank_part = f"_rank{rank}" if world > 1 else ""
    return os.path.join(config["SAVE_PATH"], env, f"{alg}_{env}_seed{config['SEED']}{rank_part}_state.safetensors")


def dist_placement():
    """(rank, world) of this process in the torch.distributed group, (0, 1) outside one."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def check_meta(meta: dict, config: dict, script: str, rank: int, world: int, path: str = "the state file"):
    """Refuse a state file that does not continue this run: another format version, script or rank, a finished run,
    or any RUN_KEYS value that differs from the config's (the message names the key)."""
    if meta.get("format") != FORMAT_VERSION:
        raise ValueError(f"{path}: state format {meta.get('format')!r}, this version reads format {FORMAT_VERSION}")
    if meta.get("script") != script:
        raise ValueError(f"{path} was written by {meta.get('script')!r}, not {script!r}")
    if (meta.get("rank"), meta.get("world")) != (rank, world):
        raise ValueError(f"{path} holds rank {meta.get('rank')} of {meta.get('world')}; this process is rank {rank} "
                         f"of {world} (world size); under a multi-GPU launch, write {{rank}} in RESUME_FROM")
    want = run_keys(config)
    for k, v in want.items():
        saved = meta["config"].get(k, _jsonable(RUN_KEYS[k]))      # a key the saving version lacked: its default
        if saved != v:
            raise ValueError(f"RESUME_FROM: {k}={v!r} differs from the saved run's {k}={saved!r} "
                             f"({path}); a resumed run must keep every key that shapes it")
    if int(meta["n_done"]) >= int(meta["num_updates"]):
        raise ValueError(f"{path}: the saved run is finished ({meta['n_done']} of {meta['num_updates']} updates)")


def load_for_resume(config: dict, script: str):
    """The state file RESUME_FROM names (None when it is null), checked against `config` before any device work.
    ``{rank}`` in the path stands for this process's rank, so that every rank of a multi-GPU job reads its own file."""
    from .utils.save_load import load_state, read_state_meta
    save_interval(config)
    path = config.get("RESUME_FROM")
    if path is None:
        return None
    rank, world = dist_placement()
    path = str(path).replace("{rank}", str(rank))
    meta = read_state_meta(path)
    check_meta(meta, config, script, rank, world, path)
    st = load_state(path)
    st["path"] = path
    return st


def check_placement(meta: dict, data_parallel: str, seed_lo: int, S: int, path: str = "the state file"):
    """Refuse a state saved for another seed slice or data-parallel mode than the one this rank trains."""
    got = (data_parallel, seed_lo, S)
    saved = (meta.get("data_parallel"), meta.get("seed_lo"), meta.get("num_seeds_local"))
    if got != saved:
        raise ValueError(f"{path} holds (data-parallel mode, first seed, seeds) = {saved}; this rank trains {got}")
