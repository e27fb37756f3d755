"""single_run / tune / main shared by pqn_minatar.py and pqn_gymnax.py
(purejaxql/pqn_minatar.py:435-541; pqn_gymnax.py is the same modulo names)."""
from __future__ import annotations

import copy
import os
import sys
import time

import torch

from . import config_loader, jaxrandom as jr, pbt, sweep


def init_distributed():
    """Under torchrun (RANK / LOCAL_RANK / WORLD_SIZE set) bind this process to its GPU and join the process
    group; a plain `python -m purejaxql_b200.pqn_minatar` run is left untouched.  Returns (rank, world)."""
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1:
        return 0, 1
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if torch.cuda.is_available():
        torch.cuda.set_device(local_rank)
    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if torch.cuda.is_available():
            dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
        else:
            dist.init_process_group("gloo")
    return dist.get_rank(), dist.get_world_size()


def seed_slice(num_seeds, rank, world):
    """Contiguous slice [lo, hi) of the seed axis owned by `rank` (may be empty when num_seeds < world)."""
    per = (num_seeds + world - 1) // world
    lo = min(num_seeds, rank * per)
    return lo, min(num_seeds, lo + per)


def pick_data_parallel(config, world, env_sharding=True):
    """"seeds" | "envs" for this run: DATA_PARALLEL (this repo's key, not in the reference) = "seeds" shards the
    independent seeds over the ranks (no collective); "envs" shards NUM_ENVS of every seed and all-reduces the
    gradient once per minibatch step; "auto" (default) picks "envs" when there are fewer seeds than GPUs (the
    shipped default is NUM_SEEDS=1, config/config.yaml:2), counting every seed of a hyperparameter grid
    (G points x NUM_SEEDS, sweep.Grid).  A script whose engine has no env-sharded mode
    (``env_sharding=False``: the recurrent one) always shards seeds, and refuses an explicit "envs"."""
    if world <= 1:
        return "seeds"
    dp = config.get("DATA_PARALLEL", "auto")
    if dp not in ("auto", "seeds", "envs"):
        raise ValueError(f"DATA_PARALLEL={dp!r}: expected auto, seeds or envs")
    if not env_sharding:
        if dp == "envs":
            raise ValueError("DATA_PARALLEL=envs: this script's engine has no env-sharded mode; use "
                             "DATA_PARALLEL=seeds (one seed per GPU)")
        return "seeds"
    if dp == "auto":
        dp = "envs" if sweep.Grid(config).total_seeds < world else "seeds"
    if dp == "envs":
        ne = int(config["NUM_ENVS"])
        if ne % world or (int(config["NUM_STEPS"]) * ne // world) % int(config["NUM_MINIBATCHES"]):
            raise ValueError(f"DATA_PARALLEL=envs: NUM_ENVS={ne} must split evenly over {world} ranks and "
                             f"NUM_MINIBATCHES must divide NUM_STEPS*NUM_ENVS/{world}")
    return dp


def _shard_seeds(rngs):
    """Seeds are independent runs (jax.vmap over rngs, pqn_minatar.py:459-461):
    under torchrun each rank trains a contiguous slice of the same split(key, NUM_SEEDS) (tiled over the points of a
    hyperparameter grid)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return rngs, 0, 1
    r, w = dist.get_rank(), dist.get_world_size()
    lo, hi = seed_slice(rngs.shape[0], r, w)
    return rngs[lo:hi], r, w


def single_run(config, make_train, alg_file_name="pqn", env_sharding=True):
    config = {**config, **config["alg"]}                              # :437
    print(config)
    alg_name = config.get("ALG_NAME", "pqn")
    env_name = config["ENV_NAME"]
    env_names = sweep.env_names(config)                               # a list of envs: one run trains them all
    use_wandb = config.get("WANDB_MODE", "disabled") != "disabled"
    d_rank, d_world = init_distributed()
    if env_names is not None:                                         # refused before a wandb run is started
        from . import env_list
        env_list.refuse(config, d_world, env_sharding)
    if use_wandb:
        import wandb
        label = "+".join(env_names) if env_names is not None else env_name
        wandb.init(entity=config["ENTITY"], project=config["PROJECT"],
                   tags=[alg_name.upper(), *(n.upper() for n in env_names or [env_name]), "b200_native"],
                   name=f'{config["ALG_NAME"]}_{label}', config=config, mode=config["WANDB_MODE"])
    grid = sweep.Grid(config)                                         # lists of LR, GAMMA, ...: one batched sweep
    env_sharded = pick_data_parallel(config, d_world, env_sharding) == "envs"
    pbt.settings(config, d_world, env_sharded)                        # a population must live in one process
    rng = jr.PRNGKey(config["SEED"])                                  # :456
    t0 = time.time()
    rngs = jr.split(rng, config["NUM_SEEDS"], int(config.get("JAX_THREEFRY_PARTITIONABLE", 0)))   # :459
    rngs = grid.tile(rngs)                                            # the same keys for every grid point
    if env_sharded:
        local_rngs, rank, world = rngs, 0, 1                          # every rank trains every seed on its env shard;
    else:                                                             # rank 0 alone saves (parameters are replicated)
        local_rngs, rank, world = _shard_seeds(rngs)
    seed_lo = seed_slice(rngs.shape[0], rank, world)[0]               # global index of this rank's first seed
    if local_rngs.shape[0] == 0:
        # fewer seeds than ranks in the seed-sharded mode: this rank has no run of its own (the env-sharded
        # mode, DATA_PARALLEL=envs, is what uses every GPU for a single seed)
        print(f"rank {rank}: no seeds assigned ({grid.total_seeds} seeds < world size {world})")
        return None
    train = make_train(config)
    engines = getattr(train, "engines", None) or {env_name: train.engine}
    for engine in engines.values():
        engine.seed_lo = seed_lo
        if env_sharded:
            engine.env_shard = (d_rank, d_world)
    outs = train(local_rngs)                                          # :460-461 (seed axis is native)
    torch.cuda.synchronize()
    print(f"Took {time.time() - t0} seconds to complete.")
    if config.get("SAVE_PATH", None) is not None and not (env_sharded and d_rank != 0):   # :464-483
        if env_names is None:
            _save(config, grid, outs, alg_name, rank, seed_lo, local_rngs.shape[0])
        else:                                     # every env where and as its standalone run saves it
            for name, engine in engines.items():
                _save(engine.cfg, grid, outs[name], alg_name, rank, seed_lo, local_rngs.shape[0])
    return outs


def _save(config, grid, outs, alg_name, rank, seed_lo, num_local):
    """The run's config (and sweep table) yaml and one checkpoint per local seed under <SAVE_PATH>/<ENV_NAME>."""
    from .utils.save_load import save_params
    env_name = config["ENV_NAME"]
    model_state = outs["runner_state"][0]
    save_dir = os.path.join(config["SAVE_PATH"], env_name)
    os.makedirs(save_dir, exist_ok=True)
    prefix = f'{alg_name}_{env_name}_seed{config["SEED"]}'
    if rank == 0:
        config_loader.save_yaml({k: v for k, v in config.items() if k != "alg"},
                                os.path.join(save_dir, f'{prefix}_config.yaml'))
        if grid.G > 1:                                                # the values every checkpoint trained with
            config_loader.save_yaml({"axes": {k: v for k, v in grid.axes}, "num_seeds": grid.num_seeds,
                                     "seeds": grid.table(0, grid.total_seeds)},
                                    os.path.join(save_dir, f'{prefix}_sweep.yaml'))
        if "pbt" in outs:                                             # the population's lineage
            config_loader.save_yaml(pbt.lineage_yaml(outs["pbt"], pbt.settings(config)),
                                    os.path.join(save_dir, f'{prefix}_pbt.yaml'))
    for i in range(num_local):
        def pick(d):
            return {k: (pick(v) if isinstance(v, dict) else v[i]) for k, v in d.items()}
        gi = seed_lo + i
        name = f"vmap{gi}" if grid.G == 1 else f"g{gi // grid.num_seeds}_vmap{gi % grid.num_seeds}"
        save_params(pick(model_state.params), os.path.join(save_dir, f'{prefix}_{name}.safetensors'))


def tune(default_config, make_train):
    """wandb Bayesian sweep over LR (pqn_minatar.py:486-531)."""
    default_config = {**default_config, **default_config["alg"]}
    pbt.settings({**default_config, "HYP_TUNE": True})
    if sweep.env_names(default_config) is not None:
        from . import env_list
        env_list.refuse({**default_config, "HYP_TUNE": True}, 1)
    import wandb
    print(default_config)
    alg_name = default_config.get("ALG_NAME", "pqn")
    env_name = default_config["ENV_NAME"]

    def wrapped_make_train():
        wandb.init(project=default_config["PROJECT"])
        config = copy.deepcopy(default_config)
        for k, v in dict(wandb.config).items():
            config[k] = v
        print("running experiment with params:", config)
        rng = jr.PRNGKey(config["SEED"])
        rngs = jr.split(rng, config["NUM_SEEDS"])
        make_train(config)(rngs)
        torch.cuda.synchronize()

    sweep_config = {
        "name": f"{alg_name}_{env_name}",
        "method": "bayes",
        "metric": {"name": "returned_episode_returns", "goal": "maximize"},
        "parameters": {"LR": {"values": [0.001, 0.0005, 0.0001, 0.00005]}},
    }
    wandb.login()
    sweep_id = wandb.sweep(sweep_config, entity=default_config["ENTITY"], project=default_config["PROJECT"])
    wandb.agent(sweep_id, wrapped_make_train, count=1000)


def main(make_train, argv=None, env_sharding=True):
    """`python -m purejaxql_b200.pqn_minatar +alg=pqn_minatar alg.NUM_ENVS=4096 NUM_SEEDS=8`"""
    argv = sys.argv[1:] if argv is None else argv
    config = config_loader.compose(argv)
    import yaml
    print("Config:\n", yaml.safe_dump(config, sort_keys=False))
    if config.get("HYP_TUNE", False):
        tune(config, make_train)
    else:
        return single_run(config, make_train, env_sharding=env_sharding)
