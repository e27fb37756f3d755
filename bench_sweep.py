"""Time a hyperparameter grid trained as one batched run against the same configs trained one after another.

    python bench_sweep.py [--presets pqn_rnn_cartpole,pqn_cartpole,pqn_minatar] [--updates 40] [--seeds 1] [--reps 3]

For each preset: G = 4 LR values (the LR values of the reference's HYP_TUNE sweep, pqn_minatar.py:486-531) x NUM_SEEDS
seeds.  "sweep" is one make_train + train of the list-valued config on the tiled keys (S = 4 * NUM_SEEDS); "sequential"
is four make_train + train calls, one per LR, on NUM_SEEDS seeds each.  Both end in a device synchronise and are timed
on the host clock around the whole call (set-up, every update, no evaluation); the two alternate over --reps
repetitions after one untimed warm-up of each, and the medians are reported.  One JSON line per preset, with the card's
name and power limit.  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import time

LRS = [0.001, 0.0005, 0.0001, 0.00005]
SCRIPTS = {"pqn_rnn_cartpole": "pqn_rnn_gymnax", "pqn_cartpole": "pqn_gymnax", "pqn_minatar": "pqn_minatar",
           "pqn_rnn_memory_chain": "pqn_rnn_gymnax"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def config(preset, updates, seeds, lr):
    from purejaxql_b200 import config_loader
    c = config_loader.compose([f"+alg={preset}", f"NUM_SEEDS={seeds}", "SAVE_PATH=null"])
    c = {**c, **c["alg"]}
    steps = float(updates * c["NUM_STEPS"] * c["NUM_ENVS"])
    c.update(TOTAL_TIMESTEPS=steps, TOTAL_TIMESTEPS_DECAY=steps, TEST_DURING_TRAINING=False, LR=lr)
    return c


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--presets", default="pqn_rnn_cartpole,pqn_cartpole,pqn_minatar")
    ap.add_argument("--updates", type=int, default=40)
    ap.add_argument("--seeds", type=int, default=1, help="NUM_SEEDS of every grid point")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import importlib

    import torch
    from purejaxql_b200 import jaxrandom as jr, sweep
    if not torch.cuda.is_available():
        raise SystemExit("bench_sweep.py measures on the GPU; there is none")
    info = card()
    for preset in args.presets.split(","):
        mod = importlib.import_module(f"purejaxql_b200.{SCRIPTS[preset]}")
        keys = jr.split(jr.PRNGKey(0), args.seeds)
        grid_cfg = config(preset, args.updates, args.seeds, LRS)
        tiled = sweep.Grid(grid_cfg).tile(keys)

        def run_sweep(cfg=grid_cfg):
            mod.make_train(dict(cfg))(tiled)

        def run_sequential():
            for lr in LRS:
                mod.make_train(config(preset, args.updates, args.seeds, lr))(keys)
        run_sweep(config(preset, 3, args.seeds, LRS))                      # warm-up: module loads, graph capture
        for lr in LRS[:1]:
            mod.make_train(config(preset, 3, args.seeds, lr))(keys)
        t_sweep, t_seq = [], []
        for r in range(args.reps):                                          # alternate the two, start order flips
            pair = [(t_sweep, run_sweep), (t_seq, run_sequential)]
            for out, fn in (pair if r % 2 == 0 else pair[::-1]):
                out.append(timed(fn))
        c = grid_cfg
        env_steps = args.updates * c["NUM_STEPS"] * c["NUM_ENVS"] * len(LRS) * args.seeds
        ms, mq = statistics.median(t_sweep), statistics.median(t_seq)
        print(json.dumps({"preset": preset, "env": c["ENV_NAME"], "grid": {"LR": LRS}, "num_seeds": args.seeds,
                          "updates": args.updates, "sweep_s": round(ms, 3), "sequential_s": round(mq, 3),
                          "speedup": round(mq / ms, 2), "sweep_env_steps_per_s": round(env_steps / ms),
                          "sequential_env_steps_per_s": round(env_steps / mq),
                          "sweep_runs_s": [round(x, 3) for x in t_sweep],
                          "sequential_runs_s": [round(x, 3) for x in t_seq], **info}), flush=True)


if __name__ == "__main__":
    main()
