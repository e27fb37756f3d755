"""Time a list of envs trained as one run against the same envs trained one after another.

    python bench_env_list.py [--workloads cartpole6,rnn3,minatar5] [--updates 20] [--reps 3]

Workloads (each a shipped preset, evaluation off):
  cartpole6  pqn_cartpole (32 envs x 64 steps, MLP) over six float envs, 1 seed;
  rnn3       pqn_rnn_cartpole (32 envs x 64 steps, GRU) over CartPole-v1, Acrobot-v1 and MemoryChain-bsuite, 1 seed;
  minatar5   pqn_minatar's five games at NUM_ENVS=1024, NUM_SEEDS=16 (the MinAtar 5-game suite of BASELINE.json).
"list" is one make_train + train of the list-valued config: one engine per env, each on its own CUDA stream.
"sequential" is one make_train + train per env, one after another, on the default stream.  Both are timed on the host
clock around the whole call (set-up, graph capture, every update), ending in a device synchronise; they alternate over
--reps repetitions after one untimed warm-up of each, and the medians are reported.  The first two workloads launch
thousands of small kernels per update and leave most of the GPU idle, so their envs can overlap; the 1024-env MinAtar
updates fill more of it.  One JSON line per workload, with the card's name, power limit and SM clocks, read right after
its timed runs.  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import time

WORKLOADS = {
    "cartpole6": ("pqn_cartpole", "pqn_gymnax", 1, {},
                  ["CartPole-v1", "Acrobot-v1", "MountainCar-v0", "Catch-bsuite", "DeepSea-bsuite", "FourRooms-misc"]),
    "rnn3": ("pqn_rnn_cartpole", "pqn_rnn_gymnax", 1, {}, ["CartPole-v1", "Acrobot-v1", "MemoryChain-bsuite"]),
    "minatar5": ("pqn_minatar", "pqn_minatar", 16, {"NUM_ENVS": 1024},
                 ["Breakout-MinAtar", "Asterix-MinAtar", "SpaceInvaders-MinAtar", "Freeway-MinAtar", "Seaquest-MinAtar"]),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock, max_clock = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}


def config(preset, seeds, overrides, updates, env_name):
    from purejaxql_b200 import config_loader
    c = config_loader.compose([f"+alg={preset}", f"NUM_SEEDS={seeds}", "SAVE_PATH=null"])
    c = {**c, **c["alg"], **overrides}
    steps = float(updates * c["NUM_STEPS"] * c["NUM_ENVS"])
    c.update(TOTAL_TIMESTEPS=steps, TOTAL_TIMESTEPS_DECAY=steps, TEST_DURING_TRAINING=False, ENV_NAME=env_name)
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
    ap.add_argument("--workloads", default="cartpole6,rnn3,minatar5")
    ap.add_argument("--updates", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import importlib

    import torch
    from purejaxql_b200 import jaxrandom as jr
    if not torch.cuda.is_available():
        raise SystemExit("bench_env_list.py measures on the GPU; there is none")
    for wl in args.workloads.split(","):
        preset, script, seeds, overrides, names = WORKLOADS[wl]
        mod = importlib.import_module(f"purejaxql_b200.{script}")
        keys = jr.split(jr.PRNGKey(0), seeds)

        def run_list(updates=args.updates):
            mod.make_train(config(preset, seeds, overrides, updates, list(names)))(keys)

        def run_sequential(updates=args.updates):
            for name in names:
                mod.make_train(config(preset, seeds, overrides, updates, name))(keys)
        run_list(3)                                                         # warm-up: module loads, graph capture
        run_sequential(3)
        t_list, t_seq = [], []
        for r in range(args.reps):                                          # alternate the two, start order flips
            pair = [(t_list, run_list), (t_seq, run_sequential)]
            for out, fn in (pair if r % 2 == 0 else pair[::-1]):
                out.append(timed(fn))
        info = card()
        c = config(preset, seeds, overrides, args.updates, names[0])
        env_steps = args.updates * c["NUM_STEPS"] * c["NUM_ENVS"] * seeds * len(names)
        ml, mq = statistics.median(t_list), statistics.median(t_seq)
        print(json.dumps({"workload": wl, "preset": preset, "envs": names, "num_envs": c["NUM_ENVS"],
                          "num_seeds": seeds, "updates": args.updates, "list_s": round(ml, 3),
                          "sequential_s": round(mq, 3), "speedup": round(mq / ml, 2),
                          "list_env_steps_per_s": round(env_steps / ml),
                          "sequential_env_steps_per_s": round(env_steps / mq),
                          "list_runs_s": [round(x, 3) for x in t_list],
                          "sequential_runs_s": [round(x, 3) for x in t_seq], **info}), flush=True)


if __name__ == "__main__":
    main()
