"""Seaquest-MinAtar measurements (the game is not in `bench.py --config minatar5`, which runs the four games gymnax
0.0.6 registers).

    python bench_seaquest.py [--steps 3] [--warmup 3]           # pqn_minatar @1024 envs x 16 seeds + env.step roofline
    python bench_seaquest.py --curve 5e6                        # a short learning curve of the pqn_minatar preset

The first form prints one JSON line in the shape of a `--config minatar5` line: env steps per second over the timed
updates (CUDA events), the end-to-end rate, SM clocks sampled in the timed region, and the standalone env.step kernel
at 2^20 envs against the HBM roofline.  The second trains the pqn_minatar preset on Seaquest with 4 seeds for the
given number of env steps and prints the mean training return per update next to the return of a uniformly random
policy over the same number of steps.  The D = 1000 MLP is measured by `bench_shapes.py --env Seaquest-MinAtar`.
Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json

import numpy as np

import bench

NAME = "Seaquest-MinAtar"


def throughput(args):
    import torch
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    from purejaxql_b200 import config_loader, jaxrandom as jr, pqn_minatar

    def cfg_for(n):
        c = config_loader.compose(["+alg=pqn_minatar", f"alg.ENV_NAME={NAME}", "NUM_SEEDS=16", "SAVE_PATH=null",
                                   "alg.NUM_ENVS=1024", "alg.TEST_DURING_TRAINING=False"])
        c = {**c, **c["alg"]}
        c["TOTAL_TIMESTEPS"] = float(n * c["NUM_STEPS"] * 1024)
        return c
    rngs = np.ascontiguousarray(jr.to_numpy_u32(jr.split(jr.PRNGKey(0, dev), 16)))
    ms, launches, clocks, out, _, eng = bench.timed_train(pqn_minatar, cfg_for(args.warmup + args.steps), rngs,
                                                          args.warmup, dev, 1, 0)
    env_steps = 16 * args.steps * 32 * 1024
    e2e_s, _, _ = bench.e2e_train(pqn_minatar, cfg_for(args.steps), rngs, dev, 1)
    roof = bench.env_step_roofline(dev, 0, bench.load_peaks(), names=(NAME,))
    print(json.dumps({"metric": f"{NAME} pqn_minatar env steps/sec @1024 envs x16 seeds", "value": env_steps / (ms / 1e3),
                      "unit": bench.UNIT, "ms_per_step": ms / args.steps, "steps": args.steps, "warmup": args.warmup,
                      "clocks": clocks, "e2e": env_steps / e2e_s, "gpu_launches": launches,
                      "cuda_graph": bool(eng.graph_captured), "card": card(),
                      "td_loss_finite": bool(torch.isfinite(out["metrics"]["td_loss"]).all()),
                      "env_step": roof[NAME]}), flush=True)


def curve(total):
    import torch
    from purejaxql_b200 import config_loader, envs, jaxrandom as jr, pqn_minatar
    c = config_loader.compose(["+alg=pqn_minatar", f"alg.ENV_NAME={NAME}", "NUM_SEEDS=4", "SAVE_PATH=null",
                               f"alg.TOTAL_TIMESTEPS={total}", "alg.TEST_DURING_TRAINING=False"])
    out = pqn_minatar.single_run(c)
    ret = out["metrics"]["returned_episode_returns"].cpu().numpy()          # [seeds, updates]
    # a uniformly random policy over 1024 envs x 2,000 steps
    dev = torch.device("cuda", 0)
    env, params = envs.make(NAME)
    n = 1024
    _, st = env.reset(jr.split(jr.PRNGKey(1, dev), n), params)
    done_ret = []
    g = torch.Generator(device=dev).manual_seed(0)
    for t in range(2000):
        a = torch.randint(0, env.num_actions, (n,), dtype=torch.int32, device=dev, generator=g)
        _, st, _, d, info = env.step(jr.split(jr.PRNGKey(10_000 + t, dev), n), st, a, params, inplace=True)
        done_ret.append(info["returned_episode_returns"][d].cpu())
    rand = float(torch.cat(done_ret).mean())
    k = max(1, ret.shape[1] // 20)
    print(json.dumps({"metric": f"{NAME} pqn_minatar preset training return (mean over 4 seeds), unpinned",
                      "env_steps": float(total), "updates": int(ret.shape[1]),
                      "return_every_k_updates": [round(float(v), 3) for v in ret.mean(0)[::k]], "k": k,
                      "final_mean_last_5pct": float(ret[:, -k:].mean()), "random_policy_return": rand,
                      "card": card()}), flush=True)


def card():
    import bench_shapes
    return bench_shapes.card()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--curve", type=float, default=0.0, help="env steps of a learning curve (0: measure throughput)")
    args = ap.parse_args()
    if args.curve > 0:
        curve(args.curve)
    else:
        throughput(args)


if __name__ == "__main__":
    main()
