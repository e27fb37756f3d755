"""Acrobot-v1 pqn_gymnax at 65,536 envs, 1 seed (BASELINE configs[3]: the same workload as
`bench.py --config acrobot65536`) for MLP Q-networks of other widths and depths than the shipped 256 x 2.

    python bench_shapes.py [--steps 3] [--warmup 2] [--shapes 64x2,256x2,512x2,256x4,512x4] [--profile 512x4]
    python bench_shapes.py --env Breakout-MinAtar --shapes 256x2 --profile 256x2 --paths 2,0

`--env` runs the same pqn_cartpole preset on another env (a MinAtar game: the MLP on packed observation bits);
`--paths` repeats every shape for each tensor-core path (pqn_set_tensor_core_path; default 2).

Prints one JSON line per shape: env steps per second over the timed updates (CUDA events around the updates after
`--warmup` untimed ones), the card's name and power limit, and for the `--profile` shape the per-kernel breakdown
(a separate run with launch events on, as bench.py takes it).  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import subprocess

import numpy as np

import bench


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in q.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, subprocess.SubprocessError, IndexError, ValueError):
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "max_sm_clock": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--shapes", default="64x2,256x2,512x2,256x4,512x4")
    ap.add_argument("--profile", default="512x4", help="shape (HxL) whose per-kernel breakdown is reported")
    ap.add_argument("--env", default="Acrobot-v1")
    ap.add_argument("--paths", default="2", help="tensor-core paths to run every shape on (comma-separated)")
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    from purejaxql_b200 import _lib, config_loader, jaxrandom as jr, pqn_gymnax
    E = 65536
    rngs = np.ascontiguousarray(jr.to_numpy_u32(jr.split(jr.PRNGKey(0, dev), 1)))
    info = card()
    for shape, tc_path in [(sh, int(p)) for sh in args.shapes.split(",") for p in args.paths.split(",")]:
        H, L = (int(v) for v in shape.split("x"))
        _lib.check(_lib.lib().pqn_set_tensor_core_path(tc_path), "pqn_set_tensor_core_path")

        def cfg_for(n):
            c = config_loader.compose(["+alg=pqn_cartpole", f"alg.ENV_NAME={args.env}", "NUM_SEEDS=1", "SAVE_PATH=null",
                                       f"alg.NUM_ENVS={E}", "alg.TEST_DURING_TRAINING=False", f"alg.HIDDEN_SIZE={H}",
                                       f"alg.NUM_LAYERS={L}"])
            c = {**c, **c["alg"]}
            c["TOTAL_TIMESTEPS"] = c["TOTAL_TIMESTEPS_DECAY"] = float(n * c["NUM_STEPS"] * E)
            return c
        c = cfg_for(args.warmup + args.steps)
        T = int(c["NUM_STEPS"])
        ms, launches, clocks, out, _, eng = bench.timed_train(pqn_gymnax, c, rngs, args.warmup, dev, 1, 0)
        line = {"metric": f"{args.env} pqn_gymnax env steps/sec @{E} envs, 1 seed, MLP {H}x{L}", "tc_path": tc_path,
                "value": args.steps * T * E / (ms / 1e3), "unit": bench.UNIT, "ms_per_update": ms / args.steps,
                "steps": args.steps, "warmup": args.warmup, "card": info, "clocks": clocks, "gpu_launches": launches,
                "cuda_graph": bool(eng.graph_captured),
                "td_loss_finite": bool(torch.isfinite(out["metrics"]["td_loss"]).all())}
        if shape == args.profile:
            pc = cfg_for(3)
            pc["CUDA_GRAPH"] = False
            _, _, _, _, prof, _ = bench.timed_train(pqn_gymnax, pc, rngs, 1, dev, 1, 0, profile=True)
            total = sum(v[0] for v in prof.values()) or 1.0
            line["kernel_breakdown"] = {k: {"ms_per_update": round(v[0] / 2, 3), "share": round(v[0] / total, 4)}
                                        for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0])}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
