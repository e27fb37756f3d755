#!/usr/bin/env python
"""bench_resume.py — the cost of the training state (STATE_SAVE_INTERVAL / RESUME_FROM) at bench.py's workload.

    python bench_resume.py [--updates 50] [--warmup 2] [--seeds 128] [--envs 4096]

Breakout-MinAtar, pqn_minatar, NUM_ENVS x seeds as in bench.py.  Prints one JSON line with:

* ``state_bytes``: the size of one state file, computed from the buffer shapes (and the size of the file written);
* ``update_ms``: wall time per update over ``--updates`` updates after ``--warmup``, with STATE_SAVE_INTERVAL=0 and
  with STATE_SAVE_INTERVAL=``--updates`` (one state written inside the timed updates), in the same process;
* ``write_s``: the time of that write; ``load_s`` / ``restore_s``: make_train loading the file and train() copying it
  into the device buffers; ``resume_bit_exact``: the resumed run ends with the uninterrupted run's parameters;
* the card's name and power limit.

Files go to a temporary directory that is removed at the end.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return out


def state_bytes(eng, S, n_done):
    """Bytes of the state file's tensors after n_done updates, from the buffer shapes of a pqn_minatar engine."""
    P, stats = eng.spec.total, eng.spec.stats_total
    E, W, words = eng.E, eng.row_words, eng.env.state_words
    n_metrics = 11 + (5 if eng.test else 0)     # env_step, update_steps, env_frame, grad_steps, td_loss, qvals, 5 means
    return {"params_mu_nu": 3 * S * P * 4, "batch_stats": S * stats * 4, "env_state": words * S * E * 4,
            "last_obs": S * E * W * 4, "keys_rng_counters": 2 * S * 2 * 4 + 4 + 8,
            "metrics": n_metrics * S * n_done * 8 + (5 * S * 8 if eng.test else 0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seeds", type=int, default=128)
    ap.add_argument("--envs", type=int, default=4096)
    args = ap.parse_args()
    import torch
    import bench
    from purejaxql_b200 import jaxrandom as jr, pqn_minatar
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rngs = np.ascontiguousarray(jr.to_numpy_u32(jr.split(jr.PRNGKey(0, dev), args.seeds)))
    K, W = args.updates, args.warmup
    tmp = tempfile.mkdtemp(prefix="pqn_state_")
    try:
        def run(extra, timed=True):
            cfg = bench.base_config(W + K, num_envs=args.envs)
            cfg.update(SEED=0, SAVE_PATH=os.path.join(tmp, "models"), **extra)
            t0 = time.perf_counter()
            train = pqn_minatar.make_train(cfg)
            t_make = time.perf_counter() - t0
            eng = train.engine
            marks = {}
            writes, restores = [], []

            def begin(col):
                if timed and col == W:
                    torch.cuda.synchronize(dev)
                    marks["t0"] = time.perf_counter()
            eng.on_update_begin = begin
            save, restore = eng._save_state, eng._restore_state

            def timed_save(*a):
                torch.cuda.synchronize(dev)
                t = time.perf_counter()
                save(*a)
                writes.append(time.perf_counter() - t)

            def timed_restore(*a):
                torch.cuda.synchronize(dev)
                t = time.perf_counter()
                r = restore(*a)
                torch.cuda.synchronize(dev)
                restores.append(time.perf_counter() - t)
                return r
            eng._save_state, eng._restore_state = timed_save, timed_restore
            out = train(rngs)                                      # ends synchronised
            t1 = time.perf_counter()
            res = {"ms_per_update": 1e3 * (t1 - marks["t0"]) / K if timed else None, "make_train_s": t_make,
                   "writes_s": writes, "restore_s": restores,
                   "params": out["runner_state"][0].params_flat.cpu(), "eng": eng}
            del out, train
            return res

        plain = run({"STATE_SAVE_INTERVAL": 0})
        eng = plain.pop("eng")
        sizes = state_bytes(eng, args.seeds, K)
        del eng
        gc.collect(); torch.cuda.empty_cache()
        saving = run({"STATE_SAVE_INTERVAL": K})                   # one write, after update K (inside the timed range)
        path = saving.pop("eng").cfg
        from purejaxql_b200 import state
        path = state.state_file(path)
        file_bytes = os.path.getsize(path)
        gc.collect(); torch.cuda.empty_cache()
        resumed = run({"STATE_SAVE_INTERVAL": 0, "RESUME_FROM": path}, timed=False)
        resumed.pop("eng")
        line = {"metric": "training-state write / resume cost at the bench.py workload",
                "workload": f"Breakout-MinAtar pqn_minatar NUM_ENVS={args.envs} x {args.seeds} seeds, "
                            f"{W} + {K} updates",
                "card": card(),
                "state_bytes": sum(sizes.values()), "state_bytes_parts": sizes, "state_file_bytes": file_bytes,
                "update_ms": {"STATE_SAVE_INTERVAL=0": plain["ms_per_update"],
                              f"STATE_SAVE_INTERVAL={K}": saving["ms_per_update"]},
                "write_s": saving["writes_s"][0],
                "write_gb_s": file_bytes / saving["writes_s"][0] / 1e9,
                "load_s": resumed["make_train_s"], "restore_s": resumed["restore_s"][0],
                "resume_bit_exact": bool(torch.equal(resumed["params"], saving["params"])),
                "bit_exact_with_saving": bool(torch.equal(plain["params"], saving["params"]))}
        print(json.dumps(line), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
