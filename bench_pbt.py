"""Time population-based training: one event, and a run with an event after every update against the same run without.

    python bench_pbt.py [--seeds 128] [--events 50] [--updates 40] [--reps 3]

"event": one ``pqn_pbt_event`` on the MinAtar CNN's parameter layout (Breakout-MinAtar, layer_norm) at S = --seeds
seeds, m = S / 4, all five hyperparameters perturbed, fitness over one column; CUDA events around --events back-to-back
events after five untimed ones, reported per event.  "run": the pqn_minatar preset at 4 LR values x (S / 4) seeds for
--updates updates (no evaluation), with PBT_INTERVAL=1 and without PBT; each timed on the host clock around make_train
+ train ending in a device synchronise, alternating over --reps repetitions after an untimed warm-up of each, medians
reported.  One JSON line with the card's name and power limit.  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import statistics

from bench_sweep import LRS, card, timed


def time_event(S, n_events):
    import torch
    from purejaxql_b200 import envs, pbt
    from purejaxql_b200.networks import NET_CNN, QNetworkSpec
    dev = torch.device("cuda")
    env, _ = envs.make("Breakout-MinAtar")
    spec = QNetworkSpec(NET_CNN, env.info.obs_shape[2], env.num_actions)
    P, NU = spec.total, 100
    st = pbt.Settings(1, 0.25, tuple(pbt.PERTURB_CODES), (0.8, 1.25), "train", 0)
    hp = {"eps": torch.rand(NU, S, device=dev), "gamma": torch.full((S,), 0.99, device=dev),
          "lam": torch.full((S,), 0.65, device=dev), "max_norm": torch.full((S,), 10.0, device=dev),
          "rew_scale": torch.ones(S, device=dev)}
    pop = pbt.Population(st, S, NU + 1, hp, 0, 0, dev)
    params, mu, nu = (torch.randn(S, P, device=dev) for _ in range(3))
    stats = spec.init_stats(S, dev)
    fit = torch.randn(S, NU, dtype=torch.float64, device=dev)

    def one(n):
        pop.event(n, fit, n % NU, 1, params, mu, nu, stats)
    for n in range(1, 6):
        one(n)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for n in range(6, 6 + n_events):
        one(n)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n_events, P, pop.m


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--seeds", type=int, default=128)
    ap.add_argument("--events", type=int, default=50)
    ap.add_argument("--updates", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    from purejaxql_b200 import config_loader, jaxrandom as jr, pqn_minatar, sweep
    if not torch.cuda.is_available():
        raise SystemExit("bench_pbt.py measures on the GPU; there is none")
    info = card()
    event_ms, P, m = time_event(args.seeds, args.events)
    per_point = max(args.seeds // len(LRS), 2)

    def cfg(updates, interval):
        c = config_loader.compose(["+alg=pqn_minatar", f"NUM_SEEDS={per_point}", "SAVE_PATH=null"])
        c = {**c, **c["alg"]}
        steps = float(updates * c["NUM_STEPS"] * c["NUM_ENVS"])
        c.update(TOTAL_TIMESTEPS=steps, TOTAL_TIMESTEPS_DECAY=steps, TEST_DURING_TRAINING=False, LR=LRS,
                 PBT_INTERVAL=interval)
        return c
    keys = sweep.Grid(cfg(3, 0)).tile(jr.split(jr.PRNGKey(0), per_point))
    for interval in (1, 0):                                                 # warm-up: module loads, graph capture
        pqn_minatar.make_train(cfg(3, interval))(keys)
    t_pbt, t_base = [], []
    for r in range(args.reps):
        pair = [(t_pbt, 1), (t_base, 0)]
        for out, interval in (pair if r % 2 == 0 else pair[::-1]):
            c = cfg(args.updates, interval)
            out.append(timed(lambda c=c: pqn_minatar.make_train(c)(keys)))
    mp, mb = statistics.median(t_pbt), statistics.median(t_base)
    print(json.dumps({"bench": "pbt", "event_env": "Breakout-MinAtar", "run_env": cfg(3, 0)["ENV_NAME"],
                      "event_seeds": args.seeds, "event_replaced": m, "event_params_per_seed": P,
                      "event_ms": round(event_ms, 4), "run_seeds": len(LRS) * per_point, "run_updates": args.updates,
                      "run_pbt_interval_1_s": round(mp, 3), "run_without_pbt_s": round(mb, 3),
                      "run_overhead": round(mp / mb - 1.0, 4), "run_pbt_s": [round(x, 3) for x in t_pbt],
                      "run_base_s": [round(x, 3) for x in t_base], **info}), flush=True)


if __name__ == "__main__":
    main()
