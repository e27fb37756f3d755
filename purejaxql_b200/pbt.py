"""Population-based training (PBT) over the seed axis of a run: truncation selection every PBT_INTERVAL updates.

    python -m purejaxql_b200.pqn_minatar +alg=pqn_minatar NUM_SEEDS=8 "alg.LR=[0.001,0.0005,0.0001,0.00005]" PBT_INTERVAL=20

The S seeds of a run (G grid points x NUM_SEEDS, sweep.Grid) are the population; the grid is its initial state.  After
every k-th update n with n < NUM_UPDATES (k = PBT_INTERVAL > 0) one event runs on the device (``pqn_pbt_event``,
DESIGN.md section 3.10):

1. fitness f[s]: "train", the mean of the metric column returned_episode_returns over updates n-k+1 .. n (float64,
   summed in column order); "test", the returned_episode_returns of the evaluation taken after update n;
2. order: descending f, ties by the lower seed index, NaN last; top = its first m seeds, bottom its last m, with
   m = floor(PBT_FRACTION * S);
3. keys: a chain of its own, kp_0 = PRNGKey(PBT_SEED); event e: kp_e, ke = split(kp_{e-1}); ka, kf = split(ke);
   a = randint(ka, (m,), 0, m) picks the parents and b = randint(kf, (m, len(PBT_PERTURB)), 0, 2) the factors;
4. exploit: child bottom[j] takes the rows of parent top[a[j]] (params, RAdam mu and nu, batch_stats) and its
   hyperparameters: its eps schedule from update n+1 on, its LR schedule from the next optimizer step on, GAMMA,
   LAMBDA, MAX_GRAD_NORM and REW_SCALE.  It keeps its own env state, rollout buffers, recurrent carry, memory and
   runner key;
5. explore: phi = PBT_FACTORS[b[j, i]] for key PBT_PERTURB[i] (fp32): LR, MAX_GRAD_NORM and REW_SCALE are multiplied
   by phi, GAMMA and LAMBDA become clamp(1 - (1 - x) * phi, 0, 1).

Seeds outside bottom are not written.  The LR stays a schedule table per grid point (or one shared table): a seed reads
the table of seed ``sched_src[s]`` scaled by ``lr_mult[s]`` (``pqn_radam_clip_step_pbt``), so no event copies a
schedule.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np
import torch

from . import _lib, jaxrandom as jr, sweep

PERTURB_CODES = {"LR": 0, "MAX_GRAD_NORM": 1, "REW_SCALE": 2, "GAMMA": 3, "LAMBDA": 4}
DEFAULTS = {"PBT_INTERVAL": 0, "PBT_FRACTION": 0.25, "PBT_PERTURB": ["LR"], "PBT_FACTORS": [0.8, 1.25],
            "PBT_FITNESS": "train", "PBT_SEED": None}
FITNESS_METRIC = "returned_episode_returns"


@dataclasses.dataclass(frozen=True)
class Settings:
    interval: int
    fraction: float
    perturb: tuple
    factors: tuple
    fitness: str
    seed: int

    def replaced(self, S: int) -> int:
        """m: the seeds replaced per event in a population of S."""
        return int(math.floor(self.fraction * S))


def _get(config, key):
    v = config.get(key)
    return DEFAULTS[key] if v is None else v


def _is_int(v):
    return isinstance(v, (int, np.integer)) and not isinstance(v, bool)


def _is_num(v):
    return isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, bool)


def settings(config: dict, world: int = 1, env_sharded: bool = False) -> Settings | None:
    """The PBT settings of a config (None: no PBT), refusing a bad value, a population too small to replace a seed, a
    test fitness without a matching evaluation, HYP_TUNE and a seed-sharded multi-process run.  Needs nothing built."""
    k = _get(config, "PBT_INTERVAL")
    if not _is_int(k) or k < 0:
        raise ValueError(f"PBT_INTERVAL={k!r}: expected a non-negative int (0: no population-based training)")
    frac = _get(config, "PBT_FRACTION")
    if not _is_num(frac) or not 0.0 < float(frac) <= 0.5:
        raise ValueError(f"PBT_FRACTION={frac!r}: expected a number in (0, 0.5]")
    per = _get(config, "PBT_PERTURB")
    if (not isinstance(per, (list, tuple)) or any(p not in PERTURB_CODES for p in per)
            or len(set(per)) != len(per)):
        raise ValueError(f"PBT_PERTURB={per!r}: expected a list of distinct keys from {', '.join(PERTURB_CODES)}")
    fac = _get(config, "PBT_FACTORS")
    if (not isinstance(fac, (list, tuple)) or len(fac) != 2 or not all(_is_num(f) for f in fac)
            or not all(0.0 < float(f) < math.inf for f in fac)):
        raise ValueError(f"PBT_FACTORS={fac!r}: expected two positive finite numbers")
    fit = _get(config, "PBT_FITNESS")
    if fit not in ("train", "test"):
        raise ValueError(f"PBT_FITNESS={fit!r}: expected train or test")
    seed = config.get("PBT_SEED")
    if seed is None:
        seed = config.get("SEED", 0)
    if not _is_int(seed):
        raise ValueError(f"PBT_SEED={seed!r}: expected an int (default: SEED)")
    if k == 0:
        return None
    if config.get("HYP_TUNE", False):
        raise ValueError(f"PBT_INTERVAL={k} with HYP_TUNE=True: the wandb LR sweep trains one config per run; "
                         f"population-based training evolves the seeds of one run")
    if world > 1 and not env_sharded:
        raise ValueError(f"PBT_INTERVAL={k}: a seed-sharded run of {world} processes would split the population "
                         f"over the processes; run PBT in one process or with DATA_PARALLEL=envs")
    S = sweep.Grid(config).total_seeds
    m = int(math.floor(float(frac) * S))
    if m < 1:
        raise ValueError(f"PBT_FRACTION={frac} of {S} seeds replaces {m} seeds per event; PBT needs at least one "
                         f"(raise NUM_SEEDS or PBT_FRACTION)")
    if fit == "test":
        if not config.get("TEST_DURING_TRAINING", False):
            raise ValueError("PBT_FITNESS=test needs TEST_DURING_TRAINING=True: the fitness is the evaluation's return")
        nu = config.get("NUM_UPDATES")
        if nu is None:
            nu = config["TOTAL_TIMESTEPS"] // config["NUM_STEPS"] // config["NUM_ENVS"]
        every = int(nu * config["TEST_INTERVAL"])
        if every <= 0 or k % every:
            raise ValueError(f"PBT_FITNESS=test: PBT_INTERVAL={k} must be a multiple of the evaluation cadence "
                             f"int(NUM_UPDATES * TEST_INTERVAL) = {every}")
    return Settings(int(k), float(frac), tuple(per), (float(fac[0]), float(fac[1])), fit, int(seed))


def num_events(st: Settings, num_updates: int) -> int:
    """Events of a run: one after every k-th update n < NUM_UPDATES."""
    return max(num_updates - 1, 0) // st.interval


class Population:
    """The device buffers of one engine's population: the per-seed LR source and multiplier, the event key and the
    event history.  Everything an event edits is a static buffer the update reads, so a captured update graph
    replays unchanged after an event."""

    VALUE_ROWS = ("lr_mult", "gamma", "lam", "max_norm", "rew_scale")

    def __init__(self, st: Settings, S: int, num_updates: int, hp: dict, sched_stride: int, rng_mode: int, dev):
        self.st, self.S, self.m, self.rng_mode = st, S, st.replaced(S), rng_mode
        if self.m < 1 or 2 * self.m > S:
            raise ValueError(f"PBT_FRACTION={st.fraction} of {S} seeds replaces {self.m} seeds per event; PBT needs "
                             f"1 <= m <= S/2")
        self.hp, self.sched_stride = hp, sched_stride
        self.K = num_events(st, num_updates)
        self.sched_src = (torch.arange(S, dtype=torch.int32, device=dev) if sched_stride
                          else torch.zeros(S, dtype=torch.int32, device=dev))
        self.lr_mult = torch.ones(S, device=dev)
        self.kp = jr.PRNGKey(st.seed, dev)
        self.fitness = torch.zeros((max(self.K, 1), S), dtype=torch.float64, device=dev)
        self.parent = torch.zeros((max(self.K, 1), S), dtype=torch.int32, device=dev)
        self.value_hist = torch.zeros((self.K + 1, len(self.VALUE_ROWS), S), device=dev)
        self.src_hist = torch.zeros((self.K + 1, S), dtype=torch.int32, device=dev)
        self.order = torch.zeros(S, dtype=torch.int32, device=dev)
        self.ws = torch.empty(int(_lib.lib().pqn_pbt_workspace_bytes(S, self.m)), dtype=torch.uint8, device=dev)
        self._snapshot(0)

    def live(self) -> dict:
        """The buffers a training state holds (the edited eps, GAMMA, ... tables are those of ``hp``)."""
        return {"pbt/sched_src": self.sched_src, "pbt/lr_mult": self.lr_mult, "pbt/kp": self.kp,
                "pbt/eps": self.hp["eps"], "pbt/gamma": self.hp["gamma"], "pbt/lam": self.hp["lam"],
                "pbt/max_norm": self.hp["max_norm"], "pbt/rew_scale": self.hp["rew_scale"],
                "pbt/fitness": self.fitness, "pbt/parent": self.parent, "pbt/value_hist": self.value_hist,
                "pbt/src_hist": self.src_hist}

    def _snapshot(self, row):
        tabs = [self.lr_mult, self.hp["gamma"], self.hp["lam"], self.hp["max_norm"], self.hp["rew_scale"]]
        self.value_hist[row].copy_(torch.stack(tabs))
        self.src_hist[row].copy_(self.sched_src)

    def due(self, n_done: int, num_updates: int) -> bool:
        return n_done % self.st.interval == 0 and n_done < num_updates

    def event(self, n_done: int, fit_src: torch.Tensor, fit_col0: int, fit_cols: int, params, mu, nu, batch_stats):
        """The event after update n_done on the current stream: fitness from columns [fit_col0, fit_col0 + fit_cols)
        of the float64 [S, stride] fit_src; then exploit and explore in place."""
        e = n_done // self.st.interval - 1
        S, eps = self.S, self.hp["eps"]
        a = _lib.PbtEvent()
        a.S, a.m = S, self.m
        a.fit = fit_src.data_ptr() + 8 * fit_col0
        a.fit_stride, a.fit_cols = fit_src.stride(0), fit_cols
        a.rng_mode, a.key = self.rng_mode, self.kp.data_ptr()
        a.n_perturb = len(self.st.perturb)
        for i, kk in enumerate(self.st.perturb):
            a.perturb[i] = PERTURB_CODES[kk]
        a.factors[0], a.factors[1] = self.st.factors
        a.params, a.mu, a.nu, a.P = params.data_ptr(), mu.data_ptr(), nu.data_ptr(), params.shape[1]
        if batch_stats is not None and batch_stats.numel():
            a.batch_stats, a.stats_floats = batch_stats.data_ptr(), batch_stats.shape[1]
        a.eps, a.eps_rows, a.eps_from = eps.data_ptr(), eps.shape[0], n_done
        a.sched_src, a.lr_mult = self.sched_src.data_ptr(), self.lr_mult.data_ptr()
        a.gamma, a.lambda_ = self.hp["gamma"].data_ptr(), self.hp["lam"].data_ptr()
        a.max_norm, a.rew_scale = self.hp["max_norm"].data_ptr(), self.hp["rew_scale"].data_ptr()
        a.fitness, a.order, a.parent = self.fitness[e].data_ptr(), self.order.data_ptr(), self.parent[e].data_ptr()
        a.workspace = self.ws.data_ptr()
        for t in (fit_src, params, mu, nu, eps):
            assert t.is_cuda and t.is_contiguous()
        _lib.check(_lib.lib().pqn_pbt_event(a, _lib.stream_ptr()), "pqn_pbt_event")
        self._snapshot(e + 1)

    def result(self, grid: "sweep.Grid", seed_lo: int, n_done: int) -> dict:
        """train()'s "pbt": the events, their fitness [K,S] and parents [K,S] (s itself when kept), and for every grid
        key the per-seed value in force initially and after each event [K+1,S] (LR: the source point's LR x
        lr_mult)."""
        K = min(n_done // self.st.interval, self.K)
        S = self.S
        pt = grid.point_of(seed_lo, S)
        src = self.src_hist[:K + 1].cpu().numpy()
        point = pt[src] if self.sched_stride else np.zeros_like(src)
        vals = self.value_hist[:K + 1].cpu().numpy().astype(np.float64)
        rows = dict(zip(self.VALUE_ROWS, np.moveaxis(vals, 1, 0)))
        lr_pts = np.array([float(grid.value(g, "LR")) for g in range(grid.G)])
        values = {"LR": lr_pts[point] * rows["lr_mult"]}
        for key in ("EPS_START", "EPS_FINISH", "EPS_DECAY"):
            values[key] = np.array([float(grid.value(g, key)) for g in range(grid.G)])[point]
        for key, row in (("GAMMA", "gamma"), ("LAMBDA", "lam"), ("MAX_GRAD_NORM", "max_norm"),
                         ("REW_SCALE", "rew_scale")):
            values[key] = rows[row]
        return {"events": [self.st.interval * (e + 1) for e in range(K)],
                "fitness": self.fitness[:K].cpu().numpy(), "parent": self.parent[:K].cpu().numpy(),
                "values": {k: values[k] for k in sweep.SWEEP_KEYS}}


def lineage_yaml(res: dict, st: Settings) -> dict:
    """The lineage file of a run (single_run writes it beside the checkpoints)."""
    return {"settings": dataclasses.asdict(st) | {"perturb": list(st.perturb), "factors": list(st.factors)},
            "events": list(res["events"]),
            "fitness": [[None if np.isnan(f) else float(f) for f in row] for row in res["fitness"]],
            "parent": res["parent"].tolist(),
            "values": {k: v.tolist() for k, v in res["values"].items()}}
