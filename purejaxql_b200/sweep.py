"""Hyperparameter grids trained as one batched run.

Every kernel is batched over the seed axis and nothing reduces across seeds, so seeds may train with different scalar
hyperparameters in the same launches.  A config may give a YAML list instead of a scalar for the keys of
``SWEEP_KEYS``; the list-valued keys form a Cartesian grid of G points::

    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole NUM_SEEDS=4 "alg.LR=[0.001,0.0005,0.0001,0.00005]"

Layout: points are ordered by key in ``SWEEP_KEYS`` order (the first list-valued key varies slowest), then by the
order of each key's list.  Point g gets NUM_SEEDS seeds and ``train`` runs S = G * NUM_SEEDS of them: seed index
g * NUM_SEEDS + i is seed i of point g.  Every point uses the same keys ``split(PRNGKey(SEED), NUM_SEEDS)`` (common
random numbers), so the key array of a sweep is those keys tiled G times (``Grid.tile``) and the seeds of point g train
exactly what a standalone run of point g's config given the same key array trains.

``ENV_NAME`` may be a list too: not a grid axis (different envs cannot share launches) but a list of envs, each trained
by its own engine as a standalone run of its name would train it (``env_list.py``); every env trains every grid point.

The device reads the hyperparameters from per-seed arrays (``engine.seed_inputs``): the eps table [NU][S], the
RAdam schedule [S][steps][4] (one shared [steps][4] table when G == 1), and gamma, lambda, max-norm and reward scale
[S].  A config without lists gives exactly the inputs of a scalar run.
"""
from __future__ import annotations

import itertools

import numpy as np

SWEEP_KEYS = ("LR", "MAX_GRAD_NORM", "GAMMA", "LAMBDA", "REW_SCALE", "EPS_START", "EPS_FINISH", "EPS_DECAY")
MAX_SEEDS = 65535          # the seed axis is gridDim.y of the kernels
_DEFAULTS = {"REW_SCALE": 1}
LIST_SETTINGS = ("PBT_PERTURB", "PBT_FACTORS")   # list-valued settings of population-based training, not grid axes


def env_names(config: dict) -> list | None:
    """The envs of a list-valued ``ENV_NAME`` (None for a single env); refuses an empty list and duplicate names."""
    v = config.get("ENV_NAME")
    if not isinstance(v, (list, tuple)):
        return None
    if len(v) == 0:
        raise ValueError("ENV_NAME=[]: an empty list has no env to train")
    if not all(isinstance(n, str) for n in v):
        raise ValueError(f"ENV_NAME={v!r}: every entry of the list must be an env name")
    dup = sorted({n for n in v if list(v).count(n) > 1})
    if dup:
        raise ValueError(f"ENV_NAME={v!r}: {', '.join(dup)} appears more than once; each env trains once per run")
    return list(v)


class Grid:
    """The grid of a config (refuses lists it cannot train, before anything is built).  ``points[g]`` maps each
    list-valued key to point g's value; ``config(g)`` is point g's scalar config."""

    def __init__(self, config: dict):
        env_names(config)
        for k, v in config.items():
            if isinstance(v, (list, tuple)) and k not in SWEEP_KEYS and k != "ENV_NAME" and k not in LIST_SETTINGS:
                raise ValueError(f"{k}={v!r}: only {', '.join(SWEEP_KEYS)} may be a list (a grid of settings trained "
                                 f"as one batched run), and ENV_NAME (a list of envs trained side by side); {k} "
                                 f"changes the shapes or the kernels of the run")
        self.axes = []
        for k in SWEEP_KEYS:
            v = config.get(k)
            if isinstance(v, (list, tuple)):
                if len(v) == 0:
                    raise ValueError(f"{k}=[]: an empty list has no value to train with")
                self.axes.append((k, list(v)))
        self.base = config
        self.points = [dict(zip([k for k, _ in self.axes], vals))
                       for vals in itertools.product(*[vs for _, vs in self.axes])]
        self.G = len(self.points)
        self.num_seeds = int(config.get("NUM_SEEDS", 1))
        if self.G > 1 and self.G * self.num_seeds > MAX_SEEDS:
            raise ValueError(f"a grid of {self.G} points x NUM_SEEDS={self.num_seeds} is {self.G * self.num_seeds} "
                             f"seeds; one run trains at most {MAX_SEEDS}")

    @property
    def total_seeds(self):
        return self.G * self.num_seeds

    def config(self, g: int) -> dict:
        return {**self.base, **self.points[g]}

    def value(self, g: int, key: str):
        return self.config(g).get(key, _DEFAULTS.get(key))

    def tile(self, rngs):
        """The [G * NUM_SEEDS, 2] key array of the sweep from the [NUM_SEEDS, 2] keys every point shares."""
        if self.G == 1:
            return rngs
        import torch
        if isinstance(rngs, torch.Tensor):
            return rngs.repeat(self.G, 1)
        return np.tile(np.asarray(rngs), (self.G, 1))

    def point_of(self, seed_lo: int, S: int) -> np.ndarray:
        """Grid point of each of the S seeds [seed_lo, seed_lo + S) of the run (a seed-sharded rank holds a slice)."""
        if self.G == 1:
            return np.zeros(S, np.int64)
        if seed_lo < 0 or seed_lo + S > self.total_seeds:
            raise ValueError(f"seeds [{seed_lo}, {seed_lo + S}) of a sweep of {self.G} points x NUM_SEEDS="
                             f"{self.num_seeds}: train(rngs) takes the tiled key array (Grid.tile) or a slice of it")
        return (seed_lo + np.arange(S)) // self.num_seeds

    def table(self, seed_lo: int, S: int) -> dict:
        """The values each of the S seeds trains with: {"point": [S], "seed": [S] (index within its point), key: [S]
        for every key of SWEEP_KEYS}."""
        pt = self.point_of(seed_lo, S)
        out = {"point": pt.tolist(), "seed": ((seed_lo + np.arange(S)) % max(self.num_seeds, 1)).tolist()
               if self.G > 1 else list(range(seed_lo, seed_lo + S))}
        for k in SWEEP_KEYS:
            out[k] = [self.value(int(g), k) for g in pt]
        return out
