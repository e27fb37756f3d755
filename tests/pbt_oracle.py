"""NumPy restatement of one population-based training event (purejaxql_b200/pbt.py, DESIGN.md section 3.10), on the
jax.random restatement of oracle/jax_prng.py.  Test infrastructure: the product never imports it."""
from __future__ import annotations

import numpy as np

from oracle import jax_prng as jr

CODES = ("LR", "MAX_GRAD_NORM", "REW_SCALE", "GAMMA", "LAMBDA")


def fitness(cols: np.ndarray) -> np.ndarray:
    """[S, k] float64 -> the mean of each row, summed in column order."""
    cols = np.asarray(cols, np.float64)
    acc = np.zeros(cols.shape[0])
    for c in range(cols.shape[1]):
        acc = acc + cols[:, c]
    return acc / np.float64(cols.shape[1])


def order(f: np.ndarray) -> np.ndarray:
    """Seeds by descending fitness; ties by the lower index; NaN last, also by index."""
    f = np.asarray(f, np.float64)
    return np.array(sorted(range(len(f)), key=lambda i: (bool(np.isnan(f[i])), 0.0 if np.isnan(f[i]) else -f[i], i)),
                    np.int64)


def plan(f, m: int, kp, n_perturb: int, factors, partitionable=False):
    """One event's decisions: (next kp, order, parent [S], children [m], their parents [m], phi [m, n_perturb])."""
    kp = np.asarray(kp, np.uint32)
    ks = jr.split(kp, 2, partitionable)
    kp_next, ke = ks[0], ks[1]
    kk = jr.split(ke, 2, partitionable)
    ka, kf = kk[0], kk[1]
    a = jr.randint(ka, (m,), 0, m, partitionable).astype(np.int64)
    b = (jr.randint(kf, (m, n_perturb), 0, 2, partitionable).astype(np.int64) if n_perturb
         else np.zeros((m, 0), np.int64))
    o = order(f)
    S = len(o)
    top, bottom = o[:m], o[S - m:]
    parent = np.arange(S)
    parent[bottom] = top[a]
    phi = np.asarray(factors, np.float32)[b]
    return kp_next, o, parent, bottom, top[a], phi


def toward_one(x, phi):
    one = np.float32(1)
    return np.clip(one - (one - np.float32(x)) * np.float32(phi), np.float32(0), one).astype(np.float32)


def apply(tables: dict, children, parents, phi, perturb, eps=None, eps_from=0):
    """Exploit + explore on copies of the per-seed tables {lr_mult, gamma, lam, max_norm, rew_scale, sched_src}
    (float32 / int32 [S]) and of eps [rows][S]: the child takes its parent's values, then each perturbed key."""
    t = {k: np.array(v, copy=True) for k, v in tables.items()}
    for j, (c, p) in enumerate(zip(children, parents)):
        for k in t:
            t[k][c] = tables[k][p]
        for i, key in enumerate(perturb):
            ph = phi[j, i]
            if key == "LR":
                t["lr_mult"][c] = np.float32(t["lr_mult"][c]) * ph
            elif key == "MAX_GRAD_NORM":
                t["max_norm"][c] = np.float32(t["max_norm"][c]) * ph
            elif key == "REW_SCALE":
                t["rew_scale"][c] = np.float32(t["rew_scale"][c]) * ph
            elif key == "GAMMA":
                t["gamma"][c] = toward_one(t["gamma"][c], ph)
            else:
                t["lam"][c] = toward_one(t["lam"][c], ph)
    if eps is not None:
        e = np.array(eps, copy=True)
        for c, p in zip(children, parents):
            e[eps_from:, c] = eps[eps_from:, p]
        return t, e
    return t
