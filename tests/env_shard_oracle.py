"""NumPy restatement of one env-sharded `_update_step` (engine.PQNEngine.train with ``env_shard = (rank, world)``).

The rollout, the bootstrap and the Q(lambda) targets are those of ``oracle.pqn_ref.update_step`` over all E envs: the
union of the shards' rollouts is the unsharded rollout (tests/test_gpu_env_shard.py pins the sharded keys).  The learn
phase follows the engine's sharded one:

* per epoch the same ``rng`` / ``kperm`` chain as the unsharded update; rank r permutes its own T * E_l rows with
  ``split(kperm, world)[r]`` (no split at world = 1), E_l = E / world;
* rank r's rows live in ``obs_buf[s][t][e]`` of its shard, so its local row j is step ``j // E_l`` of env
  ``r * E_l + j % E_l``, global row ``(j // E_l) * E + r * E_l + j % E_l`` of the [T, E] rollout;
* every minibatch step averages the ranks' mean gradients and sums their input statistics.  Ranks hold equal row
  counts, so that is the gradient and the statistics of the union of the W local minibatches, which is what is
  computed here before ``radam_clip_step``; the loss and Q-value metrics are union means as well."""
from __future__ import annotations

import numpy as np

from oracle import jax_prng as jr
from oracle import pqn_ref as R

F32 = np.float32


def global_rows(local, rank, E, world):
    """Global rows (t * E + e) of rank `rank`'s local rows `local` (t * E_l + e_local)."""
    E_l = E // world
    local = np.asarray(local, np.int64)
    return (local // E_l) * E + rank * E_l + local % E_l


def epoch_minibatches(kperm, T, E, nmb, world):
    """[nmb, world, mb] global rows of one epoch: minibatch i of rank r is positions [i * mb, (i + 1) * mb) of rank
    r's permutation of its T * E_l rows."""
    E_l = E // world
    n = T * E_l
    assert E % world == 0 and n % nmb == 0, (T, E, nmb, world)
    keys = jr.split(kperm, world) if world > 1 else kperm[None]
    out = []
    for r in range(world):
        perm = jr.permutation_indices(keys[r], n).reshape(nmb, n // nmb)
        out.append(global_rows(perm, r, E, world))
    return np.stack(out, 1)


def update_step_sharded(env, kind, params, opt, bs, obs, st, rng, cfg, n_updates, lr_fn, world, forced_actions=None,
                        tie_log=None):
    """``oracle.pqn_ref.update_step`` for one seed with the learn phase of a `world`-rank env-sharded run.  Same
    arguments and results; ``world = 1`` is the unsharded update step."""
    fwd = R.cnn_forward if kind == "cnn" else R.mlp_forward
    lossgrad = R.cnn_loss_and_grads if kind == "cnn" else R.mlp_loss_and_grads
    T, E = cfg["NUM_STEPS"], cfg["NUM_ENVS"]
    eps = R.linear_schedule(cfg["EPS_START"], cfg["EPS_FINISH"], cfg["EPS_DECAY"] * cfg["NUM_UPDATES_DECAY"], n_updates)
    ks = jr.split(rng, 2); rng, _rng = ks[0], ks[1]
    obs, st, rng, tr, infos = R.rollout(env, fwd, params, obs, st, _rng, T, eps, cfg.get("REW_SCALE", 1),
                                        forced_actions, tie_log)
    last_q = fwd(params, tr["next_obs"][-1]).max(-1)
    targets = R.q_lambda_targets(tr["reward"], tr["done"], tr["q_val"], last_q, cfg["GAMMA"], cfg["LAMBDA"])
    ks = jr.split(rng, 2); rng = ks[0]
    losses, qvs = [], []
    flat_obs = tr["obs"].reshape((T * E,) + tr["obs"].shape[2:])
    flat_act = tr["action"].reshape(-1)
    flat_tgt = targets.reshape(-1)
    nmb = cfg["NUM_MINIBATCHES"]
    for _ in range(cfg["NUM_EPOCHS"]):
        ks = jr.split(rng, 2); rng, kperm = ks[0], ks[1]
        mbs = epoch_minibatches(kperm, T, E, nmb, world)
        ks = jr.split(rng, 2); rng = ks[0]
        for i in range(nmb):
            idx = mbs[i].reshape(-1)                                  # the union of the ranks' minibatches
            loss, q_sa, g = lossgrad(params, flat_obs[idx], flat_act[idx], flat_tgt[idx])
            bs = R.bn_batch_stats_update(bs, flat_obs[idx].astype(F32))
            params, opt, _ = R.radam_clip_step(params, g, opt, lr_fn(opt["count"]), cfg["MAX_GRAD_NORM"])
            losses.append(loss); qvs.append(q_sa.mean())
    metrics = {"td_loss": float(np.mean(losses)), "qvals": float(np.mean(qvs))}
    metrics.update({k: float(v.astype(np.float64).mean()) for k, v in infos.items()})
    return params, opt, bs, obs, st, rng, metrics, tr, targets
