"""The env-sharded oracle (tests/env_shard_oracle.py) on the CPU: at one rank it is the unsharded update step bit for
bit, and at 2 and 3 ranks the ranks' minibatches of an epoch tile the rollout's rows, each rank drawing only from its
own env shard."""
import numpy as np
import pytest

import env_shard_oracle as SO
from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R


def _cfg(env, **kw):
    c = dict(ENV_NAME=env, NUM_ENVS=16, NUM_STEPS=4, NUM_MINIBATCHES=2, NUM_EPOCHS=2, EPS_START=0.5, EPS_FINISH=0.1,
             EPS_DECAY=1.0, NUM_UPDATES_DECAY=2, LR=5e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65, REW_SCALE=1.0)
    c.update(kw)
    return c


@pytest.mark.parametrize("env_name,kind,flatten,shapes", [
    ("Breakout-MinAtar", "cnn", False, R.cnn_param_shapes(4, 3)),
    ("CartPole-v1", "mlp", True, R.mlp_param_shapes(4, 2, 64, 2)),
])
def test_one_rank_is_the_unsharded_update_step(env_name, kind, flatten, shapes):
    cfg = _cfg(env_name)
    T, E = cfg["NUM_STEPS"], cfg["NUM_ENVS"]
    total = cfg["NUM_UPDATES_DECAY"] * cfg["NUM_MINIBATCHES"] * cfg["NUM_EPOCHS"]
    lr_fn = lambda i: R.linear_schedule(cfg["LR"], 1e-20, total, i)
    p0 = R.random_params(shapes, 3)
    F = shapes["BatchNorm_0/scale"][0]
    carry = []
    for step in (R.update_step, lambda *a: SO.update_step_sharded(*a, world=1)):
        env = G.make(env_name, flatten=flatten)
        obs, st = env.reset(jr.split(jr.PRNGKey(5), E))
        params, opt = dict(p0), R.opt_init(p0)
        bs = {"mean": np.zeros(F, np.float32), "var": np.ones(F, np.float32)}
        rng = jr.PRNGKey(6)
        ms = []
        for u in range(2):
            params, opt, bs, obs, st, rng, m, tr, tg = step(env, kind, params, opt, bs, obs, st, rng, dict(cfg), u, lr_fn)
            ms.append(m)
        carry.append((params, opt, bs, obs, st, rng, ms, tr, tg))
    (p1, o1, b1, obs1, st1, r1, m1, tr1, tg1), (p2, o2, b2, obs2, st2, r2, m2, tr2, tg2) = carry
    assert o1["count"] == o2["count"] == 2 * cfg["NUM_MINIBATCHES"] * cfg["NUM_EPOCHS"]
    for k in p1:
        assert np.array_equal(p1[k], p2[k]), k
        assert np.array_equal(o1["mu"][k], o2["mu"][k]) and np.array_equal(o1["nu"][k], o2["nu"][k]), k
    for k in b1:
        assert np.array_equal(b1[k], b2[k]), k
    assert np.array_equal(r1, r2) and np.array_equal(obs1, obs2) and np.array_equal(tg1, tg2)
    for k in st1:
        assert np.array_equal(st1[k], st2[k]), k
    assert m1 == m2
    assert tr1["action"].shape == (T, E)


@pytest.mark.parametrize("partitionable", [False, True], ids=["original", "partitionable"])
@pytest.mark.parametrize("T,E,nmb,world", [(8, 390, 4, 2), (8, 390, 4, 3), (16, 64, 4, 2), (2, 6, 1, 3)])
def test_sharded_minibatches_cover_every_row_once(T, E, nmb, world, partitionable, monkeypatch):
    monkeypatch.setattr(jr, "DEFAULT_PARTITIONABLE", partitionable)
    E_l = E // world
    mb = T * E_l // nmb
    for epoch in range(2):
        kperm = jr.split(jr.PRNGKey(40 + epoch), 2)[1]
        mbs = SO.epoch_minibatches(kperm, T, E, nmb, world)
        assert mbs.shape == (nmb, world, mb)
        assert np.array_equal(np.sort(mbs.reshape(-1)), np.arange(T * E)), (T, E, world, epoch)
        for r in range(world):
            env = mbs[:, r] % E
            assert ((env >= r * E_l) & (env < (r + 1) * E_l)).all(), r          # only rank r's own envs
            # the local rows are rank r's permutation of split(kperm, world)[r]
            local = (mbs[:, r] // E) * E_l + env - r * E_l
            want = jr.permutation_indices(jr.split(kperm, world)[r], T * E_l).reshape(nmb, mb)
            assert np.array_equal(local, want), r


def test_global_rows_follow_the_rank_buffers():
    """Local row j of rank r is obs_buf[s][j // E_l][j % E_l] of its shard: step j // E_l of env r * E_l + j % E_l."""
    E, world = 12, 3
    E_l = E // world
    rows = np.arange(5 * E).reshape(5, E)                          # [T, E] global row numbers
    for r in range(world):
        shard = rows[:, r * E_l:(r + 1) * E_l].reshape(-1)         # the rank's [T, E_l] buffer, row-major
        assert np.array_equal(SO.global_rows(np.arange(5 * E_l), r, E, world), shard), r
