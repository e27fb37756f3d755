"""Hyperparameter grids on the host: grid order, seed and key layout, the sweep table, the refusals (raised by
make_train before anything is built) and the per-seed tables the engines upload (a scalar config composes exactly
what it composed before grids existed)."""
import numpy as np
import pytest

from oracle import jax_prng as jr
from purejaxql_b200 import _runner, config_loader, engine, sweep


def _cfg(**kw):
    c = config_loader.compose(["+alg=pqn_cartpole", "NUM_SEEDS=3", "SAVE_PATH=null"])
    c = {**c, **c["alg"]}
    c.update(kw)
    return c


def test_grid_order_is_by_key_then_by_value():
    g = sweep.Grid(_cfg(EPS_DECAY=[0.1, 0.3], LR=[1e-3, 5e-4, 1e-4], GAMMA=[0.99, 0.9]))
    assert [k for k, _ in g.axes] == ["LR", "GAMMA", "EPS_DECAY"]            # SWEEP_KEYS order, not the config's
    assert g.G == 12 and g.total_seeds == 36
    assert g.points[0] == {"LR": 1e-3, "GAMMA": 0.99, "EPS_DECAY": 0.1}
    assert g.points[1] == {"LR": 1e-3, "GAMMA": 0.99, "EPS_DECAY": 0.3}        # the last key varies fastest
    assert g.points[2] == {"LR": 1e-3, "GAMMA": 0.9, "EPS_DECAY": 0.1}
    assert g.points[4] == {"LR": 5e-4, "GAMMA": 0.99, "EPS_DECAY": 0.1}
    assert g.points[11] == {"LR": 1e-4, "GAMMA": 0.9, "EPS_DECAY": 0.3}
    c5 = g.config(5)
    assert c5["LR"] == 5e-4 and c5["GAMMA"] == 0.99 and c5["EPS_DECAY"] == 0.3 and c5["LAMBDA"] == 0.95


def test_seed_layout_keys_and_table():
    c = _cfg(LR=[1e-3, 1e-4], MAX_GRAD_NORM=[10, 1])
    g = sweep.Grid(c)
    n = c["NUM_SEEDS"]
    rngs = jr.split(jr.PRNGKey(c["SEED"]), n)
    tiled = g.tile(rngs)
    assert tiled.shape == (4 * n, 2)
    for p in range(4):
        assert np.array_equal(tiled[p * n:(p + 1) * n], rngs)                 # common random numbers
    t = g.table(0, 4 * n)
    assert t["point"] == [p for p in range(4) for _ in range(n)]
    assert t["seed"] == list(range(n)) * 4
    assert t["LR"] == [1e-3] * 2 * n + [1e-4] * 2 * n
    assert t["MAX_GRAD_NORM"] == ([10] * n + [1] * n) * 2
    assert t["GAMMA"] == [0.99] * 4 * n and t["REW_SCALE"] == [0.1] * 4 * n
    # a seed-sharded rank's slice: seeds [5, 9) are seeds 2 of point 1 .. 2 of point 2
    s = g.table(5, 4)
    assert s["point"] == [1, 2, 2, 2] and s["seed"] == [2, 0, 1, 2]
    with pytest.raises(ValueError, match="tiled key array"):
        g.point_of(10, 4)


def test_scalar_config_is_one_point():
    c = _cfg()
    g = sweep.Grid(c)
    assert g.G == 1 and g.axes == [] and g.total_seeds == 3
    rngs = jr.split(jr.PRNGKey(0), 3)
    assert g.tile(rngs) is rngs
    t = g.table(0, 5)                        # train(rngs) of a scalar config takes any number of seeds
    assert t["point"] == [0] * 5 and t["seed"] == list(range(5)) and t["LR"] == [1e-4] * 5
    assert sweep.Grid({k: v for k, v in c.items() if k != "NUM_SEEDS"}).total_seeds == 1


@pytest.mark.parametrize("module", ["pqn_minatar", "pqn_gymnax", "pqn_rnn_gymnax"])
@pytest.mark.parametrize("bad,match", [
    (dict(LR=[]), "empty list"),
    (dict(NUM_ENVS=[16, 32]), "NUM_ENVS"),
    (dict(HIDDEN_SIZE=[128, 256]), "HIDDEN_SIZE"),
    (dict(NORM_TYPE=["layer_norm", "batch_norm"]), "NORM_TYPE"),
    (dict(EPS_TEST=[0.0, 0.05]), "EPS_TEST"),
    (dict(NUM_SEEDS=16384, LR=[1e-3, 1e-4], GAMMA=[0.9, 0.99]), "65535"),
])
def test_make_train_refuses_before_building(module, bad, match, monkeypatch):
    import importlib
    mod = importlib.import_module(f"purejaxql_b200.{module}")
    built = []
    monkeypatch.setattr(mod.envs, "make", lambda *a, **k: built.append(a))
    c = _cfg(ENV_NAME="Breakout-MinAtar" if module == "pqn_minatar" else "CartPole-v1", MEMORY_WINDOW=4, **bad)
    with pytest.raises(ValueError, match=match):
        mod.make_train(c)
    assert built == [], "refused after the env was built"


def test_grid_seed_limit_counts_every_seed():
    sweep.Grid(_cfg(NUM_SEEDS=16383, LR=[1e-3, 1e-4], GAMMA=[0.9, 0.99], REW_SCALE=1))   # 65,532 seeds: accepted
    with pytest.raises(ValueError, match="65536 seeds"):
        sweep.Grid(_cfg(NUM_SEEDS=32768, LR=[1e-3, 1e-4]))


def _old_inputs(c, NU, nud, per_update):
    """What the engines composed before grids existed (engine.py at the parent of this feature)."""
    eps = np.array([engine.linear_schedule(c["EPS_START"], c["EPS_FINISH"], c["EPS_DECAY"] * nud, n)
                    for n in range(max(NU, 1))], np.float32)
    if c.get("LR_LINEAR_DECAY", False):
        lr_fn = lambda i: engine.linear_schedule(c["LR"], 1e-20, nud * per_update, i)
    else:
        lr_fn = lambda i: engine._f32(c["LR"])
    sched = engine.radam_schedule_table(NU * per_update, lr_fn)
    return eps, sched


@pytest.mark.parametrize("preset,decay", [("pqn_cartpole", True), ("pqn_minatar", True),
                                          ("pqn_rnn_memory_chain", False)])
def test_scalar_config_composes_the_same_engine_inputs(preset, decay):
    c = config_loader.compose([f"+alg={preset}"])
    c = {**c, **c["alg"]}
    assert bool(c["LR_LINEAR_DECAY"]) == decay
    NU, nud, per_update, S = 7, 9, 6, 5
    got = engine.seed_inputs(sweep.Grid(c), 0, S, NU, nud, per_update, decay)
    eps, sched = _old_inputs(c, NU, nud, per_update)
    assert got["eps"].dtype == np.float32 and got["eps"].shape == (NU, S)
    for s in range(S):
        assert np.array_equal(got["eps"][:, s], eps)
    assert got["sched"].shape == sched.shape and np.array_equal(got["sched"], sched)      # one shared table
    for k, key in (("gamma", "GAMMA"), ("lam", "LAMBDA"), ("max_norm", "MAX_GRAD_NORM")):
        assert np.array_equal(got[k], np.full(S, np.float32(float(c[key])))), k
    assert np.array_equal(got["rew_scale"], np.full(S, np.float32(float(c.get("REW_SCALE", 1)))))


def test_grid_inputs_are_each_points_scalar_inputs():
    c = _cfg(LR=[1e-3, 1e-4], EPS_START=[1.0, 0.5], LAMBDA=[0.95, 0.5], REW_SCALE=[0.1, 1.0])
    g = sweep.Grid(c)
    n, NU, nud, per_update = c["NUM_SEEDS"], 4, 4, 8
    got = engine.seed_inputs(g, 0, g.total_seeds, NU, nud, per_update, True)
    assert got["sched"].shape == (g.total_seeds, NU * per_update, 4)
    for p in range(g.G):
        one = engine.seed_inputs(sweep.Grid(g.config(p)), 0, n, NU, nud, per_update, True)
        sl = slice(p * n, (p + 1) * n)
        assert np.array_equal(got["eps"][:, sl], one["eps"]), p
        for s in range(p * n, (p + 1) * n):
            assert np.array_equal(got["sched"][s], one["sched"]), (p, s)
        for k in ("gamma", "lam", "max_norm", "rew_scale"):
            assert np.array_equal(got[k][sl], one[k]), (p, k)
    # a rank's slice holds the rows of the same seeds
    part = engine.seed_inputs(g, 5, 6, NU, nud, per_update, True)
    assert np.array_equal(part["eps"], got["eps"][:, 5:11]) and np.array_equal(part["sched"], got["sched"][5:11])


def test_data_parallel_auto_counts_every_seed_of_a_grid():
    c = _cfg(NUM_SEEDS=1, NUM_ENVS=32, NUM_STEPS=64, NUM_MINIBATCHES=16)
    assert _runner.pick_data_parallel(c, 2) == "envs"
    assert _runner.pick_data_parallel(dict(c, LR=[1e-3, 1e-4]), 2) == "seeds"
    assert _runner.pick_data_parallel(dict(c, LR=[1e-3, 1e-4]), 4) == "envs"
