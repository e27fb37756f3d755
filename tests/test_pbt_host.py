"""Population-based training on the host: the settings and their refusals (raised before an env is built), the grid's
list exemption, resuming a state written before PBT existed, and the NumPy oracle of an event's decisions."""
import importlib

import numpy as np
import pytest
import torch

import pbt_oracle as O
from oracle import jax_prng as jr
from purejaxql_b200 import _runner, pbt, state, sweep
from purejaxql_b200.utils import save_load

MODULES = ["pqn_minatar", "pqn_gymnax", "pqn_rnn_gymnax"]


def _cfg(module="pqn_gymnax", **kw):
    c = dict(ENV_NAME="Breakout-MinAtar" if module == "pqn_minatar" else "CartPole-v1", NUM_ENVS=64, NUM_STEPS=8,
             NUM_MINIBATCHES=4, NUM_EPOCHS=2, EPS_START=1.0, EPS_FINISH=0.05, EPS_DECAY=0.1, LR=5e-4,
             MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65, LR_LINEAR_DECAY=True, TOTAL_TIMESTEPS=5120.0,
             TOTAL_TIMESTEPS_DECAY=5120.0, SEED=0, NUM_SEEDS=4, TEST_DURING_TRAINING=False, WANDB_MODE="disabled",
             MEMORY_WINDOW=4, SAVE_PATH=None, PBT_INTERVAL=2)
    c.update(kw)
    return c


BAD = [
    (dict(PBT_INTERVAL=-1), "PBT_INTERVAL"), (dict(PBT_INTERVAL=1.5), "PBT_INTERVAL"),
    (dict(PBT_INTERVAL=True), "PBT_INTERVAL"),
    (dict(PBT_FRACTION=0.0), "PBT_FRACTION"), (dict(PBT_FRACTION=0.6), "PBT_FRACTION"),
    (dict(PBT_FRACTION="x"), "PBT_FRACTION"),
    (dict(PBT_PERTURB=["LR", "LR"]), "PBT_PERTURB"), (dict(PBT_PERTURB=["EPS_START"]), "PBT_PERTURB"),
    (dict(PBT_PERTURB="LR"), "PBT_PERTURB"),
    (dict(PBT_FACTORS=[0.8]), "PBT_FACTORS"), (dict(PBT_FACTORS=[0.8, -1.0]), "PBT_FACTORS"),
    (dict(PBT_FACTORS=[0.8, 1.25, 2.0]), "PBT_FACTORS"),
    (dict(PBT_FITNESS="eval"), "PBT_FITNESS"), (dict(PBT_SEED=1.5), "PBT_SEED"),
    (dict(NUM_SEEDS=3), "PBT_FRACTION"),                                   # floor(0.25 * 3) = 0 seeds replaced
    (dict(PBT_FITNESS="test"), "PBT_FITNESS=test needs TEST_DURING_TRAINING"),
    (dict(PBT_FITNESS="test", TEST_DURING_TRAINING=True, TEST_INTERVAL=0.3, PBT_INTERVAL=2), "PBT_INTERVAL=2 must"),
    (dict(HYP_TUNE=True), "HYP_TUNE"),
]


@pytest.mark.parametrize("module", MODULES)
@pytest.mark.parametrize("bad,match", BAD, ids=[f"{list(b)[0]}={list(b.values())[0]}" for b, _ in BAD])
def test_bad_settings_are_refused_before_an_env_is_built(module, bad, match, monkeypatch):
    mod = importlib.import_module(f"purejaxql_b200.{module}")
    built = []
    monkeypatch.setattr(mod.envs, "make", lambda *a, **k: built.append(a))
    with pytest.raises(ValueError, match=match):
        mod.make_train(_cfg(module, **bad))
    assert built == [], "refused after the env was built"


def test_settings_accept_and_default():
    assert pbt.settings(_cfg(PBT_INTERVAL=0)) is None
    assert pbt.settings({k: v for k, v in _cfg().items() if k != "PBT_INTERVAL"}) is None
    st = pbt.settings(_cfg(SEED=5))
    assert st == pbt.Settings(2, 0.25, ("LR",), (0.8, 1.25), "train", 5) and st.replaced(4) == 1
    st = pbt.settings(_cfg(PBT_FRACTION=0.5, PBT_PERTURB=["GAMMA", "LR"], PBT_FACTORS=[0.5, 2], PBT_SEED=3,
                           PBT_FITNESS="test", TEST_DURING_TRAINING=True, TEST_INTERVAL=0.2, PBT_INTERVAL=4,
                           LR=[1e-3, 1e-4]))
    assert st.perturb == ("GAMMA", "LR") and st.factors == (0.5, 2.0) and st.seed == 3 and st.replaced(8) == 4
    assert pbt.num_events(st, 9) == 2 and pbt.num_events(st, 8) == 1 and pbt.num_events(st, 4) == 0


def test_seed_sharded_processes_and_hyp_tune_are_refused():
    with pytest.raises(ValueError, match="seed-sharded run of 2 processes"):
        pbt.settings(_cfg(), world=2, env_sharded=False)
    assert pbt.settings(_cfg(), world=2, env_sharded=True) is not None
    with pytest.raises(ValueError, match="HYP_TUNE"):
        _runner.tune({"alg": _cfg()}, None)


def test_single_run_refuses_a_seed_sharded_population_before_make_train(monkeypatch):
    monkeypatch.setattr(_runner, "init_distributed", lambda: (0, 2))
    called = []
    with pytest.raises(ValueError, match="seed-sharded"):
        _runner.single_run({"alg": _cfg(DATA_PARALLEL="seeds")}, lambda c: called.append(c))
    assert not called


def test_grid_exempts_only_the_pbt_lists():
    g = sweep.Grid(_cfg(PBT_PERTURB=["LR", "GAMMA"], PBT_FACTORS=[0.5, 2.0], LR=[1e-3, 1e-4]))
    assert [k for k, _ in g.axes] == ["LR"] and g.G == 2
    for key, v in (("PBT_INTERVAL", [1, 2]), ("PBT_FRACTION", [0.25, 0.5]), ("PBT_FITNESS", ["train", "test"]),
                   ("PBT_SEED", [0, 1]), ("NUM_ENVS", [16, 32])):
        with pytest.raises(ValueError, match=f"{key}="):
            sweep.Grid(_cfg(**{key: v}))


def test_a_state_written_before_pbt_resumes_a_run_without_pbt(tmp_path, monkeypatch):
    from purejaxql_b200 import pqn_gymnax
    built = []

    class Stub:
        def __init__(self, config, *a, **kw):
            built.append(config)
    monkeypatch.setattr(pqn_gymnax, "PQNEngine", Stub)
    base = _cfg(PBT_INTERVAL=0)
    c = dict(base)
    pqn_gymnax.make_train(c)
    keys = state.run_keys(c)
    old = {k: v for k, v in keys.items() if not k.startswith("PBT_")}
    assert set(keys) - set(old) == set(pbt.DEFAULTS)
    p = str(tmp_path / "s.safetensors")
    meta = dict(format=state.FORMAT_VERSION, script="pqn_gymnax", env="CartPole-v1", n_done=2,
                num_updates=int(c["NUM_UPDATES"]), rank=0, world=1, seed_lo=0, num_seeds_local=4,
                data_parallel="seeds", config=old)
    save_load.save_state(p, {"tensors": {"keys": torch.zeros((4, 2), dtype=torch.int32)}, "meta": meta})
    built.clear()
    for run in (dict(base), {k: v for k, v in base.items() if k != "PBT_INTERVAL"}):
        train = pqn_gymnax.make_train(dict(run, RESUME_FROM=p))
        assert train.engine is not None and len(built) == 1
        built.clear()
    with pytest.raises(ValueError, match="RESUME_FROM: PBT_INTERVAL=2"):
        pqn_gymnax.make_train(dict(base, RESUME_FROM=p, PBT_INTERVAL=2))
    assert not built


# --------------------------------------------------------------------------- #
# the oracle
# --------------------------------------------------------------------------- #
def test_oracle_order_ties_and_nan():
    f = np.array([1.0, np.nan, 3.0, 3.0, -0.0, 0.0, np.nan, -np.inf, 2.0])
    assert O.order(f).tolist() == [2, 3, 8, 0, 4, 5, 7, 1, 6]
    cols = np.array([[1.0, 2.0, np.nan], [0.1, 0.2, 0.3], [3.0, 3.0, 3.0]])
    got = O.fitness(cols)
    assert np.isnan(got[0]) and got[1] == ((0.0 + 0.1) + 0.2 + 0.3) / 3 and got[2] == 3.0


@pytest.mark.parametrize("partitionable", [False, True])
def test_oracle_plan_parents_and_factors(partitionable):
    rng = np.random.default_rng(0)
    S, m = 40, 10
    f = np.round(rng.normal(size=S), 1)                    # ties
    f[[3, 17, 31]] = np.nan
    kp = jr.PRNGKey(11)
    kp1, o, parent, children, parents, phi = O.plan(f, m, kp, 3, [0.8, 1.25], partitionable)
    assert sorted(o.tolist()) == list(range(S)) and set(o[-3:].tolist()) == {3, 17, 31}
    assert set(children.tolist()) == set(o[S - m:].tolist())
    assert set(parents.tolist()) <= set(o[:m].tolist())
    kept = np.setdiff1d(np.arange(S), children)
    assert np.array_equal(parent[kept], kept) and np.array_equal(parent[children], parents)
    assert phi.dtype == np.float32 and phi.shape == (m, 3) and set(np.unique(phi).tolist()) <= {np.float32(0.8),
                                                                                                 np.float32(1.25)}
    assert len(np.unique(phi)) == 2
    # the chain: event 2 splits event 1's kp; it never depends on the fitness
    ks = jr.split(kp, 2, partitionable)
    assert np.array_equal(kp1, ks[0])
    again = O.plan(f[::-1].copy(), m, kp, 3, [0.8, 1.25], partitionable)
    assert np.array_equal(again[0], kp1) and np.array_equal(again[5], phi)
    a = jr.randint(jr.split(ks[1], 2, partitionable)[0], (m,), 0, m, partitionable)
    assert np.array_equal(parents, o[:m][a])


def test_oracle_explore_in_fp32():
    S = 6
    t = dict(lr_mult=np.ones(S, np.float32), gamma=np.full(S, 0.99, np.float32), lam=np.full(S, 0.0, np.float32),
             max_norm=np.full(S, 10.0, np.float32), rew_scale=np.full(S, 0.1, np.float32),
             sched_src=np.arange(S, dtype=np.int32))
    t["gamma"][1] = 0.5
    phi = np.array([[1.25, 1.25, 0.8, 0.8, 1.25]], np.float32)
    eps = np.arange(4 * S, dtype=np.float32).reshape(4, S)
    got, e = O.apply(t, [4], [1], phi, ["LR", "GAMMA", "LAMBDA", "MAX_GRAD_NORM", "REW_SCALE"], eps, 2)
    assert got["lr_mult"][4] == np.float32(1.25) and got["sched_src"][4] == 1
    assert got["gamma"][4] == np.float32(1) - np.float32(0.5) * np.float32(1.25)
    assert got["lam"][4] == np.float32(1) - np.float32(0.8)
    assert got["max_norm"][4] == np.float32(8.0) and got["rew_scale"][4] == np.float32(0.1) * np.float32(1.25)
    assert np.array_equal(e[:2], eps[:2]) and np.array_equal(e[2:, 4], eps[2:, 1])
    for k in t:
        assert np.array_equal(np.delete(got[k], 4), np.delete(t[k], 4)), k
    clamp = O.toward_one(np.float32(0.1), np.float32(1.25))     # 1 - 0.9 * 1.25 < 0
    assert clamp == np.float32(0)
