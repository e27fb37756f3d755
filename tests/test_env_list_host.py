"""A list-valued ENV_NAME on the host: the grid accepts it, every refusal is raised before an env is built, and the
list path (env_list.make_train, train_all, single_run) hands every env its own config copy, stream and files, exactly
where and as the standalone run of that env writes them.  The engines are stand-ins: no device is needed."""
import contextlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import jax_prng as oracle_jr
from purejaxql_b200 import _runner, config_loader, engine, env_list, pqn_gymnax, pqn_minatar, pqn_rnn_gymnax, sweep

SCRIPTS = {"pqn_minatar": (pqn_minatar, ["Breakout-MinAtar", "Freeway-MinAtar"]),
           "pqn_gymnax": (pqn_gymnax, ["CartPole-v1", "Catch-bsuite", "Breakout-MinAtar"]),
           "pqn_rnn_gymnax": (pqn_rnn_gymnax, ["CartPole-v1", "MemoryChain-bsuite"])}


def _cfg(**kw):
    c = config_loader.compose(["+alg=pqn_cartpole", "NUM_SEEDS=3", "SAVE_PATH=null"])
    c = {**c, **c["alg"]}
    c.update(kw)
    return c


def test_grid_accepts_an_env_list():
    names = ["CartPole-v1", "Acrobot-v1", "Catch-bsuite"]
    g = sweep.Grid(_cfg(ENV_NAME=names))
    assert g.G == 1 and g.axes == [] and g.total_seeds == 3
    assert sweep.env_names(_cfg(ENV_NAME=names)) == names
    assert sweep.env_names(_cfg(ENV_NAME="CartPole-v1")) is None
    g = sweep.Grid(_cfg(ENV_NAME=names, LR=[1e-3, 1e-4]))               # composes with a hyperparameter grid
    assert g.G == 2 and [k for k, _ in g.axes] == ["LR"]


@pytest.mark.parametrize("module", list(SCRIPTS))
@pytest.mark.parametrize("bad,exc,match", [
    (dict(ENV_NAME=[]), ValueError, "empty list"),
    (dict(ENV_NAME=["CartPole-v1", "Catch-bsuite", "CartPole-v1"]), ValueError, "CartPole-v1 appears more than once"),
    (dict(ENV_NAME=["Pendulum-v1", "CartPole-v1"]), KeyError, "unknown env 'Pendulum-v1'"),
    (dict(DATA_PARALLEL="envs"), ValueError, "shards seeds over the GPUs"),
    (dict(STATE_SAVE_INTERVAL=2, SAVE_PATH="/nonexistent"), ValueError, "STATE_SAVE_INTERVAL"),
    (dict(RESUME_FROM="/nonexistent/state.safetensors"), ValueError, "RESUME_FROM"),
    (dict(HYP_TUNE=True), ValueError, "HYP_TUNE"),
    (dict(NUM_ENVS=[16, 32]), ValueError, "NUM_ENVS"),                  # other lists stay refused
])
def test_list_refusals_come_before_any_env_is_built(module, bad, exc, match, monkeypatch):
    mod, names = SCRIPTS[module]
    built = []
    monkeypatch.setattr(mod.envs, "make", lambda *a, **k: built.append(a))
    c = _cfg(**{"ENV_NAME": names, "MEMORY_WINDOW": 4, **bad})
    with pytest.raises(exc, match=match):
        mod.make_train(c)
    assert built == [], "refused after an env was built"


@pytest.mark.parametrize("module,names,exc,standalone", [
    ("pqn_rnn_gymnax", ["CartPole-v1", "Seaquest-MinAtar"], NotImplementedError, "Seaquest-MinAtar"),
    ("pqn_rnn_gymnax", ["Breakout-MinAtar", "CartPole-v1"], NotImplementedError, "Breakout-MinAtar"),
    ("pqn_minatar", ["Breakout-MinAtar", "CartPole-v1"], ValueError, None),
])
def test_script_refusals_are_the_standalone_ones(module, names, exc, standalone, monkeypatch):
    """The recurrent script's MinAtar refusal is the standalone run's NotImplementedError; pqn_minatar refuses a
    non-MinAtar env with the CNN's own message."""
    mod = SCRIPTS[module][0]
    cfg = _cfg(MEMORY_WINDOW=4)
    if standalone is not None:
        with pytest.raises(exc) as one:
            mod.make_train(dict(cfg, ENV_NAME=standalone))
    built = []
    monkeypatch.setattr(mod.envs, "make", lambda *a, **k: built.append(a))
    with pytest.raises(exc) as lst:
        mod.make_train(dict(cfg, ENV_NAME=names))
    assert built == []
    assert str(lst.value) == (str(one.value) if standalone is not None else engine.CNN_NEEDS_MINATAR)


@pytest.mark.parametrize("module", ["pqn_minatar", "pqn_gymnax"])
def test_auto_env_sharding_is_refused(module, monkeypatch):
    """DATA_PARALLEL=auto with fewer seeds than GPUs would shard envs: refused in make_train and in single_run."""
    mod, names = SCRIPTS[module]
    built = []
    monkeypatch.setattr(mod.envs, "make", lambda *a, **k: built.append(a))
    monkeypatch.setattr(env_list.state, "dist_placement", lambda: (0, 2))
    with pytest.raises(ValueError, match="DATA_PARALLEL=auto picks env sharding"):
        mod.make_train(_cfg(ENV_NAME=names, NUM_SEEDS=1))
    monkeypatch.setattr(_runner, "init_distributed", lambda: (0, 2))
    c = config_loader.compose(["+alg=pqn_cartpole", "NUM_SEEDS=1", "SAVE_PATH=null"])
    c["alg"]["ENV_NAME"] = names
    with pytest.raises(ValueError, match="DATA_PARALLEL=auto picks env sharding"):
        mod.single_run(c)
    assert built == []
    env_list.refuse(_cfg(ENV_NAME=names, NUM_SEEDS=2), 2)                 # seed sharding: accepted
    env_list.refuse(_cfg(ENV_NAME=names, NUM_SEEDS=1), 2, env_sharding=False)   # the recurrent script shards seeds


def test_hyp_tune_with_a_list_is_refused_before_wandb():
    c = config_loader.compose(["+alg=pqn_cartpole", "HYP_TUNE=True"])
    c["alg"]["ENV_NAME"] = ["CartPole-v1", "Acrobot-v1"]
    with pytest.raises(ValueError, match="HYP_TUNE"):
        _runner.main(pqn_gymnax.make_train, ["+alg=pqn_cartpole", "HYP_TUNE=True", "alg.ENV_NAME=[CartPole-v1,Acrobot-v1]"])
    with pytest.raises(ValueError, match="HYP_TUNE"):
        _runner.tune(c, pqn_gymnax.make_train)


# --------------------------------------------------------------------------- #
# the list path with stand-in engines
# --------------------------------------------------------------------------- #
class _Stream:
    def __init__(self):
        self.waited = 0

    def wait_stream(self, other):
        self.waited += 1


class _FakeEngine:
    """Records its config, the stream it was built and stepped under, and returns one parameter leaf per seed."""
    log = []

    def __init__(self, config, *a, env_params=None, **k):
        self.cfg, self.env_params, self.seed_lo = config, env_params, 0
        self.built_on = _CUR[0]

    def train_steps(self, rngs):
        S = rngs.shape[0]
        for n in range(3):
            _FakeEngine.log.append((self.cfg["ENV_NAME"], n, _CUR[0]))
            yield n
        w = torch.arange(S * 2, dtype=torch.float32).reshape(S, 2) + len(self.cfg["ENV_NAME"])
        return {"runner_state": (SimpleNamespace(params={"Dense_0": {"kernel": w + self.seed_lo}}),),
                "env": self.cfg["ENV_NAME"]}

    train = engine.EngineBase.train


_CUR = [None]


@contextlib.contextmanager
def _stream(s):
    prev, _CUR[0] = _CUR[0], s
    try:
        yield
    finally:
        _CUR[0] = prev


@pytest.fixture
def fake_device(monkeypatch):
    _FakeEngine.log = []
    monkeypatch.setattr(pqn_gymnax, "PQNEngine", _FakeEngine)
    monkeypatch.setattr(pqn_minatar, "PQNEngine", _FakeEngine)
    monkeypatch.setattr(pqn_rnn_gymnax, "PQNRnnEngine", _FakeEngine)
    monkeypatch.setattr(torch.cuda, "Stream", _Stream)
    monkeypatch.setattr(torch.cuda, "stream", _stream)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: _CUR[0])
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(_runner, "jr", SimpleNamespace(
        PRNGKey=oracle_jr.PRNGKey,
        split=lambda k, n, mode=0: torch.from_numpy(oracle_jr.split(k, n, bool(mode)).view(np.int32).copy())))


def test_make_train_gives_every_env_its_config_and_stream(fake_device):
    names = ["CartPole-v1", "MemoryChain-bsuite", "MetaMaze-misc"]
    c = _cfg(ENV_NAME=names, MEMORY_WINDOW=4, ENV_KWARGS={"memory_length": 7}, LR=[1e-3, 1e-4])
    caller_before = dict(c)
    train = pqn_rnn_gymnax.make_train(c)
    assert list(train.engines) == names
    # the caller's config gets the update counts; each engine's copy holds its env and its TEST_NUM_STEPS
    assert c["NUM_UPDATES"] == 5e5 // 64 // 32 and "NUM_UPDATES_DECAY" in c
    assert c["ENV_NAME"] == names and ("TEST_NUM_STEPS" in c) == ("TEST_NUM_STEPS" in caller_before)
    for name, eng in train.engines.items():
        want = dict(caller_before, ENV_NAME=name)
        pqn_rnn_gymnax.prepare_config(want, pqn_rnn_gymnax.envs.make(name)[1].max_steps_in_episode, True)
        assert eng.cfg == want and eng.cfg is not c, name
        assert eng.log_prefix == f"{name}/"
    assert train.engines["MemoryChain-bsuite"].env_params.memory_length == 7      # ENV_KWARGS: its entry only
    for name in ("CartPole-v1", "MetaMaze-misc"):
        assert train.engines[name].env_params == pqn_rnn_gymnax.envs.make(name)[1], name
    built = [eng.built_on for eng in train.engines.values()]
    assert all(s is not None for s in built) and len(set(map(id, built))) == len(names)
    outs = train(torch.zeros((6, 2), dtype=torch.int32))
    assert list(outs) == names and [o["env"] for o in outs.values()] == names
    # lockstep: update n of every env before update n + 1 of any, each stepped on the stream it was built on
    assert [(e, n) for e, n, _ in _FakeEngine.log] == [(e, n) for n in range(3) for e in names]
    for e, _, s in _FakeEngine.log:
        assert s is train.engines[e].built_on
    assert all(s.waited == 1 for s in built)                            # each waited for the caller's stream


@pytest.mark.parametrize("module,preset", [("pqn_gymnax", "pqn_cartpole"), ("pqn_rnn_gymnax", "pqn_rnn_cartpole"),
                                           ("pqn_minatar", "pqn_minatar")])
@pytest.mark.parametrize("grid", [False, True], ids=["one_point", "lr_grid"])
def test_single_run_writes_what_the_standalone_runs_write(module, preset, grid, fake_device, tmp_path):
    mod, names = SCRIPTS[module]
    extra = ["alg.LR=[0.001,0.0001]"] if grid else []

    def run(env):
        c = config_loader.compose([f"+alg={preset}", "NUM_SEEDS=2", f"SAVE_PATH={tmp_path / 'models'}", *extra])
        c["alg"]["ENV_NAME"] = env
        c["alg"]["ENV_KWARGS"] = {"memory_length": 6}
        return mod.single_run(c)

    outs = run(names)
    assert list(outs) == names
    (tmp_path / "models").rename(tmp_path / "list")
    for name in names:
        assert run(name)["env"] == name
    (tmp_path / "models").rename(tmp_path / "one")
    files = sorted(p.relative_to(tmp_path / "list") for p in (tmp_path / "list").rglob("*") if p.is_file())
    want = sorted(p.relative_to(tmp_path / "one") for p in (tmp_path / "one").rglob("*") if p.is_file())
    assert files == want and len(files) == len(names) * (1 + grid + 2 * (1 + grid))
    for f in files:
        a, b = (tmp_path / "list" / f).read_bytes(), (tmp_path / "one" / f).read_bytes()
        assert a == b, f
