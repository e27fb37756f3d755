"""The evaluation rollouts and recurrent training with eps < 1 against oracle replays.

(B) ``PQNRnnEngine.get_test_metrics`` (pqn_rnn_gymnax.py:442-502: the learning-curve number of the recurrent script)
against ``rnn_get_test_metrics`` below, on the fp64 GRU oracle; and two feed-forward evaluations that
tests/test_gpu_parity_r2.py lacks (pqn_gymnax on Breakout-MinAtar's packed-bit MLP and on MemoryChain-bsuite).
(C) Whole recurrent updates with eps going from 0.6 to 0.1, so that argmax over GRU Q-values picks actions inside the
rollout, eagerly and under CUDA-graph replay.

Greedy actions may flip on a numerical Q tie.  A disagreement between the engine's action and the oracle's own is
tolerated only when the two Q-values differ by less than TIE_GAP; every one is counted and printed, and the oracle then
follows the engine's action so that everything downstream is still compared."""
import numpy as np
import pytest
import torch

import bsuite_oracle as MC
import rnn_norm_oracle as RO
from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_rnn_ref as RR

pytestmark = pytest.mark.gpu
TIE_GAP = 1e-4


def dev():
    return torch.device("cuda:0")


def keys_t(k):
    return torch.from_numpy(np.ascontiguousarray(k, np.uint32).view(np.int32)).to(dev())


def follow(own, engine_action, q, ties, where):
    """The engine's action, after logging every disagreement with the oracle's own as (where, env, own, engine's,
    |Q gap|); a gap of TIE_GAP or more is not a tie and fails."""
    engine_action = np.asarray(engine_action, np.int32)
    for e in np.nonzero(engine_action != own)[0]:
        gap = float(abs(q[e, own[e]] - q[e, engine_action[e]]))
        assert gap < TIE_GAP, f"{where} env {e}: engine action {engine_action[e]} vs oracle {own[e]}, Q gap {gap}"
        ties.append(where + (int(e), int(own[e]), int(engine_action[e]), gap))
    return engine_action


def report(what, ties, n_actions):
    print(f"\n[{what}] {len(ties)} argmax flips on Q ties out of {n_actions} actions", ties[:5])


# --------------------------------------------------------------------------- #
# (B) the recurrent evaluation
# --------------------------------------------------------------------------- #
def rnn_get_test_metrics(env, forward, rng, num_envs, num_steps, eps_test, hidden, engine_actions, ties, tag=()):
    """``get_test_metrics(train_state, rng)`` of pqn_rnn_gymnax.py:442-502 for one seed:

    * ``rng, _rng = split(rng)``; the reset uses ``split(_rng, N)`` and the scan carry starts at the same ``_rng``;
    * every step: ``rng, rng_a, rng_s = split(rng, 3)``; the actions are eps-greedy with ``split(rng_a, N)`` on
      ``network.apply(hs, obs, last_done, last_action, train=False)``, whose GRU zeroes the carry where ``last_done``
      is set; the envs step with ``split(rng_s, N)`` (``vmap_step``);
    * the carry starts from zero hidden state, ``last_done`` False and ``last_action`` 0;
    * result: for every info leaf, ``nanmean(where(returned_episode, x, nan))`` over all steps and envs.

    ``forward(hs, obs, last_done, last_action) -> (new_hs, q)`` is one network step over the N envs.
    ``engine_actions[t]`` are the engine's actions (see ``follow``)."""
    _rng = jr.split(rng, 2)[1]
    obs, state = env.reset(jr.split(_rng, num_envs))
    hs = np.zeros((num_envs, hidden))
    last_done = np.zeros(num_envs, bool)
    last_action = np.zeros(num_envs, np.int32)
    carry = _rng
    infos = {}
    for t in range(num_steps):
        ks = jr.split(carry, 3)
        carry, rng_a, rng_s = ks[0], ks[1], ks[2]
        hs, q = forward(hs, obs, last_done, last_action)
        own = R.eps_greedy(jr.split(rng_a, num_envs), q, eps_test)
        action = follow(own, engine_actions[t], q, ties, tag + (t,))
        obs, state, _, done, info = env.step(jr.split(rng_s, num_envs), state, action)
        last_done, last_action = done, action
        for k, v in info.items():
            infos.setdefault(k, []).append(np.asarray(v))
    mask = np.stack(infos["returned_episode"]).astype(bool)
    out = {}
    for k in R.INFO_KEYS:
        sel = np.stack(infos[k]).astype(np.float64)[mask]
        out[k] = float(sel.mean()) if sel.size else float("nan")
    return out


def rnn_params(spec, S, norm_type="layer_norm", with_stats=False, seed=0):
    """Random parameters (recurrent kernels at half scale), and for the BatchNorm variants norm parameters away from
    (1, 0) and non-trivial running statistics: per seed fp64 trees for the oracle, flat device buffers for the engine."""
    D, A, H, Ls = spec.in_c, spec.num_actions, spec.hidden, spec.layers
    rng = np.random.default_rng(seed)
    ps, sts = [], []
    for s in range(S):
        p = R.random_params(RO.rnn_param_shapes(D, A, H, Ls, norm_type), 90 + 7 * seed + s)
        for g in ("hr", "hz", "hn"):
            p[RR.G + g + "/kernel"] = (p[RR.G + g + "/kernel"] * 0.5).astype(np.float32)
        st = None
        if with_stats:
            for k in p:
                if k.startswith(("BatchNorm_", "LayerNorm_")):
                    p[k] = (p[k] + rng.standard_normal(p[k].shape) * 0.2).astype(np.float32)
            st = RO.rnn_init_stats(D, H, Ls, norm_type)
            for v in st.values():
                v["mean"] = (rng.standard_normal(v["mean"].shape) * 0.3).astype(np.float32)
                v["var"] = rng.uniform(0.5, 2.0, v["var"].shape).astype(np.float32)
        ps.append(p)
        sts.append(st)
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    stats = torch.cat([spec.flatten_stats(st, 1, dev()) for st in sts], 0).contiguous() if with_stats else None
    return ps, sts, flat, stats


def rnn_forward_fp64(p, norm_type, norm_input, stats):
    p64 = {k: v.astype(np.float64) for k, v in p.items()}
    if stats is None:
        def forward(hs, obs, ld, la):
            h, q = RR.rnn_forward(p64, hs, obs[None].astype(np.float64), ld[None], la[None])
            return h, q[0]
        return forward
    st64 = {k: {kk: vv.astype(np.float64) for kk, vv in v.items()} for k, v in stats.items()}

    def forward(hs, obs, ld, la):
        h, q = RO.rnn_forward(p64, hs, obs[None].astype(np.float64), ld[None], la[None], norm_type=norm_type,
                              norm_input=norm_input, batch_stats=st64, train=False)
        return h, q[0]
    return forward


def _leaf(tree, path, s):
    d = tree
    for k in path:
        d = d[k]
    return d[s].cpu().numpy()


def record_actions(eng):
    """Hook on the engine's fused act step: a copy of the [S, N] actions of every step."""
    actions = []
    orig = eng._act_step

    def hook(*a):
        orig(*a)
        actions.append(a[7].clone())            # (S, N, step_keys, q, eps, state, obs_next, action, ...)
    eng._act_step = hook
    return actions


def _rnn_eval_cfg(env_name, **kw):
    c = dict(ENV_NAME=env_name, NUM_ENVS=8, NUM_STEPS=8, MEMORY_WINDOW=2, NUM_MINIBATCHES=2, NUM_EPOCHS=1,
             EPS_START=1.0, EPS_FINISH=0.1, EPS_DECAY=0.5, LR=1e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.95,
             NORM_TYPE="layer_norm", NORM_INPUT=False, HIDDEN_SIZE=128, NUM_LAYERS=2, LR_LINEAR_DECAY=True,
             REW_SCALE=1.0, WANDB_MODE="disabled", TEST_DURING_TRAINING=True, TEST_INTERVAL=0.5)
    c.update(kw)
    c["TOTAL_TIMESTEPS"] = c["TOTAL_TIMESTEPS_DECAY"] = float(4 * c["NUM_STEPS"] * c["NUM_ENVS"])
    return c


def _preset_cfg(preset):
    from purejaxql_b200 import config_loader
    c = config_loader.compose([f"+alg={preset}", "NUM_SEEDS=2", "SAVE_PATH=null"])
    return {**c, **c["alg"]}


RNN_EVAL_CASES = {
    "cartpole_greedy": lambda: (_rnn_eval_cfg("CartPole-v1", TEST_NUM_ENVS=48, TEST_NUM_STEPS=150, EPS_TEST=0.0),
                                lambda: G.make("CartPole-v1", flatten=True)),
    "cartpole_eps0.5": lambda: (_rnn_eval_cfg("CartPole-v1", TEST_NUM_ENVS=48, TEST_NUM_STEPS=150, EPS_TEST=0.5),
                                lambda: G.make("CartPole-v1", flatten=True)),
    # the shipped preset: memory_length 100 (episodes of 101 steps), 1000 steps, 128 envs, HIDDEN_SIZE 256
    "memory_chain_preset": lambda: (_preset_cfg("pqn_rnn_memory_chain"), lambda: MC.make(100, flatten=True)),
    "cartpole_batch_norm_norm_input": lambda: (
        _rnn_eval_cfg("CartPole-v1", TEST_NUM_ENVS=48, TEST_NUM_STEPS=150, EPS_TEST=0.0, NORM_TYPE="batch_norm",
                      NORM_INPUT=True), lambda: G.make("CartPole-v1", flatten=True)),
    # no episode of 101 steps ends within 60: every mean is NaN
    "memory_chain_no_episode_ends": lambda: (
        _rnn_eval_cfg("MemoryChain-bsuite", ENV_KWARGS={"memory_length": 100}, TEST_NUM_ENVS=16, TEST_NUM_STEPS=60,
                      EPS_TEST=0.0), lambda: MC.make(100, flatten=True)),
}


@pytest.mark.parametrize("case", list(RNN_EVAL_CASES))
def test_rnn_eval_matches_oracle(case):
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg, make_env = RNN_EVAL_CASES[case]()
    train = pqn_rnn_gymnax.make_train(cfg)
    eng = train.engine
    N, steps, eps_test = int(cfg["TEST_NUM_ENVS"]), int(cfg["TEST_NUM_STEPS"]), float(cfg["EPS_TEST"])
    if case == "memory_chain_preset":
        assert (N, steps, eng.env_params.memory_length, eng.H) == (128, 1000, 100, 256)
    S = 2
    ps, sts, flat, stats = rnn_params(eng.spec, S, eng.spec.norm_type, eng.with_stats,
                                      seed=list(RNN_EVAL_CASES).index(case))
    if eng.with_stats:
        eng.batch_stats = stats
    actions = record_actions(eng)
    keys = jr.split(jr.PRNGKey(17), S)
    got = eng.get_test_metrics(flat, keys_t(keys))
    assert len(actions) == steps
    engine_actions = torch.stack(actions, 1).cpu().numpy()                     # [S, steps, N]
    ties, ended = [], False
    for s in range(S):
        forward = rnn_forward_fp64(ps[s], eng.spec.norm_type, eng.spec.norm_input, sts[s])
        want = rnn_get_test_metrics(make_env(), forward, keys[s], N, steps, eps_test, eng.H, engine_actions[s], ties,
                                    (case, s))
        for k in R.INFO_KEYS:
            g = float(got[k][s])
            if np.isnan(want[k]):
                assert np.isnan(g), (s, k, g)
            else:
                ended = True
                assert abs(g - want[k]) <= 1e-6 * max(1.0, abs(want[k])), (s, k, g, want[k])
    report(f"recurrent eval {case}", ties, S * steps * N)
    assert ended == (case != "memory_chain_no_episode_ends")


FF_EVAL_CASES = [
    ("Breakout-MinAtar", 0.0, 120, lambda: G.make("Breakout-MinAtar", flatten=True)),
    ("MemoryChain-bsuite", 0.0, 60, lambda: MC.make(5, flatten=True)),
    ("MemoryChain-bsuite", 0.5, 60, lambda: MC.make(5, flatten=True)),
]


@pytest.mark.parametrize("env_name,eps_test,steps,make_env", FF_EVAL_CASES,
                         ids=["breakout_bits_greedy", "memory_chain_greedy", "memory_chain_eps0.5"])
def test_feed_forward_eval_matches_oracle(env_name, eps_test, steps, make_env):
    """pqn_gymnax's get_test_metrics (shared action / env key, reset-key carry) against oracle.pqn_ref's on the MLP:
    Breakout-MinAtar reads packed observation bits (PQN_NET_MLP_BITS), MemoryChain-bsuite's eval reset must carry
    the memory_length word (gymnax's default 5: episodes of 6 steps)."""
    from purejaxql_b200 import pqn_gymnax
    N = 48
    cfg = dict(ENV_NAME=env_name, NUM_ENVS=64, NUM_STEPS=8, NUM_MINIBATCHES=4, NUM_EPOCHS=2, EPS_START=1.0,
               EPS_FINISH=0.05, EPS_DECAY=0.1, LR=5e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65,
               NORM_TYPE="layer_norm", LR_LINEAR_DECAY=True, WANDB_MODE="disabled", TEST_DURING_TRAINING=True,
               TEST_INTERVAL=0.5, TEST_NUM_ENVS=N, EPS_TEST=eps_test, TEST_NUM_STEPS=steps, HIDDEN_SIZE=128,
               NUM_LAYERS=2)
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(4 * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_gymnax.make_train(cfg)
    eng = train.engine
    S = 2
    keys = jr.split(jr.PRNGKey(11), S)
    flat = eng.spec.init(keys_t(jr.split(jr.PRNGKey(12), S)), dev())
    got = eng.get_test_metrics(flat, keys_t(keys))
    tree = eng.spec.unflatten(flat)
    ended = False
    for s in range(S):
        params = {"/".join(p): _leaf(tree, p, s).astype(np.float32) for p, *_ in eng.spec.entries}
        want = R.get_test_metrics(make_env(), R.mlp_forward, params, keys[s], N, steps, eps_test)
        for k in R.INFO_KEYS:
            g = float(got[k][s])
            if np.isnan(want[k]):
                assert np.isnan(g), (s, k, g)
            else:
                ended = True
                assert abs(g - want[k]) <= 1e-6 * max(1.0, abs(want[k])), (s, k, g, want[k])
    assert ended, "no episode ended in the evaluation rollout: the means were never compared"


# --------------------------------------------------------------------------- #
# (C) recurrent training with eps < 1
# --------------------------------------------------------------------------- #
def _oracle_step(env, p, hs, obs, ld, la, st, rng, eps, rew_scale, E, engine_action=None, ties=None, where=()):
    """_step_env / _random_step (pqn_rnn_gymnax.py:192-236, :514-529) for one seed."""
    ks = jr.split(rng, 3)
    rng, rng_a, rng_s = ks[0], ks[1], ks[2]
    new_hs, q = RR.rnn_forward(p, hs, obs[None], ld[None], la[None])
    act = R.eps_greedy(jr.split(rng_a, E), q[0], eps)
    if engine_action is not None:
        act = follow(act, engine_action, q[0], ties, where)
    new_obs, st, reward, done, info = env.step(jr.split(rng_s, E), st, act)
    tr = dict(last_hs=hs, obs=obs, action=act, reward=(np.float32(rew_scale) * reward).astype(np.float32), done=done,
              last_done=ld, last_action=la)
    return (new_hs.astype(np.float32), new_obs, done, act, st, rng), tr, info


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda_graph"])
@pytest.mark.parametrize("env_name", ["CartPole-v1", "MemoryChain-bsuite"])
def test_rnn_train_with_eps_schedule_matches_oracle(env_name, graph):
    """Three whole updates of pqn_rnn_gymnax.make_train/train with eps 0.6 -> 0.1 against an oracle replay (memory
    warm-up at eps 1, key chain, env-axis minibatches, in-loss Q(lambda), RAdam): per-update td_loss, qvals and
    episode metrics, the final parameters and the final key of every seed."""
    from purejaxql_b200 import pqn_rnn_gymnax
    nupd = 3
    cfg = dict(ENV_NAME=env_name, NUM_ENVS=16, NUM_STEPS=12, MEMORY_WINDOW=3, NUM_MINIBATCHES=4, NUM_EPOCHS=2,
               EPS_START=0.6, EPS_FINISH=0.1, EPS_DECAY=1.0, LR=1e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.95,
               NORM_TYPE="layer_norm", NORM_INPUT=False, HIDDEN_SIZE=128, NUM_LAYERS=2, LR_LINEAR_DECAY=True,
               REW_SCALE=0.1, WANDB_MODE="disabled", TEST_DURING_TRAINING=False, CUDA_GRAPH=graph)
    if env_name == "MemoryChain-bsuite":
        cfg.update(ENV_KWARGS={"memory_length": 4}, REW_SCALE=1.0)            # episodes of 5 steps
        make_env = lambda: MC.make(4, flatten=True)
    else:
        make_env = lambda: G.make("CartPole-v1", flatten=True)
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_rnn_gymnax.make_train(cfg)
    eng = train.engine
    T, E, W, nmb, H = cfg["NUM_STEPS"], cfg["NUM_ENVS"], cfg["MEMORY_WINDOW"], cfg["NUM_MINIBATCHES"], cfg["HIDDEN_SIZE"]
    Bm = E // nmb
    S = 2
    rngs = jr.split(jr.PRNGKey(41), S)
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    snaps = []                                   # the update's own actions: memory slots W .. W+T-1
    eng.on_update_end = lambda n, b: snaps.append(b["mem"].action[:, W:W + T].clone())
    out = train(rngs)
    assert eng.graph_captured == graph and len(snaps) == nupd
    m = out["metrics"]
    ts = out["runner_state"][0]
    tree0 = eng.spec.unflatten(cap["flat"])
    ties = []
    for s in range(S):
        params = {"/".join(p): _leaf(tree0, p, s).astype(np.float32) for p, *_ in eng.spec.entries}
        env = make_env()
        rng = jr.split(rngs[s], 2)[0]                                      # :255 (init key = rng)
        rng = jr.split(rng, 2)[0]                                          # :505 (test key unused)
        k = jr.split(rng, 2); rng, kR = k[0], k[1]                         # :508
        obs, st = env.reset(jr.split(kR, E))
        hs = np.zeros((E, H), np.float32); ld = np.zeros(E, bool); la = np.zeros(E, np.int32)
        carry = jr.split(rng, 2)[1]                                        # :531
        mem = []
        for _ in range(W + T):                                             # warm-up: eps = 1
            (hs, obs, ld, la, st, carry), tr, _ = _oracle_step(env, params, hs, obs, ld, la, st, carry, 1.0,
                                                               cfg["REW_SCALE"], E)
            mem.append(tr)
        rng = jr.split(carry, 2)[1]                                        # :532, :541
        opt = R.opt_init(params)
        total = cfg["NUM_UPDATES_DECAY"] * nmb * cfg["NUM_EPOCHS"]
        lr_fn = lambda i: R.linear_schedule(cfg["LR"], 1e-20, total, i)
        for u in range(nupd):
            eps = R.linear_schedule(cfg["EPS_START"], cfg["EPS_FINISH"], cfg["EPS_DECAY"] * cfg["NUM_UPDATES_DECAY"], u)
            assert 0.1 <= eps <= 0.6
            engine_actions = snaps[u][s].cpu().numpy()                     # [T, E]
            carry = jr.split(rng, 2)[1]                                    # :222
            new, infos = [], []
            for t in range(T):
                (hs, obs, ld, la, st, carry), tr, info = _oracle_step(
                    env, params, hs, obs, ld, la, st, carry, eps, cfg["REW_SCALE"], E, engine_actions[t], ties,
                    (env_name, s, u, t))
                new.append(tr)
                infos.append(info)
            rng = carry
            mem = mem[T:] + new                                            # :239-243
            stack = {kk: np.stack([x[kk] for x in mem]) for kk in mem[0]}
            r = jr.split(rng, 2)[0]                                        # :381
            losses, qvals = [], []
            for _ in range(cfg["NUM_EPOCHS"]):
                k = jr.split(r, 2); r, kperm = k[0], k[1]                  # :368
                perm = jr.permutation_indices(kperm, E)
                r = jr.split(r, 2)[0]                                      # :375
                for mb in range(nmb):
                    idx = perm[mb * Bm:(mb + 1) * Bm]
                    loss, chosen, g = RR.rnn_loss_and_grads(
                        params, stack["last_hs"][0][idx], stack["obs"][:, idx], stack["last_done"][:, idx],
                        stack["last_action"][:, idx], stack["action"][:, idx], stack["reward"][:, idx],
                        stack["done"][:, idx], cfg["GAMMA"], cfg["LAMBDA"])
                    params, opt, _ = R.radam_clip_step(params, g, opt, lr_fn(opt["count"]), cfg["MAX_GRAD_NORM"])
                    losses.append(loss)
                    qvals.append(chosen.mean())
            rng = r
            where = (env_name, graph, s, u)
            for name, want in (("td_loss", np.mean(losses)), ("qvals", np.mean(qvals))):
                got = float(m[name][s, u])
                assert abs(got - want) < 2e-3 * max(1.0, abs(want)), where + (name, got, want)
            for kk in R.INFO_KEYS:
                want = float(np.mean([x[kk].astype(np.float64).mean() for x in infos]))
                got = float(m[kk][s, u])
                assert abs(got - want) <= 1e-5 * max(1.0, abs(want)), where + (kk, got, want)
        for p, *_ in eng.spec.entries:
            d = np.abs(_leaf(ts.params, p, s) - params["/".join(p)])
            assert np.quantile(d, 0.99) < 1e-4 and d.max() < 1e-3, (p, d.max())
        assert np.array_equal(out["runner_state"][4][s].cpu().numpy().view(np.uint32), rng)
    assert (m["returned_episode"] > 0).all(), "an update without a finished episode"
    report(f"recurrent train eps<1 {env_name} {'graph' if graph else 'eager'}", ties, S * nupd * T * E)
