"""Round-2 parity tests (VERDICT r1 "Next round" item 1): the evaluation rollout against its oracle, whole-engine
parity with eps < 1 (greedy branch + eps schedule through train()), and the BASELINE.json configurations at their
real geometry (configs[2]: 4 MinAtar games x NUM_ENVS=1024 x 16 seeds; configs[3]: Acrobot-v1, NUM_ENVS=65536).

Everything is "bit-exact / within tolerance AGAINST THE ORACLE" (oracle/): parity with a live gymnax is unpinned,
see tests/golden/README.md and DESIGN.md section 5."""
import numpy as np
import pytest
import torch

from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def tkeys(k):
    return torch.from_numpy(np.ascontiguousarray(k).view(np.int32)).to(dev())


def _cfg(env, **kw):
    c = dict(ENV_NAME=env, TOTAL_TIMESTEPS=0, TOTAL_TIMESTEPS_DECAY=0, NUM_ENVS=64, NUM_STEPS=8, NUM_MINIBATCHES=4,
             NUM_EPOCHS=2, EPS_START=1.0, EPS_FINISH=0.05, EPS_DECAY=0.1, LR=5e-4, MAX_GRAD_NORM=10, GAMMA=0.99,
             LAMBDA=0.65, NORM_TYPE="layer_norm", LR_LINEAR_DECAY=True, WANDB_MODE="disabled",
             TEST_DURING_TRAINING=False)
    c.update(kw)
    return c


def _seed_params(eng, tree, s):
    def leaf(path):
        d = tree
        for k in path:
            d = d[k]
        return d[s].cpu().numpy().astype(np.float32)
    return {"/".join(p): leaf(p) for p, *_ in eng.spec.entries}


# --------------------------------------------------------------------------- #
# (a) get_test_metrics  (pqn_minatar.py:371-413)
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("env_name,kind,module,flatten,eps_test,steps", [
    ("Breakout-MinAtar", "cnn", "pqn_minatar", False, 0.0, 120),
    ("Breakout-MinAtar", "cnn", "pqn_minatar", False, 0.3, 120),
    ("CartPole-v1", "mlp", "pqn_gymnax", True, 0.0, 80),
    ("CartPole-v1", "mlp", "pqn_gymnax", True, 0.5, 80),
])
def test_eval_rollout_matches_oracle(env_name, kind, module, flatten, eps_test, steps):
    """engine.get_test_metrics against oracle get_test_metrics on the same parameters and key: all five info
    means over the steps where an episode ended, incl. the shared action/env key and the reset-key scan carry."""
    import importlib
    mod = importlib.import_module(f"purejaxql_b200.{module}")
    N = 48
    cfg = _cfg(env_name, TEST_DURING_TRAINING=True, TEST_INTERVAL=0.5, TEST_NUM_ENVS=N, EPS_TEST=eps_test,
               TEST_NUM_STEPS=steps, HIDDEN_SIZE=128, NUM_LAYERS=2)
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(4 * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = mod.make_train(cfg)
    eng = train.engine
    steps = int(cfg["TEST_NUM_STEPS"])            # pqn_minatar overrides it with max_steps_in_episode (:105)
    S = 2
    from purejaxql_b200 import jaxrandom
    keys = jr.split(jr.PRNGKey(11), S)
    flat = eng.spec.init(tkeys(jr.split(jr.PRNGKey(12), S)), dev())
    got = eng.get_test_metrics(flat, tkeys(keys))
    tree = eng.spec.unflatten(flat)
    fwd = R.cnn_forward if kind == "cnn" else R.mlp_forward
    saw_episode = False
    for s in range(S):
        env = G.make(env_name, flatten=flatten)
        want = R.get_test_metrics(env, fwd, _seed_params(eng, tree, s), keys[s], N, steps, eps_test)
        for k in R.INFO_KEYS:
            g = float(got[k][s])
            if np.isnan(want[k]):
                assert np.isnan(g), (k, g)
            else:
                saw_episode = True
                assert abs(g - want[k]) <= 1e-6 * max(1.0, abs(want[k])), (s, k, g, want[k])
    assert saw_episode, "no episode ended in the evaluation rollout: the means were never compared"


def test_eval_rollout_is_nan_when_no_episode_ends():
    from purejaxql_b200 import pqn_minatar
    cfg = _cfg("Breakout-MinAtar", TEST_DURING_TRAINING=True, TEST_INTERVAL=0.5, TEST_NUM_ENVS=4, EPS_TEST=0.0)
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(4 * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_minatar.make_train(cfg)
    eng = train.engine
    eng.cfg["TEST_NUM_STEPS"] = 2                  # Breakout cannot terminate in 2 steps
    flat = eng.spec.init(tkeys(jr.split(jr.PRNGKey(1), 1)), dev())
    got = eng.get_test_metrics(flat, tkeys(jr.split(jr.PRNGKey(2), 1)))
    assert all(torch.isnan(got[k]).all() for k in R.INFO_KEYS)


# --------------------------------------------------------------------------- #
# (b) whole-engine parity with eps < 1: actions step by step, Q ties reported
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("env_name,kind,module,flatten,extra", [
    ("Breakout-MinAtar", "cnn", "pqn_minatar", False, {}),
    ("CartPole-v1", "mlp", "pqn_gymnax", True, dict(HIDDEN_SIZE=128, NUM_LAYERS=2, REW_SCALE=0.1, NUM_ENVS=32,
                                                    NUM_STEPS=16)),
])
def test_train_with_eps_schedule_matches_oracle(env_name, kind, module, flatten, extra):
    """EPS 0.6 -> 0.1 over the run: the greedy branch (argmax over CUDA Q-values) and the eps table feed integer env
    state through train().  The oracle computes its own eps-greedy action at every step; a disagreement is only
    tolerated on a numerical Q tie (|Q[a] - Q[a']| < 1e-4) and is REPORTED; the oracle then follows the engine's
    action so that everything downstream (reward, done, next obs, targets, parameters) is still compared."""
    import importlib
    mod = importlib.import_module(f"purejaxql_b200.{module}")
    nupd = 3
    cfg = _cfg(env_name, EPS_START=0.6, EPS_FINISH=0.1, EPS_DECAY=1.0, CUDA_GRAPH=False, **extra)
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = mod.make_train(cfg)
    eng = train.engine
    S = 2
    rngs = jr.split(jr.PRNGKey(3), S)
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    snaps = []
    eng.on_update_end = lambda n, b: snaps.append({k: b[k].clone() for k in ("action", "reward", "done", "targets")})
    out = train(rngs)
    ts = out["runner_state"][0]
    tree0 = eng.spec.unflatten(cap["flat"])
    T, E = cfg["NUM_STEPS"], cfg["NUM_ENVS"]
    ties = []
    for s in range(S):
        params = _seed_params(eng, tree0, s)
        K1 = jr.split(rngs[s], 2)[0]
        K2 = jr.split(K1, 2)[0]
        k = jr.split(K2, 2); K3, kR = k[0], k[1]
        env = G.make(env_name, flatten=flatten)
        obs, st = env.reset(jr.split(kR, E))
        rng = jr.split(K3, 2)[1]
        opt = R.opt_init(params)
        F = eng.spec.in_c
        bs = {"mean": np.zeros(F, np.float32), "var": np.ones(F, np.float32)}
        total = cfg["NUM_UPDATES_DECAY"] * cfg["NUM_MINIBATCHES"] * cfg["NUM_EPOCHS"]
        lr_fn = lambda i: R.linear_schedule(cfg["LR"], 1e-20, total, i)
        for u in range(nupd):
            forced = snaps[u]["action"][s].cpu().numpy()                       # [T,E]
            log = []
            params, opt, bs, obs, st, rng, m, tr, tg = R.update_step(env, kind, params, opt, bs, obs, st, rng,
                                                                     dict(cfg), u, lr_fn, forced_actions=forced,
                                                                     tie_log=log)
            for (t, e, a_own, a_forced, gap) in log:
                assert gap < 1e-4, f"seed {s} update {u} step {t} env {e}: action {a_forced} vs oracle {a_own}, Q gap {gap}"
            ties += [(s, u) + x for x in log]
            if kind == "cnn":                                                  # integer env: exact under equal actions
                assert np.array_equal(snaps[u]["done"][s].cpu().numpy().astype(bool), tr["done"].astype(bool)), (s, u)
                assert np.array_equal(snaps[u]["reward"][s].cpu().numpy(), tr["reward"]), (s, u)
                assert np.abs(snaps[u]["targets"][s].cpu().numpy() - tg).max() < 1e-4, (s, u)
            got_loss = float(out["metrics"]["td_loss"][s, u])
            assert abs(got_loss - m["td_loss"]) < 2e-4 * max(1.0, abs(m["td_loss"])), (s, u, got_loss, m["td_loss"])
        if kind == "cnn":
            def leaf(path):
                d = ts.params
                for kk in path:
                    d = d[kk]
                return d[s].cpu().numpy()
            for p, *_ in eng.spec.entries:
                assert np.abs(leaf(p) - params["/".join(p)]).max() < 5e-5, p
            assert np.array_equal(out["runner_state"][3][s].cpu().numpy().view(np.uint32), rng)
    frac = len(ties) / float(S * nupd * T * E)
    print(f"\n[eps<1 parity] {env_name}: {len(ties)} argmax flips on Q ties out of {S * nupd * T * E} actions "
          f"({100 * frac:.4f} %)", ties[:5])
    assert frac < 2e-3


# --------------------------------------------------------------------------- #
# (c) BASELINE configs at their geometry
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("env_name", ["Breakout-MinAtar", "Asterix-MinAtar", "SpaceInvaders-MinAtar",
                                      "Freeway-MinAtar"])
def test_config3_geometry_one_update_matches_oracle(env_name):
    """BASELINE configs[2]: NUM_ENVS=1024, 16 seeds, shipped pqn_minatar.yaml (T=32, 32 minibatches x 2 epochs,
    eps starts at 1).  One whole update through train(); two of the 16 seeds (first and last: seed striding)
    are replayed by the oracle: exact rollout bookkeeping + final key; parameters after the 64 clipped-RAdam steps
    agree to 5e-6 in the median, 2e-4 on 99.5 % of the coordinates and 1e-3 (two learning-rate steps) everywhere: RAdam divides by
    sqrt(v), so on coordinates whose gradient is ~1e-5 of the largest one the split-precision kernels' error
    (<= 2e-5 of the gradient's scale, tests/test_gpu_net.py) decides the update direction.  (An fp64-gradient
    oracle against the fp32 oracle stays within 3e-8 over the same 64 steps, so this is the kernels' error, not
    fp32 noise; it is reported here, not hidden.)"""
    from purejaxql_b200 import config_loader, pqn_minatar
    c = config_loader.compose(["+alg=pqn_minatar", f"alg.ENV_NAME={env_name}", "NUM_SEEDS=16", "SAVE_PATH=null",
                               "alg.NUM_ENVS=1024", "alg.TEST_DURING_TRAINING=False"])
    cfg = {**c, **c["alg"]}
    cfg["TOTAL_TIMESTEPS"] = float(cfg["NUM_STEPS"] * cfg["NUM_ENVS"])          # one update; decay horizon as shipped
    train = pqn_minatar.make_train(cfg)
    eng = train.engine
    S = 16
    rngs = jr.split(jr.PRNGKey(cfg["SEED"]), S)
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    out = train(rngs)
    assert out["metrics"]["td_loss"].shape == (S, 1)
    ts = out["runner_state"][0]
    tree0 = eng.spec.unflatten(cap["flat"])
    T, E = cfg["NUM_STEPS"], cfg["NUM_ENVS"]
    assert (T, E, cfg["NUM_MINIBATCHES"], cfg["NUM_EPOCHS"]) == (32, 1024, 32, 2)
    for s in (0, S - 1):
        params = _seed_params(eng, tree0, s)
        K1 = jr.split(rngs[s], 2)[0]
        K2 = jr.split(K1, 2)[0]
        k = jr.split(K2, 2); K3, kR = k[0], k[1]
        env = G.make(env_name)
        obs, st = env.reset(jr.split(kR, E))
        rng = jr.split(K3, 2)[1]
        total = cfg["NUM_UPDATES_DECAY"] * cfg["NUM_MINIBATCHES"] * cfg["NUM_EPOCHS"]
        lr_fn = lambda i: R.linear_schedule(cfg["LR"], 1e-20, total, i)
        C = eng.spec.in_c
        bs = {"mean": np.zeros(C, np.float32), "var": np.ones(C, np.float32)}
        p2, opt, bs, obs, st, rng2, m, tr, tg = R.update_step(env, "cnn", params, R.opt_init(params), bs, obs, st, rng,
                                                              dict(cfg), 0, lr_fn)
        for kk in R.INFO_KEYS:
            assert abs(float(out["metrics"][kk][s, 0]) - m[kk]) < 1e-6 * max(1, abs(m[kk])), (s, kk)
        assert abs(float(out["metrics"]["td_loss"][s, 0]) - m["td_loss"]) < 1e-4 * max(1.0, abs(m["td_loss"]))

        def leaf(path):
            d = ts.params
            for q in path:
                d = d[q]
            return d[s].cpu().numpy()
        worst = {}
        for p, *_ in eng.spec.entries:
            d = np.abs(leaf(p) - p2["/".join(p)]).ravel()
            worst["/".join(p)] = (float(d.max()), float(np.quantile(d, 0.995)))
            assert np.median(d) < 5e-6 and np.quantile(d, 0.995) < 2e-4, (s, p, worst["/".join(p)])
            assert d.max() < 1e-3, (s, p, worst["/".join(p)])
        print(f"\n[config3 {env_name} seed {s}] max / q99.5 |param - oracle| after 64 RAdam steps:",
              {k: (f"{a:.1e}", f"{b:.1e}") for k, (a, b) in worst.items() if a > 2e-5})
        assert np.array_equal(out["runner_state"][3][s].cpu().numpy().view(np.uint32), rng2)


def test_config4_acrobot_65536_env_step_and_train():
    """BASELINE configs[3]: Acrobot-v1 with NUM_ENVS=65536.  (i) the env operator at N=65536, teacher-forced against
    the oracle for 24 steps with a 20-step time limit (resets + truncation exercised), 2e-5 per step; (ii) two
    updates through pqn_gymnax.make_train/train at that geometry: finite loss, exact step bookkeeping, and update 1
    teacher-forced on its own buffers:
      - rollout Q-values: maxq[t, e] is max_a of the fp64 MLP on obs[t, e] under the parameters update 0 ended with,
        within 1e-5, on every 16th env (a different residue at each t) at all 64 steps;
      - Q(lambda) targets of all 65,536 envs against the fp64 recurrence on the engine's reward / done / maxq,
        bootstrapped by the fp64 MLP on obs[T]: within 4x the distance of the same computation in fp32 NumPy (fp32
        bootstrap forward + fp32 recurrence) from fp64, or 4 fp32 ulps of max |target| if that is larger;
      - transition rows: actions in [0, 3), done in {0, 1}, reward fp32 -0.1 (REW_SCALE x -1) where done is 0 and
        -0.0 at a terminal.  No episode reaches the 500-step limit in 128 steps, so every done is a terminal.
    Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): worst |maxq - fp64| 6.6e-7; targets worst error
    1.84e-6 = 1.00x the fp32 spread.  The kernel's recurrence does the fp32 NumPy recurrence's operations in the same
    order without FMA contraction (pqn_env.cu), so the two agree away from the bootstrap and share their worst element.
    Replacing gamma * lambda * delta by gamma * delta in the kernel misses by 1.9e6x the spread."""
    from purejaxql_b200 import config_loader, envs, pqn_gymnax
    name, n, atol = "Acrobot-v1", 65536, 2e-5
    oenv = G.make(name)
    env, params = envs.make(name)
    params = envs.EnvParams(max_steps_in_episode=20)
    oenv.env.core.max_steps_in_episode = 20
    try:
        key = jr.PRNGKey(9)
        ks = jr.split(key, 2); key, kr = ks[0], ks[1]
        rk = jr.split(kr, n)
        o_obs, o_st = oenv.reset(rk)
        obs, st = env.reset(tkeys(rk), params)
        assert np.allclose(obs.cpu().numpy(), o_obs, atol=atol, rtol=0)
        ndone = 0
        for t in range(24):
            ks = jr.split(key, 3); key, ka, kst = ks[0], ks[1], ks[2]
            act = jr.randint(jr.split(ka, n), (), 0, oenv.num_actions)
            sk = jr.split(kst, n)
            st = envs.fields_to_state(name, {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in o_st.items()}).to(dev())
            o_obs, o_st, o_r, o_d, o_info = oenv.step(sk, o_st, act)
            obs, st, r, d, info = env.step(tkeys(sk), st, torch.from_numpy(act).to(dev()), params)
            assert np.array_equal(d.cpu().numpy(), o_d), t
            assert np.allclose(r.cpu().numpy(), o_r, atol=atol, rtol=0)
            assert np.allclose(obs.cpu().numpy(), o_obs, atol=atol, rtol=0), t
            ndone += int(o_d.sum())
        assert ndone >= n, "every env should have hit the 20-step limit once"
    finally:
        oenv.env.core.max_steps_in_episode = 500
    c = config_loader.compose(["+alg=pqn_cartpole", "alg.ENV_NAME=Acrobot-v1", "NUM_SEEDS=1", "SAVE_PATH=null",
                               "alg.NUM_ENVS=65536", "alg.TEST_DURING_TRAINING=False"])
    cfg = {**c, **c["alg"]}
    T = cfg["NUM_STEPS"]
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(2 * T * 65536)   # SURVEY 8: must override (0 updates)
    train = pqn_gymnax.make_train(cfg)
    eng = train.engine
    snap = {}

    def grab(n_upd, b):                              # static buffers: copy them before the next update rewrites them
        if n_upd == 0:
            snap["params"] = b["params"].clone()     # update 1 rolls out and bootstraps with these
        else:
            snap.update({k: b[k][0].cpu().numpy() for k in ("obs", "reward", "done", "maxq", "targets", "action")})
    eng.on_update_end = grab
    out = train(jr.split(jr.PRNGKey(0), 1))
    m = out["metrics"]
    assert m["td_loss"].shape == (1, 2) and torch.isfinite(m["td_loss"]).all()
    assert m["env_step"][0].tolist() == [T * 65536, 2 * T * 65536]
    assert m["grad_steps"][0].tolist() == [cfg["NUM_MINIBATCHES"] * cfg["NUM_EPOCHS"],
                                           2 * cfg["NUM_MINIBATCHES"] * cfg["NUM_EPOCHS"]]
    assert "env_frame" not in m                                           # pqn_gymnax.py:324-331 has no env_frame
    # Acrobot: reward -1 per step, timestep of the LogWrapper advances by one per env per step
    assert float(m["timestep"][0, 0]) > 0 and float(m["returned_episode_returns"][0, -1]) <= 0.0

    # ---- update 1, teacher-forced on its own buffers
    E = 65536
    obs, reward, done, maxq, targets, action = (snap[k] for k in ("obs", "reward", "done", "maxq", "targets", "action"))
    assert obs.shape[:2] == (T + 1, E) and reward.shape == done.shape == maxq.shape == targets.shape == (T, E)
    p32 = _seed_params(eng, eng.spec.unflatten(snap["params"]), 0)
    p64 = {k: v.astype(np.float64) for k, v in p32.items()}
    assert eng.A == 3
    assert ((action >= 0) & (action < 3)).all()
    assert np.isin(done, (0, 1)).all()
    want_bits = np.where(done == 1, np.float32(-0.0).view(np.uint32), np.float32(-0.1).view(np.uint32))
    assert np.array_equal(reward.view(np.uint32), want_bits)
    worst_q = 0.0
    for t in range(T):
        e = np.arange(t % 16, E, 16)
        q64 = R.mlp_forward(p64, obs[t, e].astype(np.float64)).max(-1)
        worst_q = max(worst_q, float(np.abs(maxq[t, e] - q64).max()))
    assert worst_q < 1e-5, worst_q
    gamma, lam = cfg["GAMMA"], cfg["LAMBDA"]
    assert (gamma, lam) == (0.99, 0.95)
    last64 = R.mlp_forward(p64, obs[T].astype(np.float64)).max(-1)
    want = R.q_lambda_targets(reward.astype(np.float64), done, maxq.astype(np.float64)[..., None], last64, gamma, lam)
    want32 = R.q_lambda_targets(reward, done, maxq[..., None], R.mlp_forward(p32, obs[T]).max(-1), gamma, lam)
    err = float(np.abs(targets - want).max())
    spread = float(np.abs(want32 - want).max())
    bound = max(4 * spread, 4 * 2.0 ** -23 * float(np.abs(want).max()))
    print(f"\n[config4 update 1] {int(done.sum())} terminals; worst |maxq - fp64| {worst_q:.2e}; targets: worst err "
          f"{err:.2e}, fp32 spread {spread:.2e}, err / spread {err / max(spread, 1e-30):.2f}, bound {bound:.2e}")
    assert err <= bound, (err, spread, bound)
