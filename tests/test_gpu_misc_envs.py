"""SimpleBandit-bsuite, BernoulliBandit-misc, FourRooms-misc and MetaMaze-misc on the GPU, against the NumPy oracles of
tests/bsuite_bandit_oracle.py and tests/misc_envs_oracle.py.

- The env operator (reset, step, obs, auto-reset, LogWrapper words) at N = 100,003 and the fused
  ``pqn_rollout_act_step`` at 3 x 33,335 envs, with both threefry layouts: bit for bit.
- The networks' new edge cases: the MLP and GRU Q-networks at D = 1 with A = 11 (SimpleBandit), D = 4 with A = 4 and
  D = 15 with A = 4, for HIDDEN_SIZE 64 to 512 where the limits allow, on tensor-core paths 2 and 0, against the fp64
  oracles with the bars of tests/test_gpu_gymnax_extra.py; every NORM_TYPE x NORM_INPUT with batch_stats at D = 1,
  whose only input column is constant (variance 0), and at D = 15.
- SimpleBandit's 11 actions at HIDDEN_SIZE 512 are refused before anything is allocated.
- Two whole updates through make_train on SimpleBandit and on MetaMaze against an oracle replay for both scripts,
  CUDA-graph replay of the GRU against the eager run, bit-identical repeated runs, and a save-and-evaluate smoke run
  per script and env."""
import numpy as np
import pytest
import torch

import misc_envs_oracle as M
import rnn_norm_oracle as RO
import test_gpu_gymnax_extra as GX
import test_gpu_net_shapes as NS
import test_gpu_rnn_norm as RNS
from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_ref_norm as RN
from oracle import pqn_rnn_ref as RR
from test_misc_envs_host import MAX_STEPS, fields

pytestmark = pytest.mark.gpu
SB, BERN, ROOMS, MAZE = "SimpleBandit-bsuite", "BernoulliBandit-misc", "FourRooms-misc", "MetaMaze-misc"
NAMES = [SB, BERN, ROOMS, MAZE]
N_BIG = 100_003
dev, t_, keys_t, np_state, to_dev_state = GX.dev, GX.t_, GX.keys_t, GX.np_state, GX.to_dev_state


def assert_state(name, st, o_st, where):
    f = fields(name, np_state(st))
    for k, v in o_st.items():
        assert np.array_equal(f[k].astype(v.dtype).reshape(v.shape), v), (where, k)


def _near_the_end(name, o_st, rng, window):
    """Moves every env's time to within `window` steps of max_steps_in_episode, so that the episodes of the envs with
    long episodes end (and auto-reset) inside a short test."""
    if name != SB:
        o_st["time"] = rng.integers(MAX_STEPS[name] - window, MAX_STEPS[name], o_st["time"].shape[0]).astype(np.int32)


@pytest.fixture(params=[2, 0], ids=["tc_path2", "ffma_path0"])
def tc_path(request):
    from purejaxql_b200 import _lib
    _lib.check(_lib.lib().pqn_set_tensor_core_path(request.param))
    yield request.param
    _lib.lib().pqn_set_tensor_core_path(2)


# --------------------------------------------------------------------------- #
# env operator
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("name", NAMES)
def test_env_operator_bit_exact(name, part):
    """reset / step / obs at N = 100,003 over 24 steps of random actions from times 1-23 steps before the time limit
    (auto-resets included): obs, reward, done, info and every state field bit for bit; pqn_env_obs returns the obs the
    step returned; SimpleBandit's unflattened observation is gymnax's (N, 1, 1)."""
    from purejaxql_b200 import _lib, envs
    n, L = N_BIG, _lib.lib()
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env, params = envs.make(name, flatten_obs=True, rng_mode=part)
        oenv = M.make(name)
        D, A = env.obs_dim, env.num_actions
        key, kr = jr.split(jr.PRNGKey(12), 2)
        rk = jr.split(kr, n)
        obs, st = env.reset(keys_t(rk), params)
        o_obs, o_st = oenv.reset(rk)
        assert np.array_equal(obs.cpu().numpy().view(np.int32), o_obs.view(np.int32))
        assert_state(name, st, o_st, "reset")
        if name == SB:
            ones, _ = envs.make(SB, rng_mode=part)[0].reset(keys_t(rk), params)
            assert ones.shape == (n, 1, 1) and bool((ones == 1).all())
        rng = np.random.default_rng(part)
        _near_the_end(name, o_st, np.random.default_rng(7), 23)
        st = to_dev_state(name, o_st)
        dones = np.zeros(n, np.int64)
        for t in range(24):
            key, ks = jr.split(key, 2)
            sk = jr.split(ks, n)
            act = rng.integers(0, A, n).astype(np.int32)
            obs, st, r, d, info = env.step(keys_t(sk), st, t_(act), params)
            o_obs, o_st, o_r, o_d, o_info = oenv.step(sk, o_st, act)
            assert np.array_equal(d.cpu().numpy(), o_d), t
            assert np.array_equal(r.cpu().numpy().view(np.int32), o_r.view(np.int32)), t
            assert np.array_equal(obs.cpu().numpy().view(np.int32), o_obs.view(np.int32)), t
            for k in ("discount", "returned_episode_returns", "returned_episode_lengths", "timestep"):
                assert np.array_equal(info[k].cpu().numpy(), o_info[k]), (t, k)
            assert_state(name, st, o_st, t)
            ob2 = torch.empty((n, D), device=dev())
            _lib.check(L.pqn_env_obs(env.env_id, _lib.p(st), _lib.p(ob2), n, _lib.stream_ptr()), "pqn_env_obs")
            assert torch.equal(ob2, obs), t
            dones += o_d
        assert (dones >= 1).all()
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("done_only", [0, 1])
def test_rollout_act_step_matches_oracle(name, done_only, part):
    """The fused eps-greedy + step + LogWrapper launch over 3 seeds x 33,335 envs (100,005 in all; not a multiple of
    the block), in both threefry layouts: actions (eps-greedy over SimpleBandit's 11 q values included), rewards,
    dones, max q, the obs rows, every state field and the info sums, bit for bit.  The envs start 1-10 steps before
    their time limit, so that every episode ends inside the window."""
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        _rollout_act_step_against_oracle(name, done_only, part)
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def _rollout_act_step_against_oracle(name, done_only, part):
    from purejaxql_b200 import _lib, envs
    L = _lib.lib()
    S, E, eps, rew_scale, T = 3, 33_335, 0.4, 0.5, 12
    env, _ = envs.make(name, flatten_obs=True, rng_mode=part)
    oenv = M.make(name)
    D, A = env.obs_dim, env.num_actions
    seeds = jr.split(jr.PRNGKey(78), S)
    rk = np.stack([jr.split(seeds[s], E) for s in range(S)])
    o = [oenv.reset(rk[s]) for s in range(S)]
    o_obs, o_st = [x[0] for x in o], [x[1] for x in o]
    for s in range(S):
        _near_the_end(name, o_st[s], np.random.default_rng(s), 10)
    state = torch.cat([to_dev_state(name, o_st[s]) for s in range(S)], 1).contiguous()
    obs_buf = torch.zeros((S, T + 1, E, D), device=dev())
    act = torch.zeros((S, T, E), dtype=torch.int32, device=dev())
    rew = torch.zeros((S, T, E), device=dev())
    done = torch.zeros((S, T, E), dtype=torch.uint8, device=dev())
    maxq = torch.zeros((S, T, E), device=dev())
    sums = torch.zeros((S, 5), dtype=torch.float64, device=dev())
    o_sums = np.zeros((S, 5))
    eps_d = torch.full((1,), eps, device=dev())
    rng = np.random.default_rng(6)
    for t in range(T):
        q = rng.standard_normal((S * E, A)).astype(np.float32)
        step_keys = np.stack([np.stack(jr.split(jr.PRNGKey(1000 * t + s), 2)) for s in range(S)])
        keys_d, q_d = keys_t(step_keys), t_(q)
        _lib.check(L.pqn_rollout_act_step(env.env_id, _lib.p(keys_d), _lib.p(q_d), _lib.p(eps_d),
                                          _lib.p(state), _lib.raw(obs_buf[:, t + 1]), (T + 1) * E, _lib.raw(act[:, t]),
                                          _lib.raw(rew[:, t]), _lib.raw(done[:, t]), _lib.raw(maxq[:, t]), T * E,
                                          _lib.p(sums), done_only, S, E, 0, 0, 0, rew_scale, part, _lib.stream_ptr()),
                   "pqn_rollout_act_step")
        for s in range(S):
            qs = q.reshape(S, E, A)[s]
            a = R.eps_greedy(jr.split(step_keys[s, 0], E), qs, eps)
            o_obs[s], o_st[s], r, d, info = oenv.step(jr.split(step_keys[s, 1], E), o_st[s], a)
            assert np.array_equal(act[s, t].cpu().numpy(), a), (t, s)
            assert np.array_equal(rew[s, t].cpu().numpy().view(np.int32),
                                  (np.float32(rew_scale) * r).astype(np.float32).view(np.int32)), (t, s)
            assert np.array_equal(done[s, t].cpu().numpy().astype(bool), d), (t, s)
            assert np.array_equal(maxq[s, t].cpu().numpy(), qs.max(-1)), (t, s)
            assert np.array_equal(obs_buf[s, t + 1].cpu().numpy().view(np.int32), o_obs[s].view(np.int32)), (t, s)
            assert_state(name, state[:, s * E:(s + 1) * E], o_st[s], (t, s))
            m = d if done_only else np.ones(E, bool)
            o_sums[s] += [info["returned_episode_returns"][m].astype(np.float64).sum(),
                          info["returned_episode_lengths"][m].sum(), info["timestep"][m].sum(), d.sum(),
                          info["discount"][m].sum()]
    assert np.array_equal(sums.cpu().numpy(), o_sums)
    assert o_sums[:, 3].min() >= E
    if name == SB:   # every one of the 11 actions was taken, greedy and random
        assert set(np.unique(act.cpu().numpy()).tolist()) == set(range(11))


# --------------------------------------------------------------------------- #
# networks: D = 1 / A = 11, D = 4 / A = 4, D = 15 / A = 4
# --------------------------------------------------------------------------- #
SHAPES = [(D, A, H) for D, A in ((1, 11), (4, 4), (15, 4)) for H in (64, 128, 256, 512) if not (A > 9 and H == 512)]


def _inputs(rng, shape, D):
    """Random normal rows, or at D = 1 SimpleBandit's constant ones."""
    return np.ones(shape + (D,), np.float32) if D == 1 else rng.standard_normal(shape + (D,)).astype(np.float32)


@pytest.mark.parametrize("D,A,H", SHAPES)
def test_mlp_forward_and_loss_grad(D, A, H, tc_path):
    """As test_gpu_gymnax_extra checks D = 2 and 50 at A = 3: eval forward, loss, mean chosen q and every gradient
    against the fp64 oracle (2e-5 of each gradient's scale)."""
    from purejaxql_b200 import _lib
    S, total, rows, Ls = 2, 1400, 515, 2
    spec, ps, flat = NS._mlp_setup(D, H, Ls, A, S, 40)
    rng = np.random.default_rng(D + H + A)
    obs = _inputs(rng, (S, total), D)
    L = _lib.lib()
    q = torch.zeros((S * total, A), device=dev())
    to_, ws_f, ws_l = t_(obs, torch.float32), NS._ws(spec, S, total), NS._ws(spec, S, rows)
    _lib.check(L.pqn_qnet_forward(spec.desc, _lib.p(flat), None, _lib.p(to_), None, total, _lib.p(q), S, total,
                                  _lib.p(ws_f), _lib.stream_ptr()), "pqn_qnet_forward")
    qn = q.cpu().numpy().reshape(S, total, A)
    gather = np.stack([rng.permutation(total)[:rows] for _ in range(S)]).astype(np.int32)
    act = rng.integers(0, A, (S, total)).astype(np.int32)
    tgt = rng.standard_normal((S, total)).astype(np.float32)
    grads = torch.zeros_like(flat)
    ls, qs, bn = torch.zeros(S, device=dev()), torch.zeros(S, device=dev()), torch.zeros((S, 2 * D), device=dev())
    tg_, ta_, tt_ = t_(gather, torch.int32), t_(act, torch.int32), t_(tgt, torch.float32)
    _lib.check(L.pqn_qnet_loss_grad(spec.desc, _lib.p(flat), None, _lib.p(to_), _lib.p(tg_), total, _lib.p(ta_),
                                    _lib.p(tt_), total, _lib.p(grads), _lib.p(ls), _lib.p(qs), _lib.p(bn), S, rows,
                                    _lib.p(ws_l), _lib.stream_ptr()), "pqn_qnet_loss_grad")
    torch.cuda.synchronize()
    gtree = spec.unflatten(grads)
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        assert np.abs(qn[s] - R.mlp_forward(p64, obs[s].astype(np.float64))).max() < 1e-5
        loss, q_sa, g = R.mlp_loss_and_grads(p64, obs[s][gather[s]].astype(np.float64), act[s][gather[s]],
                                             tgt[s][gather[s]].astype(np.float64))
        assert abs(float(ls[s]) - loss) < 1e-5 * max(1, abs(loss)) and abs(float(qs[s]) - q_sa.mean()) < 1e-5
        for path, *_ in spec.entries:
            ref = g["/".join(path)]
            scale = max(np.abs(ref).max(), 1e-3)
            err = np.abs(NS._leaf(gtree, path, s) - ref).max()
            assert err < 2e-5 * scale + 1e-7, (path, err, scale)


@pytest.mark.parametrize("D,A,H", SHAPES)
def test_rnn_step_and_window_loss_grad(D, A, H, tc_path):
    """The GRU's step (one-hot last action over A inputs) and window loss / gradients against the fp64 oracle, as
    test_gpu_gymnax_extra checks them at A = 3."""
    from purejaxql_b200 import _lib
    S, Ls, E, T, B = 2, 2, 37, 9, 5
    spec, ps, flat = NS._rnn_setup(S, D, A, H, Ls)
    rng = np.random.default_rng(D * H + A)
    hs = rng.standard_normal((S, E, H)).astype(np.float32) * 0.5
    obs = _inputs(rng, (S, E), D)
    ld = rng.random((S, E)) < 0.3
    la = rng.integers(0, A, (S, E)).astype(np.int32)
    la[:, :A] = np.arange(A)                                 # every last action, the largest included
    hs_d, obs_d = t_(hs, torch.float32), t_(obs, torch.float32)
    ld_d, la_d = t_(ld.astype(np.uint8), torch.uint8), t_(la, torch.int32)
    q, ws = torch.zeros((S * E, A), device=dev()), NS._ws(spec, S, E)
    _lib.check(_lib.lib().pqn_rnn_step(spec.desc, _lib.p(flat), _lib.p(hs_d), _lib.p(obs_d), E, _lib.p(ld_d),
                                       _lib.p(la_d), _lib.p(q), S, E, _lib.p(ws), _lib.stream_ptr()), "pqn_rnn_step")
    torch.cuda.synchronize()
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        new_h, qq = RR.rnn_forward(p64, hs[s].astype(np.float64), obs[s][None].astype(np.float64), ld[s][None],
                                   la[s][None])
        assert np.abs(q.cpu().numpy().reshape(S, E, A)[s] - qq[0]).max() < 1e-5
        assert np.abs(hs_d.cpu().numpy()[s] - new_h).max() < 1e-5
    w, bufs = RNS._window(S, T, B, D, A, H, seed=D + H + A)
    if D == 1:
        w["obs"] = np.ones_like(w["obs"])
        bufs[1] = t_(w["obs"], torch.float32)
    grads = torch.zeros_like(flat)
    ls, qs = torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
    _lib.check(RNS._loss(spec, flat, None, bufs, grads, ls, qs, S, T, B, NS._ws(spec, S, T * B), fn="pqn_rnn_loss_grad"),
               "pqn_rnn_loss_grad")
    torch.cuda.synchronize()
    gtree = spec.unflatten(grads)
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        loss, chosen, g = RR.rnn_loss_and_grads(p64, w["hs0"][s].astype(np.float64), w["obs"][s].astype(np.float64),
                                                w["ld"][s], w["la"][s], w["ac"][s], w["rw"][s].astype(np.float64),
                                                w["dn"][s], 0.99, 0.95)
        assert abs(float(ls[s]) - loss) < 1e-5 * max(1.0, abs(loss)), (float(ls[s]), loss)
        assert abs(float(qs[s]) - chosen.mean()) < 1e-5 * max(1.0, abs(chosen.mean()))
        scale = max(np.abs(v).max() for v in g.values())
        for path, *_ in spec.entries:
            err = np.abs(NS._leaf(gtree, path, s) - g["/".join(path)]).max()
            assert err < 2e-5 * scale, (path, err, scale)


# At D = 1 every hidden pre-activation column is constant too, so a hidden BatchNorm's batch variance is 0 only in
# exact arithmetic: fp32 column sums leave (z - mean) at the rounding of the sum, and rstd = 1 / sqrt(eps) ~ 316
# amplifies it in the backward.  Any fp32 BatchNorm shares this; the gradients behind the first hidden BatchNorm
# (Dense_0, and the input BatchNorm_0) were measured at most 1.9e-2 of the scale from fp64 on the H100.
CONSTANT_COLUMN_BAR = 5e-2


def _stats_bar(norm_type, D, want):
    """2e-6, as the existing tests; at D = 1 under batch_norm the batch statistics of a layer behind a hidden
    BatchNorm carry that amplified rounding, and the running statistic takes 1 - momentum = 0.01 of it."""
    if norm_type == "batch_norm" and D == 1:
        return 2e-6 + 0.01 * CONSTANT_COLUMN_BAR * max(1.0, float(np.abs(want).max()))
    return 2e-6


def _norm_obs(rng, shape, D):
    """D = 1: SimpleBandit's constant ones.  D = 15: MetaMaze-like rows (a 0/1 wall field, a one-hot action, a reward
    of 0 or 10 and a time in [-1, 3))."""
    if D == 1:
        return np.ones(shape + (1,), np.float32)
    n = int(np.prod(shape))
    o = np.zeros((n, 15), np.float32)
    o[:, :9] = rng.random((n, 9)) < 0.4
    o[np.arange(n), 9 + rng.integers(0, 4, n)] = 1
    o[:, 13] = np.where(rng.random(n) < 0.05, 10.0, 0.0)
    o[:, 14] = (2 * rng.integers(0, 200, n) / 100 - 1).astype(np.float32)
    return o.reshape(shape + (15,))


@pytest.mark.parametrize("D,A", [(1, 11), (15, 4)])
@pytest.mark.parametrize("norm_type,norm_input", GX.NORMS6)
def test_mlp_norm_variants(norm_type, norm_input, D, A, tc_path):
    """Eval forward, loss / gradients and the updated batch_stats at D = 1 (a constant input column: the input
    BatchNorm's batch variance is 0, so its xhat is exactly 0, its scale's gradient exactly 0 and every running
    statistic finite) and at D = 15."""
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_MLP, QNetworkSpec
    H, Ls, S, total, rows = 256, 2, 2, 300, 257
    spec = QNetworkSpec(NET_MLP, D, A, H, Ls, norm_type=norm_type, norm_input=norm_input)
    ps = [R.random_params(RN.mlp_param_shapes(D, A, H, Ls, norm_type), 30 + s) for s in range(S)]
    if norm_type == "batch_norm":
        for p in ps:
            for layer in range(Ls):
                p[f"Dense_{layer}/bias"] = np.zeros_like(p[f"Dense_{layer}/bias"])
    sts = [NS._rand_stats(RN.mlp_batch_stats(D, H, Ls, norm_type), 50 + s) for s in range(S)]
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    stf = torch.cat([spec.flatten_stats(st, 1, dev()) for st in sts], 0).contiguous()
    rng = np.random.default_rng(4)
    obs = _norm_obs(rng, (S, total), D)
    dev_obs = t_(obs, torch.float32)
    L_ = _lib.lib()
    q = torch.zeros((S * total, A), device=dev())
    ws_f, ws_l = NS._ws(spec, S, total), NS._ws(spec, S, rows)
    _lib.check(L_.pqn_qnet_forward(spec.desc, _lib.p(flat), _lib.p(stf), _lib.p(dev_obs), None, total, _lib.p(q), S,
                                   total, _lib.p(ws_f), _lib.stream_ptr()), "pqn_qnet_forward")
    torch.cuda.synchronize()
    qn = q.cpu().numpy().reshape(S, total, A)
    for s in range(S):
        ref, _ = RN.mlp_forward(ps[s], sts[s], obs[s], False, norm_type, norm_input)
        assert np.abs(qn[s] - ref).max() < 1e-5 * max(1.0, np.abs(ref).max()), (s, np.abs(qn[s] - ref).max())
    gather = np.stack([rng.permutation(total)[:rows] for _ in range(S)]).astype(np.int32)
    act = rng.integers(0, A, (S, total)).astype(np.int32)
    tgt = rng.standard_normal((S, total)).astype(np.float32)
    grads = torch.zeros_like(flat)
    ls, qs, bn = torch.zeros(S, device=dev()), torch.zeros(S, device=dev()), torch.zeros((S, 2 * D), device=dev())
    st_dev = stf.clone()
    tg_, ta_, tt_ = t_(gather, torch.int32), t_(act, torch.int32), t_(tgt, torch.float32)
    _lib.check(L_.pqn_qnet_loss_grad(spec.desc, _lib.p(flat), _lib.p(st_dev), _lib.p(dev_obs), _lib.p(tg_), total,
                                     _lib.p(ta_), _lib.p(tt_), total, _lib.p(grads), _lib.p(ls), _lib.p(qs), _lib.p(bn), S,
                                     rows, _lib.p(ws_l), _lib.stream_ptr()), "pqn_qnet_loss_grad")
    _lib.check(L_.pqn_bn_stats_update(_lib.p(st_dev), _lib.p(bn), S, D, spec.stats_total, float(rows), 0.99,
                                      _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.isfinite(grads).all() and torch.isfinite(st_dev).all()
    gtree, sttree = spec.unflatten(grads), spec.unflatten_stats(st_dev)
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        st64 = {k: {kk: vv.astype(np.float64) for kk, vv in v.items()} for k, v in sts[s].items()}
        loss, q_sa, g, new_stats = RN.mlp_loss_and_grads(p64, st64, obs[s][gather[s]].astype(np.float64),
                                                         act[s][gather[s]], tgt[s][gather[s]].astype(np.float64),
                                                         norm_type, norm_input)
        assert abs(float(ls[s]) - loss) < 5e-5 * max(1.0, abs(loss)), (float(ls[s]), loss)
        assert abs(float(qs[s]) - q_sa.mean()) < 5e-5 * max(1.0, abs(q_sa.mean()))
        scale = max(np.abs(v).max() for v in g.values())
        errs = {}
        for path, *_ in spec.entries:
            name = "/".join(path)
            tol = 2e-5
            if norm_type == "batch_norm":
                tol = 5e-2 if name.startswith("Dense_") and name.endswith("/bias") and name != f"Dense_{Ls}/bias" else 2e-4
                if D == 1 and name.startswith(("Dense_0/", "BatchNorm_0/")):
                    tol = CONSTANT_COLUMN_BAR
            errs[name] = (float(np.abs(NS._leaf(gtree, path, s) - g[name]).max() / scale), tol)
        bad = {k: v for k, v in errs.items() if not v[0] < v[1]}
        assert not bad, (bad, errs)
        if D == 1 and norm_input:   # the input BatchNorm's xhat is exactly 0, so is its scale's gradient
            assert not NS._leaf(gtree, ("BatchNorm_0", "scale"), s).any() and not g["BatchNorm_0/scale"].any()
        for path, off, n in spec.stats_entries():
            d = sttree
            for k in path:
                d = d[k]
            want = new_stats["/".join(path)]
            for k in ("mean", "var"):
                err, tol = np.abs(d[k][s].cpu().numpy() - want[k]).max(), _stats_bar(norm_type, D, want[k])
                assert err < tol, (path, k, err, tol)


@pytest.mark.parametrize("D,A", [(1, 11), (15, 4)])
@pytest.mark.parametrize("norm_type,norm_input", GX.NORMS6)
def test_rnn_norm_variants(norm_type, norm_input, D, A, tc_path):
    """The GRU's *_stats entry points at D = 1 (a constant input column) and D = 15: the eval step with the running
    statistics, and the window loss / gradients with every running statistic updated in place, as
    test_gpu_gymnax_extra checks them at D = 50."""
    from purejaxql_b200 import _lib
    S, H, Ls, E, T, B = 2, 128, 2, 37, 10, 5
    spec, ps, sts, flat, stats = RNS._setup(S, D, A, H, Ls, norm_type, norm_input)
    hs, _, ld, la = RNS._step_inputs(S, E, D, A, H, 5)
    obs = _norm_obs(np.random.default_rng(5), (S, E + 5), D)
    hs_d = t_(hs, torch.float32)
    q = torch.zeros((S * E, A), device=dev())
    stats0 = stats.clone()
    _lib.check(RNS._step(spec, flat, stats, hs_d, t_(obs, torch.float32), E + 5, t_(ld.astype(np.uint8), torch.uint8),
                         t_(la, torch.int32), q, S, E, NS._ws(spec, S, E)), "pqn_rnn_step_stats")
    torch.cuda.synchronize()
    assert torch.equal(stats, stats0)
    for s in range(S):
        new_h, qq = RO.rnn_forward(RNS._f64(ps[s]), hs[s].astype(np.float64), obs[s][None, :E].astype(np.float64),
                                   ld[s][None], la[s][None], norm_type=norm_type, norm_input=norm_input,
                                   batch_stats=RNS._st64(sts[s]), train=False)
        assert np.abs(q.cpu().numpy().reshape(S, E, A)[s] - qq[0]).max() < 1e-5
        assert np.abs(hs_d.cpu().numpy()[s] - new_h).max() < 1e-5
    w, bufs = RNS._window(S, T, B, D, A, H)
    w["obs"] = _norm_obs(np.random.default_rng(6), (S, T, B), D)
    bufs[1] = t_(w["obs"], torch.float32)
    grads = torch.zeros_like(flat)
    ls, qs = torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
    _lib.check(RNS._loss(spec, flat, stats, bufs, grads, ls, qs, S, T, B, NS._ws(spec, S, T * B)),
               "pqn_rnn_loss_grad_stats")
    torch.cuda.synchronize()
    assert torch.isfinite(grads).all() and torch.isfinite(stats).all()
    gtree, sttree = spec.unflatten(grads), spec.unflatten_stats(stats)
    dead = {f"Dense_{l}/bias" for l in range(Ls)} if norm_type == "batch_norm" else set()
    for s in range(S):
        loss, chosen, g, new_stats = RO.rnn_loss_and_grads(
            RNS._f64(ps[s]), w["hs0"][s].astype(np.float64), w["obs"][s].astype(np.float64), w["ld"][s], w["la"][s],
            w["ac"][s], w["rw"][s].astype(np.float64), w["dn"][s], 0.99, 0.95, norm_type, norm_input,
            RNS._st64(sts[s]))
        assert abs(float(ls[s]) - loss) < 5e-5 * max(1.0, abs(loss)), (float(ls[s]), loss)
        assert abs(float(qs[s]) - chosen.mean()) < 5e-5 * max(1.0, abs(chosen.mean()))
        scale = max(np.abs(v).max() for v in g.values())
        errs = {}
        for path, *_ in spec.entries:
            name = "/".join(path)
            tol = (5e-2 if name in dead else 2e-4) if norm_type == "batch_norm" else 2e-5
            if norm_type == "batch_norm" and D == 1 and name.startswith(("Dense_0/", "BatchNorm_0/")):
                tol = CONSTANT_COLUMN_BAR
            errs[name] = (float(np.abs(NS._leaf(gtree, path, s) - g[name]).max() / scale), tol)
        bad = {k: v for k, v in errs.items() if not v[0] < v[1]}
        assert not bad, (bad, errs)
        if D == 1 and norm_input:   # the input BatchNorm's xhat is exactly 0, so is its scale's gradient
            assert not NS._leaf(gtree, ("BatchNorm_0", "scale"), s).any() and not g["BatchNorm_0/scale"].any()
        for path, off, n in spec.stats_entries():
            want = new_stats["/".join(path)]
            d = sttree
            for k in path:
                d = d[k]
            for k in ("mean", "var"):
                err, tol = np.abs(d[k][s].cpu().numpy() - want[k]).max(), _stats_bar(norm_type, D, want[k])
                assert err < tol, (path, k, err, tol)


@pytest.mark.parametrize("script", ["pqn_gymnax", "pqn_rnn_gymnax"])
def test_simple_bandit_at_hidden_512_is_refused_before_allocation(script):
    """11 actions need more shared memory than the head backward has at HIDDEN_SIZE 512 (actions <= 9 there):
    make_train refuses SimpleBandit with that limit before it allocates any device memory."""
    import importlib
    from purejaxql_b200 import _lib
    mod = importlib.import_module(f"purejaxql_b200.{script}")
    cfg = NS._rnn_cfg(512, 2, env=SB) if script == "pqn_rnn_gymnax" else dict(NS._mlp_cfg(512, 2), ENV_NAME=SB)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(_lib.PqnError) as e:
        mod.make_train(cfg)
    assert "num_actions=11" in str(e.value) and "limit 227 KB" in str(e.value)
    assert torch.cuda.memory_allocated() == before


# --------------------------------------------------------------------------- #
# whole runs
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name", [SB, MAZE])
def test_mlp_two_updates_match_oracle(name, monkeypatch):
    """Two whole updates of pqn_gymnax (eps = 1) against the oracle's update_step."""
    import test_gpu_train as TT
    from purejaxql_b200 import pqn_gymnax
    monkeypatch.setitem(G._REGISTRY, name, M.CORES[name])
    cfg = TT._cfg(name, HIDDEN_SIZE=128, NUM_LAYERS=2, REW_SCALE=1.0, LAMBDA=0.95, NUM_ENVS=32, NUM_STEPS=16)
    TT._run_updates_against_oracle(pqn_gymnax, name, "mlp", True, cfg, nupd=2)


@pytest.mark.parametrize("name", [SB, MAZE])
def test_rnn_two_updates_match_oracle(name):
    """Two whole updates of pqn_rnn_gymnax (eps = 1) against the oracle replay of test_gpu_memory_chain; SimpleBandit
    ends an episode at every step and feeds the GRU 11 one-hot last actions."""
    import test_gpu_memory_chain as MCT
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = MCT._rnn_cfg(ENV_NAME=name)
    del cfg["ENV_KWARGS"]
    nupd = 2
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_rnn_gymnax.make_train(cfg)
    eng = train.engine
    assert (eng.D, eng.A) == {SB: (1, 11), MAZE: (15, 4)}[name]
    rngs = jr.split(jr.PRNGKey(32), 2)
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    out = train(rngs)
    dones = MCT._replay_rnn_updates(cfg, out, eng.spec.unflatten(cap["flat"]), eng.spec, rngs, nupd,
                                    lambda: M.make(name))
    if name == SB:
        assert dones > 0


def _rnn_run(name, graph, norm_type="layer_norm", norm_input=False):
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = NS._rnn_cfg(128, 2, env=name, nupd=5, graph=graph)
    cfg.update(NORM_TYPE=norm_type, NORM_INPUT=norm_input, TEST_NUM_STEPS=30)
    train = pqn_rnn_gymnax.make_train(cfg)
    out = train(jr.split(jr.PRNGKey(5), 2))
    assert train.engine.graph_captured == graph
    return (out["runner_state"][0].params_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy(),
            out["metrics"]["returned_episode_returns"].cpu().numpy(),
            out["metrics"]["test/returned_episode_lengths"].cpu().numpy(), out["runner_state"][4].cpu().numpy())


@pytest.mark.parametrize("name", [SB, MAZE])
@pytest.mark.parametrize("norm_type,norm_input", [("layer_norm", False), ("batch_norm", True)])
def test_rnn_cuda_graph_replay_equals_eager_and_repeats(name, norm_type, norm_input):
    eager, graph, again = (_rnn_run(name, False, norm_type, norm_input), _rnn_run(name, True, norm_type, norm_input),
                           _rnn_run(name, True, norm_type, norm_input))
    for a, b, c in zip(eager, graph, again):
        assert np.array_equal(a, b, equal_nan=True) and np.array_equal(b, c, equal_nan=True)
    assert np.isfinite(eager[1]).all()
    if name == SB:
        assert (eager[3] == 1).all()


@pytest.mark.parametrize("name", NAMES)
def test_mlp_is_bit_reproducible(name):
    from purejaxql_b200 import pqn_gymnax
    outs = []
    for _ in range(2):
        cfg = NS._mlp_cfg(256, 2)
        cfg.update(ENV_NAME=name, NORM_INPUT=True)
        out = pqn_gymnax.make_train(cfg)(jr.split(jr.PRNGKey(11), 2))
        outs.append((out["runner_state"][0].params_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy()))
    assert np.isfinite(outs[0][1]).all()
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


RETURN_RANGE = {SB: (0.0, 1.0), BERN: (0.0, 100.0), ROOMS: (0.0, 1.0), MAZE: (0.0, 2000.0)}


@pytest.mark.parametrize("script,preset", [("pqn_gymnax", "pqn_cartpole"), ("pqn_rnn_gymnax", "pqn_rnn_cartpole")])
@pytest.mark.parametrize("name", NAMES)
def test_smoke_with_eval_and_save(script, preset, name, tmp_path):
    import importlib
    from purejaxql_b200 import config_loader
    from purejaxql_b200.utils.save_load import load_params
    mod = importlib.import_module(f"purejaxql_b200.{script}")
    c = config_loader.compose([f"+alg={preset}", f"alg.ENV_NAME={name}", "NUM_SEEDS=2", f"SAVE_PATH={tmp_path}",
                               "alg.TOTAL_TIMESTEPS=2e4", "alg.TOTAL_TIMESTEPS_DECAY=2e4", "alg.TEST_NUM_ENVS=16",
                               "alg.TEST_INTERVAL=0.5"])
    out = mod.single_run(c)
    m = out["metrics"]
    assert torch.isfinite(m["td_loss"]).all() and "test/returned_episode_returns" in m
    n = m["test/returned_episode_lengths"]
    if name in (SB, BERN, MAZE):
        assert (n == MAX_STEPS[name] if name != SB else n == 1).all()
    else:
        assert ((n >= 1) & (n <= MAX_STEPS[name])).all()
    lo, hi = RETURN_RANGE[name]
    r = m["test/returned_episode_returns"]
    assert ((r >= lo - 1e-6) & (r <= hi + 1e-6)).all(), r
    files = [p for p in tmp_path.rglob("*.safetensors")]
    assert len(files) == 2, files
    tree = load_params(str(sorted(files)[0]))
    assert tree["Dense_0"]["kernel"].shape[0] == {SB: 1, BERN: 4, ROOMS: 4, MAZE: 15}[name]
