"""MountainCar-v0 and Catch-bsuite on the GPU, against the NumPy oracles of tests/gymnax_extra_oracle.py.

- The env operator (reset, step, obs, auto-reset, LogWrapper words) and the fused ``pqn_rollout_act_step`` at a ragged
  N of about 100,003 with both threefry layouts: bit for bit for Catch; teacher-forced for MountainCar, with position and velocity
  within 2 fp32 ulps of the largest magnitude their step adds (tests/test_gymnax_extra_host.py), and every integer,
  reward and done exact.  The left-wall clamp and a goal crossing are set up by hand.
- The MLP and GRU Q-networks at the new input widths, D = 2 and D = 50, for HIDDEN_SIZE 64 to 512 on tensor-core
  paths 2 and 0, against the fp64 oracles with the existing bars (2e-5 of the gradients' scale; the BatchNorm variants
  the bars of test_gpu_norm / test_gpu_rnn_norm), and at D = 50 every NORM_TYPE x NORM_INPUT with batch_stats, for
  the GRU also at D = 300 and 1024 (its per-channel tables grown past 256 channels).
- Two whole updates through make_train on Catch against an oracle replay for both scripts, CUDA-graph replay of the
  GRU against the eager run, bit-identical repeated runs, and a save-and-evaluate smoke run per script and env."""
import numpy as np
import pytest
import torch

import gymnax_extra_oracle as X
import rnn_norm_oracle as RO
import test_gpu_net_shapes as NS
import test_gpu_rnn_norm as RNS
from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_ref_norm as RN
from oracle import pqn_rnn_ref as RR
from test_gymnax_extra_host import assert_mcar_close, fields

pytestmark = pytest.mark.gpu
MCAR, CATCH = "MountainCar-v0", "Catch-bsuite"
N_BIG = 100_003


def dev():
    return torch.device("cuda:0")


def t_(a, dt=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev())
    return t if dt is None else t.to(dt)


def keys_t(k):
    return t_(np.ascontiguousarray(k, np.uint32).view(np.int32))


def np_state(st):
    return st.cpu().numpy().view(np.uint32)


def to_dev_state(name, o_st):
    from purejaxql_b200 import envs
    return envs.fields_to_state(name, {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in o_st.items()}).to(dev())


def assert_catch_state(st, o_st, where):
    f = fields(CATCH, np_state(st))
    for k, v in o_st.items():
        assert np.array_equal(f[k].astype(v.dtype), v), (where, k)


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
def test_catch_env_operator_bit_exact(part):
    """reset / step / obs at N = 100,003 over two and a half episodes: obs, reward (sign of zero included), done,
    info and every state field bit for bit; pqn_env_obs returns the obs the step returned."""
    from purejaxql_b200 import _lib, envs
    n, L = N_BIG, _lib.lib()
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env, params = envs.make(CATCH, flatten_obs=True, rng_mode=part)
        oenv = X.make(CATCH)
        key, kr = jr.split(jr.PRNGKey(12), 2)
        rk = jr.split(kr, n)
        obs, st = env.reset(keys_t(rk), params)
        o_obs, o_st = oenv.reset(rk)
        assert np.array_equal(obs.cpu().numpy(), o_obs)
        assert_catch_state(st, o_st, "reset")
        board, _ = envs.make(CATCH, rng_mode=part)[0].reset(keys_t(rk), params)      # unflattened: gymnax's (10, 5)
        assert board.shape == (n, 10, 5) and np.array_equal(board.cpu().numpy().reshape(n, 50), o_obs)
        rng = np.random.default_rng(part)
        for t in range(22):
            key, ks = jr.split(key, 2)
            sk = jr.split(ks, n)
            act = rng.integers(0, 3, n).astype(np.int32)
            obs, st, r, d, info = env.step(keys_t(sk), st, t_(act), params)
            o_obs, o_st, o_r, o_d, o_info = oenv.step(sk, o_st, act)
            assert np.array_equal(d.cpu().numpy(), o_d), t
            assert np.array_equal(r.cpu().numpy().view(np.int32), o_r.view(np.int32)), t
            assert np.array_equal(obs.cpu().numpy(), o_obs), t
            for k in ("discount", "returned_episode_returns", "returned_episode_lengths", "timestep"):
                assert np.array_equal(info[k].cpu().numpy(), o_info[k]), (t, k)
            assert_catch_state(st, o_st, t)
            ob2 = torch.empty((n, 50), device=dev())
            _lib.check(L.pqn_env_obs(env.env_id, _lib.p(st), _lib.p(ob2), n, _lib.stream_ptr()), "pqn_env_obs")
            assert np.array_equal(ob2.cpu().numpy(), o_obs), t
        assert set(np.unique(o_st["log_returned_episode_returns"])) == {-1.0, 1.0}
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("part", [0, 1])
def test_mountain_car_env_operator_teacher_forced(part):
    """The reset is bit-exact at N = 100,003; then 205 teacher-forced steps of random actions (every env truncates at
    200 and auto-resets bit-exactly)."""
    from purejaxql_b200 import _lib, envs
    n, L = N_BIG, _lib.lib()
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env, params = envs.make(MCAR, flatten_obs=True, rng_mode=part)
        oenv = X.make(MCAR)
        key, kr = jr.split(jr.PRNGKey(13), 2)
        rk = jr.split(kr, n)
        obs, st = env.reset(keys_t(rk), params)
        o_obs, o_st = oenv.reset(rk)
        assert np.array_equal(obs.cpu().numpy(), o_obs)
        assert np.array_equal(np_state(st), np_state(to_dev_state(MCAR, o_st)))
        rng = np.random.default_rng(part)
        worst = 0.0
        for t in range(205):
            key, ks = jr.split(key, 2)
            sk = jr.split(ks, n)
            act = rng.integers(0, 3, n).astype(np.int32)
            prev = o_st
            obs, st, r, d, info = env.step(keys_t(sk), to_dev_state(MCAR, o_st), t_(act), params)
            o_obs, o_st, o_r, o_d, o_info = oenv.step(sk, o_st, act)
            assert np.array_equal(d.cpu().numpy(), o_d), t
            assert np.array_equal(r.cpu().numpy(), o_r), t
            hs = np_state(st)
            worst = max(worst, assert_mcar_close(hs, o_st, prev, t))
            f = fields(MCAR, hs)
            assert np.array_equal(obs.cpu().numpy(), np.stack([f["position"], f["velocity"]], 1)), t
            for k in ("discount", "returned_episode_returns", "returned_episode_lengths", "timestep"):
                assert np.array_equal(info[k].cpu().numpy(), o_info[k]), (t, k)
            if t == 199:   # random play truncates; the auto-reset is bit-exact
                assert o_d.mean() > 0.99
                assert np.array_equal(hs[:2, o_d], np_state(to_dev_state(MCAR, o_st))[:2, o_d])
            ob2 = torch.empty((n, 2), device=dev())
            _lib.check(L.pqn_env_obs(env.env_id, _lib.p(st), _lib.p(ob2), n, _lib.stream_ptr()), "pqn_env_obs")
            assert torch.equal(ob2, obs), t
        print(f"MountainCar GPU vs oracle: worst velocity error {worst:.2f} ulps")
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def test_mountain_car_left_wall_and_goal_on_device():
    """Hand-set states: cars pushed into the left wall come back at -1.2 with velocity -0.0; a car just below the goal
    moving right crosses it (done, reward -1, bit-exact auto-reset and LogWrapper words); cars at the goal moving left
    and cars at 199 steps (truncation) as the oracle says."""
    from purejaxql_b200 import envs
    n = 4096
    rng = np.random.default_rng(3)
    kind = np.arange(n) % 4
    pos = np.where(kind == 0, rng.uniform(-1.2, -1.185, n), np.where(kind == 1, rng.uniform(0.47, 0.4999, n),
                   np.where(kind == 2, 0.5, rng.uniform(-0.6, -0.4, n)))).astype(np.float32)
    vel = np.where(kind == 0, rng.uniform(-0.07, -0.02, n), np.where(kind == 1, rng.uniform(0.03, 0.07, n),
                   np.where(kind == 2, -0.004, 0.0))).astype(np.float32)
    st = dict(position=pos, velocity=vel, time=np.where(kind == 3, 199, 20).astype(np.int32),
              log_episode_returns=np.full(n, -20, np.float32), log_episode_lengths=np.full(n, 20, np.int32),
              log_returned_episode_returns=np.zeros(n, np.float32), log_returned_episode_lengths=np.zeros(n, np.int32),
              log_timestep=np.full(n, 20, np.int32))
    act = np.where(kind == 0, 0, np.where(kind == 1, 2, 1)).astype(np.int32)
    sk = jr.split(jr.PRNGKey(4), n)
    env, params = envs.make(MCAR, flatten_obs=True)
    oenv = X.make(MCAR)
    obs, dst, r, d, info = env.step(keys_t(sk), to_dev_state(MCAR, st), t_(act), params)
    o_obs, o_st, o_r, o_d, o_info = oenv.step(sk, st, act)
    d = d.cpu().numpy()
    assert np.array_equal(d, o_d) and np.array_equal(d, kind % 2 == 1)
    assert (r.cpu().numpy() == -1).all()
    f = fields(MCAR, np_state(dst))
    wall = kind == 0
    assert (f["position"][wall] == np.float32(-1.2)).all()
    assert (f["velocity"][wall].view(np.int32) == np.float32(-0.0).view(np.int32)).all()
    assert_mcar_close(np_state(dst), o_st, st, "wall/goal")
    assert np.array_equal(np_state(dst)[:, d], np_state(to_dev_state(MCAR, o_st))[:, d])
    assert (info["returned_episode_lengths"].cpu().numpy()[d] == 21).all()


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("name", [MCAR, CATCH])
@pytest.mark.parametrize("done_only", [0, 1])
def test_rollout_act_step_matches_oracle(name, done_only, part):
    """The fused eps-greedy + step + LogWrapper launch over 3 seeds x 33,335 envs (100,005 in all; not a multiple of
    the block) x 14 steps, in both threefry layouts: actions, rewards, dones, max q, the obs rows and the info sums.
    MountainCar starts at times 186-199 so that episodes truncate inside the window, and is teacher-forced (its obs
    rows within the step's ulp bar)."""
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        _rollout_act_step_against_oracle(name, done_only, part)
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def _rollout_act_step_against_oracle(name, done_only, part):
    from purejaxql_b200 import _lib, envs
    L = _lib.lib()
    S, E, T, eps, rew_scale = 3, 33_335, 14, 0.4, 0.5
    env, _ = envs.make(name, flatten_obs=True, rng_mode=part)
    oenv = X.make(name)
    D = env.obs_dim
    seeds = jr.split(jr.PRNGKey(78), S)
    rk = np.stack([jr.split(seeds[s], E) for s in range(S)])
    o = [oenv.reset(rk[s]) for s in range(S)]
    o_obs, o_st = [x[0] for x in o], [x[1] for x in o]
    if name == MCAR:
        for s in range(S):
            o_st[s]["time"] = np.random.default_rng(s).integers(186, 200, E).astype(np.int32)
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
        if name == MCAR:
            state = torch.cat([to_dev_state(name, o_st[s]) for s in range(S)], 1).contiguous()
        prev = [dict(x) for x in o_st]
        q = rng.standard_normal((S * E, 3)).astype(np.float32)
        step_keys = np.stack([np.stack(jr.split(jr.PRNGKey(1000 * t + s), 2)) for s in range(S)])
        keys_d, q_d = keys_t(step_keys), t_(q)
        _lib.check(L.pqn_rollout_act_step(env.env_id, _lib.p(keys_d), _lib.p(q_d), _lib.p(eps_d),
                                          _lib.p(state), _lib.raw(obs_buf[:, t + 1]), (T + 1) * E, _lib.raw(act[:, t]),
                                          _lib.raw(rew[:, t]), _lib.raw(done[:, t]), _lib.raw(maxq[:, t]), T * E,
                                          _lib.p(sums), done_only, S, E, 0, 0, 0, rew_scale, part, _lib.stream_ptr()),
                   "pqn_rollout_act_step")
        for s in range(S):
            qs = q.reshape(S, E, 3)[s]
            a = R.eps_greedy(jr.split(step_keys[s, 0], E), qs, eps)
            o_obs[s], o_st[s], r, d, info = oenv.step(jr.split(step_keys[s, 1], E), o_st[s], a)
            assert np.array_equal(act[s, t].cpu().numpy(), a), (t, s)
            assert np.array_equal(rew[s, t].cpu().numpy(), (np.float32(rew_scale) * r).astype(np.float32)), (t, s)
            assert np.array_equal(done[s, t].cpu().numpy().astype(bool), d), (t, s)
            assert np.array_equal(maxq[s, t].cpu().numpy(), qs.max(-1)), (t, s)
            sst = np_state(state[:, s * E:(s + 1) * E])
            if name == CATCH:
                assert np.array_equal(obs_buf[s, t + 1].cpu().numpy(), o_obs[s]), (t, s)
                assert_catch_state(state[:, s * E:(s + 1) * E], o_st[s], (t, s))
            else:
                assert_mcar_close(sst, o_st[s], prev[s], (t, s))
                f = fields(MCAR, sst)
                assert np.array_equal(obs_buf[s, t + 1].cpu().numpy(), np.stack([f["position"], f["velocity"]], 1))
            m = d if done_only else np.ones(E, bool)
            o_sums[s] += [info["returned_episode_returns"][m].astype(np.float64).sum(),
                          info["returned_episode_lengths"][m].sum(), info["timestep"][m].sum(), d.sum(),
                          info["discount"][m].sum()]
    assert np.array_equal(sums.cpu().numpy(), o_sums)
    assert o_sums[:, 3].min() > 0


# --------------------------------------------------------------------------- #
# networks at D = 2 and D = 50
# --------------------------------------------------------------------------- #
WIDTHS = [(D, H) for D in (2, 50) for H in (64, 128, 256, 512)]


@pytest.mark.parametrize("D,H", WIDTHS)
def test_mlp_forward_and_loss_grad_at_new_widths(D, H, tc_path):
    from purejaxql_b200 import _lib
    A, S, total, rows, Ls = 3, 2, 1400, 515, 2
    spec, ps, flat = NS._mlp_setup(D, H, Ls, A, S, 40)
    rng = np.random.default_rng(D + H)
    obs = rng.standard_normal((S, total, D)).astype(np.float32)
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


@pytest.mark.parametrize("D,H", WIDTHS)
def test_rnn_step_and_window_loss_grad_at_new_widths(D, H, tc_path):
    from purejaxql_b200 import _lib
    S, A, Ls, E, T, B = 2, 3, 2, 37, 9, 5
    spec, ps, flat = NS._rnn_setup(S, D, A, H, Ls)
    rng = np.random.default_rng(D * H)
    hs = rng.standard_normal((S, E, H)).astype(np.float32) * 0.5
    obs = rng.standard_normal((S, E, D)).astype(np.float32)
    ld = rng.random((S, E)) < 0.3
    la = rng.integers(0, A, (S, E)).astype(np.int32)
    # every device buffer is bound to a name, so that none is freed (and reused) before the launch
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
    w, bufs = RNS._window(S, T, B, D, A, H, seed=D + H)
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


NORMS6 = [(nt, ni) for nt in ("layer_norm", "batch_norm", "none") for ni in (False, True)]


@pytest.mark.parametrize("norm_type,norm_input", NORMS6)
def test_mlp_norm_variants_at_d50(norm_type, norm_input, tc_path):
    """Eval forward, loss / gradients and the updated batch_stats (hidden in place, input through bn_sums) at D = 50,
    as test_gpu_net_shapes checks them at D = 4."""
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_MLP, QNetworkSpec
    D, A, H, Ls, S, total, rows = 50, 3, 256, 2, 2, 300, 256
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
    obs = (rng.random((S, total, D)) < 0.04).astype(np.float32) * rng.uniform(0.5, 2.0, D).astype(np.float32)
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
            errs[name] = (float(np.abs(NS._leaf(gtree, path, s) - g[name]).max() / scale), tol)
        bad = {k: v for k, v in errs.items() if not v[0] < v[1]}
        assert not bad, (bad, errs)
        for path, off, n in spec.stats_entries():
            d = sttree
            for k in path:
                d = d[k]
            want = new_stats["/".join(path)]
            assert np.allclose(d["mean"][s].cpu().numpy(), want["mean"], atol=2e-6), path
            assert np.allclose(d["var"][s].cpu().numpy(), want["var"], atol=2e-6), path


@pytest.mark.parametrize("D", [50, 300, 1024])
@pytest.mark.parametrize("norm_type,norm_input", NORMS6)
def test_rnn_norm_variants_at_wide_inputs(norm_type, norm_input, D, tc_path):
    """The GRU's *_stats entry points at D = 50 (Catch), and at 300 and 1024, where the per-channel tables grow past
    256 channels (all three were refused before: the input BatchNorm took at most 16 features or a divisor of 256):
    the eval step with the running statistics, and the window loss / gradients with every running statistic updated
    in place, as test_gpu_rnn_norm checks them at D = 3."""
    from purejaxql_b200 import _lib
    S, A, H, Ls, E, T, B = 2, 3, 128, 2, 37, 10, 5
    spec, ps, sts, flat, stats = RNS._setup(S, D, A, H, Ls, norm_type, norm_input)
    hs, obs, ld, la = RNS._step_inputs(S, E, D, A, H, 5)
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
    grads = torch.zeros_like(flat)
    ls, qs = torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
    _lib.check(RNS._loss(spec, flat, stats, bufs, grads, ls, qs, S, T, B, NS._ws(spec, S, T * B)),
               "pqn_rnn_loss_grad_stats")
    torch.cuda.synchronize()
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
            errs[name] = (float(np.abs(NS._leaf(gtree, path, s) - g[name]).max() / scale), tol)
        bad = {k: v for k, v in errs.items() if not v[0] < v[1]}
        assert not bad, (bad, errs)
        for path, off, n in spec.stats_entries():
            want = new_stats["/".join(path)]
            d = sttree
            for k in path:
                d = d[k]
            assert np.abs(d["mean"][s].cpu().numpy() - want["mean"]).max() < 2e-6, path
            assert np.abs(d["var"][s].cpu().numpy() - want["var"]).max() < 2e-6, path


def test_rnn_stats_refuses_inputs_beyond_1024():
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_RNN, QNetworkSpec
    spec = QNetworkSpec(NET_RNN, 1025, 3, 64, 1, norm_type="batch_norm", norm_input=True)
    st = torch.zeros((1, spec.stats_total), device=dev())
    rc = _lib.lib().pqn_rnn_step_stats(spec.desc, None, _lib.p(st), None, None, 1, None, None, None, 1, 1, None,
                                       _lib.stream_ptr())
    assert rc == -3 and b"1024" in _lib.lib().pqn_last_error()


# --------------------------------------------------------------------------- #
# whole runs
# --------------------------------------------------------------------------- #
def test_mlp_catch_two_updates_match_oracle(monkeypatch):
    """Two whole updates of pqn_gymnax on Catch (eps = 1) against the oracle's update_step."""
    import test_gpu_train as TT
    from purejaxql_b200 import pqn_gymnax
    monkeypatch.setitem(G._REGISTRY, CATCH, X.Catch)
    cfg = TT._cfg(CATCH, HIDDEN_SIZE=128, NUM_LAYERS=2, REW_SCALE=1.0, LAMBDA=0.95, NUM_ENVS=32, NUM_STEPS=16)
    TT._run_updates_against_oracle(pqn_gymnax, CATCH, "mlp", True, cfg, nupd=2)


def test_rnn_catch_two_updates_match_oracle():
    """Two whole updates of pqn_rnn_gymnax on Catch (eps = 1; 9-step episodes end inside the 15-step windows)
    against the oracle replay of test_gpu_memory_chain."""
    import test_gpu_memory_chain as MCT
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = MCT._rnn_cfg(ENV_NAME=CATCH)
    del cfg["ENV_KWARGS"]
    nupd = 2
    cfg["TOTAL_TIMESTEPS"] = cfg["TOTAL_TIMESTEPS_DECAY"] = float(nupd * cfg["NUM_STEPS"] * cfg["NUM_ENVS"])
    train = pqn_rnn_gymnax.make_train(cfg)
    eng = train.engine
    assert eng.D == 50 and eng.max_steps == 1000
    rngs = jr.split(jr.PRNGKey(32), 2)
    cap = {}
    orig = eng.spec.init
    eng.spec.init = lambda k, d: cap.setdefault("flat", orig(k, d)).clone()
    out = train(rngs)
    dones = MCT._replay_rnn_updates(cfg, out, eng.spec.unflatten(cap["flat"]), eng.spec, rngs, nupd,
                                    lambda: X.make(CATCH))
    assert dones > 0


def _rnn_run(graph, norm_type="layer_norm", norm_input=False):
    from purejaxql_b200 import pqn_rnn_gymnax
    cfg = NS._rnn_cfg(128, 2, env=CATCH, nupd=5, graph=graph)
    cfg.update(NORM_TYPE=norm_type, NORM_INPUT=norm_input, TEST_NUM_STEPS=20)
    train = pqn_rnn_gymnax.make_train(cfg)
    out = train(jr.split(jr.PRNGKey(5), 2))
    assert train.engine.graph_captured == graph
    return (out["runner_state"][0].params_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy(),
            out["metrics"]["returned_episode_returns"].cpu().numpy(),
            out["metrics"]["test/returned_episode_lengths"].cpu().numpy(), out["runner_state"][4].cpu().numpy())


@pytest.mark.parametrize("norm_type,norm_input", [("layer_norm", False), ("batch_norm", True)])
def test_rnn_catch_cuda_graph_replay_equals_eager_and_repeats(norm_type, norm_input):
    eager, graph, again = _rnn_run(False, norm_type, norm_input), _rnn_run(True, norm_type, norm_input), \
        _rnn_run(True, norm_type, norm_input)
    for a, b, c in zip(eager, graph, again):
        assert np.array_equal(a, b, equal_nan=True) and np.array_equal(b, c, equal_nan=True)
    assert np.isfinite(eager[1]).all() and (eager[3] == 9).all()


def test_mlp_catch_is_bit_reproducible():
    from purejaxql_b200 import pqn_gymnax
    outs = []
    for _ in range(2):
        cfg = NS._mlp_cfg(256, 2)
        cfg.update(ENV_NAME=CATCH, NORM_INPUT=True)
        out = pqn_gymnax.make_train(cfg)(jr.split(jr.PRNGKey(11), 2))
        outs.append((out["runner_state"][0].params_flat.cpu().numpy(), out["metrics"]["td_loss"].cpu().numpy()))
    assert np.isfinite(outs[0][1]).all()
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("script,preset", [("pqn_gymnax", "pqn_cartpole"), ("pqn_rnn_gymnax", "pqn_rnn_cartpole")])
@pytest.mark.parametrize("name", [MCAR, CATCH])
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
    test_len = m["test/returned_episode_lengths"]
    if name == CATCH:
        assert (test_len == 9).all()
        r = m["test/returned_episode_returns"]
        assert ((r >= -1) & (r <= 1)).all()
    else:
        assert ((test_len > 0) & (test_len <= 200)).all()
    files = [p for p in tmp_path.rglob("*.safetensors")]
    assert len(files) == 2, files
    tree = load_params(str(sorted(files)[0]))
    D = {MCAR: 2, CATCH: 50}[name]
    assert tree["Dense_0"]["kernel"].shape[0] == D
