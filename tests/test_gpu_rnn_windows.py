"""The recurrent (GRU) Q-network on the GPU against fp64 at the shapes the recurrent presets run at: windows of
T = MEMORY_WINDOW + NUM_STEPS = 68 (CartPole) and 132 (MemoryChain) steps, the scan kernels' CTA geometry (RB = 4
batch rows per CTA, up to 9 CTAs and a ragged last one), the targets kernel's block (up to B = 1024 threads) and its
smallest window (T = 2), and the chained rollout form over MemoryChain's 1000-step evaluation.

Inputs are MemoryChain episodes (memory_length 100, random actions) from ``tests/bsuite_oracle.py``, so ``obs``,
``done``, ``last_done``, ``last_action`` and the +-1 rewards are consistent, with episode boundaries at both ends of
the window and one whole 101-step episode inside it; the CartPole case runs the CartPole oracle.  The reference is
``oracle/pqn_rnn_ref.py`` (``tests/rnn_norm_oracle.py`` for the ``_stats`` entries) in fp64; it is pinned against
torch autograd at these lengths by ``test_oracle_rnn_windows.py``.

Tolerance rule.  Every tensor (each gradient leaf, the loss, the mean chosen q, q and the carry of the rollout, the
running statistics) is held to two bars:
  - the project's global bar: ``err <= 2e-5 * max |g|`` over all gradient tensors;
  - its own scale: ``err <= max(C_SPREAD * spread32, FLOOR * max |want|)`` with ``C_SPREAD = 8`` and
    ``FLOOR = 2**-20`` (8 fp32 ulps of the tensor's largest entry).  ``spread32`` is how far the same oracle run in
    fp32 NumPy lands from fp64 on that tensor, at the same inputs; the test computes it.  ``err`` and ``spread32``
    are max-abs differences from fp64.
The floor is for scalars and tensors on which NumPy's pairwise / blocked fp32 sums land well inside one ulp of fp64:
there the ratio measures NumPy's luck, not the kernel.  On the H100 the only tensor it decides is the mean chosen q.

Measured on one NVIDIA H100 80GB HBM3 (700 W power limit), worst err / spread32 per test:
  - window loss and gradients: gradient tensors 5.9 (``iz/bias``, H = 512), the loss 4.9; the mean chosen q up to 25
    (B = 33), inside the floor (a serial fp32 sum over the window's steps against NumPy's pairwise mean);
  - the z ~ 0.95 long-range windows: 9.6 (``ir/bias``), 8.1 (``in/bias``); see that test for why they get
    ``C_SLOW_GATE = 16``;
  - the chained rollout: 1.8 (q and the carry); carry error at the last step / at step 100 (50): 0.92-1.22;
  - the ``_stats`` entries: 3.5 (``iz/kernel``), running statistics 1.0.
Numeric mutations of the kernels fail these tests by 1e5-1e7 x spread32 (a backward scan that drops the carry gradient
every 64 steps, zero gradients for batch rows >= 8, ``done`` read one step late from t = 32), while
``test_gpu_rnn.py`` and ``test_gpu_net_shapes.py`` still pass under each of them.
"""
import numpy as np
import pytest
import torch

import rnn_norm_oracle as RO
from oracle import pqn_ref as R
from oracle import pqn_rnn_ref as RR
from test_oracle_rnn_windows import EPISODE, cartpole_env, env_transitions, memory_chain_env, memory_chain_offsets, windows

pytestmark = pytest.mark.gpu

PQN_E_INVALID = -1
C_SPREAD = 8.0
FLOOR = 2.0 ** -20
C_SLOW_GATE = 16.0     # the z ~ 0.95 case only: see test_context_bit_reaches_the_query_step_100_steps_later
DRIFT = 2.0            # carry error at the last rollout step over its error at step 100 (50)
GAMMA, LAM = 0.99, 0.95
F64, F32 = np.float64, np.float32


def dev():
    return torch.device("cuda:0")


def t_(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


def _params(S, D, A, H, Ls, norm_type="layer_norm", iz_bias=None):
    """S parameter sets (different per seed) at the scales of test_gpu_rnn.py; norm scales / biases away from (1, 0)."""
    ps = []
    for s in range(S):
        p = R.random_params(RO.rnn_param_shapes(D, A, H, Ls, norm_type), 70 + s)
        for g in ("hr", "hz", "hn"):
            p[RR.G + g + "/kernel"] = (p[RR.G + g + "/kernel"] * 0.5).astype(F32)
        if norm_type != "layer_norm":
            rng = np.random.default_rng(s)
            for k in p:
                if k.startswith(("BatchNorm_", "LayerNorm_")):
                    p[k] = (p[k] + rng.standard_normal(p[k].shape) * 0.2).astype(F32)
        if iz_bias is not None:
            p[RR.G + "iz/bias"] = np.full_like(p[RR.G + "iz/bias"], iz_bias)
        ps.append(p)
    return ps


def _spec(D, A, H, Ls, norm_type="layer_norm", norm_input=False):
    from purejaxql_b200.networks import NET_RNN, QNetworkSpec
    return QNetworkSpec(NET_RNN, D, A, H, Ls, norm_type=norm_type, norm_input=norm_input)


def _flat(spec, ps):
    return torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()


def _ws(spec, S, rows):
    from purejaxql_b200 import _lib
    return torch.empty(int(_lib.lib().pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())


def _cast(p, dt):
    return {k: v.astype(dt) for k, v in p.items()}


def _bufs(w):
    return [t_(w["hs0"], torch.float32), t_(w["obs"], torch.float32), t_(w["last_done"].astype(np.uint8), torch.uint8),
            t_(w["last_action"], torch.int32), t_(w["action"], torch.int32), t_(w["reward"], torch.float32),
            t_(w["done"].astype(np.uint8), torch.uint8)]


def _leaves(spec, tree, s):
    out = {}
    for path, *_ in spec.entries:
        d = tree
        for k in path:
            d = d[k]
        out["/".join(path)] = d[s].cpu().numpy().astype(F64)
    return out


def gpu_loss_grad(spec, flat, w, stats=None, fn="pqn_rnn_loss_grad"):
    """-> per seed: {path: gradient}, loss, mean chosen q (and the running statistics with fn=..._stats)."""
    from purejaxql_b200 import _lib
    L = _lib.lib()
    S, T, B = w["action"].shape
    grads = torch.zeros_like(flat)
    ls, qs = torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
    ws = _ws(spec, S, T * B)
    ptrs = [_lib.p(b) for b in _bufs(w)]
    if fn == "pqn_rnn_loss_grad":
        rc = L.pqn_rnn_loss_grad(spec.desc, _lib.p(flat), *ptrs, _lib.p(grads), _lib.p(ls), _lib.p(qs), S, T, B, GAMMA,
                                 LAM, _lib.p(ws), _lib.stream_ptr())
    else:
        rc = L.pqn_rnn_loss_grad_stats(spec.desc, _lib.p(flat), _lib.p(stats), *ptrs, _lib.p(grads), _lib.p(ls),
                                       _lib.p(qs), S, T, B, GAMMA, LAM, _lib.p(ws), _lib.stream_ptr())
    _lib.check(rc, fn)
    torch.cuda.synchronize()
    tree = spec.unflatten(grads)
    return [dict(_leaves(spec, tree, s), loss=float(ls[s]), qsa_mean=float(qs[s])) for s in range(S)]


def oracle_loss_grad(p, w, s, dt, norm_type=None, norm_input=False, stats=None):
    """The oracle's window loss for seed s in dtype dt -> {path: gradient, loss, qsa_mean[, stats leaves]}."""
    args = (_cast(p, dt), w["hs0"][s].astype(dt), w["obs"][s].astype(dt), w["last_done"][s], w["last_action"][s],
            w["action"][s], w["reward"][s].astype(dt), w["done"][s], GAMMA, LAM)
    if norm_type is None:
        loss, chosen, g = RR.rnn_loss_and_grads(*args)
        new = None
    else:
        st = {k: {kk: vv.astype(dt) for kk, vv in v.items()} for k, v in stats.items()}
        loss, chosen, g, new = RO.rnn_loss_and_grads(*args, norm_type, norm_input, st)
    out = {k: v.astype(F64) for k, v in g.items()}
    out.update(loss=F64(loss), qsa_mean=F64(chosen.mean()))
    if new is not None:
        for k, v in new.items():
            out[k + "/mean"], out[k + "/var"] = v["mean"].astype(F64), v["var"].astype(F64)
    return out


def check_per_tensor(got, want64, want32, where, global_keys=None, c=C_SPREAD, strict=True):
    """Both bars of the module docstring.  Prints the worst err / spread32 and the worst err in fp32 ulps of the
    tensor's largest entry (the figures quoted in the docstrings); returns the failures (asserts them if strict)."""
    gk = global_keys if global_keys is not None else [k for k in want64 if k not in ("loss", "qsa_mean")]
    gscale = max(float(np.abs(want64[k]).max()) for k in gk) if gk else 0.0
    bad, worst, ulps = {}, (0.0, None), (0.0, None)
    for k, want in want64.items():
        err = float(np.abs(np.asarray(got[k], F64) - want).max())
        spread = float(np.abs(np.asarray(want32[k], F64) - want).max())
        top = float(np.abs(want).max())
        bound = max(c * spread, FLOOR * top)
        if k in gk and not err <= 2e-5 * gscale:
            bad[k] = ("global", err, 2e-5 * gscale)
        if not err <= bound:
            bad[k] = ("own", err, spread, bound)
        if spread > 0 and err / spread > worst[0]:
            worst = (err / spread, k)
        if top > 0 and err / (top * 2.0 ** -23) > ulps[0]:
            ulps = (err / (top * 2.0 ** -23), k)
    print(f"{where}: worst err/spread32 = {worst[0]:.2f} ({worst[1]}); worst err = {ulps[0]:.1f} ulps ({ulps[1]})")
    if strict:
        assert not bad, (where, bad)
    return bad


# --------------------------------------------------------------------------------------------------------------- #
# 2. the window loss and gradients at the presets' shapes
# --------------------------------------------------------------------------------------------------------------- #
WINDOW_CASES = [
    # env, H, L, D, A, T, B
    ("memory_chain", 256, 2, 3, 2, 132, 2),      # the MemoryChain preset
    ("cartpole", 256, 2, 4, 2, 68, 2),           # the CartPole preset
    ("memory_chain", 512, 2, 3, 2, 132, 2),      # 512-thread scan CTAs
    ("memory_chain", 128, 2, 3, 2, 132, 33),     # 9 scan CTAs, the last with one row; a two-warp targets block
    ("memory_chain", 128, 1, 3, 2, 3, 1024),     # the targets kernel's largest block
    ("memory_chain", 128, 2, 3, 2, 2, 7),        # one loss step
]


def _window(env, T, B, S, H, seed):
    if env == "memory_chain":
        return windows(memory_chain_env(), memory_chain_offsets(T, B, S, seed), T, seed, hs_width=H)
    w = windows(cartpole_env(), np.random.default_rng(seed).integers(0, 60, (S, B)), T, seed, hs_width=H)
    w["reward"] = (w["reward"] * F32(0.1)).astype(F32)                              # the preset's REW_SCALE
    return w


@pytest.mark.parametrize("env,H,Ls,D,A,T,B", WINDOW_CASES)
def test_window_loss_grad_per_tensor(env, H, Ls, D, A, T, B):
    """pqn_rnn_loss_grad with S = 3 seeds of different parameters: loss, mean chosen q and every gradient tensor,
    under both bars of the module docstring (C_SPREAD = 8, FLOOR = 2**-20).  Worst err / spread32 on the H100: 5.9 on
    a gradient tensor, 4.9 on the loss; the mean chosen q up to 25, inside the floor."""
    S = 3
    spec = _spec(D, A, H, Ls)
    ps = _params(S, D, A, H, Ls)
    w = _window(env, T, B, S, H, seed=H + T + B)
    got = gpu_loss_grad(spec, _flat(spec, ps), w)
    for s in range(S):
        check_per_tensor(got[s], oracle_loss_grad(ps[s], w, s, F64), oracle_loss_grad(ps[s], w, s, F32),
                         f"{env} H={H} L={Ls} T={T} B={B} seed {s}")


# --------------------------------------------------------------------------------------------------------------- #
# 3. a gradient that reaches 100 steps back
# --------------------------------------------------------------------------------------------------------------- #
def _chain_q(spec, flat, S, A, obs, ld, la, hs0, at):
    """pqn_rnn_step chained over obs [S, n, E, D] with the carry updated in place; -> q [S, E, A] after step `at`."""
    from purejaxql_b200 import _lib
    L = _lib.lib()
    E = obs.shape[2]
    hs = t_(hs0, torch.float32)
    obs_d = t_(obs.swapaxes(0, 1), torch.float32)                   # [n, S, E, D]: one contiguous block per step
    ld_d = t_(ld.swapaxes(0, 1).astype(np.uint8), torch.uint8)
    la_d = t_(la.swapaxes(0, 1), torch.int32)
    q = torch.zeros((S * E, A), device=dev())
    ws = _ws(spec, S, E)
    for t in range(at + 1):
        _lib.check(L.pqn_rnn_step(spec.desc, _lib.p(flat), _lib.p(hs), _lib.p(obs_d[t]), E, _lib.p(ld_d[t]),
                                  _lib.p(la_d[t]), _lib.p(q), S, E, _lib.p(ws), _lib.stream_ptr()), "pqn_rnn_step")
    torch.cuda.synchronize()
    return q.cpu().numpy().reshape(S, E, A).astype(F64)


def test_context_bit_reaches_the_query_step_100_steps_later():
    """The MemoryChain preset's network (H = 256, L = 2) with the update-gate bias ``iz/bias = +3`` (z ~ 0.95), so the
    carry keeps ~5 % of its signal after 64 steps and the gradient terms from far back are well above the tolerance
    (a backward scan cut after 64 steps fails the per-tensor check).  Two windows (T = 132, B = 2) differ only in
    the context bit at the first step of the episode t = 0..100 (obs column 2 at t = 0, column 0).
      - the fp64 q difference at the episode's query step (t = 100) is >= 1e-3, so the test can see the memory;
      - the GPU q difference (rollout form) matches it to 1 % of it;
      - both windows pass the per-tensor gradient check, with ``C_SLOW_GATE = 16`` in place of 8.
    Why 16: measured on the H100, the gradients of the r and n gate biases land at 9.6x (``ir/bias``) and 8.1x
    (``in/bias``) NumPy's fp32 spread, 14-19 ulps of their largest entry; every other tensor stays under 8x.  torch's
    fp32 CPU autograd lands at 1.2x and 0.65x on the same two tensors, so this is the kernels' summation order, not
    a wrong term: the backward scan forms each step's carry gradient as one serial fp32 FMA chain of 3H = 768 terms
    and the gate pre-activations as chains of H terms, where BLAS sums in blocks.  With z ~ 0.95 the carry gradient
    integrates those rounding errors over ~1 / (1 - z) = 20 steps, and the r / n gradients are scaled by (1 - z),
    so they are small next to the error they inherit.  A scan cut after 64 steps misses by 1e6x spread32."""
    S, D, A, H, Ls, T, B = 2, 3, 2, 256, 2, 132, 2
    spec = _spec(D, A, H, Ls)
    ps = _params(S, D, A, H, Ls, iz_bias=3.0)
    flat = _flat(spec, ps)
    wa = windows(memory_chain_env(), memory_chain_offsets(T, B, S, 3), T, 3, hs_width=H)
    assert wa["last_done"][:, 0, 0].all() and wa["done"][:, EPISODE - 1, 0].all()
    assert (np.abs(wa["obs"][:, 0, 0, 2]) == 1).all()
    wb = {k: v.copy() for k, v in wa.items()}
    wb["obs"][:, 0, 0, 2] *= -1
    qt = EPISODE - 1                                                              # the query (last) step
    both = {k: np.concatenate([wa[k], wb[k]], axis=2) for k in ("obs", "last_done", "last_action")}
    q_gpu = _chain_q(spec, flat, S, A, both["obs"], both["last_done"], both["last_action"],
                     np.concatenate([wa["hs0"], wb["hs0"]], axis=1), qt)
    for s in range(S):
        p64 = _cast(ps[s], F64)
        qa = RR.rnn_forward(p64, wa["hs0"][s].astype(F64), wa["obs"][s].astype(F64), wa["last_done"][s],
                            wa["last_action"][s])[1]
        qb = RR.rnn_forward(p64, wb["hs0"][s].astype(F64), wb["obs"][s].astype(F64), wb["last_done"][s],
                            wb["last_action"][s])[1]
        dq64 = qa[qt, 0] - qb[qt, 0]
        dq_gpu = q_gpu[s, 0] - q_gpu[s, B]
        print(f"seed {s}: fp64 dq = {dq64}, gpu dq = {dq_gpu}")
        assert np.abs(dq64).max() >= 1e-3, dq64
        assert np.abs(dq_gpu - dq64).max() <= 0.01 * np.abs(dq64).max(), (dq_gpu, dq64)
        assert np.array_equal(qa[:, 1], qb[:, 1])                                 # the other column is untouched
    bad = {}
    for name, w in (("a", wa), ("b", wb)):
        got = gpu_loss_grad(spec, flat, w)
        for s in range(S):
            where = f"long range window {name} seed {s}"
            bad[where] = check_per_tensor(got[s], oracle_loss_grad(ps[s], w, s, F64),
                                          oracle_loss_grad(ps[s], w, s, F32), where, c=C_SLOW_GATE, strict=False)
    assert not any(bad.values()), bad


# --------------------------------------------------------------------------------------------------------------- #
# 4. the rollout form, chained as the engine runs it
# --------------------------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize("n,E,S", [(1000, 128, 2), (132, 32, 3), (132, 1029, 1)])
def test_chained_rollout_steps(n, E, S):
    """pqn_rnn_step n times with the carry updated in place, on MemoryChain episodes started at random phases (so
    ``last_done`` resets each env every 101 steps, staggered across envs), at the MemoryChain preset's network.
    (1000, 128, 2) is the preset's evaluation; E = 1029 is ragged for RB = 4 and for the trunk's row tiles.  q and
    the carry are compared with a chained fp64 oracle every 10 steps under the per-tensor rule, and the carry error
    at the last step must stay within DRIFT = 2 x its error at step 100 (or 50 for n < 1000).
    Measured on the H100: worst err / spread32 1.8; carry error at step 1000 / step 100 = 0.99 and 0.92 (8.5e-7,
    7.2e-7 absolute), and 1.00-1.22 for the 132-step runs."""
    from purejaxql_b200 import _lib
    L = _lib.lib()
    D, A, H, Ls = 3, 2, 256, 2
    spec = _spec(D, A, H, Ls)
    ps = _params(S, D, A, H, Ls)
    flat = _flat(spec, ps)
    rng = np.random.default_rng(E)
    off = rng.integers(0, EPISODE, S * E)
    rec = env_transitions(memory_chain_env(), S * E, EPISODE + n, seed=E)
    idx = off[None, :] + np.arange(n)[:, None]
    cols = np.arange(S * E)[None, :]
    obs = rec["obs"][idx, cols].reshape(n, S, E, D).astype(F32)
    ld = rec["last_done"][idx, cols].reshape(n, S, E)
    la = rec["last_action"][idx, cols].reshape(n, S, E).astype(np.int32)
    assert ld.sum(0).min() >= n // EPISODE
    hs0 = (rng.standard_normal((S, E, H)) * 0.5).astype(F32)
    hs = t_(hs0, torch.float32)
    obs_d, ld_d, la_d = t_(obs, torch.float32), t_(ld.astype(np.uint8), torch.uint8), t_(la, torch.int32)
    q = torch.zeros((S * E, A), device=dev())
    ws = _ws(spec, S, E)
    checks = list(range(9, n, 10))
    snap_q = torch.zeros((len(checks), S * E, A), device=dev())
    snap_h = torch.zeros((len(checks), S, E, H), device=dev())
    c = 0
    for t in range(n):
        _lib.check(L.pqn_rnn_step(spec.desc, _lib.p(flat), _lib.p(hs), _lib.p(obs_d[t]), E, _lib.p(ld_d[t]),
                                  _lib.p(la_d[t]), _lib.p(q), S, E, _lib.p(ws), _lib.stream_ptr()), "pqn_rnn_step")
        if c < len(checks) and t == checks[c]:
            snap_q[c].copy_(q)
            snap_h[c].copy_(hs)
            c += 1
    torch.cuda.synchronize()
    snap_q = snap_q.cpu().numpy().reshape(len(checks), S, E, A).astype(F64)
    snap_h = snap_h.cpu().numpy().astype(F64)
    for s in range(S):
        herr = {}
        for dt in (F64, F32):
            p = _cast(ps[s], dt)
            h = hs0[s].astype(dt)
            out = []
            for t in range(n):
                h, qq = RR.rnn_forward(p, h, obs[t, s][None].astype(dt), ld[t, s][None], la[t, s][None])
                if t in checks:
                    out.append((qq[0].astype(F64), h.astype(F64)))
            if dt is F64:
                ref64 = out
            else:
                ref32 = out
        for c, t in enumerate(checks):
            check_per_tensor({"q": snap_q[c, s], "carry": snap_h[c, s]}, {"q": ref64[c][0], "carry": ref64[c][1]},
                             {"q": ref32[c][0], "carry": ref32[c][1]}, f"rollout n={n} E={E} seed {s} step {t + 1}",
                             global_keys=[])
            herr[t + 1] = float(np.abs(snap_h[c, s] - ref64[c][1]).max())
        early = 100 if n >= 1000 else 50
        print(f"rollout n={n} E={E} seed {s}: carry err at step {early} = {herr[early]:.3g}, at step {checks[-1] + 1} "
              f"= {herr[checks[-1] + 1]:.3g}, max = {max(herr.values()):.3g}")
        assert herr[checks[-1] + 1] <= DRIFT * herr[early], herr


# --------------------------------------------------------------------------------------------------------------- #
# 5. the _stats entries at the preset window
# --------------------------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize("norm_type,norm_input", [("batch_norm", True), ("layer_norm", False)])
def test_stats_entry_at_preset_window(norm_type, norm_input):
    """pqn_rnn_loss_grad_stats at (H, L, T, B) = (256, 2, 132, 2) on MemoryChain windows against
    tests/rnn_norm_oracle.py: every gradient tensor, the loss, the mean chosen q and every running statistic under
    the per-tensor rule.  ("layer_norm", False) is the default network with a non-NULL batch_stats block: only
    BatchNorm_0's statistics move, over all 264 rows of the window.
    Worst err / spread32 on the H100: 1.55 (batch_norm + NORM_INPUT), 3.5 (default network)."""
    S, D, A, H, Ls, T, B = 2, 3, 2, 256, 2, 132, 2
    spec = _spec(D, A, H, Ls, norm_type, norm_input)
    ps = _params(S, D, A, H, Ls, norm_type)
    sts = []
    rng = np.random.default_rng(7)
    for s in range(S):
        st = RO.rnn_init_stats(D, H, Ls, norm_type)
        for v in st.values():
            v["mean"] = (rng.standard_normal(v["mean"].shape) * 0.3).astype(F32)
            v["var"] = rng.uniform(0.5, 2.0, v["var"].shape).astype(F32)
        sts.append(st)
    stats = torch.cat([spec.flatten_stats(st, 1, dev()) for st in sts], 0).contiguous()
    w = windows(memory_chain_env(), memory_chain_offsets(T, B, S, 11), T, 11, hs_width=H)
    got = gpu_loss_grad(spec, _flat(spec, ps), w, stats, fn="pqn_rnn_loss_grad_stats")
    sttree = spec.unflatten_stats(stats)
    for s in range(S):
        for path, *_ in spec.stats_entries():
            d = sttree
            for k in path:
                d = d[k]
            got[s]["/".join(path) + "/mean"] = d["mean"][s].cpu().numpy()
            got[s]["/".join(path) + "/var"] = d["var"][s].cpu().numpy()
        want64 = oracle_loss_grad(ps[s], w, s, F64, norm_type, norm_input, sts[s])
        want32 = oracle_loss_grad(ps[s], w, s, F32, norm_type, norm_input, sts[s])
        assert {k for k in want64 if k.endswith(("/mean", "/var"))} == {k for k in got[s] if k.endswith(("/mean", "/var"))}
        gk = [k for k in want64 if k not in ("loss", "qsa_mean") and not k.endswith(("/mean", "/var"))]
        check_per_tensor(got[s], want64, want32, f"stats {norm_type} {norm_input} seed {s}", global_keys=gk)


# --------------------------------------------------------------------------------------------------------------- #
# 6. the refusals
# --------------------------------------------------------------------------------------------------------------- #
def test_loss_grad_refuses_one_step_window_and_1025_trajectories():
    """Both window-loss entry points return PQN_E_INVALID at T = 1 and at B = 1025 (the targets kernel runs one
    thread per trajectory in one block); nothing is launched, so the small buffers are never read."""
    from purejaxql_b200 import _lib
    L = _lib.lib()
    spec = _spec(3, 2, 128, 2)
    flat = _flat(spec, _params(1, 3, 2, 128, 2))
    buf = torch.zeros(64, device=dev())
    grads = torch.zeros_like(flat)
    ws = _ws(spec, 1, 8)
    for T, B in ((1, 2), (2, 1025), (1, 1025)):
        args = [_lib.p(buf)] * 7 + [_lib.p(grads), _lib.p(buf), _lib.p(buf), 1, T, B, GAMMA, LAM, _lib.p(ws),
                                    _lib.stream_ptr()]
        assert L.pqn_rnn_loss_grad(spec.desc, _lib.p(flat), *args) == PQN_E_INVALID, (T, B)
        assert b"B <= 1024" in L.pqn_last_error()
        assert L.pqn_rnn_loss_grad_stats(spec.desc, _lib.p(flat), None, *args) == PQN_E_INVALID, (T, B)
        assert b"T >= 2" in L.pqn_last_error()
    torch.cuda.synchronize()
    assert not grads.any()
