"""CPU checks for the recurrent network at the shipped presets' window lengths.

- ``oracle/pqn_rnn_ref.py``'s loss and BPTT against torch fp64 autograd of the same loss, written out independently
  (LayerNorm trunk, GRU cell with the ``last_done`` carry reset, Q head, the reverse-scan Q(lambda) targets under
  ``.detach()``, ``0.5 * mean`` over t < T-1), on a MemoryChain window of T = 132 steps with episode boundaries at
  both ends and one whole 101-step episode inside.  The GPU tests of ``test_gpu_rnn_windows.py`` use this oracle at
  these lengths as their reference.
- ``pqn_rnn_gymnax.make_train`` refuses the window shapes the recurrent loss does not take, before anything is built.

The window builders here (MemoryChain / CartPole transitions as the engine's memory stores them) are shared with
``test_gpu_rnn_windows.py``.
"""
import numpy as np
import pytest
import torch

import bsuite_oracle as MC
from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_rnn_ref as RR

F64 = np.float64
EPISODE = 101          # MemoryChain at memory_length 100: an episode lasts memory_length + 1 steps


def env_transitions(env, n, steps, seed):
    """``steps`` transitions of n envs from reset with uniform random actions, as the engine's memory stores them
    (``engine_rnn.py``): the obs before the step, ``last_done`` / ``last_action`` of the previous step (False / 0
    after the reset), the action, the reward and the done of the step.  -> dict of [steps, n, ...] arrays."""
    key, kr = jr.split(jr.PRNGKey(seed), 2)
    obs, st = env.reset(jr.split(kr, n))
    rng = np.random.default_rng(seed)
    ld, la = np.zeros(n, bool), np.zeros(n, np.int32)
    rec = {k: [] for k in ("obs", "last_done", "last_action", "action", "reward", "done")}
    for _ in range(steps):
        key, ks = jr.split(key, 2)
        act = rng.integers(0, env.num_actions, n).astype(np.int32)
        nobs, st, rew, done, _ = env.step(jr.split(ks, n), st, act)
        for k, v in (("obs", obs), ("last_done", ld), ("last_action", la), ("action", act), ("reward", rew),
                     ("done", done)):
            rec[k].append(np.asarray(v))
        obs, ld, la = nobs, np.asarray(done, bool), act
    return {k: np.stack(v) for k, v in rec.items()}


def windows(env, offsets, T, seed, hs_width=None):
    """One window of T transitions per column, column c starting ``offsets[c]`` steps after its env's reset.
    offsets [S, B] -> dict of [S, T, B, ...] arrays (obs float32, reward float32, flags bool, actions int32), plus
    a nonzero carry ``hs0`` [S, B, hs_width] when hs_width is given."""
    offsets = np.asarray(offsets)
    S, B = offsets.shape
    rec = env_transitions(env, S * B, int(offsets.max()) + T, seed)
    cols = np.arange(S * B)
    idx = offsets.reshape(-1)[None, :] + np.arange(T)[:, None]                      # [T, S*B]
    out = {}
    for k, v in rec.items():
        w = v[idx, cols[None, :]]                                                    # [T, S*B, ...]
        out[k] = np.ascontiguousarray(w.reshape(T, S, B, *v.shape[2:]).swapaxes(0, 1))
    out["obs"] = out["obs"].astype(np.float32)
    out["reward"] = out["reward"].astype(np.float32)
    if hs_width is not None:
        out["hs0"] = (np.random.default_rng(seed + 1).standard_normal((S, B, hs_width)) * 0.5).astype(np.float32)
    return out


def memory_chain_offsets(T, B, S=1, seed=0):
    """Per-column offsets into MemoryChain episodes (memory_length 100).  The first columns of every seed pin the
    boundaries the window code must handle: ``last_done`` at t = 0 with the whole episode t = 0..100 inside,
    ``done`` at t = T-2 (one whole episode ending there when T >= 102), ``done`` at t = T-1.  The rest are random."""
    rng = np.random.default_rng(seed)
    pinned = [EPISODE, (EPISODE - 1 - (T - 2)) % EPISODE, (EPISODE - 1 - (T - 1)) % EPISODE]
    off = rng.integers(0, 2 * EPISODE, (S, B))
    for s in range(S):
        for c in range(min(B, 3)):
            off[s, c] = pinned[c] + EPISODE * (c > 0)
    return off


def memory_chain_env():
    return MC.make(100, flatten=True, log=False)


def cartpole_env():
    return G.make("CartPole-v1", flatten=True, log=False)


# --------------------------------------------------------------------------------------------------------------- #
# the oracle against torch fp64 autograd
# --------------------------------------------------------------------------------------------------------------- #
def torch_loss(p, hs, obs, last_done, last_action, action, reward, done, gamma, lam):
    """The recurrent PQN loss (purejaxql/pqn_rnn_gymnax.py:57-105, :295-360) in torch fp64.
    -> loss, chosen q [(T-1)*B], {param path: leaf tensor with requires_grad}."""
    tp = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in p.items()
          if not k.startswith("BatchNorm_0")}
    L = sum(1 for k in p if k.startswith("LayerNorm_") and k.endswith("scale"))
    T, B, _ = obs.shape
    H = p["Dense_0/kernel"].shape[1]
    A = p[f"Dense_{L}/kernel"].shape[1]
    x = torch.tensor(obs, dtype=torch.float64)
    for l in range(L):
        z = x @ tp[f"Dense_{l}/kernel"] + tp[f"Dense_{l}/bias"]
        x = torch.relu(torch.nn.functional.layer_norm(z, (H,), tp[f"LayerNorm_{l}/scale"], tp[f"LayerNorm_{l}/bias"],
                                                      eps=1e-6))
    onehot = torch.nn.functional.one_hot(torch.tensor(np.asarray(last_action, np.int64)), A).to(torch.float64)
    xin = torch.cat([x, onehot], -1)
    w = {g: tp[RR.G + g + "/kernel"] for g in ("ir", "iz", "in", "hr", "hz", "hn")}
    b = {g: tp[RR.G + g + "/bias"] for g in ("ir", "iz", "in", "hn")}
    reset = torch.tensor(np.asarray(last_done, bool))
    h = torch.tensor(hs, dtype=torch.float64)
    ys = []
    for t in range(T):
        h = torch.where(reset[t][:, None], torch.zeros_like(h), h)
        r = torch.sigmoid(xin[t] @ w["ir"] + b["ir"] + h @ w["hr"])
        z = torch.sigmoid(xin[t] @ w["iz"] + b["iz"] + h @ w["hz"])
        n = torch.tanh(xin[t] @ w["in"] + b["in"] + r * (h @ w["hn"] + b["hn"]))
        h = (1 - z) * n + z * h
        ys.append(h)
    q = torch.stack(ys) @ tp[f"Dense_{L}/kernel"] + tp[f"Dense_{L}/bias"]                 # [T, B, A]
    # Q(lambda) targets: reverse scan over t = T-2 .. 0 of stop-gradient q values, bootstrapped from max_a q[T-1]
    maxq = q.detach().max(-1).values
    rw = torch.tensor(reward, dtype=torch.float64)
    dn = torch.tensor(np.asarray(done, bool)).to(torch.float64)
    ret = rw[T - 2] + gamma * (1 - dn[T - 2]) * maxq[T - 1]
    targets = [ret]
    for t in range(T - 3, -1, -1):
        boot = rw[t] + gamma * (1 - dn[t]) * maxq[t + 1]
        ret = boot + gamma * lam * (ret - maxq[t + 1])
        ret = (1 - dn[t]) * ret + dn[t] * rw[t]
        targets.insert(0, ret)
    target = torch.stack(targets)                                                            # [T-1, B]
    chosen = q[:-1].gather(-1, torch.tensor(np.asarray(action[:-1], np.int64))[..., None])[..., 0]
    loss = 0.5 * ((chosen - target) ** 2).mean()
    return loss, chosen.reshape(-1), tp


def test_memory_chain_window_has_the_pinned_boundaries():
    T, B = 132, 3
    w = windows(memory_chain_env(), memory_chain_offsets(T, B), T, seed=5)
    ld, dn = w["last_done"][0], w["done"][0]
    assert ld[0, 0] and dn[100, 0] and not dn[:100, 0].any()                    # whole episode t = 0..100
    assert dn[T - 2, 1] and dn[T - 2 - EPISODE, 1] and not dn[T - 1 - EPISODE:T - 2, 1].any()
    assert dn[T - 1, 2] and not dn[T - 2, 2]
    assert (w["obs"][0, 0, 0] == [1.0, 0.0, w["obs"][0, 0, 0, 2]]).all() and abs(w["obs"][0, 0, 0, 2]) == 1
    assert np.array_equal(ld[1:], dn[:-1])                                      # last_done is the previous done
    nz = w["reward"][0] != 0
    assert np.array_equal(nz, dn) and (np.abs(w["reward"][0][nz]) == 1).all()  # +-1 on the last step only


def test_oracle_bptt_matches_torch_autograd_at_long_window():
    """T = 132, B = 3, H = 16, L = 2 in fp64: the loss, the chosen q values and every gradient tensor of
    ``rnn_loss_and_grads`` agree with autograd to 1e-10 of the tensor's own largest entry."""
    T, B, D, A, H, L = 132, 3, 3, 2, 16, 2
    w = windows(memory_chain_env(), memory_chain_offsets(T, B), T, seed=5, hs_width=H)
    p = R.random_params(RR.rnn_param_shapes(D, A, H, L), seed=11, dtype=F64)
    for g in ("hr", "hz", "hn"):
        p[RR.G + g + "/kernel"] *= 0.5
    p[RR.G + "iz/bias"] += 2.0          # slow update gate: gradients reach far back along the window
    args = (w["hs0"][0].astype(F64), w["obs"][0].astype(F64), w["last_done"][0], w["last_action"][0], w["action"][0],
            w["reward"][0].astype(F64), w["done"][0], 0.99, 0.95)
    loss, chosen, g = RR.rnn_loss_and_grads(p, *args)
    tl, tchosen, tp = torch_loss(p, *args)
    tl.backward()
    assert abs(loss - tl.item()) <= 1e-12 * abs(loss)
    assert np.abs(chosen - tchosen.detach().numpy()).max() <= 1e-11 * np.abs(chosen).max()
    for k, v in g.items():
        if k.startswith("BatchNorm_0"):
            assert not v.any(), k                                          # its output is discarded (:75-76)
            continue
        want = tp[k].grad.numpy()
        assert np.abs(want).max() > 0, k
        assert np.abs(v - want).max() <= 1e-10 * np.abs(want).max(), (k, np.abs(v - want).max(), np.abs(want).max())


# --------------------------------------------------------------------------------------------------------------- #
# make_train refuses window shapes the recurrent loss does not take
# --------------------------------------------------------------------------------------------------------------- #
def _cfg(**kw):
    cfg = dict(ENV_NAME="MemoryChain-bsuite", TOTAL_TIMESTEPS=1e5, TOTAL_TIMESTEPS_DECAY=1e5, NUM_STEPS=128,
               MEMORY_WINDOW=4, NUM_ENVS=32, NUM_MINIBATCHES=16, ENV_KWARGS={"memory_length": 100})
    cfg.update(kw)
    return cfg


def test_make_train_refuses_unsupported_windows(monkeypatch):
    from purejaxql_b200 import pqn_rnn_gymnax
    built = []

    def fake_engine(config, env_params=None):
        built.append(config)
        raise RuntimeError("engine built")
    monkeypatch.setattr(pqn_rnn_gymnax, "PQNRnnEngine", fake_engine)
    for kw, limit in ((dict(NUM_ENVS=2050, NUM_MINIBATCHES=2), "1024"), (dict(NUM_ENVS=1025, NUM_MINIBATCHES=1), "1024"),
                      (dict(MEMORY_WINDOW=0, NUM_STEPS=1), "at least 2"), (dict(MEMORY_WINDOW=1, NUM_STEPS=0), "at least 2")):
        with pytest.raises(ValueError, match=limit):
            pqn_rnn_gymnax.make_train(_cfg(**kw))
    assert not built
    # the limits themselves are accepted (the engine is reached)
    for kw in (dict(NUM_ENVS=2048, NUM_MINIBATCHES=2), dict(MEMORY_WINDOW=1, NUM_STEPS=1), dict(ENV_NAME="CartPole-v1")):
        with pytest.raises(RuntimeError, match="engine built"):
            pqn_rnn_gymnax.make_train(_cfg(**kw))
    assert len(built) == 3
