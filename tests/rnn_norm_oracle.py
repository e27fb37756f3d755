"""NumPy restatement of the recurrent PQN network of purejaxql/pqn_rnn_gymnax.py for every ``NORM_TYPE`` x
``NORM_INPUT`` (``RNNQNetwork``, ``:57-94``), with the loss and its analytic backward (``:330-366``) and the running
statistics of the train-mode forward (``:362-369``).

Test-side oracle, built from ``oracle.pqn_rnn_ref`` (the GRU cell, the Q(lambda) targets) and ``oracle.pqn_ref_norm``
(BatchNorm forward / backward, the flax naming rule).  With the default arguments (layer_norm, NORM_INPUT=False) every
function computes what ``oracle.pqn_rnn_ref`` computes, in the same order of operations, so its results are identical.

flax semantics restated:
  - ``normalize`` is ``nn.LayerNorm()``, ``nn.BatchNorm(use_running_average=not train)`` or the identity;
  - the input goes through ``BatchNorm_0``; without NORM_INPUT its output is discarded, but in train mode its running
    statistics still move;
  - the hidden BatchNorms share the module counter with ``BatchNorm_0``: ``BatchNorm_1..L``;
  - a BatchNorm reduces over every axis but the last, so inside the loss it uses the statistics of all T*B rows of the
    window; the Q(lambda) targets are the stop-gradient of the same train-mode q values.
"""
from __future__ import annotations

import numpy as np

from oracle import pqn_ref_norm as RN
from oracle.pqn_ref import _layer_norm_bwd, _layer_norm_fwd
from oracle.pqn_rnn_ref import G, _sigmoid, compute_targets

NORM_TYPES = ("layer_norm", "batch_norm", "none")


def _norm_name(norm_type, l):
    return RN._norm_name(norm_type, "", l, bn_offset=1)


def rnn_param_shapes(D, A, hidden=128, layers=2, norm_type="layer_norm"):
    """Parameter tree of RNNQNetwork (:57-94) for obs size D, A actions; norm_type "none" has no norm parameters."""
    s = {"BatchNorm_0/scale": (D,), "BatchNorm_0/bias": (D,)}
    d_in = D
    for l in range(layers):
        s[f"Dense_{l}/kernel"], s[f"Dense_{l}/bias"] = (d_in, hidden), (hidden,)
        n = _norm_name(norm_type, l)
        if n:
            s[n + "/scale"], s[n + "/bias"] = (hidden,), (hidden,)
        d_in = hidden
    for g in ("ir", "iz", "in"):
        s[G + g + "/kernel"], s[G + g + "/bias"] = (hidden + A, hidden), (hidden,)
    for g in ("hr", "hz"):
        s[G + g + "/kernel"] = (hidden, hidden)
    s[G + "hn/kernel"], s[G + "hn/bias"] = (hidden, hidden), (hidden,)
    s[f"Dense_{layers}/kernel"], s[f"Dense_{layers}/bias"] = (hidden, A), (A,)
    return s


def rnn_init_stats(D, hidden=128, layers=2, norm_type="layer_norm", dtype=np.float32):
    """flax's initial batch_stats tree (mean 0, var 1): BatchNorm_0, and BatchNorm_1..L with batch_norm."""
    return RN.mlp_batch_stats(D, hidden, layers, norm_type, dtype)


def _layers(p):
    return sum(1 for k in p if k.startswith("Dense_") and k.endswith("kernel")) - 1


def rnn_forward(p, hs, obs, last_done, last_action, want_cache=False, norm_type="layer_norm", norm_input=False,
                batch_stats=None, train=False):
    """``network.apply({params, batch_stats}, hs, obs, done, last_action, train)`` (:64-94).
    hs [B,H]; obs [T,B,D]; last_done [T,B] bool; last_action [T,B] int -> (new_hs [B,H], q [T,B,A]) (+ cache).
    batch_stats is needed for batch_norm / NORM_INPUT and for train mode; in eval mode it is only read."""
    dt = p["Dense_0/kernel"].dtype
    T, B = obs.shape[:2]
    L = _layers(p)
    A = p[f"Dense_{L}/kernel"].shape[1]
    x_in = obs.astype(dt)
    x, c0, new_stats = x_in, None, None
    if batch_stats is not None:
        new_stats = dict(batch_stats)
        y0, c0, new_stats["BatchNorm_0"] = RN.batch_norm_fwd(x_in, p["BatchNorm_0/scale"], p["BatchNorm_0/bias"],
                                                             batch_stats["BatchNorm_0"], train)          # :72-76
        if norm_input:
            x = y0
    trunk = []
    for l in range(L):                                                                                   # :78-81
        z = x @ p[f"Dense_{l}/kernel"] + p[f"Dense_{l}/bias"]
        name = _norm_name(norm_type, l)
        if norm_type == "layer_norm":                         # the same calls as oracle.pqn_rnn_ref
            y, c = _layer_norm_fwd(z, p[name + "/scale"], p[name + "/bias"])
            c = ("ln", c)
        else:
            y, c, s = RN._norm_fwd(norm_type, z, p, name, batch_stats, train)
            if s is not None:
                new_stats[name] = s
        trunk.append((x, c, y, name))
        x = np.maximum(y, 0)
    onehot = np.zeros((T, B, A), dt)
    np.put_along_axis(onehot, np.asarray(last_action, np.int64)[..., None], 1.0, axis=-1)
    xin = np.concatenate([x, onehot], axis=-1)                                                           # :84-85
    h = hs.astype(dt)
    steps, ys = [], []
    for t in range(T):                                                                                   # :35-46
        h0 = np.where(np.asarray(last_done[t], bool)[:, None], dt.type(0), h)
        a_r = xin[t] @ p[G + "ir/kernel"] + p[G + "ir/bias"] + h0 @ p[G + "hr/kernel"]
        a_z = xin[t] @ p[G + "iz/kernel"] + p[G + "iz/bias"] + h0 @ p[G + "hz/kernel"]
        r, zg = _sigmoid(a_r), _sigmoid(a_z)
        hn = h0 @ p[G + "hn/kernel"] + p[G + "hn/bias"]
        n = np.tanh(xin[t] @ p[G + "in/kernel"] + p[G + "in/bias"] + r * hn)
        h = (1 - zg) * n + zg * h0
        steps.append((h0, r, zg, hn, n))
        ys.append(h)
    Y = np.stack(ys)
    q = Y @ p[f"Dense_{L}/kernel"] + p[f"Dense_{L}/bias"]                                                # :90
    if want_cache:
        return h, q, (c0, trunk, xin, steps, Y), new_stats
    return h, q


def rnn_batch_stats(p, batch_stats, hs, obs, last_done, last_action, norm_type="layer_norm", norm_input=False):
    """``updates["batch_stats"]`` of the loss's train-mode forward (:330-337, :362-369): the new running statistics."""
    return rnn_forward(p, hs, obs, last_done, last_action, True, norm_type, norm_input, batch_stats, True)[3]


def rnn_loss_and_grads(p, hs, obs, last_done, last_action, action, reward, done, gamma, lam, norm_type="layer_norm",
                       norm_input=False, batch_stats=None, target=None):
    """``_loss_fn`` (train=True, mutable batch_stats) + ``value_and_grad`` (:330-366) on one window [T,B,...].
    -> loss, chosen_action_qvals [(T-1)*B], grads, new batch_stats (None when batch_stats is None).
    ``target`` [(T-1)*B] replaces the in-loss Q(lambda) targets (they are stop-gradient values; a finite-difference
    check holds them fixed)."""
    new_h, q, (c0, trunk, xin, steps, Y), new_stats = rnn_forward(p, hs, obs, last_done, last_action, True, norm_type,
                                                                  norm_input, batch_stats, True)
    dt = q.dtype
    T, B, A = q.shape
    L = _layers(p)
    if target is None:
        last_q = q[-1].max(-1)                                                                           # :341-342
        target = compute_targets(last_q, q[:-1], reward[:-1].astype(dt), done[:-1], gamma, lam).reshape(-1)
    qsa = np.take_along_axis(q, np.asarray(action, np.int64)[..., None], axis=-1)[..., 0]
    chosen = qsa[:-1].reshape(-1)
    diff = chosen - target
    loss = dt.type(0.5) * np.mean(diff * diff, dtype=dt)
    dq = np.zeros_like(q)
    np.put_along_axis(dq[:-1], np.asarray(action[:-1], np.int64)[..., None],
                      (diff / dt.type(diff.size)).reshape(T - 1, B, 1), axis=-1)
    g = {k: np.zeros_like(v) for k, v in p.items()}
    H = Y.shape[-1]
    g[f"Dense_{L}/kernel"] = Y.reshape(-1, H).T @ dq.reshape(-1, A)
    g[f"Dense_{L}/bias"] = dq.reshape(-1, A).sum(0)
    dY = dq @ p[f"Dense_{L}/kernel"].T
    dxin = np.zeros_like(xin)
    dh = np.zeros((B, H), dt)
    for t in range(T - 1, -1, -1):                                                                       # BPTT
        h0, r, zg, hn, n = steps[t]
        dh = dh + dY[t]
        dn = dh * (1 - zg)
        dzg = dh * (h0 - n)
        dh0 = dh * zg
        da_n = dn * (1 - n * n)
        dr = da_n * hn
        dhn = da_n * r
        da_r = dr * r * (1 - r)
        da_z = dzg * zg * (1 - zg)
        for gate, da in (("ir", da_r), ("iz", da_z), ("in", da_n)):
            g[G + gate + "/kernel"] += xin[t].T @ da
            g[G + gate + "/bias"] += da.sum(0)
            dxin[t] += da @ p[G + gate + "/kernel"].T
        g[G + "hr/kernel"] += h0.T @ da_r
        g[G + "hz/kernel"] += h0.T @ da_z
        g[G + "hn/kernel"] += h0.T @ dhn
        g[G + "hn/bias"] += dhn.sum(0)
        dh0 = dh0 + da_r @ p[G + "hr/kernel"].T + da_z @ p[G + "hz/kernel"].T + dhn @ p[G + "hn/kernel"].T
        dh = np.where(np.asarray(last_done[t], bool)[:, None], dt.type(0), dh0)
    dx = dxin[..., :H]
    for l in reversed(range(L)):
        x_in, c, y, name = trunk[l]
        dy = dx * (y > 0)
        if c[0] == "ln":
            dz, g[name + "/scale"], g[name + "/bias"] = _layer_norm_bwd(dy, c[1], p[name + "/scale"])
        else:
            dz, ds, db = RN._norm_bwd(dy, c, p[name + "/scale"] if name else None)
            if name:
                g[name + "/scale"], g[name + "/bias"] = ds, db
        F = x_in.shape[-1]
        g[f"Dense_{l}/kernel"] = x_in.reshape(-1, F).T @ dz.reshape(-1, H)
        g[f"Dense_{l}/bias"] = dz.reshape(-1, H).sum(0)
        dx = dz @ p[f"Dense_{l}/kernel"].T
    if norm_input:   # BatchNorm_0 is on the path: its scale / bias get gradients (full train-mode backward)
        _, g["BatchNorm_0/scale"], g["BatchNorm_0/bias"] = RN.batch_norm_bwd(dx, c0, p["BatchNorm_0/scale"])
    return loss, chosen, g, new_stats
