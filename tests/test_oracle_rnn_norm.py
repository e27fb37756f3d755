"""The recurrent network's NORM_TYPE x NORM_INPUT oracle (tests/rnn_norm_oracle.py), on the CPU: fp64 finite
differences of its gradients for the five non-default combinations, exact agreement with oracle/pqn_rnn_ref.py on the
default one, train-mode BatchNorm over the whole [T][B] window against torch.nn.BatchNorm1d, and its parameter and
batch_stats trees against the flax-named layout of QNetworkSpec(NET_RNN, ...)."""
import numpy as np
import pytest
import torch

import rnn_norm_oracle as RO
from oracle import pqn_ref as R
from oracle import pqn_rnn_ref as RR

VARIANTS = [("layer_norm", True), ("batch_norm", False), ("batch_norm", True), ("none", False), ("none", True)]


def _window(D, A, H, Ls, T, B, norm_type, seed, dtype=np.float64):
    rng = np.random.default_rng(seed)
    p = R.random_params(RO.rnn_param_shapes(D, A, H, Ls, norm_type), seed)
    p = {k: v.astype(dtype) for k, v in p.items()}
    for g in ("hr", "hz", "hn"):
        p[RR.G + g + "/kernel"] = p[RR.G + g + "/kernel"] * dtype(0.5)
    for k in p:   # non-trivial norm scales / biases, so their gradients are not the identity's
        if k.endswith("/scale") or (k.startswith(("BatchNorm_", "LayerNorm_")) and k.endswith("/bias")):
            p[k] = (p[k] + rng.standard_normal(p[k].shape) * 0.2).astype(dtype)
    stats = RO.rnn_init_stats(D, H, Ls, norm_type, dtype)
    for v in stats.values():   # running statistics away from (0, 1)
        v["mean"] = (v["mean"] + rng.standard_normal(v["mean"].shape) * 0.3).astype(dtype)
        v["var"] = (v["var"] * rng.uniform(0.5, 2.0, v["var"].shape)).astype(dtype)
    w = dict(hs=rng.standard_normal((B, H)) * 0.5, obs=rng.standard_normal((T, B, D)) * 1.5 + 0.3,
             ld=rng.random((T, B)) < 0.2, la=rng.integers(0, A, (T, B)), ac=rng.integers(0, A, (T, B)),
             rw=rng.random((T, B)) * 0.5, dn=rng.random((T, B)) < 0.2)
    return p, stats, w


@pytest.mark.parametrize("H,Ls", [(16, 2), (8, 3)])
@pytest.mark.parametrize("norm_type,norm_input", VARIANTS)
def test_rnn_norm_grads_match_finite_differences(norm_type, norm_input, H, Ls):
    D, A, T, B = 3, 2, 6, 4
    p, stats, w = _window(D, A, H, Ls, T, B, norm_type, 11 + H + Ls)
    args = (w["hs"], w["obs"], w["ld"], w["la"], w["ac"], w["rw"], w["dn"], 0.99, 0.9, norm_type, norm_input, stats)
    loss, chosen, g, _ = RO.rnn_loss_and_grads(p, *args)
    # the in-loss targets are stop-gradient values: hold them at the unperturbed parameters' ones
    _, q = RO.rnn_forward(p, w["hs"], w["obs"], w["ld"], w["la"], False, norm_type, norm_input, stats, True)
    target = RR.compute_targets(q[-1].max(-1), q[:-1], w["rw"][:-1], w["dn"][:-1], 0.99, 0.9).reshape(-1)

    def f(pp):
        return RO.rnn_loss_and_grads(pp, *args, target=target)[0]
    assert abs(f(p) - loss) < 1e-14
    rng = np.random.default_rng(3)
    eps = 1e-6
    for k, v in p.items():
        for i in rng.choice(v.size, size=min(3, v.size), replace=False):
            pp, pm = dict(p), dict(p)
            pp[k] = v.copy().reshape(-1); pp[k][i] += eps; pp[k] = pp[k].reshape(v.shape)
            pm[k] = v.copy().reshape(-1); pm[k][i] -= eps; pm[k] = pm[k].reshape(v.shape)
            fd = (f(pp) - f(pm)) / (2 * eps)
            an = g[k].reshape(-1)[i]
            assert abs(fd - an) < 1e-6 * max(1.0, abs(fd)) + 1e-8, (k, i, fd, an)
    if not norm_input:
        assert not g["BatchNorm_0/scale"].any() and not g["BatchNorm_0/bias"].any()


def test_default_configuration_reproduces_pqn_rnn_ref_exactly():
    D, A, H, Ls, T, B = 4, 2, 16, 2, 7, 3
    p, _, w = _window(D, A, H, Ls, T, B, "layer_norm", 5)
    args = (w["hs"], w["obs"], w["ld"], w["la"], w["ac"], w["rw"], w["dn"], 0.99, 0.95)
    loss0, chosen0, g0 = RR.rnn_loss_and_grads(p, *args)
    loss1, chosen1, g1, st = RO.rnn_loss_and_grads(p, *args)
    assert st is None and loss0 == loss1 and np.array_equal(chosen0, chosen1)
    assert g0.keys() == g1.keys() and all(np.array_equal(g0[k], g1[k]) for k in g0)
    h0, q0 = RR.rnn_forward(p, w["hs"], w["obs"], w["ld"], w["la"])
    h1, q1 = RO.rnn_forward(p, w["hs"], w["obs"], w["ld"], w["la"])
    assert np.array_equal(h0, h1) and np.array_equal(q0, q1)
    assert RO.rnn_param_shapes(D, A, H, Ls) == RR.rnn_param_shapes(D, A, H, Ls)


@pytest.mark.parametrize("norm_input", [False, True])
def test_train_batch_norm_reduces_over_time_and_batch(norm_input):
    """Every BatchNorm of the train-mode forward uses the statistics of all T*B rows of the window, per feature:
    normalisation and its gradient against torch.nn.BatchNorm1d on the flattened window.  The running mean is checked
    against torch's too; the running variance against the biased variance of the rows (torch's is unbiased)."""
    D, A, H, Ls, T, B = 3, 2, 8, 2, 5, 3
    p, stats, w = _window(D, A, H, Ls, T, B, "batch_norm", 9)
    _, _, (c0, trunk, *_), new = RO.rnn_forward(p, w["hs"], w["obs"], w["ld"], w["la"], True, "batch_norm", norm_input,
                                                stats, True)
    rng = np.random.default_rng(1)
    layers = [("BatchNorm_0", w["obs"], None)]
    for l, (x_in, c, y, name) in enumerate(trunk):
        layers.append((name, x_in @ p[f"Dense_{l}/kernel"] + p[f"Dense_{l}/bias"], (c, y)))
    for name, z, cy in layers:
        F = z.shape[-1]
        bn = torch.nn.BatchNorm1d(F, eps=1e-5, momentum=0.01, dtype=torch.float64)
        with torch.no_grad():
            bn.weight.copy_(torch.from_numpy(p[name + "/scale"])); bn.bias.copy_(torch.from_numpy(p[name + "/bias"]))
            bn.running_mean.copy_(torch.from_numpy(stats[name]["mean"]))
            bn.running_var.copy_(torch.from_numpy(stats[name]["var"]))
        zt = torch.from_numpy(z.reshape(-1, F).copy()).requires_grad_(True)
        yt = bn.train()(zt)
        if cy is not None:
            c, y = cy
            assert np.abs(yt.detach().numpy().reshape(y.shape) - y).max() < 1e-12, name
            dy = rng.standard_normal(y.shape)
            dz, ds, db = RO.RN._norm_bwd(dy, c, p[name + "/scale"])
            yt.backward(torch.from_numpy(dy.reshape(-1, F)))
            assert np.abs(zt.grad.numpy().reshape(dz.shape) - dz).max() < 1e-12, name
            assert np.abs(bn.weight.grad.numpy() - ds).max() < 1e-12 and np.abs(bn.bias.grad.numpy() - db).max() < 1e-12
        assert np.abs(bn.running_mean.numpy() - new[name]["mean"]).max() < 1e-14, name
        want_var = 0.99 * stats[name]["var"] + 0.01 * z.reshape(-1, F).var(0)
        assert np.abs(new[name]["var"] - want_var).max() < 1e-13, name
    if norm_input:
        rows = w["obs"].reshape(-1, D)
        xhat = (rows - rows.mean(0)) / np.sqrt(rows.var(0) + 1e-5)
        assert np.abs(c0[0].reshape(-1, D) - xhat).max() < 1e-12


@pytest.mark.parametrize("norm_type,norm_input", VARIANTS)
def test_eval_mode_reads_running_statistics(norm_type, norm_input):
    D, A, H, Ls, T, B = 3, 2, 8, 2, 4, 3
    p, stats, w = _window(D, A, H, Ls, T, B, norm_type, 4)
    _, _, _, new = RO.rnn_forward(p, w["hs"], w["obs"], w["ld"], w["la"], True, norm_type, norm_input, stats, False)
    assert all(new[k] is stats[k] for k in stats)
    upd = RO.rnn_batch_stats(p, stats, w["hs"], w["obs"], w["ld"], w["la"], norm_type, norm_input)
    assert upd.keys() == stats.keys()
    rows = w["obs"].reshape(-1, D)
    assert np.allclose(upd["BatchNorm_0"]["mean"], 0.99 * stats["BatchNorm_0"]["mean"] + 0.01 * rows.mean(0), rtol=0,
                       atol=1e-14)


@pytest.mark.parametrize("H,Ls", [(64, 3), (512, 1), (128, 2)])
@pytest.mark.parametrize("norm_type,norm_input", VARIANTS + [("layer_norm", False)])
def test_oracle_trees_match_the_layout(norm_type, norm_input, H, Ls):
    from purejaxql_b200.networks import NET_RNN, QNetworkSpec
    D, A = 3, 2
    spec = QNetworkSpec(NET_RNN, D, A, H, Ls, norm_type=norm_type, norm_input=norm_input)
    got = {"/".join(path): tuple(shape) for path, _, shape, _ in spec.entries}
    assert got == {k: tuple(v) for k, v in RO.rnn_param_shapes(D, A, H, Ls, norm_type).items()}
    stats = RO.rnn_init_stats(D, H, Ls, norm_type)
    st_entries = {"/".join(path): (off, n) for path, off, n in spec.stats_entries()}
    assert st_entries.keys() == stats.keys()
    assert all(n == stats[k]["mean"].size for k, (_, n) in st_entries.items())
    assert spec.stats_total == sum(2 * n for _, n in st_entries.values())
    flat = spec.init_stats(1, "cpu")
    tree = spec.unflatten_stats(flat)
    for k, v in stats.items():
        d = tree
        for part in k.split("/"):
            d = d[part]
        assert np.array_equal(d["mean"][0].numpy(), v["mean"]) and np.array_equal(d["var"][0].numpy(), v["var"])
