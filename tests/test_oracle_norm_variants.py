"""CPU tests of oracle/pqn_ref_norm.py (NORM_TYPE / NORM_INPUT variants, SURVEY section 8(f) row 4): the analytic
backward agrees with central finite differences in fp64, the shared configuration (layer_norm, NORM_INPUT=False)
reproduces oracle/pqn_ref.py exactly, and BatchNorm follows flax's train/eval and running-statistics rules.  The CNN
is pinned at every channel count the library builds (CNN_SHAPES: the games' C with their action counts), since the
GPU tests compare the variant kernels with this oracle at each of them."""
import numpy as np
import pytest

from oracle import pqn_ref as R
from oracle import pqn_ref_norm as N

F64 = np.float64
VARIANTS = [("layer_norm", False), ("layer_norm", True), ("batch_norm", False), ("batch_norm", True), ("none", False)]
CNN_VARIANTS = VARIANTS + [("none", True)]
CNN_SHAPES = [(4, 3), (6, 4), (7, 3), (10, 6)]      # (C, A): Breakout, SpaceInvaders, Freeway, Seaquest


def _fd_check(loss_fn, p, keys, rng, n_probe=6, h=1e-6, rtol=2e-6):
    _, _, g, _ = loss_fn(p)
    for k in keys:
        flat = p[k].reshape(-1)
        for idx in rng.choice(flat.size, size=min(n_probe, flat.size), replace=False):
            old = flat[idx]
            flat[idx] = old + h
            lp = loss_fn(p)[0]
            flat[idx] = old - h
            lm = loss_fn(p)[0]
            flat[idx] = old
            fd = (lp - lm) / (2 * h)
            an = g[k].reshape(-1)[idx]
            assert abs(fd - an) <= rtol * max(1.0, abs(fd), abs(an)) + 1e-9, (k, idx, fd, an)


@pytest.mark.parametrize("norm_type,norm_input", CNN_VARIANTS)
@pytest.mark.parametrize("C,A", CNN_SHAPES, ids=["C%dA%d" % s for s in CNN_SHAPES])
def test_cnn_variant_grads_match_finite_differences(C, A, norm_type, norm_input):
    rng = np.random.default_rng(3 + C)
    B = 6
    p = R.random_params(N.cnn_param_shapes(C, A, norm_type), seed=1, dtype=F64)
    stats = N.cnn_batch_stats(C, norm_type, F64)
    obs = (rng.random((B, 10, 10, C)) < 0.2).astype(F64)
    act = rng.integers(0, A, B)
    tgt = rng.standard_normal(B)
    fn = lambda q: N.cnn_loss_and_grads(q, stats, obs, act, tgt, norm_type, norm_input)
    keys = [k for k in p if norm_input or not k.startswith("BatchNorm_0")]
    _fd_check(fn, p, keys, rng)
    if not norm_input:  # the dummy input BatchNorm never receives gradient (pqn_minatar.py:64-66)
        g = fn(p)[2]
        assert not g["BatchNorm_0/scale"].any() and not g["BatchNorm_0/bias"].any()


@pytest.mark.parametrize("norm_type,norm_input", VARIANTS)
def test_mlp_variant_grads_match_finite_differences(norm_type, norm_input):
    rng = np.random.default_rng(4)
    D, A, H, B = 6, 3, 16, 9
    p = R.random_params(N.mlp_param_shapes(D, A, H, 2, norm_type), seed=2, dtype=F64)
    stats = N.mlp_batch_stats(D, H, 2, norm_type, F64)
    obs = rng.standard_normal((B, D))
    act = rng.integers(0, A, B)
    tgt = rng.standard_normal(B)
    fn = lambda q: N.mlp_loss_and_grads(q, stats, obs, act, tgt, norm_type, norm_input)
    keys = [k for k in p if norm_input or not k.startswith("BatchNorm_0")]
    _fd_check(fn, p, keys, rng)


def test_shared_configuration_reproduces_pqn_ref_exactly():
    rng = np.random.default_rng(5)
    C, A, B = 4, 3, 17
    p = R.random_params(R.cnn_param_shapes(C, A), seed=7)
    assert set(p) == set(N.cnn_param_shapes(C, A, "layer_norm"))
    obs = (rng.random((B, 10, 10, C)) < 0.2).astype(np.float32)
    act = rng.integers(0, A, B)
    tgt = rng.standard_normal(B).astype(np.float32)
    stats = N.cnn_batch_stats(C)
    q, _ = N.cnn_forward(p, stats, obs, train=False)
    assert np.array_equal(q, R.cnn_forward(p, obs))
    l0, qs0, g0 = R.cnn_loss_and_grads(p, obs, act, tgt)
    l1, qs1, g1, ns = N.cnn_loss_and_grads(p, stats, obs, act, tgt)
    assert l0 == l1 and np.array_equal(qs0, qs1) and all(np.array_equal(g0[k], g1[k]) for k in g0)
    # the dummy BatchNorm's running statistics follow pqn_ref.bn_batch_stats_update (pqn_minatar.py:293-296)
    ref = R.bn_batch_stats_update(stats["BatchNorm_0"], obs)
    assert np.array_equal(ns["BatchNorm_0"]["mean"], ref["mean"]) and np.array_equal(ns["BatchNorm_0"]["var"], ref["var"])
    D, H = 4, 32
    pm = R.random_params(R.mlp_param_shapes(D, 2, H, 2), seed=8)
    assert set(pm) == set(N.mlp_param_shapes(D, 2, H, 2, "layer_norm"))
    x = rng.standard_normal((B, D)).astype(np.float32)
    assert np.array_equal(N.mlp_forward(pm, N.mlp_batch_stats(D, H, 2), x, False)[0], R.mlp_forward(pm, x))


def test_batch_norm_train_eval_and_running_statistics():
    rng = np.random.default_rng(6)
    x = rng.standard_normal((50, 3, 8)) * 2.0 + 1.0
    scale, bias = rng.standard_normal(8), rng.standard_normal(8)
    stats = {"mean": np.zeros(8), "var": np.ones(8)}
    y, _, ns = N.batch_norm_fwd(x, scale, bias, stats, train=True)
    xr = x.reshape(-1, 8)
    assert np.allclose(((y - bias) / scale).reshape(-1, 8).mean(0), 0, atol=1e-12)
    assert np.allclose(ns["mean"], 0.99 * 0 + 0.01 * xr.mean(0)) and np.allclose(ns["var"], 0.99 + 0.01 * xr.var(0))
    y_eval, _, same = N.batch_norm_fwd(x, scale, bias, ns, train=False)
    assert same is ns
    assert np.allclose(y_eval, (x - ns["mean"]) / np.sqrt(ns["var"] + 1e-5) * scale + bias)


def test_batch_norm_tree_names_follow_flax_auto_naming():
    assert "CNN_0/BatchNorm_1/scale" in N.cnn_param_shapes(4, 3, "batch_norm")
    assert "CNN_0/LayerNorm_0/scale" not in N.cnn_param_shapes(4, 3, "batch_norm")
    s = N.mlp_param_shapes(4, 2, 256, 2, "batch_norm")
    assert {"BatchNorm_0/scale", "BatchNorm_1/scale", "BatchNorm_2/scale"} <= set(s) and "LayerNorm_0/scale" not in s
    assert set(N.mlp_batch_stats(4, 256, 2, "batch_norm")) == {"BatchNorm_0", "BatchNorm_1", "BatchNorm_2"}
    assert not any("Norm_1" in k for k in N.cnn_param_shapes(4, 3, "none") if k.startswith("CNN_0"))


@pytest.mark.parametrize("norm_input", [False, True])
@pytest.mark.parametrize("C,A", CNN_SHAPES, ids=["C%dA%d" % s for s in CNN_SHAPES])
def test_cnn_batch_norm_variant_matches_torch_autograd(C, A, norm_input):
    """Independent pin: the batch_norm network built from torch primitives (batch_norm in training mode normalises
    with the biased batch variance, like flax) and differentiated by torch autograd, fp64.  The running statistics
    (new_stats) of all three BatchNorms follow flax: 0.99 of the old ones plus 0.01 of the biased batch statistics of
    each BatchNorm's input, from non-trivial old ones."""
    import torch
    rng = np.random.default_rng(12 + C)
    B = 7
    p = R.random_params(N.cnn_param_shapes(C, A, "batch_norm"), seed=13 + C, dtype=F64)
    stats = {k: {"mean": 0.1 * rng.standard_normal(v["mean"].shape), "var": 0.5 + rng.random(v["var"].shape)}
             for k, v in N.cnn_batch_stats(C, "batch_norm", F64).items()}
    obs = (rng.random((B, 10, 10, C)) < 0.25).astype(F64)
    act, tgt = rng.integers(0, A, B), rng.standard_normal(B)
    loss, _, g, new_stats = N.cnn_loss_and_grads(p, stats, obs, act, tgt, "batch_norm", norm_input)
    tp = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in p.items()}
    bn = lambda x, name: torch.nn.functional.batch_norm(x, None, None, tp[name + "/scale"], tp[name + "/bias"],
                                                        training=True, eps=1e-5)
    x0 = torch.tensor(obs).permute(0, 3, 1, 2)                        # NCHW: batch_norm reduces over N, H, W
    x = bn(x0, "BatchNorm_0") if norm_input else x0 / 255.0
    z1 = torch.nn.functional.conv2d(x, tp["CNN_0/Conv_0/kernel"].permute(3, 2, 0, 1), tp["CNN_0/Conv_0/bias"])
    h = torch.relu(bn(z1, "CNN_0/BatchNorm_0")).permute(0, 2, 3, 1).reshape(B, -1)
    z2 = h @ tp["CNN_0/Dense_0/kernel"] + tp["CNN_0/Dense_0/bias"]
    q = torch.relu(bn(z2, "CNN_0/BatchNorm_1")) @ tp["Dense_0/kernel"] + tp["Dense_0/bias"]
    tl = 0.5 * ((q[torch.arange(B), torch.tensor(act)] - torch.tensor(tgt)) ** 2).mean()
    tl.backward()
    assert abs(float(tl.detach()) - loss) < 1e-12
    for k in p:
        ref = tp[k].grad.numpy() if tp[k].grad is not None else np.zeros_like(p[k])
        assert np.allclose(g[k], ref, rtol=1e-8, atol=1e-11), k
    for name, z in (("BatchNorm_0", x0), ("CNN_0/BatchNorm_0", z1), ("CNN_0/BatchNorm_1", z2)):
        zr = z.detach().transpose(0, 1).reshape(z.shape[1], -1) if z.dim() == 4 else z.detach().T
        mean, var = zr.mean(1).numpy(), zr.var(1, unbiased=False).numpy()
        assert np.allclose(new_stats[name]["mean"], 0.99 * stats[name]["mean"] + 0.01 * mean, rtol=1e-12, atol=1e-14), name
        assert np.allclose(new_stats[name]["var"], 0.99 * stats[name]["var"] + 0.01 * var, rtol=1e-10, atol=1e-14), name
