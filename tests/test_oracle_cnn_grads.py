"""CPU checks for the MinAtar CNN's loss and gradients at every channel count the library builds.

- ``oracle.pqn_ref.cnn_loss_and_grads`` against torch fp64 autograd of the same loss, written out independently
  (``conv2d`` on the /255 input, LayerNorm with flax's fast variance and eps 1e-6, ReLU, Dense, LayerNorm, ReLU, Q head,
  ``0.5 * mean`` of the squared TD error of the chosen action), at C = 6, 7 and 10 channels and 3, 5 and 18 actions.
  The GPU tests of ``test_gpu_cnn_grads.py`` use this oracle at these widths as their fp64 reference.
- The input builders those GPU tests share, defined here: packed observation rows, the minibatch gather, the TD-error
  targets of each scale and the game-density observations with an empty board and a full channel among them.
"""
import numpy as np
import pytest
import torch

from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R

F64, F32 = np.float64, np.float32

GAMES = {4: "Breakout-MinAtar", 6: "SpaceInvaders-MinAtar", 7: "Freeway-MinAtar"}
# C = 10 (MinAtar Seaquest's channel count) has no env here: its synthetic boards set each cell of channel c
# independently with probability SYNTH_DENSITY[c], 0.5-5 %, so that a cell is empty with probability 0.82 and about one
# 3x3 patch in six is empty, between the built games' boards
SYNTH_DENSITY = (0.005, 0.005, 0.01, 0.01, 0.01, 0.02, 0.02, 0.03, 0.04, 0.05)
EMPTY_ROW, FULL_ROW = 0, 1      # the observation rows that hold an empty board and a board with one channel all set


def pack_obs(obs_bool):
    """[N,10,10,C] {0,1} -> int32[N, PW] packed rows (bit f of the row = flat index f of the HWC board), the layout
    of ``pqn_env_obs_packed``."""
    n = obs_bool.shape[0]
    flat = obs_bool.reshape(n, -1).astype(np.uint8)
    nb = flat.shape[1]
    pw = ((nb + 31) // 32 + 3) // 4 * 4
    padded = np.zeros((n, pw * 32), np.uint8)
    padded[:, :nb] = flat
    by = np.packbits(padded, axis=-1, bitorder="little")
    return np.ascontiguousarray(by).view("<u4").view(np.int32)


def game_obs(C, n, seed, steps=40):
    """n boards of C channels as training sees them: the game of that width after ``steps`` uniform random actions
    from reset (C = 4, 6, 7), or the synthetic boards of SYNTH_DENSITY (C = 10).  Row EMPTY_ROW is an empty board
    and row FULL_ROW has its last channel entirely set.  -> bool[n, 10, 10, C]"""
    if C in GAMES:
        env = G.make(GAMES[C], log=False)
        key, kr = jr.split(jr.PRNGKey(seed), 2)
        obs, st = env.reset(jr.split(kr, n))
        rng = np.random.default_rng(seed)
        for _ in range(steps):
            key, ks = jr.split(key, 2)
            obs, st, *_ = env.step(jr.split(ks, n), st, rng.integers(0, env.num_actions, n).astype(np.int32))
        obs = np.asarray(obs) != 0
    else:
        rng = np.random.default_rng(seed)
        obs = rng.random((n, 10, 10, C)) < np.asarray(SYNTH_DENSITY[:C])
    obs = obs.copy()
    obs[EMPTY_ROW] = False
    obs[FULL_ROW, :, :, C - 1] = True
    return obs


def minibatch_gather(total, rows, rng):
    """``rows`` distinct row indices out of ``total`` in random order, EMPTY_ROW and FULL_ROW among them."""
    rest = rng.permutation(np.arange(2, total))[:rows - 2]
    return rng.permutation(np.concatenate([[EMPTY_ROW, FULL_ROW], rest])).astype(np.int32)


def td_targets(q_sa, delta, rng):
    """fp32 targets whose TD error q_sa - target is delta * eps, eps ~ N(0, 1): the gradients scale with delta."""
    return (q_sa - delta * rng.standard_normal(q_sa.shape)).astype(F32)


def cast(p, dt):
    return {k: v.astype(dt) for k, v in p.items()}


def torch_cnn_loss_grads(p, obs, action, target):
    """The CNN loss and its gradients by torch fp64 autograd.  -> loss, q_sa, {path: gradient}"""
    tp = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in p.items()}

    def ln(z, scale, bias):
        mean = z.mean(-1, keepdim=True)
        var = torch.clamp((z * z).mean(-1, keepdim=True) - mean * mean, min=0.0)
        return (z - mean) / torch.sqrt(var + R.LN_EPS) * scale + bias

    x = torch.tensor(obs, dtype=torch.float64).permute(0, 3, 1, 2) / 255.0
    w = tp["CNN_0/Conv_0/kernel"].permute(3, 2, 0, 1)                       # HWIO -> OIHW
    z1 = torch.nn.functional.conv2d(x, w).permute(0, 2, 3, 1) + tp["CNN_0/Conv_0/bias"]
    h1 = torch.relu(ln(z1, tp["CNN_0/LayerNorm_0/scale"], tp["CNN_0/LayerNorm_0/bias"])).reshape(obs.shape[0], -1)
    z2 = h1 @ tp["CNN_0/Dense_0/kernel"] + tp["CNN_0/Dense_0/bias"]
    h2 = torch.relu(ln(z2, tp["CNN_0/LayerNorm_1/scale"], tp["CNN_0/LayerNorm_1/bias"]))
    q = h2 @ tp["Dense_0/kernel"] + tp["Dense_0/bias"]
    q_sa = q[torch.arange(obs.shape[0]), torch.as_tensor(action, dtype=torch.long)]
    loss = 0.5 * ((q_sa - torch.tensor(target, dtype=torch.float64)) ** 2).mean()
    loss.backward()
    # BatchNorm_0 (the input norm, off with NORM_INPUT = False) is not on the path: no gradient, zeros as in flax
    return (float(loss.detach()), q_sa.detach().numpy(),
            {k: v.grad.numpy() if v.grad is not None else np.zeros(v.shape) for k, v in tp.items()})


@pytest.mark.parametrize("A", [3, 5, 18])
@pytest.mark.parametrize("C", [6, 7, 10])
def test_cnn_oracle_matches_torch_fp64_autograd(C, A):
    rng = np.random.default_rng(100 * C + A)
    n = 96
    p = cast(R.random_params(R.cnn_param_shapes(C, A), C + A), F64)
    obs = game_obs(C, n, seed=C, steps=15)
    act = rng.integers(0, A, n)
    tgt = rng.standard_normal(n)
    loss, q_sa, g = R.cnn_loss_and_grads(p, obs.astype(F64), act, tgt)
    tloss, tq, tg = torch_cnn_loss_grads(p, obs, act, tgt)
    assert abs(loss - tloss) <= 1e-10 * abs(tloss)
    assert np.abs(q_sa - tq).max() <= 1e-10 * np.abs(tq).max()
    assert set(g) == set(tg)
    for k in tg:
        scale = np.abs(tg[k]).max()
        if k.startswith("BatchNorm_0/"):
            assert scale == 0 and not g[k].any(), k
            continue
        assert scale > 0, k
        assert np.abs(g[k] - tg[k]).max() <= 1e-10 * scale, (k, np.abs(g[k] - tg[k]).max(), scale)


@pytest.mark.parametrize("C", [4, 6, 7, 10])
def test_game_obs_density_and_edge_rows(C):
    obs = game_obs(C, 512, seed=3)
    assert obs.shape == (512, 10, 10, C) and obs.dtype == bool
    assert not obs[EMPTY_ROW].any()
    assert obs[FULL_ROW, :, :, C - 1].all()
    dens = obs[2:].mean(axis=(0, 1, 2))
    # every channel is exercised somewhere, and the boards are sparse like MinAtar's, with empty 3x3 patches
    assert (obs[2:].any(axis=(0, 1, 2))).all(), dens
    assert 0.005 < dens.mean() < 0.25, dens
    patches = R._im2col(obs[2:].astype(F32)).reshape(-1, 9 * C).any(-1)
    assert 0.05 < patches.mean() < 0.95
    if C == 10:
        assert np.allclose(dens, SYNTH_DENSITY, atol=0.01)
    # the same seed gives the same boards; another seed others
    assert np.array_equal(obs, game_obs(C, 512, seed=3))
    assert not np.array_equal(obs[2:], game_obs(C, 512, seed=4)[2:])


@pytest.mark.parametrize("C", [4, 6, 7, 10])
def test_pack_obs_roundtrip(C):
    obs = game_obs(C, 64, seed=5)
    packed = pack_obs(obs)
    pw = packed.shape[1]
    assert packed.dtype == np.int32 and pw % 4 == 0 and pw * 32 >= 100 * C and (pw - 4) * 32 < 100 * C
    bits = np.unpackbits(packed.view(np.uint8), axis=-1, bitorder="little")
    assert np.array_equal(bits[:, :100 * C].reshape(obs.shape).astype(bool), obs)
    assert not bits[:, 100 * C:].any()


def test_minibatch_gather_is_distinct_and_holds_edge_rows():
    rng = np.random.default_rng(0)
    for total, rows in ((8192, 4096), (8194, 4097), (200, 64)):
        g = minibatch_gather(total, rows, rng)
        assert g.shape == (rows,) and g.dtype == np.int32
        assert len(np.unique(g)) == rows and g.min() >= 0 and g.max() < total
        assert EMPTY_ROW in g and FULL_ROW in g
    assert not np.array_equal(minibatch_gather(100, 50, np.random.default_rng(1)),
                              minibatch_gather(100, 50, np.random.default_rng(2)))


@pytest.mark.parametrize("delta", [1e-2, 1.0, 30.0])
def test_td_targets_scale(delta):
    q = np.random.default_rng(1).standard_normal(4096) * 3
    tgt = td_targets(q, delta, np.random.default_rng(2))
    assert tgt.dtype == F32
    eps = (q - tgt.astype(F64)) / delta
    # eps ~ N(0, 1) up to the fp32 rounding of the target (|q| ~ 3: a few 1e-7 absolute, over delta)
    assert np.abs(eps - np.random.default_rng(2).standard_normal(4096)).max() < 2e-6 * (3 + 4 * delta) / delta
    assert abs(eps.std() - 1) < 0.05 and abs(eps.mean()) < 0.05
