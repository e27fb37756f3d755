"""GPU parity tests of the Q-network / optimizer kernels through the C ABI
against the fp32/fp64 oracle.  Tolerances: Q outputs 1e-5 abs (the north-star
bar); gradients 2e-5 * scale; optimizer 1e-6."""
import numpy as np
import pytest
import torch

from oracle import gymnax_envs as G
from oracle import jax_prng as jr
from oracle import pqn_ref as R

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def pack_obs(obs_bool):
    """[N,10,10,C] {0,1} -> int32[N, PW] packed rows (bit f of the row = flat index f)."""
    n = obs_bool.shape[0]
    flat = obs_bool.reshape(n, -1).astype(np.uint8)
    nb = flat.shape[1]
    pw = ((nb + 31) // 32 + 3) // 4 * 4
    padded = np.zeros((n, pw * 32), np.uint8)
    padded[:, :nb] = flat
    by = np.packbits(padded, axis=-1, bitorder="little")            # [n, pw*4] bytes, little-endian bits
    return np.ascontiguousarray(by).view("<u4").view(np.int32)      # little-endian bytes -> words


def breakout_obs(n, seed=0, steps=30):
    env = G.make("Breakout-MinAtar", log=False)
    key = jr.PRNGKey(seed)
    obs, st = env.reset(jr.split(key, n))
    rng = np.random.default_rng(seed)
    for t in range(steps):
        obs, st, *_ = env.step(jr.split(jr.PRNGKey(seed * 1000 + t), n), st, rng.integers(0, 3, n).astype(np.int32))
    return obs


def _cnn_setup(S, rows, C=4, A=3):
    from purejaxql_b200.networks import NET_CNN, QNetworkSpec
    spec = QNetworkSpec(NET_CNN, C, A)
    ps = [R.random_params(R.cnn_param_shapes(C, A), 10 + s) for s in range(S)]
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    return spec, ps, flat


def _ws(spec, S, rows):
    from purejaxql_b200 import _lib
    n = int(_lib.lib().pqn_net_workspace_bytes(spec.desc, S, rows))
    return torch.empty(n, dtype=torch.uint8, device=dev())


@pytest.fixture(params=[(2, 1), (1, 1), (0, 0), (1, 0), (2, 3)],
                ids=["tcgen05_f16split+f16_mma_conv", "tcgen05_3xtf32+f16_mma_conv", "ffma", "tcgen05_3xtf32+cuda_conv",
                     "tcgen05_f16split+tf32_mma_conv"])
def dense_path(request):
    """Runs the CNN tests on the implementation variants: dense layer on the tensor cores (wgmma on fp16-split
    planes, the default, or 3xTF32 on mma.sync; the ids keep their original names) or fp32 FFMA; conv on fp16
    warp-level MMA (default), tf32 warp-level MMA or fp32 CUDA cores."""
    from purejaxql_b200 import _lib
    _lib.check(_lib.lib().pqn_set_tensor_core_path(request.param[0]))
    _lib.check(_lib.lib().pqn_set_conv_mma_path(request.param[1]))
    yield request.param
    _lib.lib().pqn_set_tensor_core_path(2)
    _lib.lib().pqn_set_conv_mma_path(1)


@pytest.mark.parametrize("rows", [1, 130, 515])
def test_cnn_forward_matches_oracle_1e5(rows, dense_path):
    from purejaxql_b200 import _lib
    S = 3
    spec, ps, flat = _cnn_setup(S, rows)
    obs = np.stack([breakout_obs(rows, seed=s + 1) for s in range(S)])          # [S,rows,10,10,4]
    packed = torch.from_numpy(np.stack([pack_obs(obs[s] != 0) for s in range(S)])).to(dev()).contiguous()
    q = torch.zeros((S * rows, 3), device=dev())
    ws = _ws(spec, S, rows)
    _lib.check(_lib.lib().pqn_qnet_forward(spec.desc, _lib.p(flat), None, _lib.p(packed), None, rows, _lib.p(q), S, rows,
                                           _lib.p(ws), _lib.stream_ptr()))
    q = q.cpu().numpy().reshape(S, rows, 3)
    for s in range(S):
        ref32 = R.cnn_forward(ps[s], obs[s])
        ref64 = R.cnn_forward({k: v.astype(np.float64) for k, v in ps[s].items()}, obs[s].astype(np.float64))
        assert np.abs(q[s] - ref64).max() < 1e-5, np.abs(q[s] - ref64).max()
        assert np.abs(q[s] - ref32).max() < 1e-5


def test_cnn_forward_other_channel_counts_and_gather(dense_path):
    from purejaxql_b200 import _lib
    rng = np.random.default_rng(1)
    for C in (6, 7, 10):
        S, total, rows = 2, 300, 77
        spec, ps, flat = _cnn_setup(S, rows, C=C, A=5)
        obs = (rng.random((S, total, 10, 10, C)) < 0.15)
        packed = torch.from_numpy(np.stack([pack_obs(obs[s]) for s in range(S)])).to(dev()).contiguous()
        gather = np.stack([rng.permutation(total)[:rows] for _ in range(S)]).astype(np.int32)
        q = torch.zeros((S * rows, 5), device=dev())
        tg_, ws = torch.from_numpy(gather).to(dev()), _ws(spec, S, rows)
        _lib.check(_lib.lib().pqn_qnet_forward(spec.desc, _lib.p(flat), None, _lib.p(packed), _lib.p(tg_), total, _lib.p(q),
                                               S, rows, _lib.p(ws), _lib.stream_ptr()))
        q = q.cpu().numpy().reshape(S, rows, 5)
        for s in range(S):
            ref = R.cnn_forward(ps[s], obs[s][gather[s]].astype(np.float32))
            assert np.abs(q[s] - ref).max() < 1e-5, (C, np.abs(q[s] - ref).max())


@pytest.fixture(params=[2, 0], ids=["hidden_layer_tcgen05_f16split", "ffma"])
def mlp_path(request):
    """The MLP's hidden layer (Dense_1: K = N = HIDDEN_SIZE) runs on the wgmma fp16-split GEMMs by default;
    path 0 keeps everything on the fp32 FFMA kernels."""
    from purejaxql_b200 import _lib
    _lib.lib().pqn_set_tensor_core_path(request.param)
    yield request.param
    _lib.lib().pqn_set_tensor_core_path(2)


@pytest.mark.parametrize("D,H,layers,A", [(4, 256, 2, 2), (6, 256, 2, 3), (4, 128, 1, 2), (6, 128, 2, 3)])
def test_mlp_forward_matches_oracle(D, H, layers, A, mlp_path):
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_MLP, QNetworkSpec
    rng = np.random.default_rng(2)
    S, rows = 3, 203
    spec = QNetworkSpec(NET_MLP, D, A, H, layers)
    ps = [R.random_params(R.mlp_param_shapes(D, A, H, layers), 20 + s) for s in range(S)]
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    obs = rng.standard_normal((S, rows, D)).astype(np.float32)
    q = torch.zeros((S * rows, A), device=dev())
    to_, ws = torch.from_numpy(obs).to(dev()), _ws(spec, S, rows)
    _lib.check(_lib.lib().pqn_qnet_forward(spec.desc, _lib.p(flat), None, _lib.p(to_), None, rows,
                                           _lib.p(q), S, rows, _lib.p(ws), _lib.stream_ptr()))
    q = q.cpu().numpy().reshape(S, rows, A)
    for s in range(S):
        assert np.abs(q[s] - R.mlp_forward(ps[s], obs[s])).max() < 1e-5


def _loss_grad(spec, flat, obs_t, gather, total, act, tgt, S, rows, F):
    from purejaxql_b200 import _lib
    grads = torch.zeros_like(flat)
    ls = torch.zeros(S, device=dev()); qs = torch.zeros(S, device=dev())
    bn = torch.zeros((S, 2 * F), device=dev())
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)
    tg_, ta_, tt_, ws = t(gather, torch.int32), t(act, torch.int32), t(tgt, torch.float32), _ws(spec, S, rows)
    _lib.check(_lib.lib().pqn_qnet_loss_grad(
        spec.desc, _lib.p(flat), None, _lib.p(obs_t), _lib.p(tg_), total, _lib.p(ta_),
        _lib.p(tt_), total, _lib.p(grads), _lib.p(ls), _lib.p(qs), _lib.p(bn), S, rows,
        _lib.p(ws), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return grads, ls.cpu().numpy(), qs.cpu().numpy(), bn.cpu().numpy()


def _cmp_grads(spec, grads, ref_g, s, tag):
    tree = spec.unflatten(grads)
    for path, off, shape, _ in spec.entries:
        d = tree
        for k in path:
            d = d[k]
        got = d[s].cpu().numpy()
        ref = ref_g["/".join(path)]
        scale = max(np.abs(ref).max(), 1e-3)
        err = np.abs(got - ref).max()
        assert err < 2e-5 * scale + 1e-7, (tag, path, err, scale)


@pytest.mark.parametrize("rows,total", [(64, 200), (300, 1000), (1024, 4096)])
def test_cnn_loss_grad_matches_oracle(rows, total, dense_path):
    S = 2
    spec, ps, flat = _cnn_setup(S, rows)
    rng = np.random.default_rng(rows)
    obs = np.stack([breakout_obs(total, seed=s + 3, steps=20) for s in range(S)])
    packed = torch.from_numpy(np.stack([pack_obs(obs[s] != 0) for s in range(S)])).to(dev()).contiguous()
    gather = np.stack([rng.permutation(total)[:rows] for _ in range(S)])
    act = rng.integers(0, 3, (S, total))
    tgt = rng.standard_normal((S, total)).astype(np.float32)
    grads, ls, qs, bn = _loss_grad(spec, flat, packed, gather, total, act, tgt, S, rows, 4)
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        o = obs[s][gather[s]]
        loss, q_sa, g = R.cnn_loss_and_grads(p64, o.astype(np.float64), act[s][gather[s]], tgt[s][gather[s]].astype(np.float64))
        assert abs(ls[s] - loss) < 1e-5 * max(1, abs(loss)) and abs(qs[s] - q_sa.mean()) < 1e-5
        _cmp_grads(spec, grads, g, s, "cnn")
        xr = o.reshape(-1, 4)
        assert np.allclose(bn[s, :4], xr.sum(0)) and np.allclose(bn[s, 4:], (xr * xr).sum(0))


@pytest.mark.parametrize("D,H,layers,A,rows", [(4, 256, 2, 2, 32), (6, 256, 2, 3, 515), (4, 128, 1, 2, 100), (6, 128, 2, 3, 256)])
def test_mlp_loss_grad_matches_oracle(D, H, layers, A, rows, mlp_path):
    from purejaxql_b200.networks import NET_MLP, QNetworkSpec
    rng = np.random.default_rng(7)
    S, total = 2, 700
    spec = QNetworkSpec(NET_MLP, D, A, H, layers)
    ps = [R.random_params(R.mlp_param_shapes(D, A, H, layers), 30 + s) for s in range(S)]
    flat = torch.cat([spec.flatten(p, 1, dev()) for p in ps], 0).contiguous()
    obs = rng.standard_normal((S, total, D)).astype(np.float32)
    gather = np.stack([rng.permutation(total)[:rows] for _ in range(S)])
    act = rng.integers(0, A, (S, total))
    tgt = rng.standard_normal((S, total)).astype(np.float32)
    grads, ls, qs, bn = _loss_grad(spec, flat, torch.from_numpy(obs).to(dev()), gather, total, act, tgt, S, rows, D)
    for s in range(S):
        p64 = {k: v.astype(np.float64) for k, v in ps[s].items()}
        o = obs[s][gather[s]].astype(np.float64)
        loss, q_sa, g = R.mlp_loss_and_grads(p64, o, act[s][gather[s]], tgt[s][gather[s]].astype(np.float64))
        assert abs(ls[s] - loss) < 1e-5 * max(1, abs(loss)) and abs(qs[s] - q_sa.mean()) < 1e-5
        _cmp_grads(spec, grads, g, s, "mlp")
        assert np.allclose(bn[s, :D], o.sum(0), atol=1e-3) and np.allclose(bn[s, D:], (o * o).sum(0), atol=1e-3)


def test_radam_clip_matches_oracle():
    from purejaxql_b200 import _lib
    from purejaxql_b200.engine import radam_schedule_table
    rng = np.random.default_rng(4)
    S, P, steps = 3, 1028, 12
    p = rng.standard_normal((S, P)).astype(np.float32)
    tab = radam_schedule_table(steps, lambda i: np.float32(1e-3 * (1 - i / 20)))
    tp = torch.from_numpy(p.copy()).to(dev()); mu = torch.zeros_like(tp); nu = torch.zeros_like(tp)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev()); gn = torch.zeros(S * 64, device=dev())
    refs = [({"w": p[s].copy()}, R.opt_init({"w": p[s]})) for s in range(S)]
    ttab = torch.from_numpy(tab).to(dev())
    for i in range(steps):
        g = (rng.standard_normal((S, P)) * (1.0 if i % 2 else 0.05)).astype(np.float32)   # alternate clipped / unclipped
        tgr = torch.from_numpy(g).to(dev())
        _lib.check(_lib.lib().pqn_radam_clip_step(_lib.p(tp), _lib.p(tgr), _lib.p(mu),
                                                  _lib.p(nu), _lib.p(ttab), _lib.p(cnt),
                                                  _lib.p(gn), S, P, 10.0, 0.9, 0.999, 1e-8, _lib.stream_ptr()))
        torch.cuda.synchronize()
        for s in range(S):
            pp, oo = refs[s]
            pp, oo, _ = R.radam_clip_step(pp, {"w": g[s]}, oo, tab[i, 0], 10.0)
            refs[s] = (pp, oo)
    assert int(cnt.item()) == steps
    for s in range(S):
        assert np.abs(tp[s].cpu().numpy() - refs[s][0]["w"]).max() < 2e-6


def test_device_param_init_distribution_and_determinism():
    from purejaxql_b200 import jaxrandom
    from purejaxql_b200.networks import NET_CNN, NET_MLP, QNetworkSpec
    keys = jaxrandom.split(jaxrandom.PRNGKey(0, dev()), 4)
    for spec in (QNetworkSpec(NET_CNN, 4, 3), QNetworkSpec(NET_MLP, 6, 3, 256, 2)):
        a = spec.init(keys, dev())
        b = spec.init(keys, dev())
        assert torch.equal(a, b)                                   # deterministic in the keys
        tree = spec.unflatten(a)
        assert not torch.equal(a[0], a[1])                         # seeds differ
        for path, off, shape, kind in spec.entries:
            d = tree
            for k in path:
                d = d[k]
            w = d.cpu().numpy()
            if kind == "ones":
                assert (w == 1).all()
            elif kind == "zeros":
                assert (w == 0).all()
            else:
                fan_in = int(np.prod(shape[:-1]))
                target = np.sqrt((2.0 if kind == "he" else 1.0) / fan_in)
                assert np.abs(w).max() <= 2.0 * target / 0.87962566 + 1e-6       # truncated at 2 sigma
                if w.size > 4000:
                    assert abs(w.std() / target - 1.0) < 0.05, (path, w.std(), target)
                    assert abs(w.mean()) < 0.05 * target
