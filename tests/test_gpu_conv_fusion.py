"""The conv-fused dense forward of ``pqn_qnet_forward`` (``pqn_set_conv_fusion``) against the unfused kernels, bit
for bit.

With tensor-core path 2 and conv path 1 the MinAtar CNN's dense forward computes the conv output h1 itself from the
packed observations instead of reading the h1 planes a conv kernel wrote.  Every h1 element goes through the same conv
MMA chain, LayerNorm and fp16 split as in the conv kernel, and the GEMM keeps its k order and promotion, so the Q
values are expected to be identical, not merely close.

Cases: C = 4, 6, 7 and 10 channels; 100, 128, 390, 4096 and 4097 rows (partial and whole 128-row tiles); 1 and 3
seeds with their own parameters and boards; with and without a minibatch gather index; the engine's initial
parameters (conv bias 0, so an empty 3x3 patch has rstd = 1000) and random parameters.  Boards are random bits at a
density drawn per board from [0, 0.5], with an empty board and a full board among the rows read.
"""
import numpy as np
import pytest
import torch

from oracle import pqn_ref as R
from test_oracle_cnn_grads import pack_obs

pytestmark = pytest.mark.gpu

ROWS = (100, 128, 390, 4096, 4097)
SEEDS = (1, 3)
EXTRA = 37          # observation rows per seed beyond `rows`: the gather reads a subset of them
A = 6


def dev():
    return torch.device("cuda:0")


def _lib():
    from purejaxql_b200 import _lib
    return _lib


def t_(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


@pytest.fixture
def fusion():
    L = _lib().lib()
    yield lambda mode: _lib().check(L.pqn_set_conv_fusion(mode), "pqn_set_conv_fusion")
    _lib().check(L.pqn_set_conv_fusion(1))


def cnn_spec(C):
    from purejaxql_b200.networks import NET_CNN, QNetworkSpec
    return QNetworkSpec(NET_CNN, C, A)


def make_inputs(C, S, rows, regime, gathered, seed):
    """Flat parameters [S, P], packed boards [S, total, PW] and gather [S, rows] or None."""
    from purejaxql_b200 import jaxrandom
    spec = cnn_spec(C)
    rng = np.random.default_rng(seed)
    total = rows + EXTRA
    if regime == "init":
        flat = spec.init(jaxrandom.split(jaxrandom.PRNGKey(seed, dev()), S), dev())
    else:
        flat = torch.cat([spec.flatten(R.random_params(R.cnn_param_shapes(C, A), seed + s), 1, dev())
                          for s in range(S)], 0)
    boards = rng.random((S, total, 10, 10, C)) < rng.random((S, total, 1, 1, 1)) * 0.5
    boards[:, 0] = False
    boards[:, 1] = True
    packed = np.stack([pack_obs(b) for b in boards])
    gather = None
    if gathered:
        gather = np.stack([np.concatenate([[1, 0], rng.permutation(np.arange(2, total))[:rows - 2]]) for _ in range(S)])
        gather = rng.permuted(gather, axis=1).astype(np.int32)
    return spec, flat.contiguous(), packed, gather, total


def run_forward(spec, flat, packed, gather, total, S, rows):
    L = _lib().lib()
    p = _lib().p
    q = torch.zeros((S * rows, A), device=dev())
    ws = torch.empty(int(L.pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())
    g = t_(gather, torch.int32) if gather is not None else None
    _lib().check(L.pqn_qnet_forward(spec.desc, p(flat), None, p(t_(packed, torch.int32)), p(g) if g is not None else None,
                                    total, p(q), S, rows, p(ws), _lib().stream_ptr()), "pqn_qnet_forward")
    torch.cuda.synchronize()
    return {"q": q.cpu().numpy()}


def bits_differ(got, want):
    """-> names of the tensors whose fp32 bit patterns differ, with the count of differing elements"""
    out = []
    for k in want:
        d = int((got[k].view(np.uint32) != want[k].view(np.uint32)).sum())
        if d:
            out.append((k, d, float(np.abs(got[k] - want[k]).max())))
    return out


@pytest.mark.parametrize("gathered", [True, False], ids=["gather", "nogather"])
@pytest.mark.parametrize("regime", ["init", "random"])
@pytest.mark.parametrize("C", [4, 6, 7, 10])
def test_forward_bit_identical(fusion, C, regime, gathered):
    bad = []
    for rows in ROWS:
        for S in SEEDS:
            spec, flat, packed, gather, total = make_inputs(C, S, rows, regime, gathered, 1000 * C + rows + S)
            fusion(0)
            want = run_forward(spec, flat, packed, gather, total, S, rows)
            fusion(1)
            got = run_forward(spec, flat, packed, gather, total, S, rows)
            assert np.isfinite(want["q"]).all()
            diff = bits_differ(got, want)
            if diff:
                bad.append((rows, S, diff))
    assert not bad, bad


def test_fusion_mode_checked():
    L = _lib().lib()
    assert L.pqn_set_conv_fusion(2) != 0
    assert L.pqn_set_conv_fusion(-1) != 0
    _lib().check(L.pqn_set_conv_fusion(1))
