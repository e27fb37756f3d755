"""GPU tests of the input-gradient (dgrad) epilogues of the fp16-split wgmma GEMM: the packed-bit and fp32 ReLU masks
must give exactly mask * (the unmasked product), at the shapes the Q-network's dense dgrad runs at."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_STORE, EPI_RELU_MASK, EPI_RELU_BITS = 0, 3, 4
GUARD = 4096   # floats after the output that a ragged last m-tile must not write


def dev():
    return torch.device("cuda:0")


def _planes(x):
    from purejaxql_b200 import _lib
    t = torch.from_numpy(x).to(dev())
    hi = torch.empty(t.shape, dtype=torch.float16, device=dev())
    lo = torch.empty_like(hi)
    _lib.check(_lib.lib().pqn_tc_split16(_lib.p(t), _lib.p(hi), _lib.p(lo), t.numel(), 1.0, _lib.stream_ptr()))
    return hi, lo


def _dgrad(planes, mask, bits, S, M, N, K, epi, out=None):
    from purejaxql_b200 import _lib
    if out is None:
        out = torch.full((S * M * N + GUARD,), float("nan"), device=dev())
    ptr = lambda t: _lib.p(t) if t is not None else None
    _lib.check(_lib.lib().pqn_tc_dgrad16_test(*(_lib.p(p) for p in planes), ptr(mask), ptr(bits), _lib.p(out),
                                              S, M, N, K, epi, 0.5, _lib.stream_ptr()), "pqn_tc_dgrad16_test")
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.isnan(o[S * M * N:]).all(), "rows past M were written"
    return o[:S * M * N].reshape(S, M, N)


@pytest.mark.parametrize("S,M", [(5, 4096), (2, 6536), (160, 128)])
def test_relu_epilogues_equal_masked_store(S, M):
    N, K = 1024, 128
    rng = np.random.default_rng(M + S)
    dz = rng.standard_normal((S, M, K)).astype(np.float32)
    w = (rng.standard_normal((S, N, K)) * 0.05).astype(np.float32)
    mask = rng.standard_normal((S, M, N)).astype(np.float32)
    mask[rng.random((S, M, N)) < 0.05] = 0.0
    bits = np.packbits((mask > 0).reshape(S, M, N // 32, 32), axis=-1, bitorder="little").view(np.uint32)[..., 0]
    planes = (*_planes(dz), *_planes(w))
    tmask = torch.from_numpy(mask).to(dev())
    tbits = torch.from_numpy(np.ascontiguousarray(bits)).to(dev())

    plain = _dgrad(planes, None, None, S, M, N, K, EPI_STORE)
    assert np.isfinite(plain).all()
    want = np.where(mask > 0, plain, np.float32(0.0)).view(np.uint32)

    got_bits = _dgrad(planes, None, tbits, S, M, N, K, EPI_RELU_BITS)
    assert np.array_equal(got_bits.view(np.uint32), want)
    got_mask = _dgrad(planes, tmask, None, S, M, N, K, EPI_RELU_MASK)
    assert np.array_equal(got_mask.view(np.uint32), want)
    # in place, as the network's dgrad runs when the mask is the fp32 activation itself
    inplace = torch.cat([tmask.reshape(-1), torch.full((GUARD,), float("nan"), device=dev())])
    got_inplace = _dgrad(planes, inplace, None, S, M, N, K, EPI_RELU_MASK, out=inplace)
    assert np.array_equal(got_inplace.view(np.uint32), want)
