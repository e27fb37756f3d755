"""GPU tests of the tensor-core GEMM paths (TMA ring; 3xTF32 on mma.sync, fp16-split on wgmma) against fp64."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def _run(S, M, N, K, a_mn, b_mn, split3, seed=0):
    from purejaxql_b200 import _lib
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((S, M, K)).astype(np.float32)          # logical [M,K]
    B = (rng.standard_normal((S, K, N)) * 0.05).astype(np.float32)  # logical [K,N]
    a_store = np.ascontiguousarray(A.transpose(0, 2, 1)) if a_mn else A
    b_store = B if b_mn else np.ascontiguousarray(B.transpose(0, 2, 1))
    ta, tb = torch.from_numpy(a_store).to(dev()), torch.from_numpy(b_store).to(dev())
    tal, tbl = torch.empty_like(ta), torch.empty_like(tb)
    L = _lib.lib()
    _lib.check(L.pqn_tc_split_lo(_lib.p(ta), _lib.p(tal), ta.numel(), _lib.stream_ptr()))
    _lib.check(L.pqn_tc_split_lo(_lib.p(tb), _lib.p(tbl), tb.numel(), _lib.stream_ptr()))
    d = torch.full((S, M, N), float("nan"), device=dev())
    _lib.check(L.pqn_tc_gemm_test(_lib.p(ta), _lib.p(tal), _lib.p(tb), _lib.p(tbl), _lib.p(d), S, M, N, K, a_mn, b_mn,
                                  split3, _lib.stream_ptr()), "pqn_tc_gemm_test")
    torch.cuda.synchronize()
    ref = np.matmul(A.astype(np.float64), B.astype(np.float64))
    return d.cpu().numpy(), ref, A, B, tal.cpu().numpy()


@pytest.mark.parametrize("a_mn,b_mn", [(0, 1), (1, 1), (0, 0)])
def test_tc_gemm_single_pass_tf32(a_mn, b_mn):
    d, ref, A, B, _ = _run(2, 256, 128, 96, a_mn, b_mn, 0)
    # single TF32 pass == exact product of the truncated operands (fp32 accumulate)
    trunc = lambda x: (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    ref_t = np.matmul(trunc(A).astype(np.float64), trunc(B).astype(np.float64))
    assert np.isfinite(d).all()
    assert np.abs(d - ref_t).max() < 5e-5, np.abs(d - ref_t).max()
    assert np.abs(d - ref).max() < 2e-2


@pytest.mark.parametrize("a_mn,b_mn", [(0, 1), (1, 1), (0, 0)])
@pytest.mark.parametrize("S,M,N,K", [(1, 128, 128, 32), (3, 200, 128, 1024), (2, 1024, 256, 4096)])
def test_tc_gemm_inline_a_lo_is_bitwise_the_same(a_mn, b_mn, S, M, N, K):
    """split3=2 derives A_lo inside the kernel (converter warps, smem -> smem) instead of reading it from memory:
    same operands, same MMA order, so the result must be identical to the precomputed-lo run."""
    d1, ref, *_ = _run(S, M, N, K, a_mn, b_mn, 1, seed=K)
    d2, *_ = _run(S, M, N, K, a_mn, b_mn, 2, seed=K)
    assert np.isfinite(d2).all()
    assert np.array_equal(d1, d2)
    assert np.abs(d2 - ref).max() < 4e-6 * np.abs(ref).max()


@pytest.mark.parametrize("a_mn,b_mn", [(0, 1), (1, 1), (0, 0)])
@pytest.mark.parametrize("S,M,N,K", [(1, 128, 128, 32), (3, 200, 128, 1024), (2, 1024, 256, 4096)])
def test_tc_gemm_3xtf32_fp32_accuracy(a_mn, b_mn, S, M, N, K):
    d, ref, A, B, alo = _run(S, M, N, K, a_mn, b_mn, 1, seed=K)
    assert np.isfinite(d).all()
    scale = np.abs(ref).max()
    err = np.abs(d - ref).max()
    assert err < 4e-6 * scale, (err, scale)
    # the lo operand is what the header says
    hi = (A.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    lo_ref = A - hi
    lo_ref = np.ascontiguousarray(lo_ref.transpose(0, 2, 1)) if a_mn else lo_ref
    assert np.array_equal(alo, lo_ref)


# --------------------------------------------------------------------------- #
# fp16-split path: operands as (hi, lo') fp16 planes, wgmma f16 with fp32 accumulate, 64-element k-blocks
# --------------------------------------------------------------------------- #
def _run16(S, M, N, K, a_mn, b_mn, seed=0, a_scale=1.0, a_mag=1.0, b_mag=0.05):
    from purejaxql_b200 import _lib
    rng = np.random.default_rng(seed)
    A = (rng.standard_normal((S, M, K)) * a_mag).astype(np.float32)          # logical [M,K]
    B = (rng.standard_normal((S, K, N)) * b_mag).astype(np.float32)          # logical [K,N]
    a_store = np.ascontiguousarray(A.transpose(0, 2, 1)) if a_mn else A
    b_store = B if b_mn else np.ascontiguousarray(B.transpose(0, 2, 1))
    ta, tb = torch.from_numpy(a_store).to(dev()), torch.from_numpy(b_store).to(dev())
    planes = [torch.empty(t.shape, dtype=torch.float16, device=dev()) for t in (ta, ta, tb, tb)]
    L = _lib.lib()
    _lib.check(L.pqn_tc_split16(_lib.p(ta), _lib.p(planes[0]), _lib.p(planes[1]), ta.numel(), a_scale, _lib.stream_ptr()))
    _lib.check(L.pqn_tc_split16(_lib.p(tb), _lib.p(planes[2]), _lib.p(planes[3]), tb.numel(), 1.0, _lib.stream_ptr()))
    d = torch.full((S, M, N), float("nan"), device=dev())
    _lib.check(L.pqn_tc_gemm16_test(_lib.p(planes[0]), _lib.p(planes[1]), _lib.p(planes[2]), _lib.p(planes[3]), _lib.p(d),
                                    S, M, N, K, a_mn, b_mn, 1.0 / a_scale, _lib.stream_ptr()), "pqn_tc_gemm16_test")
    torch.cuda.synchronize()
    ref = np.matmul(A.astype(np.float64), B.astype(np.float64))
    return d.cpu().numpy(), ref, ta, planes


def test_split16_planes_reconstruct_22_bits():
    from purejaxql_b200 import _lib
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(1 << 16) * np.exp(rng.uniform(-14, 8, 1 << 16))).astype(np.float32)   # 1e-6 .. 3e3
    x[:4] = [0.0, 70000.0, -1e9, 6.1e-5]
    t = torch.from_numpy(x).to(dev())
    hi = torch.empty(x.shape, dtype=torch.float16, device=dev())
    lo = torch.empty_like(hi)
    _lib.check(_lib.lib().pqn_tc_split16(_lib.p(t), _lib.p(hi), _lib.p(lo), t.numel(), 1.0, _lib.stream_ptr()))
    rec = hi.double().cpu().numpy() + lo.double().cpu().numpy() / 2048.0
    xs = np.clip(x.astype(np.float64), -65000.0, 65000.0)                                          # saturation
    assert np.isfinite(rec).all()
    err = np.abs(rec - xs)
    assert (err <= np.maximum(np.abs(xs) * 2.0 ** -21, 2.0 ** -34)).all(), err.max()


@pytest.mark.parametrize("a_mn,b_mn", [(0, 1), (1, 1), (0, 0)])
@pytest.mark.parametrize("S,M,N,K", [(1, 128, 128, 64), (3, 200, 128, 1024), (2, 1024, 256, 4096), (2, 136, 128, 200)])
def test_tc_gemm16_fp32_accuracy(a_mn, b_mn, S, M, N, K):
    d, ref, *_ = _run16(S, M, N, K, a_mn, b_mn, seed=K)
    assert np.isfinite(d).all()
    scale = np.abs(ref).max()
    err = np.abs(d - ref).max()
    assert err < 4e-6 * scale, (err, scale)


@pytest.mark.parametrize("a_mn,b_mn", [(1, 1), (0, 0)])
def test_tc_gemm16_small_gradients_with_prescale(a_mn, b_mn):
    """Gradient-sized operands (1e-6) keep fp32 accuracy through the power-of-two pre-scale (undone by out_scale)."""
    d, ref, *_ = _run16(2, 256, 128, 512, a_mn, b_mn, seed=3, a_scale=float(2 ** 16), a_mag=1e-6)
    scale = np.abs(ref).max()
    assert np.abs(d - ref).max() < 4e-6 * scale, (np.abs(d - ref).max(), scale)


@pytest.mark.parametrize("S,M,N", [(5, 4096, 1024), (3, 6536, 256), (160, 128, 384)])
def test_tc_gemm16_dgrad_shapes(S, M, N):
    """K = 128 (two k-blocks), K-major operands, several n-tiles and more (seed, m-tile) groups than SMs -- the dense
    dgrad's shape at full size; ragged M covers the row clipping.  (An A-stationary variant of the kernel for this shape
    -- A tiles loaded once per group, two-stage ring -- measured no faster in round 2 and was dropped: DESIGN.md 3.2.)"""
    d, ref, *_ = _run16(S, M, N, 128, 0, 0, seed=S + N)
    assert np.isfinite(d).all()
    scale = np.abs(ref).max()
    err = np.abs(d - ref).max()
    assert err < 4e-6 * scale, (err, scale)
