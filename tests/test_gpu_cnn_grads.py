"""The MinAtar CNN's loss and gradients (``pqn_qnet_loss_grad``) on the GPU against fp64, on every kernel variant that
entry point selects: the five (tensor-core path, conv path) pairs, the channel counts 4, 6, 7 and 10, the mixed path
of more than PQN_TC_MAX_A = 8 actions, minibatches of 4096 and 4097 rows through a gather, the parameters training
starts from, TD errors of three scales, the benchmark's 128 seeds x 4096 rows, and the NORM_TYPE / NORM_INPUT variants
at C = 7.  The fp64 reference is ``oracle/pqn_ref.py`` (``oracle/pqn_ref_norm.py`` for the variants), pinned against
torch autograd at these widths by ``test_oracle_cnn_grads.py``, whose input builders these tests share.

Inputs.  Boards of the game of each width (Breakout, SpaceInvaders, Freeway; synthetic boards for C = 10) with an
empty board and a board with one channel entirely set among the gathered rows; S = 2 seeds with their own parameters
and boards; targets ``q_sa(fp64) - delta * eps``, eps ~ N(0, 1), delta in {1e-2, 1, 30} (30 covers the lambda-returns
of the densest-reward games at init; below about 1e-3 the fp32 rounding of q dominates the gradient, in the reference
as well).  Parameters are either ``R.random_params`` (biases N(0, 0.1), scales 1 + N(0, 0.1)) or the engine's own
``spec.init`` (conv bias 0, LayerNorm scales 1): there an empty 3x3 patch has z = 0 over its 16 channels, var = 0 and
rstd = 1 / sqrt(1e-6) = 1000.

Tolerance rule.  Every tensor is compared by max-abs error ``err`` with its own fp64 scale (max |want|; max |q_sa|
for the mean chosen q), with no absolute floor, since the gradients scale with delta.  ``spread32`` is how far the
same oracle run in fp32 NumPy lands from fp64 on the same inputs; the test computes it.
  - every gradient tensor on every path: ``err <= max(2e-5 * scale, C_SPREAD * spread32)``.  At these sizes fp32 arithmetic
    itself does not meet 2e-5 everywhere: the fp32 oracle lands up to 1.2e-5 of the scale away at delta = 1 and
    1.6e-4 - 4e-4 at delta = 1e-2 (there the fp32 rounding of q sets the gradient's error), and the FFMA path up to
    7e-5 (LayerNorm_1/scale, 4097 rows);
  - FFMA path (0, 0): also ``err <= max(C_SPREAD * spread32, 2**-20 * scale)``, C_SPREAD = 8 at delta >= 1 and 16 at
    delta = 1e-2, where GPU and NumPy round q independently (LayerNorm_0/scale at C = 6: up to 3.3e-3 of the scale,
    between 8x and 16x the fp32 oracle's distance);
  - split-precision paths: ``err <= SPLIT_SPREAD * spread32``, 16;
  - the loss and the mean chosen q: ``err <= 2e-5 * scale``; NumPy's pairwise fp32 mean lands far inside one ulp of
    fp64 there, so a ratio to spread32 measures NumPy's luck, not the kernel.
Measured on one NVIDIA H100 80GB HBM3 (700 W power limit), worst err / spread32 over all gradient tensors, shapes,
regimes and deltas: FFMA 8.5 (delta = 1e-2), 3xTF32 + fp16 conv 11.2, 3xTF32 + CUDA-core conv 5.4, fp16-split +
fp16 conv 5.1, fp16-split + tf32 conv 5.1.  No gradient tensor of a split-precision path is further from fp64 than 16x
the fp32 oracle: the distance of up to 2e-5 of the scale that these paths show at 4096 rows is fp32's own.  Loss and
mean chosen q: at most 3.2e-6 and 4.9e-7 of their scale.  In the init regime at delta = 30, max |dz * gs| of the fp16
conv backward reaches 3.96e4 (C = 10, 4097 rows), 1.65x below the fp16 maximum.

The input BatchNorm's gradients are exactly zero (it is off the path with NORM_INPUT = False), and ``bn_sums`` are
integer counts, compared exactly.
"""
import functools

import numpy as np
import pytest
import torch

from oracle import pqn_ref as R
from oracle import pqn_ref_norm as RN
from test_oracle_cnn_grads import cast, game_obs, minibatch_gather, pack_obs, td_targets

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
BAR = 2e-5
C_SPREAD = 8.0
FLOOR = 2.0 ** -20
SPLIT_SPREAD = 16.0
SCALARS = ("loss", "qmean")
DELTAS = (1e-2, 1.0, 30.0)
FP16_MAX = 65504.0
PATHS = [(2, 1), (1, 1), (0, 0), (1, 0), (2, 3)]
PATH_IDS = ["f16split+f16conv", "3xtf32+f16conv", "ffma", "3xtf32+cudaconv", "f16split+tf32conv"]
SHAPES = [(4, 3), (4, 5), (6, 4), (7, 3), (10, 18), (4, 9)]
REPORT = []          # (path, C, A, rows, regime, delta, tensor, err / scale, err / spread32), printed at the end


def dev():
    return torch.device("cuda:0")


def _lib():
    from purejaxql_b200 import _lib
    return _lib


def t_(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


def set_path(path):
    L = _lib().lib()
    _lib().check(L.pqn_set_tensor_core_path(path[0]))
    _lib().check(L.pqn_set_conv_mma_path(path[1]))


@pytest.fixture(params=PATHS, ids=PATH_IDS)
def path(request):
    set_path(request.param)
    yield request.param
    set_path((2, 1))


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if not REPORT:
        return
    worst = {}
    for p, C, A, rows, regime, delta, name, rs, rsp in REPORT:
        k = (p, C, A, "%s-%d" % (regime, rows), delta, name)
        a = worst.get(k, (0.0, 0.0))
        worst[k] = (max(a[0], rs), max(a[1], rsp))
    print("\nworst err/scale and err/spread32 per (path, C, A, regime, delta, tensor):")
    for k in sorted(worst):
        print("  %-6s C=%-2d A=%-2d %-13s delta=%-5g %-26s %9.2e %9.2f" % (k[0], k[1], k[2], k[3], k[4], k[5], *worst[k]))


def cnn_spec(C, A, norm_type="layer_norm", norm_input=False):
    from purejaxql_b200.networks import NET_CNN, QNetworkSpec
    return QNetworkSpec(NET_CNN, C, A, norm_type=norm_type, norm_input=norm_input)


def leaves(spec, flat, s):
    tree = spec.unflatten(flat)
    out = {}
    for pth, *_ in spec.entries:
        d = tree
        for k in pth:
            d = d[k]
        out["/".join(pth)] = d[s].cpu().numpy()
    return out


def init_params(C, A, seed):
    """The engine's own initial parameters (``spec.init`` on the device), read back."""
    from purejaxql_b200 import jaxrandom
    spec = cnn_spec(C, A)
    flat = spec.init(jaxrandom.split(jaxrandom.PRNGKey(seed, dev()), 1), dev())
    return leaves(spec, flat, 0)


def make_set(C, A, rows, total, regime, seed):
    """One seed's (parameters, boards, gather, actions) and its fp64 q_sa on the gathered rows."""
    rng = np.random.default_rng(seed)
    p = R.random_params(R.cnn_param_shapes(C, A), seed) if regime == "random" else init_params(C, A, seed)
    obs = game_obs(C, total, seed)
    gather = minibatch_gather(total, rows, rng)
    act = rng.integers(0, A, total).astype(np.int32)
    q64 = R.cnn_forward(cast(p, F64), obs[gather].astype(F64))
    return dict(p=p, obs=obs, gather=gather, act=act, q64=q64, q_sa=q64[np.arange(rows), act[gather]])


def with_targets(st, delta, seed):
    tgt = np.zeros(st["obs"].shape[0], F32)
    tgt[st["gather"]] = td_targets(st["q_sa"], delta, np.random.default_rng(seed))
    return tgt


def oracle(st, tgt):
    """-> fp64 values, fp32-oracle values and scales of every compared tensor, and the conv's max |dz| (fp64)."""
    g_, a_ = st["gather"], st["act"][st["gather"]]
    out = []
    for dt in (F64, F32):
        loss, q_sa, g = R.cnn_loss_and_grads(cast(st["p"], dt), st["obs"][g_].astype(dt), a_, tgt[g_].astype(dt))
        g = {k: v.astype(F64) for k, v in g.items()}
        g["loss"], g["qmean"] = np.array([loss], F64), np.array([q_sa.mean()], F64)
        out.append(g)
    want, w32 = out
    scale = {k: float(np.abs(v).max()) for k, v in want.items()}
    scale["qmean"] = float(np.abs(st["q_sa"]).max())
    return want, w32, scale, conv_dz_max(st["p"], st["obs"][g_], a_, tgt[g_])


def conv_dz_max(p, obs, act, tgt):
    """max |dz| of the conv LayerNorm's input gradient in fp64: the values the fp16 conv backward scales and splits."""
    p = cast(p, F64)
    q, (cols, c1, y1, h1, c2, y2, h2) = R.cnn_forward(p, obs.astype(F64), want_cache=True)
    B = obs.shape[0]
    dq = np.zeros_like(q)
    dq[np.arange(B), act] = (q[np.arange(B), act] - tgt.astype(F64)) / B
    dz2, _, _ = R._layer_norm_bwd((dq @ p["Dense_0/kernel"].T) * (y2 > 0), c2, p["CNN_0/LayerNorm_1/scale"])
    dy1 = (dz2 @ p["CNN_0/Dense_0/kernel"].T).reshape(y1.shape) * (y1 > 0)
    dz1, _, _ = R._layer_norm_bwd(dy1, c1, p["CNN_0/LayerNorm_0/scale"])
    return float(np.abs(dz1).max())


def conv_dz_scale(rows):
    """The power-of-two scale of the fp16 conv backward's dz planes: 2^ceil(log2 rows) (pqn_qnet_loss_grad)."""
    s = 1.0
    while rows > 1:
        s *= 2.0
        rows = (rows + 1) >> 1
    return s


def gpu_loss_grad(spec, sets, tgts, S, rows):
    """pqn_qnet_loss_grad of seeds s < S holding sets[s % len(sets)].  -> [per seed {tensor: value}], bn [S, 2C]"""
    L = _lib().lib()
    C = spec.in_c
    total = sets[0]["obs"].shape[0]
    idx = [s % len(sets) for s in range(S)]
    flat = torch.cat([spec.flatten(sets[i]["p"], 1, dev()) for i in range(len(sets))], 0)[idx].contiguous()
    packed = t_(np.stack([pack_obs(st["obs"]) for st in sets])[idx], torch.int32)
    gather = t_(np.stack([st["gather"] for st in sets])[idx], torch.int32)
    act = t_(np.stack([st["act"] for st in sets])[idx], torch.int32)
    tgt = t_(np.stack(tgts)[idx], torch.float32)
    grads = torch.zeros_like(flat)
    ls, qs = torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
    bn = torch.zeros((S, 2 * C), device=dev())
    ws = torch.empty(int(L.pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())
    p = _lib().p
    _lib().check(L.pqn_qnet_loss_grad(spec.desc, p(flat), None, p(packed), p(gather), total, p(act), p(tgt), total,
                                      p(grads), p(ls), p(qs), p(bn), S, rows, p(ws), _lib().stream_ptr()),
                 "pqn_qnet_loss_grad")
    torch.cuda.synchronize()
    ls, qs = ls.cpu().numpy(), qs.cpu().numpy()
    out = []
    for s in range(S):
        d = {k: v.astype(F64) for k, v in leaves(spec, grads, s).items()}
        d["loss"], d["qmean"] = np.array([ls[s]], F64), np.array([qs[s]], F64)
        out.append(d)
    del ws
    return out, bn.cpu().numpy()


def gpu_forward(spec, sets, S, rows):
    L = _lib().lib()
    total = sets[0]["obs"].shape[0]
    idx = [s % len(sets) for s in range(S)]
    flat = torch.cat([spec.flatten(sets[i]["p"], 1, dev()) for i in range(len(sets))], 0)[idx].contiguous()
    packed = t_(np.stack([pack_obs(st["obs"]) for st in sets])[idx], torch.int32)
    gather = t_(np.stack([st["gather"] for st in sets])[idx], torch.int32)
    q = torch.zeros((S * rows, spec.num_actions), device=dev())
    ws = torch.empty(int(L.pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())
    p = _lib().p
    _lib().check(L.pqn_qnet_forward(spec.desc, p(flat), None, p(packed), p(gather), total, p(q), S, rows, p(ws),
                                    _lib().stream_ptr()), "pqn_qnet_forward")
    torch.cuda.synchronize()
    return q.cpu().numpy().reshape(S, rows, spec.num_actions)


def check_bn_sums(bn, st, C):
    x = st["obs"][st["gather"]].reshape(-1, C).astype(F64)
    assert np.array_equal(bn[:C], x.sum(0)) and np.array_equal(bn[C:], x.sum(0))


def compare(got, ref, path, tag):
    """Applies the tolerance rule of the module docstring to every tensor; records the ratios.  -> failures"""
    want, w32, scale, _ = ref
    delta = tag[-1]
    bad = []
    for name, w in want.items():
        g = got[name]
        if name.startswith("BatchNorm_0/"):
            if g.any() or w.any():
                bad.append((name, "not zero"))
            continue
        err = float(np.abs(g - w).max())
        spread = float(np.abs(w32[name] - w).max())
        sc = scale[name]
        REPORT.append((path, *tag, name, err / sc, err / spread if spread > 0 else float("inf")))
        if name in SCALARS:
            if not err <= BAR * sc:
                bad.append((name, "2e-5 bar", err / sc))
            continue
        c_glob = C_SPREAD if delta >= 1 else 2 * C_SPREAD
        if not err <= max(BAR * sc, c_glob * spread):
            bad.append((name, "global bar", err / sc))
        c = c_glob if path == (0, 0) else SPLIT_SPREAD
        if not err <= max(c * spread, FLOOR * sc):
            bad.append((name, "spread bar", err / spread))
    return [(tag, b) for b in bad]


@functools.lru_cache(maxsize=None)
def grad_inputs(C, A, rows, regime):
    """S = 2 sets gathered from 2 x rows boards, with the oracle's results for every delta."""
    sets = [make_set(C, A, rows, 2 * rows, regime, 1000 * C + 10 * A + s + (0 if regime == "random" else 500))
            for s in range(2)]
    tgts = {d: [with_targets(st, d, 7 + s) for s, st in enumerate(sets)] for d in DELTAS}
    refs = {d: [oracle(st, tg) for st, tg in zip(sets, tgts[d])] for d in DELTAS}
    return sets, tgts, refs


@pytest.mark.parametrize("regime", ["random", "init"])
@pytest.mark.parametrize("rows", [4096, 4097])
@pytest.mark.parametrize("C,A", SHAPES, ids=["C%dA%d" % s for s in SHAPES])
def test_cnn_loss_grad_matches_fp64(C, A, rows, regime, path):
    """Loss, mean chosen q, every gradient tensor and bn_sums at the channel counts / actions the library builds.
    rows = 4097 doubles the fp16 gradient scale against rows; A = 9 and 18 take the mixed path (FFMA dense layer,
    fp16 conv backward when the conv path is 1).  In the init regime at delta = 30, max |dz * gs| of the conv
    backward's fp16 planes stays below the fp16 maximum (conversions saturate silently)."""
    spec = cnn_spec(C, A)
    sets, tgts, refs = grad_inputs(C, A, rows, regime)
    bad = []
    for d in DELTAS:
        got, bn = gpu_loss_grad(spec, sets, tgts[d], 2, rows)
        for s in range(2):
            bad += compare(got[s], refs[d][s], path, (C, A, rows, regime, d))
            check_bn_sums(bn[s], sets[s], C)
            dzs = refs[d][s][3] * conv_dz_scale(rows)
            REPORT.append((path, C, A, rows, regime, d, "max|dz*gs|", dzs, 0.0))
            assert dzs < FP16_MAX, (C, A, rows, regime, d, dzs)
    assert not bad, (path, bad)


# --------------------------------------------------------------------------------------------------------------------
# the benchmark's geometry: 128 seeds x 4096 rows gathered from 8192 per seed
# --------------------------------------------------------------------------------------------------------------------
BENCH_ROWS, BENCH_TOTAL, NSETS = 4096, 8192, 8
BENCH_DELTAS = (1e-2, 1.0, 30.0, 1.0)
CONV_ATOMIC = ["CNN_0/Conv_0/kernel", "CNN_0/Conv_0/bias", "CNN_0/LayerNorm_0/scale", "CNN_0/LayerNorm_0/bias"]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def wgrad_regime(path, S, rows):
    """The dense weight gradient's K split on the current device, restated from pqn_net.cu: wgrad_ksplit
    (tensor-core paths; 8 output tiles per seed, k-blocks of 64 rows for fp16) or wgrad_splits (FFMA)."""
    sms = _sms()
    if path[0] == 0:
        s = (2 * sms + 8 * S - 1) // (8 * S)
        return max(1, min(s, (rows + 255) // 256))
    tiles, kb = 8 * S, (rows + 63) // 64
    if tiles >= sms:
        return 1
    ks = max(1, min(sms // tiles, kb // 8))
    while ks > 1 and (ks - 1) * ((kb + ks - 1) // ks) >= kb:
        ks -= 1
    return ks


def conv_mma_ctas(S, rows, per_sm):
    """CTAs per seed of the conv / row-backward grids (pqn_net.cu conv_mma_ctas)."""
    resident = _sms() * per_sm
    maxc = (rows + 7) // 8
    best, best_eff = 1, 0.0
    lim = (6 * resident + S - 1) // S
    for per_seed in range(1, min(lim, maxc) + 1):
        total = per_seed * S
        waves = (total + resident - 1) // resident
        if waves > 6:
            break
        eff = total / (waves * resident)
        if eff > best_eff + 0.01 or (eff > best_eff - 0.01 and waves <= 4):
            best_eff, best = max(eff, best_eff), per_seed
    return best


def final_slices(count):
    return 32 if count > 48 else 8


@functools.lru_cache(maxsize=None)
def bench_inputs():
    sets = [make_set(4, 3, BENCH_ROWS, BENCH_TOTAL, "random" if k % 2 == 0 else "init", 9000 + k) for k in range(NSETS)]
    tgts = [with_targets(st, BENCH_DELTAS[k % 4], 77 + k) for k, st in enumerate(sets)]
    refs = [oracle(st, tg) for st, tg in zip(sets, tgts)]
    return sets, tgts, refs


def test_bench_geometry_selects_both_regimes():
    """S = 1, 8, 9 and 128 at 4096 rows cover both regimes of the dense weight gradient (split-K / not) and both
    finalize kernels (8 / 32 slices) on this device; on a 132-SM H100, S <= 8 is split and S >= 9 is not."""
    Ss = (1, 8, 9, 128)
    split = {S: wgrad_regime((2, 1), S, BENCH_ROWS) > 1 for S in Ss}
    slices = {S: final_slices(conv_mma_ctas(S, BENCH_ROWS, 2)) for S in Ss}
    assert set(split.values()) == {True, False}, split
    assert set(slices.values()) == {8, 32}, slices
    if _sms() == 132:
        assert split == {1: True, 8: True, 9: False, 128: False}, split
        assert slices[128] == 8 and slices[1] == 32, slices


@pytest.mark.parametrize("S", [1, 8, 9, 128])
@pytest.mark.parametrize("bpath", [(2, 1), (0, 0)], ids=["f16split+f16conv", "ffma"])
def test_bench_geometry_loss_grad(S, bpath):
    """Seed s holds input set s mod 8: every seed is bit-identical to the first seed of its set (per-seed work
    depends on gridDim.x only, so a seed-offset or 64-bit-offset bug shows as a mismatch; at S = 128 the saved conv
    xhat alone is 2^29 floats), and the 8 distinct sets meet the fp64 bars."""
    set_path(bpath)
    try:
        spec = cnn_spec(4, 3)
        sets, tgts, refs = bench_inputs()
        got, bn = gpu_loss_grad(spec, sets, tgts, S, BENCH_ROWS)
    finally:
        set_path((2, 1))
    for s in range(NSETS, S):
        first = got[s % NSETS]
        diff = [k for k in first if not np.array_equal(got[s][k], first[k])]
        if bpath[1] == 0:
            # the CUDA-core conv backward adds its CTA partials into the gradients with float atomics: its four tensors
            # differ between replicas in the last bits (the order of the atomics), everything else is bit-identical
            for k in CONV_ATOMIC:
                if k in diff:
                    diff.remove(k)
                    assert np.abs(got[s][k] - first[k]).max() <= FLOOR * 16 * np.abs(first[k]).max(), (s, k)
        assert not diff, (s, diff)
        assert np.array_equal(bn[s], bn[s % NSETS]), s
    bad = []
    for k in range(min(S, NSETS)):
        bad += compare(got[k], refs[k], bpath, (4, 3, BENCH_ROWS, "bench-S%d" % S, BENCH_DELTAS[k % 4]))
        check_bn_sums(bn[k], sets[k], 4)
    assert not bad, (bpath, bad)


@pytest.mark.parametrize("bpath", [(2, 1), (0, 0)], ids=["f16split+f16conv", "ffma"])
def test_bench_geometry_eval_forward(bpath):
    """pqn_qnet_forward at 128 seeds x 4096 gathered rows: replicas bit-identical, q within 1e-5 of fp64."""
    set_path(bpath)
    try:
        sets, _, _ = bench_inputs()
        q = gpu_forward(cnn_spec(4, 3), sets, 128, BENCH_ROWS)
    finally:
        set_path((2, 1))
    for s in range(NSETS, 128):
        assert np.array_equal(q[s], q[s % NSETS]), s
    for k in range(NSETS):
        assert np.abs(q[k] - sets[k]["q64"]).max() < 1e-5, (k, np.abs(q[k] - sets[k]["q64"]).max())


# --------------------------------------------------------------------------------------------------------------------
# NORM_TYPE / NORM_INPUT variants at C = 7 (Freeway)
# --------------------------------------------------------------------------------------------------------------------
BN_DEAD_BIASES = ("CNN_0/Conv_0/bias", "CNN_0/Dense_0/bias")   # biases that feed a BatchNorm: exact gradient zero


@pytest.mark.parametrize("norm_type,norm_input", [("batch_norm", False), ("none", True), ("batch_norm", True)])
def test_norm_variants_c7_match_fp64(norm_type, norm_input, path):
    """conv_eff_kernel / conv_grad_finish_kernel and the batch-statistics kernels at C = 7, 1024 rows, against
    oracle/pqn_ref_norm.py with test_gpu_norm.py's bars; the running statistics updated with bn_count = rows x 100."""
    L = _lib().lib()
    C, A, S, total, rows = 7, 3, 2, 2048, 1024
    spec = cnn_spec(C, A, norm_type, norm_input)
    shapes = RN.cnn_param_shapes(C, A, norm_type)
    ps = [R.random_params(shapes, 40 + s) for s in range(S)]
    if norm_type == "batch_norm":
        # a bias in front of a BatchNorm is a no-op; a non-zero one only makes the fast variance cancel in fp32
        for pp in ps:
            for k in BN_DEAD_BIASES:
                pp[k] = np.zeros_like(pp[k])
    rng = np.random.default_rng(3)
    stats0 = RN.cnn_batch_stats(C, norm_type)
    sts = [{k: {"mean": (0.1 * rng.standard_normal(v["mean"].shape)).astype(F32),
                "var": (0.5 + rng.random(v["var"].shape)).astype(F32)} for k, v in stats0.items()} for _ in range(S)]
    obs = np.stack([game_obs(C, total, 60 + s) for s in range(S)])
    gather = np.stack([minibatch_gather(total, rows, rng) for _ in range(S)])
    act = rng.integers(0, A, (S, total)).astype(np.int32)
    tgt = rng.standard_normal((S, total)).astype(F32)
    flat = torch.cat([spec.flatten(pp, 1, dev()) for pp in ps], 0).contiguous()
    stf = torch.cat([spec.flatten_stats(st, 1, dev()) for st in sts], 0).contiguous()
    grads = torch.zeros_like(flat)
    ls, qs = torch.zeros(S, device=dev()), torch.zeros(S, device=dev())
    bn = torch.zeros((S, 2 * C), device=dev())
    packed = t_(np.stack([pack_obs(o) for o in obs]), torch.int32)
    tg_, ta_, tt_ = t_(gather, torch.int32), t_(act, torch.int32), t_(tgt, torch.float32)
    ws = torch.empty(int(L.pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())
    p = _lib().p
    _lib().check(L.pqn_qnet_loss_grad(spec.desc, p(flat), p(stf), p(packed), p(tg_), total, p(ta_), p(tt_), total,
                                      p(grads), p(ls), p(qs), p(bn), S, rows, p(ws), _lib().stream_ptr()),
                 "pqn_qnet_loss_grad")
    _lib().check(L.pqn_bn_stats_update(p(stf), p(bn), S, C, spec.stats_total, float(rows * 100), 0.99,
                                       _lib().stream_ptr()))
    torch.cuda.synchronize()
    sttree = spec.unflatten_stats(stf)
    for s in range(S):
        st64 = {k: {kk: vv.astype(F64) for kk, vv in v.items()} for k, v in sts[s].items()}
        x = obs[s][gather[s]].astype(F64)
        loss, q_sa, g, new_stats = RN.cnn_loss_and_grads(cast(ps[s], F64), st64, x, act[s][gather[s]],
                                                         tgt[s][gather[s]].astype(F64), norm_type, norm_input)
        assert abs(float(ls[s]) - loss) < 5e-5 * max(1.0, abs(loss)), (float(ls[s]), loss)
        assert abs(float(qs[s]) - q_sa.mean()) < 5e-5 * max(1.0, abs(q_sa.mean()))
        scale = max(np.abs(v).max() for v in g.values())
        got = leaves(spec, grads, s)
        errs = {}
        for name, want in g.items():
            tol = 2e-5
            if norm_type == "batch_norm":
                tol = 5e-2 if name in BN_DEAD_BIASES else 2e-4   # test_gpu_norm.py: fp32 batch statistics
            errs[name] = (float(np.abs(got[name] - want).max() / scale), tol)
        bad = {k: v for k, v in errs.items() if not v[0] < v[1]}
        assert not bad, (bad, errs)
        for pth, off, n in spec.stats_entries():
            d = sttree
            for k in pth:
                d = d[k]
            want = new_stats["/".join(pth)]
            assert np.allclose(d["mean"][s].cpu().numpy(), want["mean"], atol=2e-6), pth
            assert np.allclose(d["var"][s].cpu().numpy(), want["var"], atol=2e-6), pth
