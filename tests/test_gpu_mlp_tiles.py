"""The default MLP Q-networks (layer_norm, NORM_INPUT False) against fp64 in the rollout buffer's layout, at the seed
counts and minibatch sizes where their kernels change branch: the fp32 ``PQN_NET_MLP`` of ``pqn_gymnax`` on the
classic-control and bsuite envs, and ``PQN_NET_MLP_BITS`` (``csrc/pqn_bits.cuh``) on the MinAtar games.

The older MLP tests pass one value as both row strides of ``pqn_qnet_loss_grad`` and run at most 3 seeds and 515 fp32
rows (65,536 packed-bit rows).  Here every case takes the engine's layout (``engine.update_body``): per seed (T+1) E
observation rows (fp32 rows, or packed words) and T E action / target rows, the gather one minibatch of
``jaxrandom.permutation_indices(..., chunk=rows)``.  Rows outside the minibatch hold NaN observations (all-ones words
for the bits kind), NaN targets and valid actions that differ from the gathered rows', so a wrong stride reads a NaN,
a full board or another action.  ``grads``, ``loss_sum``, ``qsa_sum``, ``bn_sums`` and the forward's q carry NaN
guard tails.  Cases (S seeds x minibatch rows; the counts at 132 SMs):

  cartpole   MLP 4 x 256 x 2, A 2     128 x 128      pqn_cartpole (E 32, T 64, 16 minibatches) at 128 seeds: the thin
                                                      first-layer wgrad in one chunk, wgmma hidden wgrad unsplit
  acrobot    MLP 6 x 256 x 2, A 3       1 x 262,144  configs[3] (E 65,536, T 64, 16 minibatches): 256 thin-wgrad
                                                      chunks (wgrad_split_reduce_kernel<32>), hidden wgrad split-K 33
  ragged64   MLP 3 x 64 x 3, A 2        5 x 4,097    FFMA hidden layers (H 64); 33 thin chunks, the last of one row
  wide       MLP 50 x 128 x 2, A 3      9 x 4,097    Catch-sized: tiled FFMA first-layer wgrad (D > 8) in 17 row
                                                      splits, hidden wgmma wgrad split-K 8
  breakout   bits 400 x 256 x 2, A 3  128 x 128      pqn_minatar (E 128, T 32, 32 minibatches) at 128 seeds: the
                                                      unsplit bits::wgrad_kernel writing at seed stride P
  breakout16 bits 400 x 256 x 2, A 3   16 x 2,048    configs[2] (E 1,024, T 32, 16 minibatches): 3 bits-wgrad splits
  seaquest   bits 1000 x 256 x 2, A 6   1 x 262,144  configs[3]-sized: fwd_kernel<4>, 17 bits-wgrad splits, 4,096
                                                      rows per popcount block
  spaceinv   bits 600 x 64 x 1, A 4     9 x 4,097    bits::wgrad_kernel<64> in 6 splits, the head on layer 0

Each case runs on tensor-core path 2 and on path 0 (FFMA; the bits kind expands its rows to fp32 there).  The split
and chunk counts follow the host dispatch (``wgrad_ksplit``, ``wgrad_splits``, ``run_wgrad_first``,
``bits::wgrad_splits``), restated in ``branches`` from the device's SM count: each case asserts the branch it is
named for, and the launch counters (``pqn_profile_enable``) must show exactly the kernels that branch launches.

Seeds 0 and S-1 hold the same parameters and data (set 0), seed 1 set 1, the others two more sets: seeds with one
set must agree bit for bit (the path has no float atomics).  Sets 0 and 1 are checked against ``oracle/pqn_ref.py``
in fp64: loss and mean Q(s, a) within 1e-5 of max(1, |value|), every gradient tensor within max(2e-5 x scale,
MLP_SPREAD_K x spread32) (spread32: the same oracle in fp32 from fp64, as in ``test_gpu_norm_tiles.py``), bn_sums
exact for the bits (popcounts) and within 1e-6 of the column sums of |x| and x^2 for fp32.  The rollout's forward
(``pqn_qnet_forward`` on the E rows of step t = 0 and t = T, stride (T+1) E, no gather) within 1e-5 of fp64.

Inputs: fp32 rows with per-feature offsets N(0, 1) and scales e^-1.5 - e^2.5 (an Acrobot velocity reaches 9 pi);
packed rows half real observations of the game (a pool of 2,048 boards), half dense random bits.  Set 0 has
``R.random_params``, set 1 the engine's ``spec.init``; TD errors of scale 1 and 30.  No ReLU input of a checked set
lies within 2e-6 of zero: the LayerNorm bias in front of each ReLU is moved per channel as in
``test_gpu_norm_tiles.py`` (no row is dropped).

Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): see DESIGN.md section 5.
"""
import functools
import time

import numpy as np
import pytest
import torch

import test_gpu_mlp_minatar as TM
import test_gpu_norm_tiles as NT
from oracle import pqn_ref as R
from test_oracle_cnn_grads import td_targets

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
GUARD = 1024
MLP_SPREAD_K = 8.0
DELTAS = (1.0, 30.0, 1.0, 30.0)
POOL = 2048               # real boards per set; the minibatch draws from them with replacement
# name: kind, D, H, L, A, S, T, E, minibatch rows, game (bits)
CASES = {
    "cartpole": ("mlp", 4, 256, 2, 2, 128, 64, 32, 128, None),
    "acrobot": ("mlp", 6, 256, 2, 3, 1, 64, 65536, 262144, None),
    "ragged64": ("mlp", 3, 64, 3, 2, 5, 17, 241, 4097, None),
    "wide": ("mlp", 50, 128, 2, 3, 9, 17, 241, 4097, None),
    "breakout": ("bits", 400, 256, 2, 3, 128, 32, 128, 128, "Breakout-MinAtar"),
    "breakout16": ("bits", 400, 256, 2, 3, 16, 32, 1024, 2048, "Breakout-MinAtar"),
    "seaquest": ("bits", 1000, 256, 2, 6, 1, 64, 65536, 262144, "Seaquest-MinAtar"),
    "spaceinv": ("bits", 600, 64, 1, 4, 9, 17, 241, 4097, "SpaceInvaders-MinAtar"),
}
# the branch each case is named for, as predicates on branches() (path 2, path 0)
WANT = {
    "cartpole": {"thin_chunks": lambda v: v == 1, "tc_ksplit": lambda v: v == 1},
    "acrobot": {"thin_chunks": lambda v: v > 48, "tc_ksplit": lambda v: v > 1, "ffma_hidden_splits": lambda v: v > 1},
    "ragged64": {"thin_chunks": lambda v: v > 1, "thin_last_rows": lambda v: v == 1, "hidden_tc": lambda v: not v},
    "wide": {"ffma_first_splits": lambda v: v > 1, "tc_ksplit": lambda v: v > 1},
    "breakout": {"bits_splits": lambda v: v == 1, "tc_ksplit": lambda v: v == 1},
    "breakout16": {"bits_splits": lambda v: v > 1},
    "seaquest": {"bits_fwd_nt": lambda v: v == 4, "bits_splits": lambda v: v > 1,
                 "count_rows": lambda v: v == 4096},
    "spaceinv": {"bits_splits": lambda v: v > 1, "hidden_tc": lambda v: not v},
}
REPORT = []               # (case, path, what, value)


def dev():
    return torch.device("cuda:0")


def _lib():
    from purejaxql_b200 import _lib
    return _lib


def t_(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


def guarded(n, fill=0.0):
    out = torch.full((n + GUARD,), float("nan"), device=dev())
    out[:n] = fill
    return out


def spec_of(case):
    from purejaxql_b200.networks import NET_MLP, NET_MLP_BITS, QNetworkSpec
    kind, D, H, L, A = CASES[case][:5]
    return QNetworkSpec(NET_MLP_BITS if kind == "bits" else NET_MLP, D, A, H, L)


def packed_words(D):
    return ((D + 31) // 32 + 3) // 4 * 4


# --------------------------------------------------------------------------------------------------------------------
# the host dispatch, restated
# --------------------------------------------------------------------------------------------------------------------
def cdiv(a, b):
    return (a + b - 1) // b


def ffma_splits(tiles, S, rows, sms):                     # pqn_net.cu wgrad_splits
    return max(1, min(cdiv(2 * sms, tiles * S), cdiv(rows, 256)))


def ffma_tiles(kin, n):
    return cdiv(kin, 128) * (n // (128 if n % 128 == 0 else 64))


def tc_ksplit(tiles_total, k_blocks, sms):                # pqn_net.cu wgrad_ksplit
    if tiles_total >= sms:
        return 1
    ks = max(1, min(sms // tiles_total, k_blocks // 8))
    while ks > 1 and (ks - 1) * cdiv(k_blocks, ks) >= k_blocks:
        ks -= 1
    return ks


def branches(case, sms):
    kind, D, H, L, A, S, T, E, rows, _ = CASES[case]
    b = {"hidden_tc": H >= 128}                             # on path 2
    chunks = max(1, min((2 * sms) // S, cdiv(rows, 128)))   # run_wgrad_first, D <= 8
    per = cdiv(cdiv(rows, chunks), 128) * 128
    b["thin_chunks"] = cdiv(rows, per)
    b["thin_last_rows"] = rows - (b["thin_chunks"] - 1) * per
    b["ffma_first_splits"] = ffma_splits(ffma_tiles(D, H), S, rows, sms)
    b["ffma_hidden_splits"] = ffma_splits(ffma_tiles(H, H), S, rows, sms)
    b["tc_ksplit"] = tc_ksplit(S * (H // 128) ** 2, cdiv(rows, 64), sms) if H >= 128 else 0
    bnc = 128 if H >= 128 else 64                           # pqn_bits.cuh wgrad_splits / split_rows
    sp = max(1, min(cdiv(2 * sms, cdiv(D, 128) * (H // bnc) * S), cdiv(rows, 256), 64))
    rps = cdiv(cdiv(rows, sp), 64) * 64
    b["bits_splits"] = cdiv(rows, rps)
    ks = cdiv(D, 16)                                        # fwd_ntiles
    b["bits_fwd_nt"] = 8 if ks * 8 * 32 * 16 + 128 * (ks | 1) * 8 <= 227 * 1024 else 4
    b["count_rows"] = cdiv(rows, 64)
    return b


def expected_launches(case, path, b):
    """{profiler kernel name: launches} of one pqn_qnet_loss_grad of the default MLP (pqn_net.cu, MLP branch)."""
    kind, D, H, L = CASES[case][:4]
    bits, tc = kind == "bits", path == 2
    tcl = tc and b["hidden_tc"]
    hid = L - 1
    n = {"row_bwd": L}
    if tcl:
        n.update(tc_split=2 * hid, tc_dense_fwd=hid, norm_fwd=hid, tc_wgrad=hid, tc_dgrad=hid)
        hidden_reduce = hid * (b["tc_ksplit"] > 1)
    else:
        n.update(dense_fwd=hid, wgrad=hid, dgrad=hid)
        hidden_reduce = hid * (b["ffma_hidden_splits"] > 1)
    if bits and tc:
        n["tc_split"] = n.get("tc_split", 0) + 1            # wfrag
        n["norm_fwd"] = n.get("norm_fwd", 0) + 1            # layer 0's LayerNorm
        n["bits_dense_fwd"] = n["bits_wgrad"] = 1
        first_reduce = int(b["bits_splits"] > 1)
    else:
        n["gather_rows"] = 1                                # gather, or the bits' expand
        n["dense_fwd"] = n.get("dense_fwd", 0) + 1
        n["wgrad"] = n.get("wgrad", 0) + 1
        first_reduce = 1 if D <= 8 else int(b["ffma_first_splits"] > 1)
    n["norm_reduce"] = 1 if bits else 2                     # popcounts, or colsum2 of the gathered rows
    n["grad_finalize"] = L + first_reduce + hidden_reduce + bits
    return {k: v for k, v in n.items() if v}


# --------------------------------------------------------------------------------------------------------------------
# sets: parameters, rows, actions, targets and their oracle
# --------------------------------------------------------------------------------------------------------------------
def nsets(S):
    return 1 if S == 1 else min(S, 4)


def seed_assign(S):
    a = np.array([2 + s % 2 for s in range(S)])
    a[0] = a[-1] = 0
    if S > 2:
        a[1] = 1
    return np.minimum(a, nsets(S) - 1)


@functools.lru_cache(maxsize=None)
def board_pool(game, seed):
    if game == "Seaquest-MinAtar":
        return NT.seaquest_boards(POOL, seed).reshape(POOL, -1).astype(np.uint8)
    return TM._env_bits(game, POOL, seed)


def set_rows(case, j, rng):
    kind, D, H, L, A, S, T, E, rows, game = CASES[case]
    if kind == "mlp":
        f_rng = np.random.default_rng(D)                    # per-feature offsets and scales shared by the sets
        off, scl = f_rng.standard_normal(D), np.exp(f_rng.uniform(-1.5, 2.5, D))
        return (off + rng.standard_normal((rows, D)) * scl).astype(F32)
    pool = board_pool(game, 50 + j)
    x = np.concatenate([pool[rng.integers(0, POOL, rows // 2)],
                        (rng.random((rows - rows // 2, D)) < 0.5).astype(np.uint8)])
    return x[rng.permutation(rows)]


def fwd_cached_z0(p64, x64):
    """relu_inputs for NT.clear_relu_kink: Dense_0's product is computed once (only LayerNorm biases move)."""
    L = sum(1 for k in p64 if k.startswith("LayerNorm_") and k.endswith("/bias"))
    z0 = x64 @ p64["Dense_0/kernel"] + p64["Dense_0/bias"]

    def f(p):
        ys, h = [], None
        for l in range(L):
            z = z0 if l == 0 else h @ p[f"Dense_{l}/kernel"].astype(F64) + p[f"Dense_{l}/bias"].astype(F64)
            y, _ = R._layer_norm_fwd(z, p[f"LayerNorm_{l}/scale"].astype(F64), p[f"LayerNorm_{l}/bias"].astype(F64))
            ys.append((f"LayerNorm_{l}/bias", y))
            h = np.maximum(y, 0)
        return h @ p[f"Dense_{L}/kernel"].astype(F64) + p[f"Dense_{L}/bias"].astype(F64), ys
    return f


@functools.lru_cache(maxsize=None)
def case_set(case, j):
    """Set j of a case: fp32 parameters, rows, actions, targets; for j < 2 (checked) also the oracle in fp64 and fp32,
    the fp64 bn_sums and the fp64 q of the first E rows."""
    kind, D, H, L, A, S, T, E, rows, _ = CASES[case]
    spec = spec_of(case)
    seed = 9000 + 100 * j + D + H + L
    rng = np.random.default_rng(seed)
    p = NT.set_params(spec, "mlp", R.mlp_param_shapes(D, A, H, L), "random" if j % 2 == 0 else "init", seed,
                      "layer_norm")
    x = set_rows(case, j, rng)
    act = rng.integers(0, A, rows).astype(np.int32)
    out = dict(p=p, x=x, act=act)
    if j >= 2:
        out["tgt"] = rng.standard_normal(rows).astype(F32)
        return out
    x64 = x.astype(F64)
    q64 = NT.clear_relu_kink(p, fwd_cached_z0(NT.cast_tree(p, F64), x64))
    tgt = td_targets(q64[np.arange(rows), act], DELTAS[j], rng)
    p64 = NT.cast_tree(p, F64)
    out.update(tgt=tgt, ref=R.mlp_loss_and_grads(p64, x64, act, tgt.astype(F64)),
               ref32=R.mlp_loss_and_grads(p, x.astype(F32), act, tgt), q_fwd=R.mlp_forward(p64, x64[:E]))
    if kind == "bits":
        cnt = x.sum(0, dtype=np.int64).astype(F32)
        out["bn"] = (np.concatenate([cnt, cnt]), None)
    else:
        out["bn"] = (np.concatenate([x64.sum(0), (x64 * x64).sum(0)]),
                     np.concatenate([np.abs(x64).sum(0), (x64 * x64).sum(0)]))
    del x64
    return out


def obs_rows(case, x):
    """The observation rows as the engine stores them: fp32, or packed int32 words."""
    return x if CASES[case][0] == "mlp" else TM._pack(x)


def params_and_assign(case, spec):
    S = CASES[case][5]
    sets = [case_set(case, j) for j in range(nsets(S))]
    assign = seed_assign(S)
    flat = torch.cat([spec.flatten(s["p"], 1, dev()) for s in sets], 0)[t_(assign, torch.int64)].contiguous()
    return sets, assign, flat


def poison(case):
    return float("nan") if CASES[case][0] == "mlp" else -1


# --------------------------------------------------------------------------------------------------------------------
# the rollout buffers and the calls
# --------------------------------------------------------------------------------------------------------------------
def rollout_buffers(case, sets, assign):
    """obs [S][(T+1) E][W], action / target [S][T E] and the gather [S][rows]: the last minibatch of a device
    permutation of [0, T E) per seed (own key); set assign[s]'s rows at the gathered positions in minibatch order."""
    from purejaxql_b200 import jaxrandom
    kind, D, H, L, A, S, T, E, rows, _ = CASES[case]
    n = T * E
    perm = jaxrandom.permutation_indices(jaxrandom.split(jaxrandom.PRNGKey(D + H + S, dev()), S), n, chunk=rows)
    gather = perm[n // rows - 1].contiguous()
    del perm
    a = t_(assign, torch.int64)
    sel = (torch.arange(S, device=dev())[:, None], gather.long())
    o = torch.from_numpy(np.stack([obs_rows(case, s["x"]) for s in sets])).to(dev())
    obs = torch.full((S, (T + 1) * E, o.shape[-1]), poison(case), dtype=o.dtype, device=dev())
    obs[sel] = o[a]
    del o
    act_sets = t_(np.stack([s["act"] for s in sets]), torch.int32)[a]
    action = ((act_sets[:, torch.arange(n, device=dev()) % rows] + 1) % A).to(torch.int32)   # not the gathered rows'
    action[sel] = act_sets
    target = torch.full((S, n), float("nan"), device=dev())
    target[sel] = t_(np.stack([s["tgt"] for s in sets]), torch.float32)[a]
    return obs, action, target, gather


def loss_grad(case, spec, flat, bufs):
    """pqn_qnet_loss_grad at the rollout strides into guarded outputs, profiled.
    -> (grads [S, P], loss [S], qsa [S], bn_sums [S, 2D]), {kernel: launches}"""
    L_, p = _lib().lib(), _lib().p
    kind, D, H, L, A, S, T, E, rows, _ = CASES[case]
    obs, action, target, gather = bufs
    P = flat.shape[1]
    grads, ls, qs, bn = guarded(S * P, float("nan")), guarded(S), guarded(S), guarded(S * 2 * D, float("nan"))
    ws = torch.empty(int(L_.pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())
    torch.cuda.synchronize()
    L_.pqn_profile_enable(1)
    try:
        _lib().profile_read(reset=True)
        _lib().check(L_.pqn_qnet_loss_grad(spec.desc, p(flat), None, p(obs), p(gather), (T + 1) * E, p(action),
                                           p(target), T * E, p(grads), p(ls), p(qs), p(bn), S, rows, p(ws),
                                           _lib().stream_ptr()), "pqn_qnet_loss_grad")
        torch.cuda.synchronize()
        launches = {k: v[1] for k, v in _lib().profile_read(reset=True).items()}
    finally:
        L_.pqn_profile_enable(0)
    del ws
    for name, t, m in (("grads", grads, S * P), ("loss_sum", ls, S), ("qsa_sum", qs, S), ("bn_sums", bn, S * 2 * D)):
        assert bool(torch.isnan(t[m:]).all()), (name, "written past its end")
    return (grads[:S * P].view(S, P), ls[:S], qs[:S], bn[:S * 2 * D].view(S, 2 * D)), launches


def replica_failures(outs, assign):
    bad = []
    for j in np.unique(assign):
        seeds = np.flatnonzero(assign == j)
        for name, t in outs.items():
            b = t[t_(seeds, torch.int64)].contiguous().view(torch.int32)
            d = (b != b[:1]).reshape(len(seeds), -1).any(1)
            if bool(d.any()):
                bad.append(("replicas of set %d differ in %s" % (j, name), seeds[d.cpu().numpy()][:8].tolist()))
    return bad


@pytest.fixture
def tc_path():
    yield lambda p: _lib().check(_lib().lib().pqn_set_tensor_core_path(p))
    _lib().lib().pqn_set_tensor_core_path(2)


@pytest.fixture(scope="module", autouse=True)
def report():
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    if not REPORT:
        return
    worst = {}
    for case, path, what, v in REPORT:
        k = (case, path, what)
        worst[k] = max(worst.get(k, 0.0), v)
    print("\nworst per (case, path):")
    for k in sorted(worst):
        print("  %-10s path %d  %-28s %10.3g" % (*k, worst[k]))
    print("module wall time %.1f s, peak device memory %.2f GB"
          % (time.time() - t0, torch.cuda.max_memory_allocated() / 2 ** 30))


IDS = {
    "cartpole": "cartpole-128x128-thin1chunk-wgmma-unsplit",
    "acrobot": "acrobot-1x262144-thin-reduce32-splitK",
    "ragged64": "ragged64-5x4097-ffma-hidden-thin-last1row",
    "wide": "wide-9x4097-ffma-first-splits-splitK",
    "breakout": "bits-breakout-128x128-unsplit-strideP",
    "breakout16": "bits-breakout-16x2048-3splits",
    "seaquest": "bits-seaquest-1x262144-fwd4-17splits",
    "spaceinv": "bits-spaceinv-9x4097-wgrad64-head0",
}


# --------------------------------------------------------------------------------------------------------------------
# loss and gradients
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", [2, 0], ids=["path2", "path0"])
@pytest.mark.parametrize("case", list(CASES), ids=[IDS[c] for c in CASES])
def test_loss_grad_in_rollout_layout(case, path, tc_path):
    kind, D, H, L, A, S, T, E, rows, _ = CASES[case]
    tc_path(path)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    b = branches(case, sms)
    for name, pred in WANT[case].items():
        assert pred(b[name]), (case, name, b[name], sms)
    spec = spec_of(case)
    sets, assign, flat = params_and_assign(case, spec)
    bufs = rollout_buffers(case, sets, assign)
    (grads, ls, qs, bn), launches = loss_grad(case, spec, flat, bufs)
    del bufs
    assert launches == expected_launches(case, path, b), (launches, expected_launches(case, path, b), b)
    bad = replica_failures({"grads": grads, "loss_sum": ls, "qsa_sum": qs, "bn_sums": bn}, assign)
    for j in range(min(2, len(sets))):
        s, sd = sets[j], int(np.flatnonzero(assign == j)[0])
        loss, q_sa, g = s["ref"]
        g32 = s["ref32"][2]
        for what, got, want in (("loss", float(ls[sd]), loss), ("qmean", float(qs[sd]), q_sa.mean())):
            e = abs(got - want) / max(1.0, abs(want))
            REPORT.append((case, path, what + " err", e))
            if not e < 1e-5:
                bad.append((j, what, got, want))
        got = NT.leaves(spec, grads, sd)
        scale = max(np.abs(v).max() for v in g.values())
        for name, want in g.items():
            err = float(np.abs(got[name] - want).max())
            spread = float(np.abs(g32[name].astype(F64) - want).max())
            REPORT.append((case, path, "grad err / scale", err / scale))
            REPORT.append((case, path, "grad err / spread32", err / spread if spread > 0 else (0.0 if err == 0 else np.inf)))
            if not (err < 2e-5 * scale or err <= MLP_SPREAD_K * spread):
                bad.append((j, name, err / scale, err / spread if spread > 0 else np.inf))
        bgot = bn[sd].cpu().numpy()
        bwant, bscale = s["bn"]
        if bscale is None:
            if not np.array_equal(bgot, bwant):
                bad.append((j, "bn_sums", int(np.abs(bgot - bwant).max())))
        else:
            e = float((np.abs(bgot - bwant) / bscale).max())
            REPORT.append((case, path, "bn_sums err / sum|x|", e))
            if not e <= 1e-6:
                bad.append((j, "bn_sums", e))
    assert not bad, bad[:20]


# --------------------------------------------------------------------------------------------------------------------
# the rollout's forward: E rows of step t in the (T+1) E-row buffer
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", [2, 0], ids=["path2", "path0"])
@pytest.mark.parametrize("case", list(CASES), ids=[IDS[c] for c in CASES])
def test_rollout_forward(case, path, tc_path):
    L_, p = _lib().lib(), _lib().p
    kind, D, H, L, A, S, T, E, rows, _ = CASES[case]
    tc_path(path)
    spec = spec_of(case)
    sets, assign, flat = params_and_assign(case, spec)
    o = torch.from_numpy(np.stack([obs_rows(case, s["x"][:E]) for s in sets])).to(dev())[t_(assign, torch.int64)]
    ws = torch.empty(int(L_.pqn_net_workspace_bytes(spec.desc, S, E)), dtype=torch.uint8, device=dev())
    bad = []
    for t in (0, T):
        buf = torch.full((S, T + 1, E, o.shape[-1]), poison(case), dtype=o.dtype, device=dev())
        buf[:, t] = o
        q = torch.full((S * E * A + GUARD,), float("nan"), device=dev())
        _lib().check(L_.pqn_qnet_forward(spec.desc, p(flat), None, _lib().raw(buf[:, t]), None, (T + 1) * E, p(q), S,
                                         E, p(ws), _lib().stream_ptr()), "pqn_qnet_forward")
        torch.cuda.synchronize()
        assert bool(torch.isnan(q[S * E * A:]).all()), ("q written past its end", t)
        qs = q[:S * E * A].view(S, E * A)
        del buf
        bad += [(t,) + f for f in replica_failures({"q": qs}, assign)]
        for j in range(min(2, len(sets))):
            ref = sets[j]["q_fwd"]
            got = qs[int(np.flatnonzero(assign == j)[0])].view(E, A).cpu().numpy()
            e = float(np.abs(got - ref).max() / max(1.0, np.abs(ref).max()))
            REPORT.append((case, path, "forward err", e))
            if not e < 1e-5:
                bad.append((t, j, "q", e))
    assert not bad, bad[:20]
