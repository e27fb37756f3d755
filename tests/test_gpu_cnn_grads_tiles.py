"""The MinAtar CNN's loss and gradients (``pqn_qnet_loss_grad``) against fp64 where every warp of the training step's
conv kernels runs many samples, at the channel counts 6, 7 and 10 as well as 4, with the rollout buffer's seed strides.

The conv kernels of the training step are grid-stride loops: warp w of CTA b takes the rows b * WARPS + w,
+ row_stride, ... with row_stride = gridDim.x * WARPS and gridDim.x from ``conv_mma_ctas`` / ``conv_bwd_ctas``
(``pqn_net.cu``).  Only a warp's third row reaches the steady state of the two-deep prefetch of
``conv_fwd_mma16_kernel`` and ``conv_bwd_mma16_kernel`` (the observation whose gather index was itself prefetched), and
only many rows build up the per-warp accumulators (``wrun``, ``a_dsc``, ``a_dbi``, ``a_dcb``, the ``bn_sums``
popcounts) and make the backward rebuild the conv LayerNorm of many samples in turn into one stage.  At 2 x 4,096 rows
(``test_gpu_cnn_grads.py``) a warp of the fp16 conv backward runs 2 rows; here it runs up to 86.  Cases (S x rows,
T, E; the channel counts and action counts of the games):

  - many: 128 x 4,096, T = 32, E = 4,096: C = 6 (A 4), 7 (3), 10 (5), 10 (18: the mixed path), 4 (5); 32 dense tiles
    per CTA, 8 finalize slices, the headline layout; at C = 10 the observation buffer is 2.2 GB, so its byte offsets
    pass 2^31;
  - odd: 37 x 4,097, T = 16, E = 257: C = 6, 7, 10; a one-row last dense tile, CTAs whose tiles change seed;
  - minatar5: 16 x 1,024, T = 32, E = 1,024: C = 4 (5), 6 (4), 7 (3), ``bench.py --config minatar5``'s minibatch;
  - grid: 512 x 128, T = 32, E = 128: C = 6, 7; a four-point hyperparameter grid of 128 seeds each of the preset.
Kernel paths (``pqn_set_tensor_core_path``, ``pqn_set_conv_mma_path``): many runs (2, 1) fp16-split dense + fp16 conv
(the default), (0, 0) FFMA + CUDA-core conv backward, (2, 3) the tf32 conv backward and (1, 1) 3xTF32; the other cases
(2, 1) and (0, 0).  ``test_geometry_rows_per_warp`` restates the grid sizing and checks that these cases reach the
regimes above on this device.

Inputs, as ``engine.update_body`` passes them.  NSETS = 8 sets of parameters, boards and targets per case: set j has
``R.random_params`` (even j) or the engine's ``spec.init`` (odd j: rstd = 1000 on empty patches), TD errors of scale
1e-2, 1 or 30 (j mod 3), and boards of the game of that width (synthetic at C = 10) with an empty board and a board
with one channel full.  A set's boards come from a pool of 6,000; boards where some ReLU input (the output of
LayerNorm_0 or LayerNorm_1) lies within RELU_MARGIN = 2e-6 of zero but is not exactly zero are left out.  At such a
board the gradient is discontinuous within fp32 rounding: any fp32 evaluation may take the other side of the kink, and
in sets drawn without this rule, one flipped element moved the fp16-split and 3xTF32 paths' gradients by 2e-3 to 3e-3
of their scale (550 to 3,300x spread32), at 8 seeds as at 128.

Seeds take the sets in a fixed pseudo-random order.  Per seed, ``obs_buf`` is [(T+1) E][PW] and ``action`` /
``target`` are [T E]: the seed's gather is one ``rows``-long chunk of a device permutation of [0, T E)
(``jaxrandom.permutation_indices``, as the engine draws it), each seed with its own key, and the set's boards, actions
and targets sit at the gathered positions.  Every other observation row holds all-ones words and
every other target is NaN, so a wrong row or seed stride reads other boards or a NaN instead of passing.  The
minibatch rows are in the same order in every replica of a set, so replicas must agree bit for bit although they read
different buffer rows.  ``grads``, ``loss_sum``, ``qsa_sum`` and ``bn_sums`` carry a NaN guard tail.

Checks, per case and path:
  - seeds holding the same set are bit-identical; the four conv tensors of the CUDA-core conv backward (float
    atomics) within 2^-16 of their scale, as in ``test_bench_geometry_loss_grad``;
  - the first seed of each set meets the tolerance rule of ``test_gpu_cnn_grads.py`` (``compare``): every gradient
    within max(2e-5 * scale, 8 * spread32) (16 at delta = 1e-2), split-precision paths within 16 * spread32, the loss
    and the mean chosen q within 2e-5 of their scale; ``bn_sums`` exact;
  - max |dz * gs| of the fp16 conv backward's dz planes (fp64, ``conv_dz_max`` through ``oracle``) stays below the
    fp16 maximum;
  - the guard tails are untouched.
The worst err / scale and err / spread32 per (path, C, A, case), the rows per warp, max |dz * gs| per C and the peak
device memory are printed at the end of the module.

Measured on one NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit).  Rows per warp (most / fewest): fp16 conv
backward 86 / 85 (many, C != 4), 25 / 24 (odd), 11 / 10 (grid), 3 / 2 (minatar5); fp16 conv forward 52 / 51, 15 / 14,
7 / 6, 3 / 2; CUDA-core conv backward 57 / 56 (many); dense GEMM tiles per CTA 32, 10 and 4.  Replicas bit-identical
on every path.  Worst err / spread32 over the gradient tensors: fp16-split + fp16 conv 8.8 (C = 7), fp16-split + tf32
conv 8.8 (C = 7), 3xTF32 8.7 (C = 4), FFMA 8.2 (C = 4); per C at most 8.7 (C = 4), 6.0 (6), 8.8 (7), 7.5 (10).  Loss
and mean chosen q within 2e-5 of their scale.  max |dz * gs| of the fp16 conv backward: 1.5e4 (C = 4), 3.4e4 (6),
4.02e4 (7: 1.63x below the fp16 maximum), 3.4e4 (10).  Up to 113 of a pool's 6,000 boards were left out for the
ReLU margin, 3.2 on average.  The module takes about 4.5 minutes; peak device memory 9.7 GB.
"""
import functools

import numpy as np
import pytest
import torch

from oracle import pqn_ref as R
from test_gpu_cnn_grads import (CONV_ATOMIC, FLOOR, FP16_MAX, REPORT as CMP_REPORT, _sms, check_bn_sums, cnn_spec,
                                compare, conv_dz_scale, conv_mma_ctas, final_slices, init_params, leaves,
                                oracle, set_path)
from test_oracle_cnn_grads import EMPTY_ROW, FULL_ROW, cast, game_obs, minibatch_gather, pack_obs, td_targets

pytestmark = pytest.mark.gpu

F64 = np.float64
NSETS = 8
POOL = 6000           # boards per (C, set); a case's set takes `rows` of them, the empty and the full board included
GUARD = 1024          # NaN floats after grads, loss_sum, qsa_sum and bn_sums
DELTAS = (1e-2, 1.0, 30.0)
CASES = {             # S, rows, T, E
    "many": (128, 4096, 32, 4096),
    "odd": (37, 4097, 16, 257),
    "minatar5": (16, 1024, 32, 1024),
    "grid": (512, 128, 32, 128),
}
CASE_SHAPES = {
    "many": [(6, 4), (7, 3), (10, 5), (10, 18), (4, 5)],
    "odd": [(6, 4), (7, 3), (10, 5)],
    "minatar5": [(4, 5), (6, 4), (7, 3)],
    "grid": [(6, 4), (7, 3)],
}
PATH_NAMES = {(2, 1): "f16split+f16conv", (0, 0): "ffma", (2, 3): "f16split+tf32conv", (1, 1): "3xtf32+f16conv"}
CASE_PATHS = {"many": [(2, 1), (0, 0), (2, 3), (1, 1)], "odd": [(2, 1), (0, 0)], "minatar5": [(2, 1), (0, 0)],
              "grid": [(2, 1), (0, 0)]}
PARAMS = [(case, C, A) for case in CASES for C, A in CASE_SHAPES[case]]
RELU_MARGIN = 2e-6    # no ReLU input of the minibatch closer to the kink than this (fp64; LayerNorm outputs are O(1))
MAX_DRAWS = 8
REPORT = []           # (path, C, A, case, tensor, err / scale, err / spread32)
EXCLUDED = []         # pool boards per set left out for a ReLU input within RELU_MARGIN of zero
DZ = {}               # C -> max |dz * gs| over every set of every case


def dev():
    return torch.device("cuda:0")


def _lib():
    from purejaxql_b200 import _lib
    return _lib


def t_(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


def cdiv(a, b):
    return (a + b - 1) // b


# --------------------------------------------------------------------------------------------------------------------
# grid sizing of the training step, restated from pqn_net.cu / pqn_tc.cu
# --------------------------------------------------------------------------------------------------------------------
def conv_bwd_ctas(S, rows):
    """CTAs per seed of the CUDA-core conv backward (conv_bwd_ctas): about 4 waves of 2 CTAs per SM."""
    return max(1, min((_sms() * 2 * 4 + S - 1) // S, (rows + 7) // 8))


def geometry(S, rows, C):
    """Rows per warp (fewest, most) of the training step's row loops, the conv-backward finalize slices and the dense
    GEMMs' tiles per CTA (fewest, most) for S seeds x rows at C channels."""
    def per_warp(ctas, warps):
        return rows // (ctas * warps), cdiv(rows, ctas * warps)
    mma2 = conv_mma_ctas(S, rows, 2)
    tiles = S * cdiv(rows, 128)
    grid = min(tiles, _sms())
    return dict(bwd16=per_warp(mma2, 8 if C == 4 else 6),       # conv_bwd_mma16_kernel, ConvBwd16<C>::WARPS
                fwd16=per_warp(conv_mma_ctas(S, rows, 5), 4),   # conv_fwd_mma16_kernel, CONV16_WARPS x 5 CTAs / SM
                bwd_tf32=per_warp(mma2, 8),                     # conv_bwd_mma_kernel
                bwd_cc=per_warp(conv_bwd_ctas(S, rows), 8),     # conv_bwd_kernel
                row_bwd=per_warp(conv_mma_ctas(S, rows, 4), 8),
                slices=final_slices(mma2),
                tiles=(tiles // grid, cdiv(tiles, grid)))


def test_geometry_rows_per_warp():
    """Every many and odd case at C = 6, 7, 10 runs at least 3 rows on every warp of both fp16 conv kernels, both
    finalize kernels (8 and 32 slices) run at some C != 4, and the dense GEMMs run more than one tile on every CTA in
    many, odd and grid.  On a 132-SM H100 also the exact counts, including those of the existing tests' shapes."""
    for case in ("many", "odd"):
        S, rows = CASES[case][:2]
        for C in (6, 7, 10):
            g = geometry(S, rows, C)
            assert g["bwd16"][0] >= 3 and g["fwd16"][0] >= 3, (case, C, g)
    slices = {geometry(*CASES[case][:2], C)["slices"] for case in CASES for C, _ in CASE_SHAPES[case] if C != 4}
    assert slices == {8, 32}, slices
    for case in ("many", "odd", "grid"):
        assert geometry(*CASES[case][:2], 6)["tiles"][0] >= 2, case
    if _sms() == 132:
        # (S, rows, C): most rows per warp of the fp16 conv backward / fp16 conv forward / CUDA-core conv backward,
        # finalize slices, most tiles per CTA; the first four are test_gpu_cnn_grads.py's and test_gpu_train.py's
        want = {(2, 4096, 4): (2, 4, 1, 32, 1), (2, 4096, 6): (2, 4, 1, 32, 1), (2, 4097, 6): (2, 4, 1, 32, 1),
                (1, 128, 4): (1, 2, 1, 8, 1), (1, 128, 6): (2, 2, 1, 8, 1), (128, 4096, 4): (64, 52, 57, 8, 32),
                (128, 4096, 6): (86, 52, 57, 8, 32), (37, 4097, 6): (25, 15, 18, 8, 10),
                (16, 1024, 4): (2, 3, 2, 32, 1), (16, 1024, 6): (3, 3, 2, 32, 1), (512, 128, 6): (11, 7, 6, 8, 4)}
        got = {}
        for S, rows, C in want:
            g = geometry(S, rows, C)
            got[(S, rows, C)] = (g["bwd16"][1], g["fwd16"][1], g["bwd_cc"][1], g["slices"], g["tiles"][1])
        assert got == want, got


# --------------------------------------------------------------------------------------------------------------------
# inputs
# --------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def pool_boards(C, j):
    return game_obs(C, POOL, 3000 + 10 * C + j)


def relu_margins(y):
    """Per row, the smallest |y| over its non-zero ReLU inputs (exact zeros, the init regime's empty patches, are
    exact on every path too)."""
    a = np.abs(y.reshape(y.shape[0], -1))
    return np.where(a == 0, np.inf, a).min(1)


def make_set(C, A, case, j):
    """Set j of a case: parameters, the boards / actions / targets of the minibatch rows in order, and the oracle's
    results (test_gpu_cnn_grads.oracle on a state whose gather is the identity).  Boards with a ReLU input within
    RELU_MARGIN of zero are left out of the minibatch (module docstring)."""
    rows = CASES[case][1]
    regime = "random" if j % 2 == 0 else "init"
    delta = DELTAS[j % 3]
    rng = np.random.default_rng(5000 + 100 * C + 10 * A + j + 7 * rows)
    pool = pool_boards(C, j)
    for k in range(MAX_DRAWS):
        seed = 5000 + 100 * C + 10 * A + j + 100000 * k
        p = R.random_params(R.cnn_param_shapes(C, A), seed) if regime == "random" else init_params(C, A, seed)
        _, cache = R.cnn_forward(cast(p, F64), pool.astype(F64), want_cache=True)
        ok = np.minimum(relu_margins(cache[2]), relu_margins(cache[5])) >= RELU_MARGIN
        if ok[EMPTY_ROW] and ok[FULL_ROW] and ok.sum() >= rows:
            break
    else:
        raise AssertionError((case, C, A, j, "no parameter draw keeps the empty and full boards off the ReLU kink"))
    eligible = np.flatnonzero(ok)                  # starts with EMPTY_ROW, FULL_ROW
    EXCLUDED.append(int((~ok).sum()))
    obs = pool[eligible[minibatch_gather(len(eligible), rows, rng)]]
    act = rng.integers(0, A, rows).astype(np.int32)
    q64 = R.cnn_forward(cast(p, F64), obs.astype(F64))
    st = dict(p=p, obs=obs, gather=np.arange(rows), act=act, q_sa=q64[np.arange(rows), act])
    tgt = td_targets(st["q_sa"], delta, rng)
    return dict(st=st, tgt=tgt, ref=oracle(st, tgt), delta=delta, regime=regime)


def seed_sets(S, case):
    """Set of each seed: a fixed pseudo-random order in which every set occurs; -> (set of seed, first seed of set)."""
    assign = np.random.default_rng(S + len(case)).permutation(np.arange(S) % NSETS)
    return assign, [int(np.flatnonzero(assign == j)[0]) for j in range(NSETS)]


def rollout_buffers(spec, sets, assign, case, key):
    """obs_buf [S][(T+1) E][PW], action / target [S][T E] and the gather [S][rows] of one case (module docstring)."""
    from purejaxql_b200 import jaxrandom
    S, rows, T, E = CASES[case]
    n = T * E
    perm = jaxrandom.permutation_indices(jaxrandom.split(jaxrandom.PRNGKey(key, dev()), S), n)
    chunk = n // rows - 1                                   # the last whole minibatch of the permutation
    gather = perm[:, chunk * rows:(chunk + 1) * rows].contiguous()
    del perm
    srt = torch.sort(gather, 1)[0]
    assert bool((srt[:, 1:] > srt[:, :-1]).all()) and int(srt.min()) >= 0 and int(srt.max()) < n
    del srt
    a = t_(assign, torch.int64)
    sel = (torch.arange(S, device=dev())[:, None], gather.long())
    packed = t_(np.stack([pack_obs(s["st"]["obs"]) for s in sets]), torch.int32)
    obs_buf = torch.full((S, (T + 1) * E, packed.shape[-1]), -1, dtype=torch.int32, device=dev())
    obs_buf[sel] = packed[a]
    gen = torch.Generator(device=dev())
    gen.manual_seed(key)
    action = torch.randint(0, spec.num_actions, (S, n), generator=gen, device=dev(), dtype=torch.int32)
    action[sel] = t_(np.stack([s["st"]["act"] for s in sets]), torch.int32)[a]
    target = torch.full((S, n), float("nan"), device=dev())
    target[sel] = t_(np.stack([s["tgt"] for s in sets]), torch.float32)[a]
    return obs_buf, action, target, gather


def guarded(n, dev_):
    out = torch.full((n + GUARD,), float("nan"), device=dev_)
    out[:n] = 0.0
    return out


def loss_grad(spec, flat, bufs, case, ws):
    """pqn_qnet_loss_grad at the case's strides into guarded outputs; -> grads [S, P], loss [S], qsa [S], bn [S, 2C]"""
    L, p = _lib().lib(), _lib().p
    S, rows, T, E = CASES[case]
    obs_buf, action, target, gather = bufs
    P, C = flat.shape[1], spec.in_c
    grads, ls, qs, bn = guarded(S * P, dev()), guarded(S, dev()), guarded(S, dev()), guarded(S * 2 * C, dev())
    grads[:S * P] = float("nan")                            # the entry point clears them itself
    _lib().check(L.pqn_qnet_loss_grad(spec.desc, p(flat), None, p(obs_buf), p(gather), (T + 1) * E, p(action),
                                      p(target), T * E, p(grads), p(ls), p(qs), p(bn), S, rows, p(ws),
                                      _lib().stream_ptr()), "pqn_qnet_loss_grad")
    torch.cuda.synchronize()
    for name, t, n in (("grads", grads, S * P), ("loss_sum", ls, S), ("qsa_sum", qs, S), ("bn_sums", bn, S * 2 * C)):
        assert bool(torch.isnan(t[n:]).all()), (case, name, "written past its end")
    return grads[:S * P].view(S, P), ls[:S], qs[:S], bn[:S * 2 * C].view(S, 2 * C)


def replica_failures(spec, out, assign, first, path):
    """Seeds holding the same set against the set's first seed, bit for bit (the CUDA-core conv backward's four
    atomically summed tensors within 2^-16 of their scale).  -> failures"""
    grads, ls, qs, bn = out
    S = grads.shape[0]
    ref = t_(np.asarray(first)[assign], torch.int64)
    bits = grads.view(torch.int32)
    diff = bits != bits[ref]
    bad = []
    if path[1] == 0:
        for pth, off, shape, _ in spec.entries:
            if "/".join(pth) in CONV_ATOMIC:
                n = int(np.prod(shape))
                g, w = grads[:, off:off + n], grads[ref, off:off + n]
                bound = FLOOR * 16 * w.abs().amax(1)
                over = ((g - w).abs().amax(1) > bound) | torch.isnan(g).any(1)
                if bool(over.any()):
                    bad.append(("replicas", "/".join(pth), torch.nonzero(over).flatten()[:8].tolist()))
                diff[:, off:off + n] = False
    seeds = torch.nonzero(diff.any(1)).flatten()
    if len(seeds):
        bad.append(("replicas differ in grads", seeds[:8].tolist()))
    for name, t in (("loss_sum", ls), ("qsa_sum", qs), ("bn_sums", bn)):
        b = t.view(torch.int32)
        d = (b != b[ref]) if b.dim() == 1 else (b != b[ref]).any(1)
        if bool(d.any()):
            bad.append(("replicas differ in " + name, torch.nonzero(d).flatten()[:8].tolist()))
    return bad


@pytest.fixture(scope="module", autouse=True)
def report():
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    if not REPORT:
        return
    print("\n%d SMs; most (fewest) rows per warp: fp16 conv bwd, fp16 conv fwd, tf32 conv bwd, CUDA-core conv bwd, "
          "row_bwd; finalize slices; dense tiles per CTA" % _sms())
    for case, (S, rows, T, E) in CASES.items():
        for C in sorted({c for c, _ in CASE_SHAPES[case]}):
            g = geometry(S, rows, C)
            print("  %-8s %3d x %-5d C=%-2d %3d (%3d) %3d (%3d) %3d (%3d) %3d (%3d) %3d (%3d)  %2d  %2d (%2d)" % (
                case, S, rows, C, g["bwd16"][1], g["bwd16"][0], g["fwd16"][1], g["fwd16"][0], g["bwd_tf32"][1],
                g["bwd_tf32"][0], g["bwd_cc"][1], g["bwd_cc"][0], g["row_bwd"][1], g["row_bwd"][0], g["slices"],
                g["tiles"][1], g["tiles"][0]))
    worst = {}
    for path, C, A, case, name, rs, rsp in REPORT:
        k = (PATH_NAMES[path], C, A, case)
        rsp = 0.0 if name in ("loss", "qmean") else rsp     # held to 2e-5 of the scale only
        a = worst.get(k, (0.0, 0.0, "", ""))
        worst[k] = (max(a[0], rs), max(a[1], rsp), name if rs >= a[0] else a[2], name if rsp >= a[1] else a[3])
    print("worst err/scale (gradients, loss, mean q) and err/spread32 (gradients) per (path, C, A, case):")
    for k in sorted(worst):
        print("  %-18s C=%-2d A=%-2d %-9s %9.2e %7.2f  (%s; %s)" % (*k, *worst[k]))
    print("max |dz * gs| of the fp16 conv backward: " + ", ".join("C=%d %.3g" % kv for kv in sorted(DZ.items())))
    print("pool boards left out per set for a ReLU input within %g of zero: up to %d of %d, %.1f on average" % (
        RELU_MARGIN, max(EXCLUDED), POOL, float(np.mean(EXCLUDED))))
    print("peak device memory: %.2f GB" % (torch.cuda.max_memory_allocated() / 2 ** 30))


@pytest.mark.parametrize("case,C,A", PARAMS, ids=["%s-C%dA%d" % p for p in PARAMS])
def test_many_rows_per_warp_loss_grad(case, C, A):
    S, rows, T, E = CASES[case]
    spec = cnn_spec(C, A)
    sets = [make_set(C, A, case, j) for j in range(NSETS)]
    assign, first = seed_sets(S, case)
    for j, s in enumerate(sets):
        dzs = s["ref"][3] * conv_dz_scale(rows)
        DZ[C] = max(DZ.get(C, 0.0), dzs)
        assert dzs < FP16_MAX, (case, C, A, j, dzs)
    flat = torch.cat([spec.flatten(s["st"]["p"], 1, dev()) for s in sets], 0)[t_(assign, torch.int64)].contiguous()
    bufs = rollout_buffers(spec, sets, assign, case, 100 * C + A)
    L = _lib().lib()
    ws = torch.empty(int(L.pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())
    bad = []
    for path in CASE_PATHS[case]:
        set_path(path)
        try:
            out = loss_grad(spec, flat, bufs, case, ws)
        finally:
            set_path((2, 1))
        bad += [(PATH_NAMES[path],) + b for b in replica_failures(spec, out, assign, first, path)]
        grads = out[0]
        ls, qs, bn = out[1].cpu().numpy(), out[2].cpu().numpy(), out[3].cpu().numpy()
        for j, s in enumerate(sets):
            r = first[j]
            got = {k: v.astype(F64) for k, v in leaves(spec, grads, r).items()}
            got["loss"], got["qmean"] = np.array([ls[r]], F64), np.array([qs[r]], F64)
            n0 = len(CMP_REPORT)
            bad += compare(got, s["ref"], path, (C, A, rows, "%s-%s" % (case, s["regime"]), s["delta"]))
            REPORT.extend((path, C, A, case, e[6], e[7], e[8]) for e in CMP_REPORT[n0:])
            del CMP_REPORT[n0:]
            try:
                check_bn_sums(bn[r], s["st"], C)
            except AssertionError:
                bad.append((PATH_NAMES[path], "bn_sums", j))
        del out, grads
    assert not bad, (case, C, A, bad[:20])
