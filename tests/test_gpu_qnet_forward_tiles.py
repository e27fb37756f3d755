"""The MinAtar CNN's Q-value forward (``pqn_qnet_forward``) against fp64 at shapes where every CTA of the persistent
dense GEMMs runs several 128-row tiles, on the four kernel paths of that entry point.

Both ``tc_conv_gemm_kernel`` (the conv fused into the dense GEMM, the default) and ``tc_gemm_kernel`` launch
``min(tiles, SMs)`` CTAs and step ``tile += gridDim.x``.  Only a second tile on the same CTA exercises the second
observation buffer, the W1 ring's stage and phase carried into a new tile, the conv-weight reload when the seed changes
(and skipping it when it does not), and one tile's LayerNorm epilogue overlapping the next tile's MMAs.  Cases:

  - S x rows = 37 x 1,000 (every tile a CTA moves on to belongs to a different seed, and to a different parameter
    set), 2 x 40,000 (more tiles per seed than SMs: consecutive tiles of one seed, no weight reload) and 17 x 8,193
    (a one-row last tile), each with and without a minibatch gather, at C = 4, 6, 7 and 10 channels (A = 3, 4, 3, 5;
    C = 10 has no game here that the fused kernel serves, Seaquest's 18 actions take the mixed path);
  - A = 1 ... 9 at C = 4, 37 x 1,000 (A <= PQN_TC_MAX_A = 8 through the fused LayerNorm + Q-head epilogue, A = 9 the
    first count of the mixed path: FFMA dense layer), and C = 10 with A = 18;
  - the rollout's layout: ``obs_buf[S][T+1][E][PW]`` with S = 128, T = 32, E = 4,096 read at steps 0 and T with a
    seed stride of (T+1) E rows and no gather, as ``engine.py`` calls it (4,096 tiles); every other step holds
    all-ones words, so that a wrong row stride reads boards with other Q values;
  - the evaluation's layout: ``obs[S][2][N][PW]``, read at slot 1 with a seed stride of 2N (S = 16, N = 2,100);
    in both layouts the three sets hold initial, random and small-variance parameters.

Paths: fused (fp16-split tensor cores, fp16 conv, ``pqn_set_conv_fusion(1)``), unfused (the same arithmetic in two
kernels, ``pqn_set_conv_fusion(0)``), 3xTF32 (tensor-core path 1) and FFMA (path 0, CUDA-core conv).

Parameters: the engine's ``spec.init`` (conv bias 0: rstd = 1000 on empty patches), ``R.random_params``, and two
regimes of the 128-wide LayerNorm_1 derived from the random ones: *small variance* (the kernel and bias of
CNN_0/Dense_0 scaled so that the median row std of its 128 outputs is 3e-4, 1e-3 or 3e-3 in the three sets, which
puts the variance at 0.1, 1 and 9 times eps = 1e-6) and *large mean* (30 added to every CNN_0/Dense_0 bias, where
the fast variance E[x^2] - E[x]^2 that flax, the oracle and the kernels use loses about ten bits).  Boards are the
game's (synthetic at C = 10), with an empty board, a board with one channel full and a board with every cell set among
the rows read.

Seed s holds parameter and board set s mod 3, so the fp64 oracle runs on three sets only; each set's observation rows
are drawn from its own pool of 1,024 boards, whose fp64 Q values the oracle computes once.

Checks, per case and path:
  - seeds that hold the same set are bit-identical;
  - the first three seeds against fp64: |q - q64| <= 1e-5 (DESIGN sections 3.2 and 5).  In the large-mean regime the
    fp32 oracle itself lands further than that (``spread32``, computed here), so there the rule of
    ``test_gpu_cnn_grads.py`` holds: err <= max(1e-5 * max|q64|, 8 * spread32);
  - the fused and the unfused path agree bit for bit;
  - ``q`` is allocated with a NaN guard tail: nothing past S * rows * A is written and no NaN is left in ``q``.
The worst errors per (path, C, A, regime) are printed at the end of the module, with the SM count and the tiles per CTA
of each case.

Measured on one NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit; 2-3, 4-5, 8-9, 31-32 and 2-3 tiles per CTA in the
cases above), worst |q - q64| outside the large-mean regime: fused kernel 1.8e-6 (A <= 8), 3xTF32 2.4e-6, FFMA 2.2e-6,
the mixed path (A = 9, 18) 2.2e-6; at most 2.6x the fp32 oracle's own distance on any path.  Fused and unfused are
bit-identical in every case.  In the small-variance sets the LayerNorm_1 variance runs from 0.09 to 9.1 times eps.
Large mean: the fp32 oracle lands 8e-5 - 3.2e-4 from fp64 (q scale 0.6 - 2.3); FFMA 0.98x that distance, the three
tensor-core paths up to 5.7x (1.6e-3 at C = 7).  Their LayerNorm epilogue (``epilogue_ln_row``) adds the 128 values
and squares of a row in one sequential chain per thread, where the FFMA kernel adds 16 partial sums of 8 lanes in a
butterfly, and the cancellation in E[x^2] - E[x]^2 magnifies the difference.  The module takes about 30 s.
"""
import contextlib
import functools

import numpy as np
import pytest
import torch

from oracle import pqn_ref as R
from test_oracle_cnn_grads import cast, game_obs, pack_obs

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
BAR = 1e-5
C_SPREAD = 8.0
NSETS = 3             # distinct (parameters, boards) sets; seed s holds set s % NSETS
POOL = 1024           # boards per set; observation rows are drawn from them
EXTRA = 37            # observation rows per seed beyond `rows`: the seed stride is never the row count
GUARD = 1024          # NaN floats after the S * rows * A outputs of q
SMALL_STD = (3e-4, 1e-3, 3e-3)   # median row std of the LayerNorm_1 input of set j in the small-variance regime
BIG_MEAN = 30.0
GAME_A = {4: 3, 6: 4, 7: 3, 10: 5}
SHAPES = [(37, 1000), (2, 40000), (17, 8193)]
ROLLOUT = (128, 32, 4096)      # S, T, E
EVAL = (16, 2100)              # S, N
PATHS = {"fused": (2, 1, 1), "unfused": (2, 1, 0), "3xtf32": (1, 1, 1), "ffma": (0, 0, 1)}
REGIMES = ("init", "random", "smallvar", "largemean")
REPORT = []           # (path, C, A, regime, case, err, err / spread32)
VAR_EPS = {}          # (C, A) -> (min, max) of the LayerNorm_1 variance over eps in the small-variance regime


def dev():
    return torch.device("cuda:0")


def _lib():
    from purejaxql_b200 import _lib
    return _lib


def t_(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def cta_tiles(S, rows):
    """-> (tiles, grid, [tiles of CTA b]) of the persistent dense GEMMs: grid = min(tiles, SMs), tile += grid."""
    tiles = S * ((rows + 127) // 128)
    grid = min(tiles, sms())
    return tiles, grid, [list(range(b, tiles, grid)) for b in range(grid)]


@contextlib.contextmanager
def kernel_path(name):
    L, check = _lib().lib(), _lib().check
    tc, conv, fuse = PATHS[name]
    try:
        check(L.pqn_set_tensor_core_path(tc))
        check(L.pqn_set_conv_mma_path(conv))
        check(L.pqn_set_conv_fusion(fuse))
        yield
    finally:
        check(L.pqn_set_tensor_core_path(2))
        check(L.pqn_set_conv_mma_path(1))
        check(L.pqn_set_conv_fusion(1))


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    n = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 0
    if not n:
        return
    print("\n%d SMs; tiles per CTA (min-max) of each case:" % n)
    cases = [("%d x %d" % s, s) for s in SHAPES] + [("rollout %d x %d" % (ROLLOUT[0], ROLLOUT[2]),
                                                     (ROLLOUT[0], ROLLOUT[2])), ("evaluation %d x %d" % EVAL, EVAL)]
    for name, (S, rows) in cases:
        tiles, grid, per = cta_tiles(S, rows)
        print("  %-22s %5d tiles, %3d CTAs, %d-%d tiles per CTA" % (name, tiles, grid, min(map(len, per)),
                                                                     max(map(len, per))))
    for k, v in sorted(VAR_EPS.items()):
        print("  small variance C=%d A=%d: LayerNorm_1 var / eps from %.3g to %.3g" % (*k, *v))
    if not REPORT:
        return
    worst = {}
    for path, C, A, regime, case, err, rsp in REPORT:
        k = (path, C, A, regime)
        a = worst.get(k, (0.0, 0.0, ""))
        worst[k] = (max(a[0], err), max(a[1], rsp), case if err >= a[0] else a[2])
    print("worst |q - q64| and its ratio to spread32 per (path, C, A, regime):")
    for k in sorted(worst):
        print("  %-8s C=%-2d A=%-2d %-10s %9.2e %7.2f  (%s)" % (*k, *worst[k]))


def cnn_spec(C, A):
    from purejaxql_b200.networks import NET_CNN, QNetworkSpec
    return QNetworkSpec(NET_CNN, C, A)


@functools.lru_cache(maxsize=None)
def pool_boards(C, j):
    """POOL boards of set j: row 0 empty, row 1 with its last channel full (game_obs), row 2 with every cell set."""
    obs = game_obs(C, POOL, 7000 + 10 * C + j)
    obs[2] = True
    return obs


@functools.lru_cache(maxsize=None)
def packed_pool(C, j):
    return pack_obs(pool_boards(C, j))


def init_params(C, A, seed):
    """The engine's own initial parameters (``spec.init`` on the device), read back as the oracle's dict."""
    from purejaxql_b200 import jaxrandom
    spec = cnn_spec(C, A)
    flat = spec.init(jaxrandom.split(jaxrandom.PRNGKey(seed, dev()), 1), dev())
    tree = spec.unflatten(flat)
    out = {}
    for pth, *_ in spec.entries:
        d = tree
        for k in pth:
            d = d[k]
        out["/".join(pth)] = d[0].cpu().numpy()
    return out


def dense0_preact(p, obs):
    """fp64 input of LayerNorm_1 (the 128 outputs of CNN_0/Dense_0) for the boards `obs`."""
    p64 = cast(p, F64)
    _, cache = R.cnn_forward(p64, obs.astype(F64), want_cache=True)
    return cache[3] @ p64["CNN_0/Dense_0/kernel"] + p64["CNN_0/Dense_0/bias"]


@functools.lru_cache(maxsize=None)
def param_set(C, A, regime, j):
    """Set j of a regime: (fp32 parameter dict, fp64 q of its pool boards [POOL, A], max |q32 - q64| over the pool)."""
    seed = 1000 * C + 10 * A + j + 100 * REGIMES.index(regime)
    obs = pool_boards(C, j)
    if regime == "init":
        p = init_params(C, A, seed)
    else:
        p = R.random_params(R.cnn_param_shapes(C, A), seed)
        if regime == "smallvar":
            z = dense0_preact(p, obs)
            f = SMALL_STD[j] / float(np.median(z.std(-1)))
            for k in ("CNN_0/Dense_0/kernel", "CNN_0/Dense_0/bias"):
                p[k] = (p[k].astype(F64) * f).astype(F32)
            r = dense0_preact(p, obs).var(-1) / R.LN_EPS
            lo, hi = VAR_EPS.get((C, A), (np.inf, 0.0))
            VAR_EPS[(C, A)] = (min(lo, float(r.min())), max(hi, float(r.max())))
        elif regime == "largemean":
            p["CNN_0/Dense_0/bias"] = (p["CNN_0/Dense_0/bias"] + F32(BIG_MEAN)).astype(F32)
    q64 = R.cnn_forward(cast(p, F64), obs.astype(F64))
    q32 = R.cnn_forward(cast(p, F32), obs.astype(F32))
    return p, q64, float(np.abs(q32.astype(F64) - q64).max())


def flat_params(spec, sets, S):
    flat = torch.cat([spec.flatten(p, 1, dev()) for p, _, _ in sets], 0)
    return flat[torch.arange(S, device=dev()) % len(sets)].contiguous()


def board_rows(rng, total):
    """Pool board of each observation row of one set; rows 0-2 hold the empty, one-channel and full boards."""
    return np.concatenate([[0, 1, 2], rng.integers(0, POOL, total - 3)])


def make_case(C, A, regime, S, rows, gathered, seed):
    """-> spec, flat [S, P], packed observations [S, total, PW], gather [S, rows] or None, total, fp64 q of the
    first NSETS seeds [NSETS, rows, A], spread32 of each set"""
    spec = cnn_spec(C, A)
    sets = [param_set(C, A, regime, j) for j in range(NSETS)]
    rng = np.random.default_rng(seed)
    total = rows + EXTRA
    boards = [board_rows(rng, total) for _ in range(NSETS)]
    pool = t_(np.stack([packed_pool(C, j) for j in range(NSETS)]), torch.int32)
    obs = torch.stack([pool[j][t_(boards[j], torch.int64)] for j in range(NSETS)])
    idx = torch.arange(S, device=dev()) % NSETS
    obs = obs[idx].contiguous()
    if gathered:
        gsets = [rng.permutation(np.concatenate([[0, 1, 2], rng.permutation(np.arange(3, total))[:rows - 3]]))
                 for _ in range(NSETS)]
        read = [g.astype(np.int64) for g in gsets]
        gather = t_(np.stack(gsets).astype(np.int32), torch.int32)[idx].contiguous()
    else:
        read = [np.arange(rows)] * NSETS
        gather = None
    want = np.stack([sets[j][1][boards[j][read[j]]] for j in range(NSETS)])
    return spec, flat_params(spec, sets, S), obs, gather, total, want, [s[2] for s in sets]


def run_forward(spec, flat, obs, gather, stride, S, rows, tag):
    """pqn_qnet_forward into a q with a NaN guard tail.  -> q [S, rows, A]"""
    L, p = _lib().lib(), _lib().p
    A = spec.num_actions
    n = S * rows * A
    q = torch.full((n + GUARD,), float("nan"), device=dev())
    ws = torch.empty(int(L.pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())
    _lib().check(L.pqn_qnet_forward(spec.desc, p(flat), None, _lib().raw(obs), p(gather), stride, p(q), S, rows,
                                    p(ws), _lib().stream_ptr()), "pqn_qnet_forward")
    torch.cuda.synchronize()
    del ws
    q = q.cpu().numpy()
    assert np.isnan(q[n:]).all(), (tag, "written past S * rows * A", int((~np.isnan(q[n:])).sum()))
    assert np.isfinite(q[:n]).all(), (tag, "NaN or inf left in q", int((~np.isfinite(q[:n])).sum()))
    return q[:n].reshape(S, rows, A)


def check_q(q, want, spread, regime, tag):
    """Replicas bit for bit, the first NSETS seeds against fp64 (module docstring).  -> failures"""
    S = q.shape[0]
    bad = []
    bits = q.view(np.uint32)
    rep = np.arange(NSETS, S)
    if len(rep):
        diff = (bits[rep] != bits[rep % NSETS]).any(axis=(1, 2))
        if diff.any():
            bad.append((tag, "replicas differ", rep[diff][:8].tolist()))
    for j in range(min(S, NSETS)):
        err = float(np.abs(q[j].astype(F64) - want[j]).max())
        REPORT.append((tag[0], *tag[1:4], tag[4], err, err / spread[j]))
        bar = max(BAR * float(np.abs(want[j]).max()), C_SPREAD * spread[j]) if regime == "largemean" else BAR
        if not err <= bar:
            bad.append((tag, "set %d" % j, err, bar))
    return bad


def bits_equal(a, b):
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


def run_paths(spec, flat, obs, gather, stride, S, rows, want, spread, regime, tag):
    """Every kernel path on one input: fp64 and replica checks, then fused == unfused.  -> failures"""
    got, bad = {}, []
    for name in PATHS:
        with kernel_path(name):
            got[name] = run_forward(spec, flat, obs, gather, stride, S, rows, (name,) + tag)
        bad += check_q(got[name], want, spread, regime, (name,) + tag)
    if not bits_equal(got["fused"], got["unfused"]):
        ndiff = int((got["fused"].view(np.uint32) != got["unfused"].view(np.uint32)).sum())
        bad.append((tag, "fused != unfused", ndiff))
    return bad


def test_geometry_runs_many_tiles_per_cta():
    """Every case of this module puts at least two tiles on every CTA, on whatever SM count this device has; the
    37 x 1,000 case moves every CTA to another seed and parameter set, 2 x 40,000 keeps some CTAs on one seed."""
    n = sms()
    for S, rows in SHAPES + [(ROLLOUT[0], ROLLOUT[2]), EVAL]:
        tiles, grid, per = cta_tiles(S, rows)
        assert min(map(len, per)) >= 2, (S, rows, n)
        assert rows % 128 or rows == ROLLOUT[2], (S, rows)   # a ragged last tile in every seed but the rollout's
    tps = (1000 + 127) // 128
    _, _, per = cta_tiles(37, 1000)
    steps = [(a, b) for ts in per for a, b in zip(ts, ts[1:])]
    assert steps and all(a // tps != b // tps and (a // tps) % NSETS != (b // tps) % NSETS for a, b in steps)
    tps = (40000 + 127) // 128
    assert tps > n
    _, _, per = cta_tiles(2, 40000)
    assert any(a // tps == b // tps for ts in per for a, b in zip(ts, ts[1:]))
    assert any(a // tps != b // tps for ts in per for a, b in zip(ts, ts[1:]))
    if n == 132:
        got = {s: (cta_tiles(*s)[0], min(map(len, cta_tiles(*s)[2])), max(map(len, cta_tiles(*s)[2])))
               for s in SHAPES + [(ROLLOUT[0], ROLLOUT[2]), EVAL]}
        assert got == {(37, 1000): (296, 2, 3), (2, 40000): (626, 4, 5), (17, 8193): (1105, 8, 9),
                       (128, 4096): (4096, 31, 32), (16, 2100): (272, 2, 3)}, got


@pytest.mark.parametrize("gathered", [True, False], ids=["gather", "nogather"])
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("C", [4, 6, 7, 10])
def test_multi_tile_forward_matches_fp64(C, regime, gathered):
    A = GAME_A[C]
    bad = []
    for S, rows in SHAPES:
        spec, flat, obs, gather, total, want, spread = make_case(C, A, regime, S, rows, gathered, S * rows + C)
        bad += run_paths(spec, flat, obs, gather, total, S, rows, want, spread, regime,
                         (C, A, regime, "%dx%d%s" % (S, rows, "g" if gathered else "")))
    assert not bad, bad


ACTION_SHAPES = [(4, a) for a in range(1, 10)] + [(10, 18)]


@pytest.mark.parametrize("regime", ["init", "random"])
@pytest.mark.parametrize("C,A", ACTION_SHAPES, ids=["C%dA%d" % s for s in ACTION_SHAPES])
def test_action_counts_match_fp64(C, A, regime):
    """A = 1 ... 8 through the tensor-core LayerNorm + Q-head epilogue, A = 9 and 18 through the mixed path."""
    S, rows = SHAPES[0]
    spec, flat, obs, gather, total, want, spread = make_case(C, A, regime, S, rows, True, 77 * A + C)
    bad = run_paths(spec, flat, obs, gather, total, S, rows, want, spread, regime,
                    (C, A, regime, "%dx%dg" % (S, rows)))
    assert not bad, bad


LAYOUT_REGIMES = ("init", "random", "smallvar")   # regime of set j in the rollout and evaluation cases ("layout")


def layout_sets(C, A):
    return [param_set(C, A, LAYOUT_REGIMES[j], j) for j in range(NSETS)]


@pytest.mark.parametrize("C", [4, 10])
def test_rollout_layout_matches_fp64(C):
    """``obs_buf[:, t]`` for t = 0 and T with the seed stride (T+1) E, no gather, as the rollout and the bootstrap
    read it: 128 seeds x 4,096 envs, 4,096 tiles."""
    S, T, E = ROLLOUT
    A = GAME_A[C]
    spec = cnn_spec(C, A)
    sets = layout_sets(C, A)
    rng = np.random.default_rng(C)
    boards = {t: [rng.integers(0, POOL, E) for _ in range(NSETS)] for t in (0, T)}
    for t in (0, T):
        for b in boards[t]:
            b[:3] = (0, 1, 2)
    pw = packed_pool(C, 0).shape[1]
    slab = torch.full((NSETS, T + 1, E, pw), -1, dtype=torch.int32, device=dev())   # all-ones words, padding included
    for j in range(NSETS):
        pool = t_(packed_pool(C, j), torch.int32)
        for t in (0, T):
            slab[j, t] = pool[t_(boards[t][j], torch.int64)]
    obs_buf = slab[torch.arange(S, device=dev()) % NSETS].contiguous()
    del slab
    flat = flat_params(spec, sets, S)
    bad = []
    for t in (0, T):
        want = np.stack([sets[j][1][boards[t][j]] for j in range(NSETS)])
        bad += run_paths(spec, flat, obs_buf[:, t], None, (T + 1) * E, S, E, want, [s[2] for s in sets], "layout",
                         (C, A, "layout", "rollout t=%d" % t))
    assert not bad, bad


@pytest.mark.parametrize("C", [4, 6, 7, 10])
def test_evaluation_layout_matches_fp64(C):
    """The greedy evaluation's ping-pong rows ``obs[:, cur]``, cur = 1, seed stride 2N, no gather."""
    S, N = EVAL
    A = GAME_A[C]
    spec = cnn_spec(C, A)
    sets = layout_sets(C, A)
    rng = np.random.default_rng(10 + C)
    boards = [board_rows(rng, N) for _ in range(NSETS)]
    pw = packed_pool(C, 0).shape[1]
    two = torch.full((NSETS, 2, N, pw), -1, dtype=torch.int32, device=dev())
    for j in range(NSETS):
        two[j, 1] = t_(packed_pool(C, j), torch.int32)[t_(boards[j], torch.int64)]
    obs = two[torch.arange(S, device=dev()) % NSETS].contiguous()
    want = np.stack([sets[j][1][boards[j]] for j in range(NSETS)])
    bad = run_paths(spec, flat_params(spec, sets, S), obs[:, 1], None, 2 * N, S, N, want, [s[2] for s in sets],
                    "layout", (C, A, "layout", "eval"))
    assert not bad, bad
