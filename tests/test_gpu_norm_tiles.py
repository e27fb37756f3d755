"""The NORM_TYPE / NORM_INPUT Q-networks other than the default (the "modular" fp32 path of ``csrc/pqn_norm.cuh``)
against fp64 at the training minibatches, at every MinAtar channel count and in the layouts the engine passes.

The modular path reduces across rows in two stages: RED_BLOCKS = 64 row chunks per seed (``colsum2_partial_kernel``,
``head_bwd_kernel``, ``obs_counts_kernel``, ``conv_dw_kernel``), then one block per seed adds the 64 partials in order.
``test_gpu_norm.py`` runs 256 rows (4 per chunk) at C = 4 and ``test_norm_variants_c7_match_fp64`` 1,024 at C = 7,
both with one value for the observation and the action / target row strides.  Here:

  - loss and gradients (``pqn_qnet_loss_grad``) of the CNN, cases S x rows, T, E:
      minatar5  16 x 1,024, 32, 1,024   C = 4 (5 actions), 6 (4), 7 (3), 10 (6), all five variants: 16 rows per chunk
      odd        9 x 4,097, 16, 257     C = 6, 10; (batch_norm, T), (none, F), (layer_norm, T): 63 chunks of 65 rows
                                        and one of 2; rows not a multiple of 4 (``conv_raw_kernel``) or 8 (the head)
      tiny       5 x 37, 4, 16          C = 6, 10; (batch_norm, T), (none, T): 27 of the 64 chunks empty
      big      128 x 4,096, 32, 4,096   C = 10, (batch_norm, T): the benchmark's minibatch; the observation buffer is
                                        2.2 GB, so its byte offsets pass 2^31
  - the eval forward (``pqn_qnet_forward`` with the running statistics) at the rollout's layout (step t's E rows at
    row t * E of a (T+1) E-row buffer) and at the evaluation's (ping-pong rows, stride 2 N, N = TEST_NUM_ENVS), every
    C and variant, with one channel of every running variance at 1e-4 (rstd ~ 100);
  - the MLP's loss and gradients at 8 x 4,097 rows with the rollout strides: H = 512 with A = 9 (the two-channels-
    per-thread branch of ``colsum2_partial_kernel``, a 512-thread ``head_bwd_kernel`` at the most actions
    ``check_desc`` allows at H = 512), H = 128 with A = HEAD_MAX_A = 32 (H = 256 allows at most 22), H = 64; inputs
    D = 6 (the G <= 16 branch: D = 4 divides 256 and takes the first), 50 (16 < G, not dividing 256) and 64;
  - two whole ``pqn_minatar`` updates at C = 6 and 10 against the oracle replay, and a Seaquest batch_norm run
    resumed after update 2 of 5.

Inputs follow ``engine.update_body``: ``obs_buf`` is [S][(T+1) E][row], action / target [S][T E]; the gather is one
chunk of a device permutation (``jaxrandom.permutation_indices``), each seed with its own key.  Every observation row
outside the minibatch is all-ones words (CNN) or NaN (MLP), every target there NaN, so a wrong stride reads another
board or a NaN.  ``grads``, ``loss_sum``, ``qsa_sum``, ``bn_sums`` and the running statistics carry NaN guard tails.
NSETS sets per run (4; 2 at 4,096 and 4,097 rows, where the fp64 oracle dominates the module's time): set j has
``R.random_params`` (even j; biases in front of a BatchNorm zeroed, as in ``test_gpu_norm.py``) or the engine's
``spec.init`` (odd j), TD errors of scale 1 (j = 0, 3) or 30 (j = 1, 2), and running statistics of mean
0.1 N(0, 1) and var 0.5 - 1.5.  Boards are the games' (at C = 10 half synthetic, half Seaquest's) with an empty board
and one with a full channel.  Seeds take the sets in a pseudo-random order; the path has no float atomics, so seeds
holding one set agree bit for bit, the running statistics included.

ReLU kink.  Where a ReLU input lies within fp32 rounding of zero the fp32 gradient is ill-defined (see
``test_gpu_cnn_grads_tiles.py``).  That module leaves such boards out; with batch statistics that does not work,
since leaving a board out moves every other board's ReLU inputs.  Instead, the per-channel additive parameter of each
ReLU's input (the norm's bias, or the layer's own bias with NORM_TYPE none) is moved by the smallest amount that puts
every ReLU input of the minibatch at least RELU_MARGIN = 2e-6 from zero (exact zeros stay), layer by layer, in fp64.

Checks, per run, on the first seed of each set against ``oracle/pqn_ref_norm.py`` in fp64: loss and mean chosen q
within 5e-5 of max(1, |value|); every gradient tensor within ``test_gpu_norm.py``'s bars of the largest gradient
(2e-5; batch_norm 2e-4, and 5e-2 on a bias in front of a BatchNorm, whose exact gradient is 0); ``bn_sums`` exact
(CNN: integer popcounts); the running statistics within 2e-6 after ``pqn_bn_stats_update``.  Every gradient's error
is also reported in units of spread32, the distance of the same oracle run in fp32 from fp64.  For the MLP those bars
do not hold at 4,097 rows: its inputs here have per-feature means of N(0, 1) and scales of e^-1.5 - e^1.5, the
kernels land up to 3.3e-3 of the scale from fp64 (D = 6, H = 512, batch_norm), and the fp32 oracle lands as far
(err / spread32 at most 1.4).  So an MLP gradient also passes within MLP_SPREAD_K = 8 x spread32.

Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): see DESIGN.md section 5.
"""
import functools

import numpy as np
import pytest
import torch

import seaquest_oracle as SQ
import test_gpu_norm as TN
import test_gpu_resume as RS
from oracle import jax_prng as jr
from oracle import pqn_ref as R
from oracle import pqn_ref_norm as RN
from test_gpu_seaquest import registered  # noqa: F401  (fixture: the oracle's registry knows Seaquest)
from test_oracle_cnn_grads import game_obs, pack_obs, td_targets

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32
NSETS = {"minatar5": 4, "odd": 2, "tiny": 4, "big": 2, "mlp": 2}
DELTAS = (1.0, 30.0, 30.0, 1.0)
GUARD = 1024
RELU_MARGIN = 2e-6
ALL = [("batch_norm", False), ("batch_norm", True), ("none", False), ("none", True), ("layer_norm", True)]
GAME_A = {4: 5, 6: 4, 7: 3, 10: 6}
CASES = {                 # S, rows, T, E
    "minatar5": (16, 1024, 32, 1024),
    "odd": (9, 4097, 16, 257),
    "tiny": (5, 37, 4, 16),
    "big": (128, 4096, 32, 4096),
}
CASE_RUNS = {             # C, variants
    "minatar5": [(C, ALL) for C in (4, 6, 7, 10)],
    "odd": [(C, [("batch_norm", True), ("none", False), ("layer_norm", True)]) for C in (6, 10)],
    "tiny": [(C, [("batch_norm", True), ("none", True)]) for C in (6, 10)],
    "big": [(10, [("batch_norm", True)])],
}
CNN_PARAMS = [(case, C, nt, ni) for case, runs in CASE_RUNS.items() for C, vs in runs for nt, ni in vs]
MLP_SHAPES = [(512, 2, 9), (128, 3, 32), (64, 1, 3)]      # H, L, A
MLP_D = [6, 50, 64]
MLP_CASE = (8, 4097, 16, 257)
MLP_SPREAD_K = 8.0        # the MLP's gradients may also lie within 8 x spread32 of fp64 (module docstring)
REPORT = []               # (net, case, C or D/H, variant, tensor, err / scale, err / spread32)


def dev():
    return torch.device("cuda:0")


def _lib():
    from purejaxql_b200 import _lib
    return _lib


def t_(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), dt)


def vid(nt, ni):
    return "%s-%s" % (nt, "T" if ni else "F")


# --------------------------------------------------------------------------------------------------------------------
# parameters, statistics and boards
# --------------------------------------------------------------------------------------------------------------------
def cnn_spec(C, A, nt, ni):
    from purejaxql_b200.networks import NET_CNN, QNetworkSpec
    return QNetworkSpec(NET_CNN, C, A, norm_type=nt, norm_input=ni)


def mlp_spec(D, A, H, L, nt, ni):
    from purejaxql_b200.networks import NET_MLP, QNetworkSpec
    return QNetworkSpec(NET_MLP, D, A, H, L, norm_type=nt, norm_input=ni)


def dead_biases(kind, nt, layers=2):
    """Biases that feed a BatchNorm directly: a no-op whose exact gradient is zero."""
    if nt != "batch_norm":
        return ()
    return TN.BN_DEAD_BIASES["cnn"] if kind == "cnn" else tuple("Dense_%d/bias" % l for l in range(layers))


def set_params(spec, kind, shapes, regime, seed, nt, layers=2):
    if regime == "init":
        from purejaxql_b200 import jaxrandom
        flat = spec.init(jaxrandom.split(jaxrandom.PRNGKey(seed, dev()), 1), dev())
        tree = spec.unflatten(flat)
        out = {}
        for pth, *_ in spec.entries:
            d = tree
            for k in pth:
                d = d[k]
            out["/".join(pth)] = d[0].cpu().numpy()
        return out
    p = R.random_params(shapes, seed)
    for k in dead_biases(kind, nt, layers):
        p[k] = np.zeros_like(p[k])
    return p


def cast_tree(p, dt):
    return {k: v.astype(dt) for k, v in p.items()}


def cast_stats(st, dt):
    return {k: {kk: vv.astype(dt) for kk, vv in v.items()} for k, v in st.items()}


@functools.lru_cache(maxsize=None)
def seaquest_boards(n, seed, steps=40):
    env = SQ.make(log=False)
    key, kr = jr.split(jr.PRNGKey(seed), 2)
    obs, st = env.reset(jr.split(kr, n))
    rng = np.random.default_rng(seed)
    for _ in range(steps):
        key, ks = jr.split(key, 2)
        obs, st, *_ = env.step(jr.split(ks, n), st, rng.integers(0, 6, n).astype(np.int32))
    return np.asarray(obs) != 0


@functools.lru_cache(maxsize=None)
def boards(C, n, seed):
    """n boards of the game of width C in a pseudo-random order, an empty board and a full channel among them; at
    C = 10 half of them Seaquest's.  -> bool[n, 10, 10, C]"""
    obs = game_obs(C, n, seed).copy()
    if C == 10 and n > 4:
        half = n // 2
        obs[2:2 + half] = seaquest_boards(half, seed)
    return obs[np.random.default_rng(seed).permutation(n)]


def relu_shift(v, m):
    """The smallest |delta| (0 or one of -v +- 1.2 m) such that every non-zero value of v + delta lies at least m
    from zero, with 0.1 m to spare for the fp32 rounding of the shifted parameter; exact zeros stay at delta = 0 and
    must clear m like the rest otherwise."""
    nz = v[v != 0]
    if not len(nz) or np.abs(nz).min() >= m:
        return 0.0
    kinks = np.sort(-(np.concatenate([nz, [0.0]]) if (v == 0).any() else nz))   # delta = -v puts v on the kink
    cand = np.concatenate([kinks - 1.2 * m, kinks + 1.2 * m])
    i = np.searchsorted(kinks, cand)
    near = np.minimum(np.abs(cand - kinks[np.maximum(i - 1, 0)]), np.abs(kinks[np.minimum(i, len(kinks) - 1)] - cand))
    ok = cand[near >= 1.1 * m]
    return float(ok[np.argmin(np.abs(ok))])


def clear_relu_kink(p, relu_inputs):
    """Moves the additive parameter in front of each ReLU (fp32, in place in p) until no ReLU input of the batch lies
    within RELU_MARGIN of zero.  relu_inputs(p) -> q, [(parameter name, ReLU input [..., channels] in fp64)] in layer
    order; a layer's values are read after the layers before it are cleared.  -> q (fp64) of the final parameters"""
    q, ys = relu_inputs(p)
    for layer in range(len(ys)):
        name, y = ys[layer]
        y = y.reshape(-1, y.shape[-1])
        delta = np.array([relu_shift(y[:, c], RELU_MARGIN) for c in range(y.shape[1])])
        if delta.any():
            p[name] = (p[name].astype(F64) + delta).astype(F32)
            q, ys = relu_inputs(p)
    for name, y in ys:
        a = np.abs(y)
        assert not ((a > 0) & (a < RELU_MARGIN)).any(), (name, float(a[a > 0].min()))
    return q


def rand_stats(stats0, seed, small_var=False):
    st = TN._rand_stats(stats0, seed)
    if small_var:                              # one channel per BatchNorm with rstd ~ 100
        for k, v in st.items():
            v["var"][seed % len(v["var"])] = 1e-4
    return st


# --------------------------------------------------------------------------------------------------------------------
# the rollout buffers and the call
# --------------------------------------------------------------------------------------------------------------------
def seed_sets(S, n):
    assign = np.random.default_rng(S + 7 * n).permutation(np.arange(S) % n)
    return assign, [int(np.flatnonzero(assign == j)[0]) for j in range(n)]


def rollout_buffers(rows_of, fill, A, S, rows, T, E, assign, key):
    """obs_buf [S][(T+1) E][W] (`fill` outside the minibatch), action / target [S][T E] (NaN targets outside) and the
    gather [S][rows]: one chunk of a device permutation of [0, T E) per seed (its own key), set assign[s]'s rows at
    the gathered positions in minibatch order.  rows_of: [set] -> (obs rows [rows, W], actions, targets)."""
    from purejaxql_b200 import jaxrandom
    n = T * E
    perm = jaxrandom.permutation_indices(jaxrandom.split(jaxrandom.PRNGKey(key, dev()), S), n)
    chunk = n // rows - 1
    gather = perm[:, chunk * rows:(chunk + 1) * rows].contiguous()
    del perm
    srt = torch.sort(gather, 1)[0]
    assert bool((srt[:, 1:] > srt[:, :-1]).all()) and int(srt.min()) >= 0 and int(srt.max()) < n
    del srt
    a = t_(assign, torch.int64)
    sel = (torch.arange(S, device=dev())[:, None], gather.long())
    o = torch.from_numpy(np.stack([r[0] for r in rows_of])).to(dev())
    obs_buf = torch.full((S, (T + 1) * E, o.shape[-1]), fill, dtype=o.dtype, device=dev())
    obs_buf[sel] = o[a]
    del o
    gen = torch.Generator(device=dev())
    gen.manual_seed(key)
    action = torch.randint(0, A, (S, n), generator=gen, device=dev(), dtype=torch.int32)
    action[sel] = t_(np.stack([r[1] for r in rows_of]), torch.int32)[a]
    target = torch.full((S, n), float("nan"), device=dev())
    target[sel] = t_(np.stack([r[2] for r in rows_of]), torch.float32)[a]
    return obs_buf, action, target, gather


def guarded(n, fill=0.0):
    out = torch.full((n + GUARD,), float("nan"), device=dev())
    out[:n] = fill
    return out


def loss_grad(spec, flat, stats, bufs, S, rows, T, E, bn_count):
    """pqn_qnet_loss_grad at the rollout strides into guarded outputs, then pqn_bn_stats_update.
    -> grads [S, P], loss [S], qsa [S], bn_sums [S, 2F], running statistics after the update [S, stats_total]"""
    L, p = _lib().lib(), _lib().p
    obs_buf, action, target, gather = bufs
    P, F, ST = flat.shape[1], spec.in_c, spec.stats_total
    grads, ls, qs, bn = guarded(S * P, float("nan")), guarded(S), guarded(S), guarded(S * 2 * F)
    st = guarded(S * ST)
    st[:S * ST] = stats.reshape(-1)
    ws = torch.empty(int(L.pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())
    _lib().check(L.pqn_qnet_loss_grad(spec.desc, p(flat), p(st), p(obs_buf), p(gather), (T + 1) * E, p(action),
                                      p(target), T * E, p(grads), p(ls), p(qs), p(bn), S, rows, p(ws),
                                      _lib().stream_ptr()), "pqn_qnet_loss_grad")
    bn_host = bn[:S * 2 * F].view(S, 2 * F).clone()            # pqn_bn_stats_update clears bn_sums
    _lib().check(L.pqn_bn_stats_update(p(st), p(bn), S, F, ST, float(bn_count), 0.99, _lib().stream_ptr()))
    torch.cuda.synchronize()
    del ws
    for name, t, n in (("grads", grads, S * P), ("loss_sum", ls, S), ("qsa_sum", qs, S), ("bn_sums", bn, S * 2 * F),
                       ("batch_stats", st, S * ST)):
        assert bool(torch.isnan(t[n:]).all()), (name, "written past its end")
    return grads[:S * P].view(S, P), ls[:S], qs[:S], bn_host, st[:S * ST].view(S, ST)


def replica_failures(out, assign, first):
    ref = t_(np.asarray(first)[assign], torch.int64)
    bad = []
    for name, t in zip(("grads", "loss_sum", "qsa_sum", "bn_sums", "batch_stats"), out):
        b = t.contiguous().view(torch.int32)
        d = (b != b[ref]) if b.dim() == 1 else (b != b[ref]).any(1)
        if bool(d.any()):
            bad.append(("replicas differ in " + name, torch.nonzero(d).flatten()[:8].tolist()))
    return bad


def leaves(spec, flat, s):
    tree = spec.unflatten(flat)
    out = {}
    for pth, *_ in spec.entries:
        d = tree
        for k in pth:
            d = d[k]
        out["/".join(pth)] = d[s].cpu().numpy().astype(F64)
    return out


def stats_leaves(spec, st, s):
    tree = spec.unflatten_stats(st)
    out = {}
    for pth, *_ in spec.stats_entries():
        d = tree
        for k in pth:
            d = d[k]
        out["/".join(pth)] = {k: v[s].cpu().numpy() for k, v in d.items()}
    return out


def check_set(spec, out, s, ref, ref32, dead, tag, spread_k=None):
    """The first seed s of a set against the fp64 oracle (module docstring); with spread_k, a gradient also passes
    within spread_k x spread32.  -> failures"""
    grads, ls, qs, bn, st = out
    loss, q_sa, g, new_stats, bn_want = ref
    g32 = ref32[2]
    bad = []
    if not abs(float(ls[s]) - loss) < 5e-5 * max(1.0, abs(loss)):
        bad.append(("loss", float(ls[s]), loss))
    if not abs(float(qs[s]) - q_sa.mean()) < 5e-5 * max(1.0, abs(q_sa.mean())):
        bad.append(("qmean", float(qs[s]), q_sa.mean()))
    got = leaves(spec, grads, s)
    scale = max(np.abs(v).max() for v in g.values())
    for name, want in g.items():
        err = float(np.abs(got[name] - want).max())
        spread = float(np.abs(g32[name].astype(F64) - want).max())
        tol = 2e-5
        if spec.norm_type == "batch_norm":
            tol = 5e-2 if name in dead else 2e-4
        REPORT.append(tag + (name, err / scale, err / spread if spread > 0 else (0.0 if err == 0 else np.inf)))
        if not (err < tol * scale or (spread_k is not None and err <= spread_k * spread)):
            bad.append((name, err / scale, tol, err / spread if spread > 0 else np.inf))
    if bn_want is not None and not np.array_equal(bn[s].cpu().numpy(), bn_want):
        bad.append(("bn_sums",))
    for name, v in stats_leaves(spec, st, s).items():
        w = new_stats[name]
        for k in ("mean", "var"):
            e = float(np.abs(v[k] - w[k]).max())
            if not e <= 2e-6:
                bad.append(("stats", name, k, e))
    return [(tag, b) for b in bad]


@pytest.fixture(scope="module", autouse=True)
def report():
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    if not REPORT:
        return
    worst = {}
    for net, case, w, v, name, rs, rsp in REPORT:
        k = (net, case, w, v)
        a = worst.get(k, (0.0, 0.0, "", ""))
        worst[k] = (max(a[0], rs), max(a[1], rsp), name if rs >= a[0] else a[2], name if rsp >= a[1] else a[3])
    print("\nworst gradient err / scale and err / spread32 per (net, case, width, variant):")
    for k in sorted(worst):
        print("  %-4s %-9s %-12s %-14s %9.2e %8.2f  (%s; %s)" % (*k, *worst[k]))
    print("peak device memory: %.2f GB" % (torch.cuda.max_memory_allocated() / 2 ** 30))


# --------------------------------------------------------------------------------------------------------------------
# CNN: loss and gradients at the training geometries
# --------------------------------------------------------------------------------------------------------------------
def cnn_relu_inputs(nt, ni, st64, obs64):
    n0 = {"layer_norm": "CNN_0/LayerNorm_0/bias", "batch_norm": "CNN_0/BatchNorm_0/bias"}.get(nt, "CNN_0/Conv_0/bias")
    n1 = {"layer_norm": "CNN_0/LayerNorm_1/bias", "batch_norm": "CNN_0/BatchNorm_1/bias"}.get(nt, "CNN_0/Dense_0/bias")

    def f(p):
        q, cache, _ = RN.cnn_forward(cast_tree(p, F64), st64, obs64, True, nt, ni, want_cache=True)
        return q, [(n0, cache[3]), (n1, cache[6])]
    return f


def cnn_set(C, A, nt, ni, rows, j):
    """Set j: parameters (kink-cleared), running statistics, boards, actions, targets and the oracle in fp64 / fp32."""
    spec = cnn_spec(C, A, nt, ni)
    seed = 7000 + 100 * C + 10 * j + rows
    rng = np.random.default_rng(seed)
    p = set_params(spec, "cnn", RN.cnn_param_shapes(C, A, nt), "random" if j % 2 == 0 else "init", seed, nt)
    st = rand_stats(RN.cnn_batch_stats(C, nt), seed)
    obs = boards(C, rows, 100 * C + j)
    obs64 = obs.astype(F64)
    st64 = cast_stats(st, F64)
    q64 = clear_relu_kink(p, cnn_relu_inputs(nt, ni, st64, obs64))
    act = rng.integers(0, A, rows).astype(np.int32)
    tgt = td_targets(q64[np.arange(rows), act], DELTAS[j], rng)
    ref = RN.cnn_loss_and_grads(cast_tree(p, F64), st64, obs64, act, tgt.astype(F64), nt, ni)
    ref32 = RN.cnn_loss_and_grads(p, st, obs.astype(F32), act, tgt, nt, ni)
    x = obs.reshape(-1, C).sum(0).astype(F32)
    return dict(p=p, st=st, obs=obs, act=act, tgt=tgt, ref=ref + (np.concatenate([x, x]),), ref32=ref32)


@pytest.mark.parametrize("case,C,nt,ni", CNN_PARAMS, ids=["%s-C%d-%s" % (c, C, vid(nt, ni)) for c, C, nt, ni in CNN_PARAMS])
def test_cnn_loss_grad_at_training_geometry(case, C, nt, ni):
    S, rows, T, E = CASES[case]
    A = GAME_A[C]
    spec = cnn_spec(C, A, nt, ni)
    sets = [cnn_set(C, A, nt, ni, rows, j) for j in range(NSETS[case])]
    assign, first = seed_sets(S, NSETS[case])
    a = t_(assign, torch.int64)
    flat = torch.cat([spec.flatten(s["p"], 1, dev()) for s in sets], 0)[a].contiguous()
    stats = torch.cat([spec.flatten_stats(s["st"], 1, dev()) for s in sets], 0)[a].contiguous()
    bufs = rollout_buffers([(pack_obs(s["obs"]), s["act"], s["tgt"]) for s in sets], -1, A, S, rows, T, E, assign,
                           100 * C + A)
    out = loss_grad(spec, flat, stats, bufs, S, rows, T, E, rows * 100)
    del bufs
    bad = replica_failures(out, assign, first)
    for j, s in enumerate(sets):
        bad += check_set(spec, out, first[j], s["ref"], s["ref32"], dead_biases("cnn", nt),
                         ("cnn", case, "C=%d" % C, vid(nt, ni)))
    assert not bad, bad[:20]


# --------------------------------------------------------------------------------------------------------------------
# CNN: eval forward at the rollout's and the evaluation's layouts
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nt,ni", ALL, ids=[vid(*v) for v in ALL])
@pytest.mark.parametrize("C", [4, 6, 7, 10])
def test_cnn_eval_forward_at_rollout_and_evaluation_layouts(C, nt, ni):
    """q with the running statistics (one variance per BatchNorm at 1e-4) within 1e-5 of max(1, |q|) of fp64; the
    forward leaves the running statistics as they were."""
    L, p = _lib().lib(), _lib().p
    A = GAME_A[C]
    spec = cnn_spec(C, A, nt, ni)
    S, T, E, t, N = 3, 4, 300, 2, 128
    ps = [set_params(spec, "cnn", RN.cnn_param_shapes(C, A, nt), "init" if s == 1 else "random", 500 + s, nt)
          for s in range(S)]
    sts = [rand_stats(RN.cnn_batch_stats(C, nt), 60 + s, small_var=True) for s in range(S)]
    flat = torch.cat([spec.flatten(q, 1, dev()) for q in ps], 0).contiguous()
    stf = torch.cat([spec.flatten_stats(st, 1, dev()) for st in sts], 0).contiguous()
    st0 = stf.clone()
    for rows, layout in ((E, "rollout"), (N, "evaluation")):
        obs = [boards(C, rows, 900 + 10 * C + s) for s in range(S)]
        packed = torch.from_numpy(np.stack([pack_obs(o) for o in obs])).to(dev())
        if layout == "rollout":
            buf = torch.full((S, T + 1, E, packed.shape[-1]), -1, dtype=torch.int32, device=dev())
            buf[:, t] = packed
            view, orps = buf[:, t], (T + 1) * E
        else:
            buf = torch.full((S, 2, N, packed.shape[-1]), -1, dtype=torch.int32, device=dev())
            buf[:, 1] = packed
            view, orps = buf[:, 1], 2 * N
        q = torch.full((S * rows + GUARD, A), float("nan"), device=dev())
        ws = torch.empty(int(L.pqn_net_workspace_bytes(spec.desc, S, rows)), dtype=torch.uint8, device=dev())
        _lib().check(L.pqn_qnet_forward(spec.desc, p(flat), p(stf), _lib().raw(view), None, orps, p(q), S, rows, p(ws),
                                        _lib().stream_ptr()), "pqn_qnet_forward")
        torch.cuda.synchronize()
        assert bool(torch.isnan(q[S * rows:]).all())
        assert torch.equal(stf.view(torch.int32), st0.view(torch.int32)), "the eval forward changed the statistics"
        got = q[:S * rows].cpu().numpy().reshape(S, rows, A)
        for s in range(S):
            ref, _ = RN.cnn_forward(cast_tree(ps[s], F64), cast_stats(sts[s], F64), obs[s].astype(F64), False, nt, ni)
            err = np.abs(got[s] - ref).max()
            assert err < 1e-5 * max(1.0, np.abs(ref).max()), (layout, s, err, np.abs(ref).max())


# --------------------------------------------------------------------------------------------------------------------
# MLP: the reductions at 65 rows per chunk
# --------------------------------------------------------------------------------------------------------------------
MLP_PARAMS = [(H, L, A, D, nt, ni) for H, L, A in MLP_SHAPES for D in MLP_D
              for nt, ni in (("batch_norm", True), ("none", True))]


def mlp_set(D, A, H, L, nt, ni, rows, j):
    spec = mlp_spec(D, A, H, L, nt, ni)
    seed = 8000 + 1000 * L + H + 7 * D + j
    rng = np.random.default_rng(seed)
    p = set_params(spec, "mlp", RN.mlp_param_shapes(D, A, H, L, nt), "random" if j % 2 == 0 else "init", seed, nt, L)
    st = rand_stats(RN.mlp_batch_stats(D, H, L, nt), seed)
    f_rng = np.random.default_rng(D)                      # per-feature offsets and scales shared by the sets
    obs = (f_rng.standard_normal(D) + rng.standard_normal((rows, D)) * np.exp(f_rng.uniform(-1.5, 1.5, D))).astype(F32)
    obs64 = obs.astype(F64)
    st64 = cast_stats(st, F64)
    names = [("BatchNorm_%d/bias" if nt == "batch_norm" else "Dense_%d/bias") % (l + (nt == "batch_norm"))
             for l in range(L)]

    def relu_inputs(p_):
        q, (_, caches, _), _ = RN.mlp_forward(cast_tree(p_, F64), st64, obs64, True, nt, ni, want_cache=True)
        return q, [(n, c[2]) for n, c in zip(names, caches)]
    q64 = clear_relu_kink(p, relu_inputs)
    act = rng.integers(0, A, rows).astype(np.int32)
    tgt = td_targets(q64[np.arange(rows), act], DELTAS[j], rng)
    ref = RN.mlp_loss_and_grads(cast_tree(p, F64), st64, obs64, act, tgt.astype(F64), nt, ni)
    ref32 = RN.mlp_loss_and_grads(p, st, obs, act, tgt, nt, ni)
    return dict(p=p, st=st, obs=obs, act=act, tgt=tgt, ref=ref + (None,), ref32=ref32)


@pytest.mark.parametrize("H,L,A,D,nt,ni", MLP_PARAMS,
                         ids=["H%dL%dA%d-D%d-%s" % (H, L, A, D, vid(nt, ni)) for H, L, A, D, nt, ni in MLP_PARAMS])
def test_mlp_loss_grad_at_many_rows_per_chunk(H, L, A, D, nt, ni):
    S, rows, T, E = MLP_CASE
    spec = mlp_spec(D, A, H, L, nt, ni)
    sets = [mlp_set(D, A, H, L, nt, ni, rows, j) for j in range(NSETS["mlp"])]
    assign, first = seed_sets(S, NSETS["mlp"])
    a = t_(assign, torch.int64)
    flat = torch.cat([spec.flatten(s["p"], 1, dev()) for s in sets], 0)[a].contiguous()
    stats = torch.cat([spec.flatten_stats(s["st"], 1, dev()) for s in sets], 0)[a].contiguous()
    bufs = rollout_buffers([(s["obs"], s["act"], s["tgt"]) for s in sets], float("nan"), A, S, rows, T, E, assign,
                           H + 10 * D + A)
    out = loss_grad(spec, flat, stats, bufs, S, rows, T, E, rows)
    bad = replica_failures(out, assign, first)
    for j, s in enumerate(sets):
        bad += check_set(spec, out, first[j], s["ref"], s["ref32"], dead_biases("mlp", nt, L),
                         ("mlp", "8x4097", "D=%d H=%d" % (D, H), vid(nt, ni)), MLP_SPREAD_K)
    assert not bad, bad[:20]


# --------------------------------------------------------------------------------------------------------------------
# whole updates and a resumed run
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nt,ni", [("batch_norm", True), ("none", False)], ids=["batch_norm-T", "none-F"])
@pytest.mark.parametrize("env_name", ["SpaceInvaders-MinAtar", "Seaquest-MinAtar"])
def test_minatar_updates_match_oracle(env_name, nt, ni, registered, monkeypatch):  # noqa: F811
    """two pqn_minatar updates at C = 6 and 10 against the oracle replay (test_gpu_norm.py's test and tolerances)"""
    TN.test_norm_variant_update_step_matches_oracle(env_name, "cnn", "pqn_minatar", False, nt, ni, monkeypatch)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_seaquest_batch_norm_resume_is_bit_identical(graph, tmp_path):
    """a pqn_minatar run on Seaquest with (batch_norm, NORM_INPUT): its CNN batch_stats block is saved and resumed"""
    cfg = RS._cfg("Seaquest-MinAtar", NUM_ENVS=128, NORM_TYPE="batch_norm", NORM_INPUT=True, CUDA_GRAPH=graph)
    rngs = jr.split(jr.PRNGKey(7), cfg["NUM_SEEDS"])
    a, b, eng_a, eng_b = RS._a_then_b("pqn_minatar", cfg, rngs, str(tmp_path))
    RS._assert_same_bits(a, b, "seaquest batch_norm")
    assert a["batch_stats"].shape == (2, 2 * 10 + 2 * 16 + 2 * 128)
    assert eng_a.graph_captured == graph and eng_b.graph_captured == graph
