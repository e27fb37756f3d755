"""The PQN training program: ``make_train(config) -> train(rngs)``.

Host-side restatement of ``make_train`` in purejaxql/pqn_minatar.py:89-431 and
purejaxql/pqn_gymnax.py:78-424 (identical modulo the network and the flatten
wrapper), with the seed axis taken natively — the reference wraps ``train`` in
``jax.jit(jax.vmap(...))`` over ``rngs[S,2]`` (pqn_minatar.py:459-461); here
``train(rngs)`` receives the whole ``[S,2]`` key array and every kernel launch
covers all S seeds.

All compute is libpqn_b200 kernels (include/pqn_b200.h).  This module only
allocates buffers (torch), walks the reference's PRNG key chain (SURVEY
Appendix B) and sequences the launches:

  per update (``_update_step``, :176-369):
    rollout   T x [ Q-network forward ; fused eps-greedy + env step + stores ]
    bootstrap forward on the last obs ; Q(lambda) reverse scan
    epochs x minibatches x [ permutation gather ; loss/grad ; clip+RAdam ; BN stats ]
"""
from __future__ import annotations

import dataclasses
import os
from types import SimpleNamespace

import numpy as np
import torch

from . import _lib, envs, jaxrandom as jr, pbt, state as runstate, sweep
from .networks import NET_CNN, NET_MLP, NET_MLP_BITS, NET_RNN, QNetworkSpec

CNN_NEEDS_MINATAR = "the MinAtar CNN needs a (10,10,C) binary-observation env"
INFO_KEYS = ("returned_episode_returns", "returned_episode_lengths", "timestep", "returned_episode", "discount")


def _f32(x):
    return np.float32(x)


def linear_schedule(init, end, transition_steps, count):
    """optax.linear_schedule evaluated in float32 (pqn_minatar.py:134-146)."""
    if transition_steps <= 0:
        return _f32(init)
    c = np.clip(_f32(count), _f32(0), _f32(transition_steps))
    frac = _f32(1) - c / _f32(transition_steps)
    return _f32(_f32(init - end) * frac + _f32(end))


def radam_schedule_table(num_steps, lr_fn, b1=0.9, b2=0.999, threshold=5.0):
    """[num_steps,4] float32 rows (lr_t, 1-b1^t, 1-b2^t, rect_t or 0) of
    optax.scale_by_radam + scale_by_learning_rate for optimizer steps t=1..

    Evaluated in float32 in optax's operation order (the traced program computes ``b2t = b2**count_inc``,
    ``ro = ro_inf - 2*count_inc*b2t/(1-b2t)`` and the rectification term on weak-typed float32 scalars): the
    cancellation in ``ro`` is visible in float32 for the first few hundred steps, so a float64 table would not
    match the reference optimizer to 1e-5 there.  (XLA's f32 pow may still differ from numpy's by an ulp, which
    the cancellation amplifies; this cannot be pinned without an optax install -- DESIGN.md section 5.)"""
    f = np.float32
    tab = np.zeros((max(num_steps, 1), 4), np.float32)
    ro_inf = f(2.0) / (f(1.0) - f(b2)) - f(1.0)
    for i in range(num_steps):
        t = f(i + 1)
        b2t = np.power(f(b2), t, dtype=np.float32)
        b1t = np.power(f(b1), t, dtype=np.float32)
        ro = ro_inf - f(2.0) * t * b2t / (f(1.0) - b2t)
        rect = f(0.0)
        if ro >= f(threshold):
            rect = np.sqrt((ro - f(4)) * (ro - f(2)) * ro_inf / ((ro_inf - f(4)) * (ro_inf - f(2)) * ro), dtype=np.float32)
        tab[i] = (lr_fn(i), f(1.0) - b1t, f(1.0) - b2t, rect)
    return tab


def seed_inputs(grid: "sweep.Grid", seed_lo: int, S: int, num_updates: int, updates_decay: int,
                grad_steps_per_update: int, lr_linear_decay: bool) -> dict:
    """The per-seed hyperparameter tables the device reads, for the S seeds [seed_lo, seed_lo + S) of a run (numpy
    float32; a seed takes the values of its grid point, sweep.Grid):

      eps        [max(NU,1)][S]  eps_scheduler(n_updates) (pqn_minatar.py:134-139)
      sched      RAdam rows (lr_t, 1-b1^t, 1-b2^t, rect_t): [steps][4] shared by every seed when the grid has one point,
                 else [S][steps][4], each seed its point's table (:140-147)
      gamma, lam, max_norm, rew_scale  [S]
    """
    pt = grid.point_of(seed_lo, S)
    nud, total_grad_steps = updates_decay, num_updates * grad_steps_per_update
    eps_pts, sched_pts = [], []
    for g in range(grid.G):
        c = grid.config(g)
        eps_pts.append([linear_schedule(c["EPS_START"], c["EPS_FINISH"], c["EPS_DECAY"] * nud, n)
                        for n in range(max(num_updates, 1))])
        if lr_linear_decay:
            lr_fn = lambda i, lr=c["LR"]: linear_schedule(lr, 1e-20, nud * grad_steps_per_update, i)
        else:
            lr_fn = lambda i, lr=c["LR"]: _f32(lr)
        sched_pts.append(radam_schedule_table(total_grad_steps, lr_fn))
    eps = np.ascontiguousarray(np.asarray(eps_pts, np.float32).T[:, pt])
    sched = sched_pts[0] if grid.G == 1 else np.stack([sched_pts[g] for g in pt])

    def per_seed(key):
        return np.array([grid.value(int(g), key) for g in pt], np.float32)
    return dict(eps=eps, sched=sched, gamma=per_seed("GAMMA"), lam=per_seed("LAMBDA"),
                max_norm=per_seed("MAX_GRAD_NORM"), rew_scale=per_seed("REW_SCALE"))


def seed_tensors(inputs: dict, dev):
    """seed_inputs on the device, and the RAdam schedule's per-seed stride in floats (0: one shared table)."""
    t = {k: torch.from_numpy(v).to(dev) for k, v in inputs.items()}
    sched = t["sched"]
    return t, (0 if sched.dim() == 2 else sched.shape[1] * 4)


class TrainState(SimpleNamespace):
    """Mirror of CustomTrainState (pqn_minatar.py:82-86): params / batch_stats
    nested dicts with a leading seed axis, plus timesteps, n_updates, grad_steps
    and the optimizer moments."""


def network_spec(env, network: str, c: dict):
    """(QNetworkSpec, int32/float32 words per stored obs row, their torch dtype) of the engine's Q-network on `env`
    (host-side: allocates nothing).  "cnn": the MinAtar CNN on packed rows; "mlp": the MLP QNetwork, on float rows for
    classic control / bsuite and on the packed rows of a MinAtar env behind FlattenObservationWrapper
    (PQN_NET_MLP_BITS)."""
    norm_type, norm_input = c.get("NORM_TYPE", "layer_norm"), bool(c.get("NORM_INPUT", False))
    if network == "cnn":
        if not env.binary_obs:
            raise ValueError(CNN_NEEDS_MINATAR)
        spec = QNetworkSpec(NET_CNN, env.info.obs_shape[2], env.num_actions, norm_type=norm_type, norm_input=norm_input)
        return spec, env.packed_obs_words, torch.int32
    kind = NET_MLP_BITS if env.binary_obs else NET_MLP
    spec = QNetworkSpec(kind, env.obs_dim, env.num_actions, int(c.get("HIDDEN_SIZE", 128)), int(c.get("NUM_LAYERS", 2)),
                        norm_type=norm_type, norm_input=norm_input)
    if env.binary_obs:
        return spec, env.packed_obs_words, torch.int32
    return spec, env.obs_dim, torch.float32


class EngineBase:
    """What the feed-forward and the recurrent engine share: the config, the per-seed hyperparameter tables, the
    optimiser and update-step buffers, the fused act step, the update loop (eager, then a captured CUDA graph), the
    metrics, the evaluation means and the assembly of train()'s result.  A subclass owns its network, its key chain
    and its ``update_body``."""

    def __init__(self, config: dict, flatten_obs: bool, device=None, env_params: envs.EnvParams | None = None):
        self.cfg = c = config
        self.grid = sweep.Grid(config)       # per-seed hyperparameters: a grid of G points x NUM_SEEDS
        self.pbt = pbt.settings(config)      # population-based training (None: off); train() builds the population
        self.population = None
        self.seed_lo = 0            # global index of this run's first seed (a seed-sharded rank trains a slice)
        self.env_shard = None       # (rank, world): train envs [rank*E/world, (rank+1)*E/world) of every seed
        self.device = torch.device(device or "cuda")
        if self.device.type != "cuda" or not torch.cuda.is_available():
            raise _lib.PqnError("purejaxql_b200 needs a CUDA device: there is no CPU fallback")
        self.rng_mode = int(c.get("JAX_THREEFRY_PARTITIONABLE", 0))
        self.env, self.env_params = envs.make(c["ENV_NAME"], flatten_obs=flatten_obs, rng_mode=self.rng_mode)
        if env_params is not None:                                   # e.g. MemoryChain's memory_length
            self.env_params = env_params
        self.max_steps = int(self.env_params.max_steps_in_episode)
        self.T, self.E, self.NU = int(c["NUM_STEPS"]), int(c["NUM_ENVS"]), int(c["NUM_UPDATES"])
        self.A = self.env.num_actions
        self.nmb, self.epochs = int(c["NUM_MINIBATCHES"]), int(c["NUM_EPOCHS"])
        self.test = bool(c.get("TEST_DURING_TRAINING", False))
        self.batch_stats = None     # [S][stats_total] running statistics; train() sets them
        # hooks (bench / tests), called on the host outside the captured region so they do not prevent graph replay:
        # on_update_begin(n) before update n, on_update_end(n, payload) with the engine's static buffers after it
        self.on_update_begin = None
        self.on_update_end = None
        self.log_prefix = ""        # prepended to every wandb key (an env list logs each env under "<env>/")
        self.graph_captured = False
        self.graph_replays = 0
        self.graph_launches_per_replay = 0
        self._ws = None
        # training state (purejaxql_b200.state): written after every state_every-th update (0: never); `resume`, which
        # make_train loads from RESUME_FROM, is copied into the static buffers before the first update this run runs
        self.state_every = runstate.save_interval(c)
        self.resume = None

    def _workspace(self, S, rows):
        need = int(_lib.lib().pqn_net_workspace_bytes(self.spec.desc, S, rows))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

    def _seed_tables(self, S):
        """seed_tensors of this run's S seeds: ({eps, sched, gamma, lam, max_norm, rew_scale}, sched stride)."""
        c = self.cfg
        return seed_tensors(seed_inputs(self.grid, self.seed_lo, S, self.NU, c["NUM_UPDATES_DECAY"],
                                        self.nmb * self.epochs, c.get("LR_LINEAR_DECAY", False)), self.device)

    def _population(self, hp, sched_stride, S):
        """The run's pbt.Population over its S seeds (None without PBT).  The event edits hp's tables in place."""
        self.population = None
        if self.pbt is None:
            return None
        dp, _, world = self._placement()
        if dp == "seeds" and world > 1:
            raise ValueError(f"PBT_INTERVAL={self.pbt.interval}: a seed-sharded run of {world} processes would split "
                             f"the population over the processes; run PBT in one process or with DATA_PARALLEL=envs")
        self.population = pbt.Population(self.pbt, S, self.NU, hp, sched_stride, self.rng_mode, self.device)
        return self.population

    def _radam_step(self, params, u, hp, sched_stride, S, P):
        """clip + RAdam of every seed (pqn_minatar.py:292): pqn_radam_clip_step_seeds, or with PBT
        pqn_radam_clip_step_pbt, which reads each seed's schedule source and LR multiplier."""
        L, pop, sp = _lib.lib(), self.population, _lib.stream_ptr
        if pop is None:
            _lib.check(L.pqn_radam_clip_step_seeds(_lib.p(params), _lib.p(u.grads), _lib.p(u.mu), _lib.p(u.nu),
                                                   _lib.p(hp["sched"]), sched_stride, _lib.p(u.step_counter),
                                                   _lib.p(u.gnorm), S, P, _lib.p(hp["max_norm"]), 0.9, 0.999, 1e-8,
                                                   sp()), "pqn_radam_clip_step_seeds")
        else:
            _lib.check(L.pqn_radam_clip_step_pbt(_lib.p(params), _lib.p(u.grads), _lib.p(u.mu), _lib.p(u.nu),
                                                 _lib.p(hp["sched"]), sched_stride, _lib.p(pop.sched_src),
                                                 _lib.p(pop.lr_mult), _lib.p(u.step_counter), _lib.p(u.gnorm), S, P,
                                                 _lib.p(hp["max_norm"]), 0.9, 0.999, 1e-8, sp()),
                       "pqn_radam_clip_step_pbt")

    def _update_buffers(self, params, rng):
        """The optimiser state and the static buffers every update reads and writes (so that it can be replayed
        from a CUDA graph): the runner key, the evaluation key and the update index on the device, and the sums
        the metrics are taken from."""
        S, dev = rng.shape[0], self.device
        return SimpleNamespace(
            mu=torch.zeros_like(params), nu=torch.zeros_like(params), grads=torch.zeros_like(params),
            step_counter=torch.zeros(1, dtype=torch.int32, device=dev),
            gnorm=torch.zeros(S * 64, device=dev),                   # block partials of the squared gradient norm
            rng=rng.clone(),                                          # runner rng, updated in place
            kT=torch.zeros((S, 2), dtype=torch.int32, device=dev),    # eval key of this update
            idx=torch.zeros(1, dtype=torch.int64, device=dev),        # n_updates on the device
            m=torch.zeros((S, 7), dtype=torch.float64, device=dev),   # td_loss, qvals, 5 info means
            loss_sum=torch.zeros(S, device=dev), qsa_sum=torch.zeros(S, device=dev))

    def _end_update(self, u, r, info_sums):
        """The end of every update body: the evaluation key (rng, _rng = split(rng)), the runner key and the
        update's means."""
        if self.test:
            k = jr.split(r, 2, self.rng_mode)
            r = k[:, 0].contiguous()
            u.kT.copy_(k[:, 1])
        u.rng.copy_(r)
        denom = float(self.epochs * self.nmb)
        u.m[:, 0] = u.loss_sum.double() / denom
        u.m[:, 1] = u.qsa_sum.double() / denom
        u.m[:, 2:7] = info_sums / float(self.T * self.E)
        u.idx.add_(1)

    def _act_step(self, S, N, step_keys, q, eps, state, obs_next, action, reward, done, maxq, sums, done_only,
                  rew_scale, obs_stride, tr_stride, env_total, env_offset):
        """Fused eps-greedy + env step + stores (pqn_rollout_act_step_seeds) for S seeds x N envs.  eps and
        rew_scale are float32[S] device values of each seed; obs_next and the transition buffers may be strided
        views (obs_stride / tr_stride rows per seed); the N envs are [env_offset, env_offset + N) of env_total."""
        _lib.check(_lib.lib().pqn_rollout_act_step_seeds(
            self.env.env_id, _lib.p(step_keys), _lib.p(q), _lib.p(eps), _lib.p(state), _lib.raw(obs_next), obs_stride,
            _lib.raw(action), _lib.raw(reward), _lib.raw(done), _lib.raw(maxq), tr_stride, _lib.p(sums), done_only,
            S, N, env_total, env_offset, self.max_steps, _lib.p(rew_scale), self.rng_mode, _lib.stream_ptr()),
            "pqn_rollout_act_step_seeds")

    @staticmethod
    def _episode_means(sums):
        """INFO_KEYS means over the episodes that ended (sums[:, 3] of them); NaN where none did."""
        cnt = sums[:, 3]
        return {kk: torch.where(cnt > 0, sums[:, j] / cnt.clamp(min=1), torch.full_like(cnt, float("nan")))
                for j, kk in enumerate(INFO_KEYS)}

    def train(self, rngs):
        """The whole run: ``train_steps(rngs)`` driven to its end."""
        steps = self.train_steps(rngs)
        while True:
            try:
                next(steps)
            except StopIteration as done:
                return done.value

    def _run_updates(self, keys, params, u, update_body, payload, graph_auto, test_metrics, frame_channels=None,
                     live=None):
        """NUM_UPDATES x update_body, with the metrics (pqn_minatar.py:329-338), the evaluation (:340-350) and the
        wandb log (:353-365) of every update.  A generator: it yields the update's index after each update, so that a
        driver (env_list.py) can interleave the updates of several engines, and returns its result at the end.  The
        first update this process runs is eager (it warms every code path); when CUDA_GRAPH is true, or "auto" and
        graph_auto holds, later updates replay a graph captured after it.
        `live` names the engine's buffers that carry a run from one update to the next besides ``u``'s: they are what
        the training state holds.  On resume the state is copied into them and into the metric columns first, and
        the loop starts at the column after the saved update.  Returns (metrics, test_hist, test_metrics): [S, NU]
        float64 columns and the last evaluation."""
        c, dev, L, NU = self.cfg, self.device, _lib.lib(), self.NU
        S = keys.shape[0]
        # pqn_minatar.py:330-338 reports env_frame; pqn_gymnax.py:324-331 and pqn_rnn_gymnax.py:401-408 do not
        metric_names = ["env_step", "update_steps", *(["env_frame"] if frame_channels else []), "grad_steps",
                        "td_loss", "qvals", *INFO_KEYS]
        metrics = {m: torch.zeros((S, max(NU, 1)), dtype=torch.float64, device=dev) for m in metric_names}
        test_hist = None
        if self.test:
            test_every = int(NU * c["TEST_INTERVAL"])
            test_hist = {kk: torch.zeros((S, max(NU, 1)), dtype=torch.float64, device=dev) for kk in INFO_KEYS}
        live = {**(live or {}), "mu": u.mu, "nu": u.nu, "step_counter": u.step_counter, "rng": u.rng, "idx": u.idx}
        pop = self.population
        if pop is not None:
            live.update(pop.live())
        n0 = 0
        if self.resume is not None:
            n0, test_metrics = self._restore_state(live, metrics, test_hist)
        want_graph = c.get("CUDA_GRAPH", "auto")
        use_graph = (graph_auto if want_graph == "auto" else bool(want_graph)) and NU - n0 > 2
        graph = None
        self.graph_captured = False
        self.graph_replays = 0
        self.graph_launches_per_replay = 0
        for col in range(n0, NU):
            if self.on_update_begin is not None:
                self.on_update_begin(col)
            if graph is not None:
                graph.replay()
                self.graph_replays += 1
            else:
                update_body()
                if use_graph and col == n0:
                    try:
                        torch.cuda.synchronize(dev)
                        g = torch.cuda.CUDAGraph()
                        l0 = L.pqn_launch_count()
                        with torch.cuda.graph(g):
                            update_body()
                        self.graph_launches_per_replay = int(L.pqn_launch_count() - l0)
                        graph = g
                        self.graph_captured = True
                    except Exception as e:                            # capture is an optimisation only
                        import warnings
                        warnings.warn(f"CUDA graph capture of the update step failed ({e!r}); running eagerly")
                        graph = None
                        use_graph = False
                        torch.cuda.synchronize(dev)
            n_done = col + 1
            timesteps = n_done * self.T * self.E                      # :222-225
            metrics["env_step"][:, col] = timesteps
            metrics["update_steps"][:, col] = n_done
            if frame_channels:
                metrics["env_frame"][:, col] = timesteps * frame_channels
            metrics["grad_steps"][:, col] = n_done * self.nmb * self.epochs
            metrics["td_loss"][:, col] = u.m[:, 0]
            metrics["qvals"][:, col] = u.m[:, 1]
            for j, kk in enumerate(INFO_KEYS):
                metrics[kk][:, col] = u.m[:, 2 + j]
            if self.on_update_end is not None:
                self.on_update_end(col, payload)
            if self.test:
                if test_every > 0 and n_done % test_every == 0:
                    test_metrics = self.get_test_metrics(params, u.kT.clone())
                for kk in INFO_KEYS:
                    test_hist[kk][:, col] = test_metrics[kk]
            if c.get("WANDB_MODE", "disabled") != "disabled":
                self._wandb_log(metrics, test_hist, col, jr.to_numpy_u32(keys)[:, 0])
            if pop is not None and pop.due(n_done, NU):         # eager, on the static buffers the graph replays
                if pop.st.fitness == "test":
                    fit, c0, cols = test_metrics[pbt.FITNESS_METRIC].contiguous(), 0, 1
                else:
                    fit, c0, cols = metrics[pbt.FITNESS_METRIC], n_done - pop.st.interval, pop.st.interval
                pop.event(n_done, fit, c0, cols, params, u.mu, u.nu, self.batch_stats)
            if self.state_every and n_done % self.state_every == 0:
                self._save_state(keys, live, metrics, test_hist, test_metrics, n_done)
            yield col
        torch.cuda.synchronize(dev)
        return metrics, test_hist, test_metrics

    # ---- training state (purejaxql_b200.state) ------------------------------------------------------------------ #
    def _placement(self):
        """(data-parallel mode, rank, world) of this engine's run."""
        shard = self.env_shard
        if shard is not None and shard[1] > 1:
            return "envs", int(shard[0]), int(shard[1])
        return ("seeds", *runstate.dist_placement())

    def _resume_begin(self, keys):
        """Whether this train() resumes from ``self.resume``; refuses keys, a seed slice or a data-parallel mode other
        than the saved run's before anything is allocated."""
        rs = self.resume
        if rs is None:
            return False
        runstate.check_placement(rs["meta"], self._placement()[0], self.seed_lo, keys.shape[0], rs["path"])
        if not torch.equal(keys.cpu(), rs["tensors"]["keys"]):
            raise ValueError(f"train(rngs): the keys differ from those the run in {rs['path']} was trained with")
        return True

    def _save_state(self, keys, live, metrics, test_hist, test_metrics, n_done):
        """Write the state after update n_done to runstate.state_file (host-side, outside any graph capture)."""
        from .utils.save_load import save_state
        dp, rank, world = self._placement()
        S, spec = keys.shape[0], self.spec
        t = {"keys": keys, **live}
        t.update({f"metrics/{m}": v[:, :n_done] for m, v in metrics.items()})
        if test_hist is not None:
            t.update({f"test_hist/{kk}": v[:, :n_done] for kk, v in test_hist.items()})
        if test_metrics is not None:
            t.update({f"test_metrics/{kk}": v for kk, v in test_metrics.items()})
        kind = {NET_CNN: "cnn", NET_MLP: "mlp", NET_MLP_BITS: "mlp_bits", NET_RNN: "rnn"}[spec.kind]
        meta = dict(format=runstate.FORMAT_VERSION, script=self.script, env=self.cfg["ENV_NAME"],
                    env_params=dataclasses.asdict(self.env_params),
                    network=dict(kind=kind, D=spec.in_c, A=spec.num_actions, H=spec.hidden, L=spec.layers,
                                 norm_type=spec.norm_type, norm_input=spec.norm_input),
                    n_done=n_done, num_updates=self.NU, rng_mode=self.rng_mode, sweep=self.grid.table(self.seed_lo, S),
                    seed_lo=self.seed_lo, num_seeds_local=S, data_parallel=dp, rank=rank, world=world,
                    config=runstate.run_keys(self.cfg))
        path = runstate.state_file(self.cfg, rank, world)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        save_state(path, {"tensors": t, "meta": meta})

    def _restore_state(self, live, metrics, test_hist):
        """Copy the state of ``self.resume`` into the freshly built buffers and metric columns.  Returns (n0,
        test_metrics): the first update to run and the last evaluation."""
        rs = self.resume
        t, n0 = rs["tensors"], int(rs["meta"]["n_done"])

        def put(dst, name):
            src = t.get(name)
            if src is None or src.shape != dst.shape or src.dtype != dst.dtype:
                got = "missing" if src is None else f"{src.dtype}{list(src.shape)}"
                raise ValueError(f"{rs['path']}: {name} is {got}; this run's is {dst.dtype}{list(dst.shape)}")
            dst.copy_(src)
        for name, buf in live.items():
            put(buf, name)
        for m, v in metrics.items():
            put(v[:, :n0], f"metrics/{m}")
        test_metrics = None
        if test_hist is not None:
            for kk, v in test_hist.items():
                put(v[:, :n0], f"test_hist/{kk}")
            test_metrics = {kk: t[f"test_metrics/{kk}"].to(self.device) for kk in INFO_KEYS}
        if self._placement()[0] == "envs":
            self._check_replicated(t)
        return n0, test_metrics

    def _check_replicated(self, t):
        """Env-sharded ranks hold replicas of the parameters and optimiser state: refuse files that disagree."""
        import hashlib
        import torch.distributed as dist
        h = hashlib.sha256()
        for name in ("params", "batch_stats", "mu", "nu", "step_counter", "rng", "idx"):
            if name in t:
                h.update(t[name].numpy().tobytes())
        d = torch.tensor(list(h.digest()), dtype=torch.int64, device=self.device)
        hi, lo = d.clone(), d.clone()
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        if not torch.equal(hi, lo):
            raise ValueError(f"{self.resume['path']}: the replicated parameters and optimiser state of the env-sharded "
                             f"ranks' state files differ")

    def _wandb_log(self, metrics, test_hist, col, seed_labels):
        import wandb
        S = metrics["td_loss"].shape[0]
        row = {m: v[:, col].mean().item() for m, v in metrics.items()}
        if test_hist is not None:
            row.update({f"test/{kk}": v[:, col].nanmean().item() for kk, v in test_hist.items()})
        if self.cfg.get("WANDB_LOG_ALL_SEEDS", False):
            for s in range(S):
                for m, v in metrics.items():
                    row[f"rng{int(seed_labels[s])}/{m}"] = v[s, col].item()
        wandb.log({self.log_prefix + k: v for k, v in row.items()}, step=int(row["update_steps"]))

    def _result(self, params, batch_stats, u, metrics, test_hist, runner_tail):
        """train()'s result: {"runner_state": (TrainState, *runner_tail), "metrics", "sweep"}."""
        NU, spec, S = self.NU, self.spec, params.shape[0]
        out_metrics = {m: v[:, :NU].float() if m in ("td_loss", "qvals", *INFO_KEYS) else v[:, :NU].to(torch.int64)
                       for m, v in metrics.items()}
        if test_hist is not None:
            out_metrics.update({f"test/{kk}": v[:, :NU].float() for kk, v in test_hist.items()})
        timesteps, grad_steps = NU * self.T * self.E, NU * self.nmb * self.epochs
        train_state = TrainState(
            params=spec.unflatten(params), params_flat=params,
            batch_stats=spec.unflatten_stats(batch_stats), batch_stats_flat=batch_stats,
            opt_state=SimpleNamespace(mu=u.mu, nu=u.nu, count=grad_steps),
            timesteps=torch.full((S,), timesteps, dtype=torch.int64), n_updates=torch.full((S,), NU),
            grad_steps=torch.full((S,), grad_steps))
        out = {"runner_state": (train_state, *runner_tail), "metrics": out_metrics,
               "sweep": self.grid.table(self.seed_lo, S)}
        if self.population is not None:
            out["pbt"] = self.population.result(self.grid, self.seed_lo, NU)
        return out


class PQNEngine(EngineBase):
    def __init__(self, config: dict, network: str, flatten_obs: bool, device=None):
        super().__init__(config, flatten_obs, device)
        self.network = network
        self.spec, self.row_words, self.obs_dtype = network_spec(self.env, network, config)

    @property
    def script(self):
        """The training script of this engine, as a state file records it."""
        return "pqn_minatar" if self.network == "cnn" else "pqn_gymnax"

    def forward(self, params, obs, S, rows, obs_rows_per_seed, q_out, gather=None, batch_stats=None):
        """network.apply({"params", "batch_stats"}, obs, train=False) (pqn_minatar.py:184-191)."""
        ws = self._workspace(S, rows)
        _lib.check(_lib.lib().pqn_qnet_forward(self.spec.desc, _lib.p(params), _lib.p(batch_stats), _lib.raw(obs),
                                               _lib.p(gather),
                                               obs_rows_per_seed, _lib.p(q_out), S, rows, _lib.p(ws),
                                               _lib.stream_ptr()), "pqn_qnet_forward")
        return q_out

    # ------------------------------------------------------------------ #
    def train_steps(self, rngs):
        """train(rngs), one update per ``next``: a generator that yields after every update and returns train's
        result."""
        dev, L = self.device, _lib.lib()
        T, E, A = self.T, self.E, self.A
        keys = jr.as_key_tensor(rngs, dev)
        assert keys.dim() == 2 and keys.shape[1] == 2, "train(rngs) takes the [NUM_SEEDS, 2] key array"
        S = keys.shape[0]
        mode = self.rng_mode
        # ---- env-sharded data parallelism (SURVEY 8(e): needed when NUM_SEEDS < #GPUs).  Rank r owns envs
        # [r*E/W, (r+1)*E/W) of EVERY seed; rollouts are local (per-env keys are those of the unsharded vmap), each
        # minibatch step all-reduces (mean) the flat [S][P] gradient once before clip + RAdam, so parameters stay
        # bit-identical across ranks.  The minibatch permutation is per rank (statistically equivalent to the
        # reference's global shuffle, not sample-identical).
        shard = self.env_shard
        E_total, env_lo, world, rank = E, 0, 1, 0
        if shard is not None and shard[1] > 1:
            import torch.distributed as dist
            rank, world = int(shard[0]), int(shard[1])
            assert E % world == 0, f"NUM_ENVS={E} must be divisible by the {world} env shards"
            E = E // world
            env_lo = rank * E
            assert (T * E) % self.nmb == 0, "NUM_MINIBATCHES must divide NUM_STEPS * NUM_ENVS / world"
            if self.spec.norm_type == "batch_norm" or self.spec.norm_input:
                raise NotImplementedError("env-sharded data parallelism with batch statistics on the path "
                                          "(NORM_TYPE=batch_norm / NORM_INPUT) would need their all-reduce; use "
                                          "DATA_PARALLEL=seeds")
        mb = T * E // self.nmb                                        # minibatch rows of THIS rank
        spec, P = self.spec, self.spec.total
        W = self.row_words

        # ---- schedules (pqn_minatar.py:134-147) and the other per-seed hyperparameters
        hp, sched_stride = self._seed_tables(S)
        eps_table = hp["eps"]
        self._population(hp, sched_stride, S)

        # ---- key chain (SURVEY Appendix B; pqn_minatar.py:172-173,415-423).  A resumed run (RESUME_FROM) skips the
        # initialiser, the first evaluation and the reset: the saved state is copied over the buffers below
        resume = self._resume_begin(keys)
        if not resume:
            k = jr.split(keys, 2, mode)
            K1 = k[:, 0].contiguous()                               # :172 rng (also the init key, :173)
            params = spec.init(K1, dev)                             # :156-170
        else:
            params = torch.empty((S, P), device=dev)
        F = spec.in_c
        batch_stats = spec.init_stats(S, dev)                       # flax BatchNorm running statistics: mean 0, var 1
        self.batch_stats = batch_stats                              # read by get_test_metrics (train=False)
        bn_sums = torch.zeros(S, 2 * F, device=dev)

        test_metrics = None
        if not resume:
            k = jr.split(K1, 2, mode)
            K2, kT0 = k[:, 0].contiguous(), k[:, 1].contiguous()    # :415
            test_metrics = self.get_test_metrics(params, kT0) if self.test else None
            k = jr.split(K2, 2, mode)
            K3, kR = k[:, 0].contiguous(), k[:, 1].contiguous()     # :418
        # ---- rollout buffers: obs rows [S][T+1][E], transitions [S][T][E]
        obs_buf = torch.zeros((S, T + 1, E, W), dtype=self.obs_dtype, device=dev)
        act_buf = torch.zeros((S, T, E), dtype=torch.int32, device=dev)
        rew_buf = torch.zeros((S, T, E), dtype=torch.float32, device=dev)
        done_buf = torch.zeros((S, T, E), dtype=torch.uint8, device=dev)
        maxq_buf = torch.zeros((S, T, E), dtype=torch.float32, device=dev)
        targets = torch.zeros((S, T, E), dtype=torch.float32, device=dev)
        q_buf = torch.zeros((S * E, A), dtype=torch.float32, device=dev)
        info_sums = torch.zeros((S, 5), dtype=torch.float64, device=dev)
        step_keys = torch.zeros((T, S, 2, 2), dtype=torch.int32, device=dev)
        eps_dev = torch.zeros((1, S), device=dev)                   # eps of every seed for this update
        # ---- reset (vmap_reset, :107-109,419)
        if not resume:
            reset_keys = jr.split(kR, E_total, mode)[:, env_lo:env_lo + E].reshape(S * E, 2).contiguous()
        state = torch.empty((self.env.state_words, S * E), dtype=torch.int32, device=dev)
        if not resume:
            envs.reset_into(self.env.env_id, reset_keys, state, None, S * E, self.env_params, mode)
            self._write_obs(state, obs_buf, T, S)                    # update_body moves row T to row 0
            rng = jr.split(K3, 2, mode)[:, 1].contiguous()          # :422-423 runner rng
        else:
            rng = torch.empty_like(keys)

        sp = _lib.stream_ptr
        seed_stride_obs = (T + 1) * E
        seed_stride_tr = T * E
        u = self._update_buffers(params, rng)                        # the whole step is CUDA-graph capturable
        ws = self._workspace(S, max(mb, E))
        perm_ws = jr.permutation_workspace(T * E, S, dev)
        bn_count = float(mb * world * (100 if self.network == "cnn" else 1))   # CNN: per channel over 10x10 pixels

        def allreduce_(t, avg):
            if world > 1:
                dist.all_reduce(t, op=dist.ReduceOp.SUM)              # in-stream: the consumer kernels just follow
                if avg:
                    t.mul_(1.0 / world)

        def update_body():
            """One `_update_step` (pqn_minatar.py:176-350) on the current stream; reads/writes only the static
            buffers above, so it can be replayed from a CUDA graph."""
            # ================= SAMPLE PHASE (:181-219)
            eps_dev.copy_(eps_table.index_select(0, u.idx))
            obs_buf[:, 0].copy_(obs_buf[:, T])                       # last_obs of this rollout = last next_obs
            carry = jr.split(u.rng, 2, mode)[:, 1].contiguous()      # :213  `_rng`
            _lib.check(L.pqn_rollout_keys(_lib.p(carry), _lib.p(step_keys), S, T, mode, sp()), "pqn_rollout_keys")
            info_sums.zero_()
            for t in range(T):
                self.forward(params, obs_buf[:, t], S, E, seed_stride_obs, q_buf, batch_stats=batch_stats)
                self._act_step(S, E, step_keys[t], q_buf, eps_dev, state, obs_buf[:, t + 1], act_buf[:, t],
                               rew_buf[:, t], done_buf[:, t], maxq_buf[:, t], info_sums, 0, hp["rew_scale"],
                               seed_stride_obs, seed_stride_tr, E_total, env_lo)
            r = carry                                                # scan's final carry (:214)
            # ================= bootstrap + Q(lambda) (:227-260)
            self.forward(params, obs_buf[:, T], S, E, seed_stride_obs, q_buf, batch_stats=batch_stats)
            _lib.check(L.pqn_qlambda_seeds(_lib.p(rew_buf), _lib.p(done_buf), _lib.p(maxq_buf), _lib.p(q_buf),
                                           _lib.p(targets), T, S, E, A, _lib.p(hp["gamma"]), _lib.p(hp["lam"]), sp()),
                       "pqn_qlambda_seeds")
            # ================= NETWORKS UPDATE (:263-327)
            r = jr.split(r, 2, mode)[:, 0].contiguous()              # :324
            u.loss_sum.zero_()
            u.qsa_sum.zero_()
            for _ in range(self.epochs):
                k = jr.split(r, 2, mode)                             # :309
                r, kperm = k[:, 0].contiguous(), k[:, 1].contiguous()
                if world > 1:                                        # a different local permutation on every rank
                    kperm = jr.split(kperm, world, mode)[:, rank].contiguous()
                perm_view = jr.permutation_indices(kperm, T * E, mode, chunk=mb, workspace=perm_ws)   # :299-321  [nmb][S][mb]
                r = jr.split(r, 2, mode)[:, 0].contiguous()          # :317
                for mbi in range(self.nmb):
                    _lib.check(L.pqn_qnet_loss_grad(
                        spec.desc, _lib.p(params), _lib.p(batch_stats), _lib.p(obs_buf), _lib.p(perm_view[mbi]),
                        seed_stride_obs,
                        _lib.p(act_buf), _lib.p(targets), seed_stride_tr, _lib.p(u.grads), _lib.p(u.loss_sum),
                        _lib.p(u.qsa_sum), _lib.p(bn_sums), S, mb, _lib.p(ws), sp()), "pqn_qnet_loss_grad")
                    allreduce_(u.grads, True)                        # the ONE collective of the data path
                    allreduce_(bn_sums, False)
                    self._radam_step(params, u, hp, sched_stride, S, P)
                    _lib.check(L.pqn_bn_stats_update(_lib.p(batch_stats), _lib.p(bn_sums), S, F, spec.stats_total,
                                                     bn_count, 0.99, sp()), "pqn_bn_stats_update")
            allreduce_(u.loss_sum, True)
            allreduce_(u.qsa_sum, True)
            allreduce_(info_sums, False)
            self._end_update(u, r, info_sums)                        # :341

        # "auto" captures the update when the run is launch-bound (small S*E)
        payload = dict(obs=obs_buf, action=act_buf, reward=rew_buf, done=done_buf, maxq=maxq_buf, targets=targets,
                       params=params, state=state, rng=u.rng)
        metrics, test_hist, test_metrics = yield from self._run_updates(
            keys, params, u, update_body, payload, S * E * T <= (1 << 21) and world == 1, test_metrics,
            frame_channels=self.env.observation_space().shape[-1] if self.network == "cnn" else None,
            live=dict(params=params, batch_stats=batch_stats, env_state=state, last_obs=obs_buf[:, T]))
        expl_state = (obs_buf[:, -1].contiguous(), state)
        return self._result(params, batch_stats, u, metrics, test_hist, (expl_state, test_metrics, u.rng))

    # ------------------------------------------------------------------ #
    def _write_obs(self, state, obs_buf, t, S):
        """obs rows of `state` into obs_buf[:, t] (the reset observation)."""
        L = _lib.lib()
        E = obs_buf.shape[2]
        tmp = torch.empty((S * E, self.row_words), dtype=self.obs_dtype, device=self.device)
        if self.env.binary_obs:
            _lib.check(L.pqn_env_obs_packed(self.env.env_id, _lib.p(state), _lib.p(tmp), S * E, _lib.stream_ptr()),
                       "pqn_env_obs_packed")
        else:
            _lib.check(L.pqn_env_obs(self.env.env_id, _lib.p(state), _lib.p(tmp), S * E, _lib.stream_ptr()),
                       "pqn_env_obs")
        obs_buf[:, t] = tmp.view(S, E, self.row_words)

    # ------------------------------------------------------------------ #
    def get_test_metrics(self, params, rng):
        """Greedy evaluation rollout (pqn_minatar.py:371-413), incl. its key quirks:
        the scan carry starts at the reset key `_rng`, and each step uses the same
        sub-key for the action keys and the env keys.  The network reads ``self.batch_stats``."""
        c, dev, mode = self.cfg, self.device, self.rng_mode
        S = rng.shape[0]
        N = int(c["TEST_NUM_ENVS"])
        steps = int(c["TEST_NUM_STEPS"])
        W, A = self.row_words, self.A
        k = jr.split(rng, 2, mode)
        kr = k[:, 1].contiguous()                                    # :396 `_rng`
        state = torch.empty((self.env.state_words, S * N), dtype=torch.int32, device=dev)
        envs.reset_into(self.env.env_id, jr.split(kr, N, mode).reshape(S * N, 2).contiguous(), state, None, S * N,
                        self.env_params, mode)
        obs = torch.zeros((S, 2, N, W), dtype=self.obs_dtype, device=dev)   # ping-pong rows
        self._write_obs(state, obs, 0, S)
        q = torch.zeros((S * N, A), dtype=torch.float32, device=dev)
        scratch_i = torch.zeros((S, N), dtype=torch.int32, device=dev)
        scratch_f = torch.zeros((S, N), dtype=torch.float32, device=dev)
        scratch_f2 = torch.zeros((S, N), dtype=torch.float32, device=dev)
        scratch_b = torch.zeros((S, N), dtype=torch.uint8, device=dev)
        sums = torch.zeros((S, 5), dtype=torch.float64, device=dev)
        eps = torch.full((S,), float(c["EPS_TEST"]), device=dev)
        ones = torch.ones(S, device=dev)                             # the evaluation's rewards are not scaled
        carry = kr                                                   # :399-401
        for t in range(steps):
            k = jr.split(carry, 2, mode)                             # :378
            carry, ku = k[:, 0].contiguous(), k[:, 1].contiguous()
            sk = torch.stack([ku, ku], 1).contiguous()               # same key for actions and env (:388-393)
            cur, nxt = t & 1, (t + 1) & 1
            self.forward(params, obs[:, cur], S, N, 2 * N, q, batch_stats=self.batch_stats)
            self._act_step(S, N, sk, q, eps, state, obs[:, nxt], scratch_i, scratch_f, scratch_b, scratch_f2, sums, 1,
                           ones, 2 * N, N, N, 0)
        return self._episode_means(sums)


def prepare_config(config: dict, env_max_steps: int, allow_test_steps_override: bool):
    """The config mutations of make_train (pqn_minatar.py:91-105 / pqn_gymnax.py:80-97)."""
    config["NUM_UPDATES"] = config["TOTAL_TIMESTEPS"] // config["NUM_STEPS"] // config["NUM_ENVS"]
    config["NUM_UPDATES_DECAY"] = config["TOTAL_TIMESTEPS_DECAY"] // config["NUM_STEPS"] // config["NUM_ENVS"]
    assert (config["NUM_STEPS"] * config["NUM_ENVS"]) % config["NUM_MINIBATCHES"] == 0, \
        "NUM_MINIBATCHES must divide NUM_STEPS*NUM_ENVS"
    if allow_test_steps_override:
        config["TEST_NUM_STEPS"] = config.get("TEST_NUM_STEPS", env_max_steps)
    else:
        config["TEST_NUM_STEPS"] = env_max_steps
    return config
