"""The recurrent (GRU) PQN training program: host-side restatement of ``make_train`` in
purejaxql/pqn_rnn_gymnax.py:117-560 with the seed axis taken natively.

All compute is libpqn_b200 kernels: ``pqn_rnn_step`` (one step of the recurrent Q-network for the rollout, the memory
warm-up and the evaluation), ``pqn_rollout_act_step_seeds`` (eps-greedy + env step + LogWrapper, shared with the
feed-forward engine), ``pqn_rnn_loss_grad_seeds`` (window forward, in-loss Q(lambda) targets, BPTT) and
``pqn_radam_clip_step_seeds``; the ``_seeds`` entries read eps, the reward scale, gamma, lambda, the clipping norm and
the RAdam schedule per seed (a hyperparameter grid, sweep.py).  The NORM_TYPE / NORM_INPUT variants other than
(layer_norm, False) call ``pqn_rnn_step_stats`` and pass a static ``batch_stats`` buffer to the loss: the loss updates the running statistics in place (:362-369), the steps read them
(train=False), so the update stays capturable in a CUDA graph.  This
module owns the buffers, walks the reference's PRNG key chain — including its re-bindings of ``rng`` to the final
carry of the rollout scans (:222-228, :531-537) — and keeps the memory of the last MEMORY_WINDOW + NUM_STEPS
transitions.  Minibatches are whole env trajectories: ``jax.random.permutation(rng, x, axis=1)`` (:368-379).
Any float-observation env of ``envs.ENV_IDS`` runs, at its own observation width (1 for SimpleBandit-bsuite up to 64
for DeepSea-bsuite); binary-observation (MinAtar) envs are refused.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch

from . import _lib, envs, jaxrandom as jr
from .engine import EngineBase
from .networks import NET_RNN, QNetworkSpec


def refuse_env(name: str):
    """The recurrent engine's refusal of an env it is not built for (raised before anything is built)."""
    if name in envs.MINATAR_GAMES + envs.MINATAR_UNREGISTERED:              # its memory buffer stores float observation rows
        raise NotImplementedError("the recurrent script is built for the float-observation envs "
                                  "(classic control, MemoryChain-bsuite)")


class PQNRnnEngine(EngineBase):
    def __init__(self, config: dict, device=None, env_params: envs.EnvParams | None = None):
        refuse_env(config["ENV_NAME"])
        super().__init__(config, True, device, env_params)           # env_params: MemoryChain's memory_length (:134-136)
        c = config
        self.W = int(c["MEMORY_WINDOW"])
        self.D = self.env.obs_dim
        self.H = int(c.get("HIDDEN_SIZE", 128))
        self.spec = QNetworkSpec(NET_RNN, self.D, self.A, self.H, int(c.get("NUM_LAYERS", 2)),
                                 norm_type=c.get("NORM_TYPE", "layer_norm"), norm_input=bool(c.get("NORM_INPUT", False)))
        # the default network keeps the entry points without running statistics (its BatchNorm_0 output is discarded)
        self.with_stats = self.spec.norm_type != "layer_norm" or self.spec.norm_input
        assert self.E % self.nmb == 0, "NUM_MINIBATCHES must divide NUM_ENVS (minibatches are whole env trajectories)"
        self.Bm = self.E // self.nmb

    @property
    def script(self):
        """The training script of this engine, as a state file records it."""
        return "pqn_rnn_gymnax"

    # ------------------------------------------------------------------ #
    def step(self, params, hs, obs, last_done, last_action, q, S, N):
        """network.apply(params, hs, obs[None], done[None], last_action[None], train=False) for S x N envs; hs in place.
        The BatchNorm variants normalise with ``self.batch_stats``."""
        L, ws = _lib.lib(), self._workspace(S, N)
        if self.with_stats:
            _lib.check(L.pqn_rnn_step_stats(self.spec.desc, _lib.p(params), _lib.p(self.batch_stats), _lib.p(hs),
                                            _lib.p(obs), N, _lib.p(last_done), _lib.p(last_action), _lib.p(q), S, N,
                                            _lib.p(ws), _lib.stream_ptr()), "pqn_rnn_step_stats")
        else:
            _lib.check(L.pqn_rnn_step(self.spec.desc, _lib.p(params), _lib.p(hs), _lib.p(obs), N, _lib.p(last_done),
                                      _lib.p(last_action), _lib.p(q), S, N, _lib.p(ws), _lib.stream_ptr()), "pqn_rnn_step")

    def _reset(self, key, S, N):
        """vmap_reset(N)(key): obs [S,N,D], state."""
        dev, mode = self.device, self.rng_mode
        state = torch.empty((self.env.state_words, S * N), dtype=torch.int32, device=dev)
        obs = torch.empty((S, N, self.D), dtype=torch.float32, device=dev)
        envs.reset_into(self.env.env_id, jr.split(key, N, mode).reshape(S * N, 2).contiguous(), state, obs, S * N,
                        self.env_params, mode)
        return obs, state

    # ------------------------------------------------------------------ #
    def train_steps(self, rngs):
        """train(rngs), one update per ``next`` (EngineBase.train drives it to its end)."""
        dev, L, mode = self.device, _lib.lib(), self.rng_mode
        T, E, A, W, H, D, Bm = self.T, self.E, self.A, self.W, self.H, self.D, self.Bm
        Tm = W + T
        keys = jr.as_key_tensor(rngs, dev)
        S = keys.shape[0]
        spec, P = self.spec, self.spec.total
        hp, sched_stride = self._seed_tables(S)
        eps_table = hp["eps"]                                        # [NU][S]
        self._population(hp, sched_stride, S)

        # ---- key chain (:255-256, :505-543).  A resumed run (RESUME_FROM) skips the initialiser, the first evaluation,
        # the reset and the memory warm-up: the saved state is copied over the buffers below
        resume = self._resume_begin(keys)
        if not resume:
            k = jr.split(keys, 2, mode)
            rng = k[:, 0].contiguous()                               # :255  rng, _rng = split(rng)
            params = spec.init(rng, dev)                             # :256  create_agent(rng)  (the CARRIED key)
        else:
            params = torch.empty((S, P), device=dev)
        self.batch_stats = spec.init_stats(S, dev) if self.with_stats else None   # mean 0, var 1
        test_metrics = None
        if not resume:
            k = jr.split(rng, 2, mode)
            rng, kT = k[:, 0].contiguous(), k[:, 1].contiguous()     # :505
            test_metrics = self.get_test_metrics(params, kT) if self.test else None
            k = jr.split(rng, 2, mode)
            rng, kR = k[:, 0].contiguous(), k[:, 1].contiguous()     # :508
            last_obs, state = self._reset(kR, S, E)                  # :509
        else:
            last_obs = torch.empty((S, E, D), dtype=torch.float32, device=dev)
            state = torch.empty((self.env.state_words, S * E), dtype=torch.int32, device=dev)
        last_done = torch.zeros((S, E), dtype=torch.uint8, device=dev)
        last_action = torch.zeros((S, E), dtype=torch.int32, device=dev)
        hs = torch.zeros((S, E, H), dtype=torch.float32, device=dev)

        mem = SimpleNamespace(
            hs=torch.zeros((S, Tm, E, H), device=dev), obs=torch.zeros((S, Tm, E, D), device=dev),
            action=torch.zeros((S, Tm, E), dtype=torch.int32, device=dev), reward=torch.zeros((S, Tm, E), device=dev),
            done=torch.zeros((S, Tm, E), dtype=torch.uint8, device=dev),
            last_done=torch.zeros((S, Tm, E), dtype=torch.uint8, device=dev),
            last_action=torch.zeros((S, Tm, E), dtype=torch.int32, device=dev))
        q = torch.zeros((S * E, A), device=dev)
        maxq = torch.zeros((S, E), device=dev)
        info_sums = torch.zeros((S, 5), dtype=torch.float64, device=dev)
        new_obs = torch.empty_like(last_obs)
        eps_one = torch.ones(S, device=dev)                          # random actions of the memory warm-up
        eps_dev = torch.zeros((1, S), device=dev)                    # eps of every seed for this update

        act_t = torch.empty((S, E), dtype=torch.int32, device=dev)
        rew_t = torch.empty((S, E), device=dev)
        done_t = torch.empty((S, E), dtype=torch.uint8, device=dev)

        def rollout(carry_key, n_steps, slot0, eps):
            """n_steps x _step_env / _random_step starting from the expl_state above; transitions go to memory slots
            slot0..; returns the scan's final carry key (the reference re-binds `rng` to it).  Only static buffers are
            touched, so the update's rollout can be replayed from a CUDA graph."""
            step_keys = torch.zeros((n_steps, S, 2, 2), dtype=torch.int32, device=dev)
            carry = carry_key.clone()
            _lib.check(L.pqn_rollout_keys(_lib.p(carry), _lib.p(step_keys), S, n_steps, mode, _lib.stream_ptr()),
                       "pqn_rollout_keys")
            for t in range(n_steps):
                s = slot0 + t
                mem.hs[:, s].copy_(hs); mem.obs[:, s].copy_(last_obs)
                mem.last_done[:, s].copy_(last_done); mem.last_action[:, s].copy_(last_action)
                self.step(params, hs, last_obs, last_done, last_action, q, S, E)
                self._act_step(S, E, step_keys[t], q, eps, state, new_obs, act_t, rew_t, done_t, maxq, info_sums, 0,
                               hp["rew_scale"], E, E, E, 0)
                mem.action[:, s].copy_(act_t); mem.reward[:, s].copy_(rew_t); mem.done[:, s].copy_(done_t)
                last_obs.copy_(new_obs)
                last_done.copy_(done_t); last_action.copy_(act_t)
            return carry

        # ---- memory warm-up with random actions (:514-537); `rng` becomes the scan's final carry
        if not resume:
            k = jr.split(rng, 2, mode)
            rng = rollout(k[:, 1].contiguous(), Tm, 0, eps_one)
            k = jr.split(rng, 2, mode)                               # :541
            rng = k[:, 1].contiguous()                               # runner rng = _rng
        else:
            rng = torch.empty_like(keys)

        u = self._update_buffers(params, rng)                        # static buffers of the update step
        ws = self._workspace(S, max(Tm * Bm, E))
        perm_ws = jr.permutation_workspace(E, S, dev)

        def update_body():
            # ================= SAMPLE PHASE (:190-236)
            eps_dev.copy_(eps_table.index_select(0, u.idx))
            k = jr.split(u.rng, 2, mode)                             # :222
            info_sums.zero_()
            for name in ("hs", "obs", "action", "reward", "done", "last_done", "last_action"):   # :239-243 shift the memory
                buf = getattr(mem, name)
                buf[:, :W].copy_(buf[:, T:T + W].clone())
            rng = rollout(k[:, 1].contiguous(), T, W, eps_dev)       # rng := final carry of the scan (:223-228)
            # ================= NETWORKS UPDATE (:246-386)
            u.loss_sum.zero_(); u.qsa_sum.zero_()
            k = jr.split(rng, 2, mode)                               # :381  (the scan carry starts at `rng`)
            r = k[:, 0].contiguous()
            for _ in range(self.epochs):
                k = jr.split(r, 2, mode)                             # :368
                r, kperm = k[:, 0].contiguous(), k[:, 1].contiguous()
                perm = jr.permutation_indices(kperm, E, mode, workspace=perm_ws).to(torch.int64)   # permutation of the ENV axis
                r = jr.split(r, 2, mode)[:, 0].contiguous()          # :375
                for mbi in range(self.nmb):
                    idx = perm[:, mbi * Bm:(mbi + 1) * Bm]                             # [S, Bm]
                    i3 = idx[:, None, :].expand(S, Tm, Bm)

                    def g3(x):
                        return x.gather(2, i3).contiguous()
                    obs_mb = mem.obs.gather(2, i3[..., None].expand(S, Tm, Bm, D)).contiguous()
                    hs0 = mem.hs[:, 0].gather(1, idx[:, :, None].expand(S, Bm, H)).contiguous()
                    ld, la, ac, rw, dn = g3(mem.last_done), g3(mem.last_action), g3(mem.action), g3(mem.reward), g3(mem.done)
                    # batch_stats = updates["batch_stats"] (:362-369); None for the default network
                    _lib.check(L.pqn_rnn_loss_grad_seeds(
                        spec.desc, _lib.p(params), _lib.p(self.batch_stats), _lib.p(hs0), _lib.p(obs_mb), _lib.p(ld),
                        _lib.p(la), _lib.p(ac), _lib.p(rw), _lib.p(dn), _lib.p(u.grads), _lib.p(u.loss_sum),
                        _lib.p(u.qsa_sum), S, Tm, Bm, _lib.p(hp["gamma"]), _lib.p(hp["lam"]), _lib.p(ws),
                        _lib.stream_ptr()), "pqn_rnn_loss_grad_seeds")
                    self._radam_step(params, u, hp, sched_stride, S, P)
            self._end_update(u, r, info_sums)                        # :398

        # these runs are launch-bound (32 envs x 64 steps: thousands of small launches per update), so "auto" always
        # captures the update
        live = dict(params=params, env_state=state, hs=hs, last_obs=last_obs, last_done=last_done,
                    last_action=last_action, **{f"mem/{k}": v for k, v in vars(mem).items()})
        if self.with_stats:
            live["batch_stats"] = self.batch_stats
        metrics, test_hist, test_metrics = yield from self._run_updates(
            keys, params, u, update_body, dict(mem=mem, params=params, rng=u.rng, batch_stats=self.batch_stats), True,
            test_metrics, live=live)
        bs = self.batch_stats if self.with_stats else spec.init_stats(S, dev)
        expl_state = (hs, last_obs, last_done, last_action, state)
        return self._result(params, bs, u, metrics, test_hist, (mem, expl_state, test_metrics, u.rng))

    # ------------------------------------------------------------------ #
    def get_test_metrics(self, params, rng):
        """Greedy evaluation (:411-503): reset with `_rng`, the scan carry starts at the same `_rng`, every step splits
        (rng, rng_a, rng_s) like the training rollout."""
        c, dev, L, mode = self.cfg, self.device, _lib.lib(), self.rng_mode
        S = rng.shape[0]
        N, steps = int(c["TEST_NUM_ENVS"]), int(c["TEST_NUM_STEPS"])
        kr = jr.split(rng, 2, mode)[:, 1].contiguous()               # :475
        obs, state = self._reset(kr, S, N)
        nxt = torch.empty_like(obs)
        hs = torch.zeros((S, N, self.H), device=dev)
        ld = torch.zeros((S, N), dtype=torch.uint8, device=dev)
        la = torch.zeros((S, N), dtype=torch.int32, device=dev)
        q = torch.zeros((S * N, self.A), device=dev)
        rw, mq = torch.zeros((S, N), device=dev), torch.zeros((S, N), device=dev)
        act = torch.zeros((S, N), dtype=torch.int32, device=dev)
        dn = torch.zeros((S, N), dtype=torch.uint8, device=dev)
        sums = torch.zeros((S, 5), dtype=torch.float64, device=dev)
        eps = torch.full((S,), float(c["EPS_TEST"]), device=dev)
        ones = torch.ones(S, device=dev)                             # the evaluation's rewards are not scaled
        step_keys = torch.zeros((steps, S, 2, 2), dtype=torch.int32, device=dev)
        carry = kr.clone()
        _lib.check(L.pqn_rollout_keys(_lib.p(carry), _lib.p(step_keys), S, steps, mode, _lib.stream_ptr()), "pqn_rollout_keys")
        for t in range(steps):
            self.step(params, hs, obs, ld, la, q, S, N)
            self._act_step(S, N, step_keys[t], q, eps, state, nxt, act, rw, dn, mq, sums, 1, ones, N, N, N, 0)
            obs, nxt = nxt, obs
            ld.copy_(dn); la.copy_(act)
        return self._episode_means(sums)
