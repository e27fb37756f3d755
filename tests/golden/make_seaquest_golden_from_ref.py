"""Seaquest-MinAtar golden trajectories FROM THE REAL GAME, to be run the first time a machine with MinAtar (and,
optionally, a gymnax that registers "Seaquest-MinAtar") is reachable.  Without them it prints why and writes nothing.

    python tests/golden/make_seaquest_golden_from_ref.py [--out tests/golden] [--steps 3000] [--envs 32]

Outputs:

    seaquest_minatar_ref.json   MinAtar's own game (minatar.Environment("seaquest", sticky_action_prob=0)):
        one record per step with the game state before the step (every attribute tests/seaquest_oracle.py names),
        the action, the random draws the step made (recorded from the game's RandomState: enemy lr, is_sub, row; diver
        lr, row; null where not drawn), the reward, the terminal flag, the state after the step and its (10, 10, 10)
        observation as a list of set (row, col, channel) cells.  Actions are uniform random; a terminal step is
        followed by a reset.
    seaquest_gymnax_<original|partitionable>_ref.npz   only if gymnax.make("Seaquest-MinAtar") works: reset_keys,
        obs0, step_keys[T], action[T], obs[T], reward[T], done[T], with the key recipe of make_golden_from_ref.py
        (key = PRNGKey(seed); (key, kr) = split(key); reset keys = split(kr, n); every step (key, ka, ks) =
        split(key, 3); action_i = randint(split(ka, n)[i], (), 0, 6); env keys = split(ks, n)).

tests/test_seaquest_golden.py replays them: MinAtar's records teacher-forced through the oracle's step (the recorded
draws in place of the oracle's jax.random ones), gymnax's through the oracle and the host-compiled device logic.
"""
import argparse
import json
import os
import sys

STATE = ("oxygen", "diver_count", "sub_x", "sub_y", "sub_or", "shot_timer", "surface", "terminal", "move_speed",
         "ramp_index", "e_spawn_speed", "e_spawn_timer", "d_spawn_timer")
LISTS = ("f_bullets", "e_bullets", "e_fish", "e_subs", "divers")


class _Recorder:
    """wraps the game's RandomState: every choice() result is appended to `log` as a plain int"""

    def __init__(self, rs):
        self.rs, self.log = rs, []

    def choice(self, *a, **kw):
        v = self.rs.choice(*a, **kw)
        self.log.append(int(v))
        return v

    def __getattr__(self, k):
        return getattr(self.rs, k)


def _game_state(g):
    d = {k: (bool(getattr(g, k)) if isinstance(getattr(g, k), (bool,)) else int(getattr(g, k))) for k in STATE}
    for k in LISTS:
        d[k] = [[int(v) for v in z] for z in getattr(g, k)]
    return d


def minatar(out, steps):
    try:
        import numpy as np
        from minatar import Environment
    except ImportError as e:
        print(f"MinAtar not importable ({e}); nothing written for it")
        return
    env = Environment("seaquest", sticky_action_prob=0.0, random_seed=0)
    g = env.env
    rec = _Recorder(g.random)
    g.random = rec
    rng = np.random.default_rng(0)
    env.reset()
    records = []
    for t in range(steps):
        a = int(rng.integers(0, 6))
        before = _game_state(g)
        spawn_enemy, spawn_diver = g.e_spawn_timer == 0, g.d_spawn_timer == 0
        rec.log = []
        r, term = env.act(a)
        log = list(rec.log)
        draws = [None] * 5
        if spawn_enemy:
            draws[0:3] = log[0:3]
            log = log[3:]
        if spawn_diver:
            draws[3:5] = log[0:2]
        obs = env.state()
        records.append(dict(before=before, action=a, draws=draws, reward=int(r), terminal=bool(term),
                            after=_game_state(g), obs=[[int(i) for i in c] for c in np.argwhere(obs)]))
        if term:
            env.reset()
    with open(os.path.join(out, "seaquest_minatar_ref.json"), "w") as f:
        json.dump({"records": records}, f)
    print(f"wrote {len(records)} MinAtar records")


def gymnax_(out, n, steps):
    try:
        import gymnax
        import jax
        import numpy as np
        from gymnax.wrappers.purerl import FlattenObservationWrapper, LogWrapper
        core, params = gymnax.make("Seaquest-MinAtar")
    except Exception as e:   # noqa: BLE001 -- any failure means this gymnax cannot make the game
        print(f"gymnax cannot make Seaquest-MinAtar ({e!r}); nothing written for it")
        return
    for part in (False, True):
        jax.config.update("jax_threefry_partitionable", part)
        env = LogWrapper(FlattenObservationWrapper(core))
        key = jax.random.PRNGKey(61)
        key, kr = jax.random.split(key)
        rk = jax.random.split(kr, n)
        obs, st = jax.vmap(env.reset, in_axes=(0, None))(rk, params)
        rec = dict(reset_keys=np.asarray(jax.random.key_data(rk) if hasattr(jax.random, "key_data") else rk),
                   obs0=np.asarray(obs))
        cols = {k: [] for k in ("step_keys", "action", "obs", "reward", "done")}
        step = jax.jit(jax.vmap(env.step, in_axes=(0, 0, 0, None)))
        for t in range(steps):
            key, ka, ks = jax.random.split(key, 3)
            act = jax.vmap(lambda k: jax.random.randint(k, (), 0, 6))(jax.random.split(ka, n))
            sk = jax.random.split(ks, n)
            obs, st, r, d, _ = step(sk, st, act, params)
            for k, v in (("step_keys", sk), ("action", act), ("obs", obs), ("reward", r), ("done", d)):
                cols[k].append(np.asarray(v))
        rec.update({k: np.stack(v) for k, v in cols.items()})
        np.savez_compressed(os.path.join(out, f"seaquest_gymnax_{'partitionable' if part else 'original'}_ref.npz"),
                            **rec)
        print(f"wrote gymnax trajectories ({'partitionable' if part else 'original'})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.dirname(os.path.abspath(__file__)))
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--envs", type=int, default=32)
    args = ap.parse_args()
    minatar(args.out, args.steps)
    gymnax_(args.out, args.envs, min(args.steps, 1005))
    return 0


if __name__ == "__main__":
    sys.exit(main())
