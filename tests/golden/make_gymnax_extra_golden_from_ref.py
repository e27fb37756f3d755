"""MountainCar-v0 and Catch-bsuite golden trajectories FROM THE REAL REFERENCE STACK (jax + gymnax==0.0.6), to be run
the first time a machine with those packages is reachable.  Without jax / gymnax it prints why and writes nothing.

    python tests/golden/make_gymnax_extra_golden_from_ref.py [--out tests/golden] [--envs 32]

Output, for both envs and both threefry layouts:

    gymnax_extra_<mountain_car|catch>_<original|partitionable>_ref.npz
        reset_keys, obs0, step_keys[T], action[T], obs[T], reward[T], done[T], discount[T], ret[T], len[T], the env
        state after every step under gymnax's field names (MountainCar: position, velocity, time; Catch: ball_x,
        ball_y, paddle_x, paddle_y, prev_done, time), and every field of the env's default EnvParams as
        ``param_<name>``

MountainCar runs T = 210 steps (past the 200-step truncation); Catch runs T = 3 * 9 + 2 steps (three whole episodes).
Actions are uniform random over the 3 actions.  The names do not match the ``*_traj_*_ref.npz`` glob of
tests/test_golden_and_abi.py; the files are replayed by tests/test_gymnax_extra_host.py::test_against_reference,
which checks the recollected points listed in tests/gymnax_extra_oracle.py.

Env construction == pqn_gymnax.py:92-94: gymnax.make(name), FlattenObservationWrapper, LogWrapper, default params.
Key recipe == make_golden_from_ref.py: key = PRNGKey(seed); (key, kr) = split(key); reset keys = split(kr, n); every
step (key, ka, ks) = split(key, 3); action_i = randint(split(ka, n)[i], (), 0, 3); env keys = split(ks, n).
"""
import argparse
import dataclasses
import os
import sys

FIELDS = {"MountainCar-v0": ("mountain_car", ("position", "velocity", "time"), 210, 31),
          "Catch-bsuite": ("catch", ("ball_x", "ball_y", "paddle_x", "paddle_y", "prev_done", "time"), 29, 32)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.dirname(os.path.abspath(__file__)))
    ap.add_argument("--envs", type=int, default=32)
    args = ap.parse_args()
    try:
        import jax
        import jax.numpy as jnp
        import gymnax
        from gymnax.wrappers.purerl import FlattenObservationWrapper, LogWrapper
    except Exception as e:  # pragma: no cover
        print(f"reference stack unavailable: {e!r}")
        return 3
    import numpy as np
    os.makedirs(args.out, exist_ok=True)
    n = args.envs

    for part in (False, True):
        jax.config.update("jax_threefry_partitionable", part)
        tag = "partitionable" if part else "original"
        for name, (short, fields, steps, seed) in FIELDS.items():
            env, params = gymnax.make(name)
            env = LogWrapper(FlattenObservationWrapper(env))
            vreset = jax.jit(jax.vmap(env.reset, in_axes=(0, None)))
            vstep = jax.jit(jax.vmap(env.step, in_axes=(0, 0, 0, None)))
            vrand = jax.jit(jax.vmap(lambda k: jax.random.randint(k, (), 0, 3)))
            key = jax.random.PRNGKey(seed)
            key, kr = jax.random.split(key)
            rkeys = jax.random.split(kr, n)
            obs, st = vreset(rkeys, params)
            out = {k: [] for k in ("step_keys", "action", "obs", "reward", "done", "discount", "ret", "len") + fields}
            for t in range(steps):
                key, ka, ks = jax.random.split(key, 3)
                act = vrand(jax.random.split(ka, n)).astype(jnp.int32)
                sk = jax.random.split(ks, n)
                obs_t, st, r, d, info = vstep(sk, st, act, params)
                for k, v in (("step_keys", sk), ("action", act), ("obs", obs_t), ("reward", r), ("done", d),
                             ("discount", info["discount"]), ("ret", info["returned_episode_returns"]),
                             ("len", info["returned_episode_lengths"])):
                    out[k].append(np.asarray(v))
                for k in fields:
                    out[k].append(np.asarray(getattr(st.env_state, k)))
            res = {k: np.stack(v) for k, v in out.items()}
            res.update(reset_keys=np.asarray(rkeys), obs0=np.asarray(obs))
            for f in dataclasses.fields(params):
                res[f"param_{f.name}"] = np.asarray(getattr(params, f.name))
            np.savez_compressed(os.path.join(args.out, f"gymnax_extra_{short}_{tag}_ref.npz"), **res)
            print("wrote", name, tag, flush=True)
    jax.config.update("jax_threefry_partitionable", False)
    return 0


if __name__ == "__main__":
    sys.exit(main())
