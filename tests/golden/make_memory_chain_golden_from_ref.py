"""MemoryChain-bsuite golden trajectories FROM THE REAL REFERENCE STACK (jax + gymnax==0.0.6), to be run the first
time a machine with those packages is reachable.  Without jax / gymnax it prints why and writes nothing.

    python tests/golden/make_memory_chain_golden_from_ref.py [--out tests/golden] [--envs 32]

Output, for memory_length L in (5, 100) and both threefry layouts:

    memory_chain_L<L>_<original|partitionable>_ref.npz
        memory_length, reset_keys, obs0, step_keys[T], action[T], obs[T], reward[T], done[T], discount[T], ret[T],
        len[T] and the env state after every step: context[T], query[T], total_perfect[T], total_regret[T], time[T]

T = 3 (L + 1) + 2 steps, i.e. three whole episodes of every env.  Actions are uniform random, so both the +1 and the
-1 reward occur.  The names do not match the ``*_traj_*_ref.npz`` glob of tests/test_golden_and_abi.py; the files
are replayed by tests/test_memory_chain_host.py::test_oracle_against_reference_memory_chain, which checks the (R)
points listed in tests/bsuite_oracle.py.

Env construction == pqn_rnn_gymnax.py:134-139: gymnax.make("MemoryChain-bsuite"), EnvParams(memory_length=L),
FlattenObservationWrapper, LogWrapper.  Key recipe == make_golden_from_ref.py: key = PRNGKey(seed);
(key, kr) = split(key); reset keys = split(kr, n); every step (key, ka, ks) = split(key, 3);
action_i = randint(split(ka, n)[i], (), 0, 2); env keys = split(ks, n).
"""
import argparse
import os
import sys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.dirname(os.path.abspath(__file__)))
    ap.add_argument("--envs", type=int, default=32)
    args = ap.parse_args()
    try:
        import jax
        import jax.numpy as jnp
        import gymnax
        from gymnax.environments.bsuite.memory_chain import EnvParams
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
        for L, seed in ((5, 21), (100, 22)):
            env, _ = gymnax.make("MemoryChain-bsuite")
            params = EnvParams(memory_length=L)
            env = LogWrapper(FlattenObservationWrapper(env))
            vreset = jax.jit(jax.vmap(env.reset, in_axes=(0, None)))
            vstep = jax.jit(jax.vmap(env.step, in_axes=(0, 0, 0, None)))
            vrand = jax.jit(jax.vmap(lambda k: jax.random.randint(k, (), 0, 2)))
            key = jax.random.PRNGKey(seed)
            key, kr = jax.random.split(key)
            rkeys = jax.random.split(kr, n)
            obs, st = vreset(rkeys, params)
            out = {k: [] for k in ("step_keys", "action", "obs", "reward", "done", "discount", "ret", "len", "context",
                                   "query", "total_perfect", "total_regret", "time")}
            for t in range(3 * (L + 1) + 2):
                key, ka, ks = jax.random.split(key, 3)
                act = vrand(jax.random.split(ka, n)).astype(jnp.int32)
                sk = jax.random.split(ks, n)
                obs_t, st, r, d, info = vstep(sk, st, act, params)
                es = st.env_state
                for k, v in (("step_keys", sk), ("action", act), ("obs", obs_t), ("reward", r), ("done", d),
                             ("discount", info["discount"]), ("ret", info["returned_episode_returns"]),
                             ("len", info["returned_episode_lengths"]), ("context", es.context), ("query", es.query),
                             ("total_perfect", es.total_perfect), ("total_regret", es.total_regret),
                             ("time", es.time)):
                    out[k].append(np.asarray(v))
            res = {k: np.stack(v) for k, v in out.items()}
            res.update(memory_length=np.int32(L), reset_keys=np.asarray(rkeys), obs0=np.asarray(obs))
            np.savez_compressed(os.path.join(args.out, f"memory_chain_L{L}_{tag}_ref.npz"), **res)
            print("wrote memory_chain", L, tag, flush=True)
    jax.config.update("jax_threefry_partitionable", False)
    return 0


if __name__ == "__main__":
    sys.exit(main())
