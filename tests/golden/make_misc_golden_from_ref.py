"""SimpleBandit-bsuite, BernoulliBandit-misc, FourRooms-misc and MetaMaze-misc golden trajectories FROM THE REAL
REFERENCE STACK (jax + gymnax==0.0.6), to be run the first time a machine with those packages is reachable.  Without
jax / gymnax it prints why and writes nothing.

    python tests/golden/make_misc_golden_from_ref.py [--out tests/golden] [--envs 32]

Output, for the four envs and both threefry layouts:

    misc_<simple_bandit|bernoulli_bandit|four_rooms|meta_maze>_<original|partitionable>_ref.npz
        reset_keys, obs0, step_keys[T], action[T], obs[T], reward[T], done[T], discount[T], ret[T], len[T], the env
        state after every step under gymnax's field names (SimpleBandit: rewards, total_regret, time; BernoulliBandit:
        last_action, last_reward, exp_reward_best, reward_probs, time; FourRooms: pos, goal, time; MetaMaze:
        last_action, last_reward, pos, goal, time), every field of the env's default EnvParams as ``param_<name>``,
        and ``obs_shape``, the shape of one unflattened observation

SimpleBandit runs T = 40 steps (every step is an episode), BernoulliBandit T = 2 * 100 + 5, FourRooms T = 2 * 500 + 5
and MetaMaze T = 2 * 200 + 5.  Actions are uniform random over the env's actions.  The files are replayed by
tests/test_misc_envs_host.py::test_against_reference, which checks the recollected points listed in
tests/bsuite_bandit_oracle.py and tests/misc_envs_oracle.py: among them the fp32 levels of jnp.linspace(0, 1, 11) (the
``rewards`` field), the time normalisation in the observations and the default EnvParams.

Env construction == pqn_gymnax.py:92-94: gymnax.make(name), FlattenObservationWrapper, LogWrapper, default params.
Key recipe == make_golden_from_ref.py: key = PRNGKey(seed); (key, kr) = split(key); reset keys = split(kr, n); every
step (key, ka, ks) = split(key, 3); action_i = randint(split(ka, n)[i], (), 0, num_actions); env keys = split(ks, n).
"""
import argparse
import dataclasses
import os
import sys

FIELDS = {
    "SimpleBandit-bsuite": ("simple_bandit", ("rewards", "total_regret", "time"), 40, 51),
    "BernoulliBandit-misc": ("bernoulli_bandit", ("last_action", "last_reward", "exp_reward_best", "reward_probs",
                                                  "time"), 205, 52),
    "FourRooms-misc": ("four_rooms", ("pos", "goal", "time"), 1005, 53),
    "MetaMaze-misc": ("meta_maze", ("last_action", "last_reward", "pos", "goal", "time"), 405, 54),
}


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
            raw, params = gymnax.make(name)
            num_actions = raw.action_space(params).n
            obs_shape = raw.reset(jax.random.PRNGKey(0), params)[0].shape
            env = LogWrapper(FlattenObservationWrapper(raw))
            vreset = jax.jit(jax.vmap(env.reset, in_axes=(0, None)))
            vstep = jax.jit(jax.vmap(env.step, in_axes=(0, 0, 0, None)))
            vrand = jax.jit(jax.vmap(lambda k: jax.random.randint(k, (), 0, num_actions)))
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
            res["reward"] = res["reward"].reshape(steps, n)       # a reward of shape (1,) per env comes out (n, 1)
            res.update(reset_keys=np.asarray(rkeys), obs0=np.asarray(obs), obs_shape=np.asarray(obs_shape))
            for f in dataclasses.fields(params):
                res[f"param_{f.name}"] = np.asarray(getattr(params, f.name))
            np.savez_compressed(os.path.join(args.out, f"misc_{short}_{tag}_ref.npz"), **res)
            print("wrote", name, tag, flush=True)
    jax.config.update("jax_threefry_partitionable", False)
    return 0


if __name__ == "__main__":
    sys.exit(main())
