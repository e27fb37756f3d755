"""jax.random.normal values and GaussianBandit-misc golden trajectories FROM THE REAL REFERENCE STACK (jax 0.4.x +
gymnax==0.0.6), to be run the first time a machine with those packages is reachable, ideally one with a CUDA device.
Without jax / gymnax it prints why and writes nothing.

    python tests/golden/make_gaussian_bandit_golden_from_ref.py [--out tests/golden] [--envs 32]

Output:

    gaussian_bandit_normal_ref.npz
        bits: a stride-97 sample of the 2^23 distinct inputs (bits >> 9 = k, low bits 0) plus the edge cases: the
        clamp at lo (k = 0), |u| -> 1 (k = 0, 1, 2^23 - 2, 2^23 - 1), the smallest |u| (u = +-2^-24 + ...: k = 2^22 - 1,
        2^22), and 8 inputs on each side of the w = 5 branch boundary on both signs;
        normal_<cpu|cuda>: jax's normal of those bits (sqrt(2) * erf_inv(uniform(lo, 1)), jitted) on each device present;
        keys_<0|1>, key_normal_<cpu|cuda>_<0|1>: jax.random.normal(key, (1001,)) at 8 keys, per threefry layout
    gaussian_bandit_<original|partitionable>_traj_ref.npz
        reset_keys, obs0, step_keys[T], action[T], obs[T], reward[T], done[T], discount[T], ret[T], len[T], every
        EnvState field after every step as ``state_<name>``, every field of the default EnvParams as ``param_<name>``,
        ``obs_shape`` and ``platform`` (the jax backend the trajectory ran on); T = 2 * 100 + 5

The files are replayed by tests/test_gaussian_bandit_host.py (test_normal_against_reference, test_against_reference)
and tests/test_gpu_gaussian_bandit.py (test_device_normal_against_reference), which check the recollected points
listed in tests/jax_normal_oracle.py and tests/gaussian_bandit_oracle.py.

Env construction == pqn_gymnax.py:92-94: gymnax.make(name), FlattenObservationWrapper, LogWrapper, default params.
Key recipe == make_golden_from_ref.py: key = PRNGKey(seed); (key, kr) = split(key); reset keys = split(kr, n); every
step (key, ka, ks) = split(key, 3); action_i = randint(split(ka, n)[i], (), 0, num_actions); env keys = split(ks, n).
"""
import argparse
import dataclasses
import os
import sys


def normal_inputs(np):
    """The recorded bits (see the module docstring)."""
    k = np.arange(1 << 23, dtype=np.int64)
    u = (2 * k * 2.0 ** -23 - (1 - 2.0 ** -24)).astype(np.float32)      # exact in fp32
    w = -np.log1p(-(u.astype(np.float64) ** 2))
    cross = np.nonzero(np.diff((w < 5).astype(np.int8)))[0]
    edges = [0, 1, (1 << 22) - 1, 1 << 22, (1 << 23) - 2, (1 << 23) - 1]
    for c in cross:
        edges += list(range(max(0, c - 7), min(1 << 23, c + 9)))
    ks = np.unique(np.concatenate([k[::97], np.array(edges, np.int64)]))
    return (ks.astype(np.uint32) << np.uint32(9)).astype(np.uint32)


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

    # ---- jax.random.normal ----
    lo = np.nextafter(np.float32(-1), np.float32(0))

    def from_bits(b):   # jax 0.4.x _normal_real on given random bits
        fb = jax.lax.bitwise_or(jax.lax.shift_right_logical(b, jnp.uint32(9)), jnp.uint32(0x3F800000))
        f = jax.lax.bitcast_convert_type(fb, jnp.float32) - jnp.float32(1)
        u = jax.lax.max(jnp.float32(lo), f * (jnp.float32(1) - jnp.float32(lo)) + jnp.float32(lo))
        return jnp.float32(np.sqrt(2)) * jax.lax.erf_inv(u)

    bits = normal_inputs(np)
    res = {"bits": bits}
    devices = {"cpu": jax.devices("cpu")}
    try:
        devices["cuda"] = jax.devices("gpu")
    except RuntimeError:
        pass
    for part in (0, 1):
        jax.config.update("jax_threefry_partitionable", bool(part))
        keys = jax.random.split(jax.random.PRNGKey(90 + part), 8)
        res[f"keys_{part}"] = np.asarray(keys)
        for name, devs in devices.items():
            with jax.default_device(devs[0]):
                if part == 0:
                    res[f"normal_{name}"] = np.asarray(jax.jit(from_bits)(jnp.asarray(bits)))
                res[f"key_normal_{name}_{part}"] = np.asarray(
                    jax.jit(jax.vmap(lambda k: jax.random.normal(k, (1001,))))(jax.device_put(keys, devs[0])))
    np.savez_compressed(os.path.join(args.out, "gaussian_bandit_normal_ref.npz"), **res)
    print("wrote normal values on", sorted(devices), flush=True)

    # ---- GaussianBandit-misc trajectories ----
    steps = 2 * 100 + 5
    for part in (False, True):
        jax.config.update("jax_threefry_partitionable", part)
        tag = "partitionable" if part else "original"
        raw, params = gymnax.make("GaussianBandit-misc")
        num_actions = raw.action_space(params).n
        obs_shape = raw.reset(jax.random.PRNGKey(0), params)[0].shape
        env = LogWrapper(FlattenObservationWrapper(raw))
        vreset = jax.jit(jax.vmap(env.reset, in_axes=(0, None)))
        vstep = jax.jit(jax.vmap(env.step, in_axes=(0, 0, 0, None)))
        vrand = jax.jit(jax.vmap(lambda k: jax.random.randint(k, (), 0, num_actions)))
        key = jax.random.PRNGKey(55)
        key, kr = jax.random.split(key)
        rkeys = jax.random.split(kr, n)
        obs, st = vreset(rkeys, params)
        names = [f.name for f in dataclasses.fields(st.env_state)]
        out = {k: [] for k in ("step_keys", "action", "obs", "reward", "done", "discount", "ret", "len")}
        out.update({f"state_{k}": [] for k in names})
        for t in range(steps):
            key, ka, ks = jax.random.split(key, 3)
            act = vrand(jax.random.split(ka, n)).astype(jnp.int32)
            sk = jax.random.split(ks, n)
            obs_t, st, r, d, info = vstep(sk, st, act, params)
            for k, v in (("step_keys", sk), ("action", act), ("obs", obs_t), ("reward", r), ("done", d),
                         ("discount", info["discount"]), ("ret", info["returned_episode_returns"]),
                         ("len", info["returned_episode_lengths"])):
                out[k].append(np.asarray(v))
            for k in names:
                out[f"state_{k}"].append(np.asarray(getattr(st.env_state, k)).reshape(n, -1).squeeze(-1))
        res = {k: np.stack(v) for k, v in out.items()}
        res["reward"] = res["reward"].reshape(steps, n)       # a reward of shape (1,) per env comes out (n, 1)
        res.update(reset_keys=np.asarray(rkeys), obs0=np.asarray(obs), obs_shape=np.asarray(obs_shape),
                   platform=np.asarray(jax.default_backend()))
        for f in dataclasses.fields(params):
            res[f"param_{f.name}"] = np.asarray(getattr(params, f.name))
        np.savez_compressed(os.path.join(args.out, f"gaussian_bandit_{tag}_traj_ref.npz"), **res)
        print("wrote GaussianBandit-misc", tag, flush=True)
    jax.config.update("jax_threefry_partitionable", False)
    return 0


if __name__ == "__main__":
    sys.exit(main())
