"""Golden vectors FROM THE REAL REFERENCE STACK (jax + gymnax==0.0.6), to be run the first time a machine with
those packages is reachable (SURVEY.md section 8(c)).  Without jax / gymnax it prints why and writes nothing.

    python tests/golden/make_golden_from_ref.py [--out tests/golden] [--steps 10000]

Output (same layout as make_golden.py, so tests/test_golden_and_abi.py checks the oracle, the host-compiled
device logic and -- under -m gpu -- the CUDA kernels against them as soon as the files exist):

    <game>_traj_original_ref.npz / <game>_traj_partitionable_ref.npz   for the MinAtar games and classic control
        reset_keys, obs0, step_keys[T], action[T], obs[T], reward[T], done[T], ret[T], len[T], final_time
    jax_prng_ref.json        split / random_bits / uniform / randint / permutation values for both threefry layouts
    optax_radam_ref.npz      40 steps of chain(clip_by_global_norm(10), radam(linear_schedule)) incl. one clipped step
    qnetwork_cnn_ref.npz     the reference's own QNetwork (imported from $PUREJAXQL_REF or /root/reference): flax init,
                             forward (train=False), loss and gradients of the _loss_fn form on 33 binary observations
    ref_versions.json        jax / jaxlib / gymnax versions and which MinAtar ids gymnax.make accepts
                             (records the Seaquest-MinAtar registration finding)

Key recipe == make_golden.py: key = PRNGKey(seed); (key, kr) = split(key); reset keys = split(kr, n); every step
(key, ka, ks) = split(key, 3); action_i = randint(split(ka, n)[i], (), 0, A); env keys = split(ks, n).
"""
import argparse
import json
import os
import sys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.dirname(os.path.abspath(__file__)))
    ap.add_argument("--steps", type=int, default=10000)
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

    versions = {"jax": jax.__version__, "gymnax": getattr(gymnax, "__version__", "?")}
    try:
        import jaxlib
        versions["jaxlib"] = jaxlib.__version__
    except Exception:
        pass
    accepted = {}
    for name in ("Breakout-MinAtar", "Asterix-MinAtar", "SpaceInvaders-MinAtar", "Freeway-MinAtar",
                 "Seaquest-MinAtar", "CartPole-v1", "Acrobot-v1"):
        try:
            env, params = gymnax.make(name)
            accepted[name] = {"ok": True, "num_actions": int(env.action_space(params).n),
                              "obs_shape": list(env.observation_space(params).shape),
                              "max_steps_in_episode": int(params.max_steps_in_episode)}
        except Exception as e:
            accepted[name] = {"ok": False, "error": repr(e)}
    versions["gymnax_make"] = accepted
    json.dump(versions, open(os.path.join(args.out, "ref_versions.json"), "w"), indent=1)

    def trajectory(name, n, steps, seed, flatten):
        env, params = gymnax.make(name)
        if flatten:
            env = FlattenObservationWrapper(env)
        env = LogWrapper(env)
        A = int(env.action_space(params).n)
        vreset = jax.jit(jax.vmap(env.reset, in_axes=(0, None)))
        vstep = jax.jit(jax.vmap(env.step, in_axes=(0, 0, 0, None)))
        vrand = jax.jit(jax.vmap(lambda k: jax.random.randint(k, (), 0, A)))
        key = jax.random.PRNGKey(seed)
        key, kr = jax.random.split(key)
        rkeys = jax.random.split(kr, n)
        obs, st = vreset(rkeys, params)
        out = {"reset_keys": np.asarray(rkeys), "obs0": np.asarray(obs), "step_keys": [], "action": [], "obs": [],
               "reward": [], "done": [], "ret": [], "len": []}
        for t in range(steps):
            key, ka, ks = jax.random.split(key, 3)
            act = vrand(jax.random.split(ka, n)).astype(jnp.int32)
            if name == "Freeway-MinAtar":
                act = jnp.where(jnp.arange(n) % 4 != 0, 1, act).astype(jnp.int32)
            sk = jax.random.split(ks, n)
            obs, st, r, d, info = vstep(sk, st, act, params)
            out["step_keys"].append(np.asarray(sk)); out["action"].append(np.asarray(act))
            out["obs"].append(np.asarray(obs)); out["reward"].append(np.asarray(r)); out["done"].append(np.asarray(d))
            out["ret"].append(np.asarray(info["returned_episode_returns"]))
            out["len"].append(np.asarray(info["returned_episode_lengths"]))
        res = {k: (np.stack(v) if isinstance(v, list) else v) for k, v in out.items()}
        if name.endswith("MinAtar"):
            res["obs0"] = np.packbits(res["obs0"].astype(bool).reshape(n, -1), axis=-1)
            res["obs"] = np.packbits(res["obs"].astype(bool).reshape(steps, n, -1), axis=-1)
        res["final_time"] = np.asarray(st.env_state.time)
        return res

    prng = {}
    for part in (False, True):
        jax.config.update("jax_threefry_partitionable", part)
        tag = "partitionable" if part else "original"
        k = jax.random.PRNGKey(1234)
        prng[tag] = {
            "split2": np.asarray(jax.random.split(k)).tolist(),
            "split5": np.asarray(jax.random.split(k, 5)).tolist(),
            "bits7": np.asarray(jax.random.bits(k, (7,), "uint32")).tolist(),
            "uniform": float(jax.random.uniform(k)),
            "randint3": int(jax.random.randint(k, (), 0, 3)),
            "permutation40": np.asarray(jax.random.permutation(k, jnp.arange(40))).tolist(),
            "choice_p": int(jax.random.choice(k, jnp.arange(4), p=jnp.array([0.1, 0.2, 0.3, 0.4]))),
        }
        for name, seed, flatten in (("Breakout-MinAtar", 2024, False), ("Asterix-MinAtar", 8, False),
                                    ("SpaceInvaders-MinAtar", 6, False), ("Freeway-MinAtar", 5, False),
                                    ("Seaquest-MinAtar", 4, False), ("CartPole-v1", 11, True),
                                    ("Acrobot-v1", 13, True)):
            if not accepted[name]["ok"]:
                continue
            res = trajectory(name, args.envs, args.steps, seed, flatten)
            short = name.split("-")[0].lower()
            np.savez_compressed(os.path.join(args.out, f"{short}_traj_{tag}_ref.npz"), **res)
            print("wrote", short, tag, flush=True)
    jax.config.update("jax_threefry_partitionable", False)
    json.dump(prng, open(os.path.join(args.out, "jax_prng_ref.json"), "w"))

    # ---- optax: chain(clip_by_global_norm, radam(linear_schedule)) over 40 steps on a small parameter tree
    try:
        import optax
        rng = np.random.default_rng(5)
        p0 = {"a": rng.standard_normal((7, 5)).astype(np.float32), "b": rng.standard_normal(11).astype(np.float32)}
        gs = [{k: (rng.standard_normal(v.shape) * (30.0 if t == 3 else 1.0)).astype(np.float32) for k, v in p0.items()}
              for t in range(40)]
        sched = optax.linear_schedule(init_value=5e-4, end_value=1e-20, transition_steps=64)
        tx = optax.chain(optax.clip_by_global_norm(10.0), optax.radam(learning_rate=sched))
        params = {k: jnp.asarray(v) for k, v in p0.items()}
        state = tx.init(params)
        traj = []
        for g in gs:
            upd, state = tx.update({k: jnp.asarray(v) for k, v in g.items()}, state, params)
            params = optax.apply_updates(params, upd)
            traj.append({k: np.asarray(v) for k, v in params.items()})
        np.savez_compressed(os.path.join(args.out, "optax_radam_ref.npz"),
                            **{f"p0_{k}": v for k, v in p0.items()},
                            **{f"g{t}_{k}": v for t, g in enumerate(gs) for k, v in g.items()},
                            **{f"p{t + 1}_{k}": v for t, tr in enumerate(traj) for k, v in tr.items()})
        versions["optax"] = optax.__version__
        print("wrote optax_radam_ref.npz", flush=True)
    except Exception as e:  # pragma: no cover
        print(f"optax vectors skipped: {e!r}")

    # ---- the reference's own QNetwork (imported, not restated): init, forward (train=False) and loss gradient
    try:
        sys.path.insert(0, os.environ.get("PUREJAXQL_REF", "/root/reference"))
        from purejaxql.pqn_minatar import QNetwork
        import flax
        from flax.traverse_util import flatten_dict
        net = QNetwork(action_dim=3, norm_type="layer_norm", norm_input=False)
        rng = np.random.default_rng(9)
        obs = (rng.random((33, 10, 10, 4)) < 0.1).astype(np.float32)
        variables = net.init(jax.random.PRNGKey(3), jnp.zeros((1, 10, 10, 4)), train=False)
        q = net.apply(variables, jnp.asarray(obs), train=False)
        act = rng.integers(0, 3, 33)
        tgt = rng.standard_normal(33).astype(np.float32)

        def loss_fn(params):
            qv, _ = net.apply({"params": params, "batch_stats": variables["batch_stats"]}, jnp.asarray(obs), train=True,
                              mutable=["batch_stats"])
            qa = jnp.take_along_axis(qv, jnp.asarray(act)[:, None], axis=-1).squeeze(-1)
            return 0.5 * jnp.square(qa - jnp.asarray(tgt)).mean()
        loss, grads = jax.value_and_grad(loss_fn)(variables["params"])
        np.savez_compressed(os.path.join(args.out, "qnetwork_cnn_ref.npz"), obs=obs, action=act, target=tgt,
                            q=np.asarray(q), loss=np.asarray(loss),
                            **{"param/" + "/".join(k): np.asarray(v) for k, v in flatten_dict(variables["params"]).items()},
                            **{"grad/" + "/".join(k): np.asarray(v) for k, v in flatten_dict(grads).items()})
        versions["flax"] = flax.__version__
        print("wrote qnetwork_cnn_ref.npz", flush=True)
    except Exception as e:  # pragma: no cover
        print(f"QNetwork vectors skipped: {e!r}")
    json.dump(versions, open(os.path.join(args.out, "ref_versions.json"), "w"), indent=1)
    print("reference golden vectors written to", args.out)
    return 0


if __name__ == "__main__":
    sys.exit(main())
