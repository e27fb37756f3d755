"""Multi-GPU tests (need >= 2 GPUs; skipped otherwise): the env-sharded
data-parallel mode (SURVEY 8(e), north star's "single NCCL gradient all-reduce") against a single-rank run."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _cfg():
    # ONE minibatch per epoch, one epoch: the minibatch is the whole rollout, so the per-rank permutation cannot
    # change WHICH samples a gradient step sees and the sharded run must reproduce the single-rank run
    return dict(ENV_NAME="Breakout-MinAtar", TOTAL_TIMESTEPS=3 * 8 * 128.0, TOTAL_TIMESTEPS_DECAY=3 * 8 * 128.0,
                NUM_ENVS=128, NUM_STEPS=8, NUM_MINIBATCHES=1, NUM_EPOCHS=1, EPS_START=1.0, EPS_FINISH=1.0,
                EPS_DECAY=0.1, LR=5e-4, MAX_GRAD_NORM=10, GAMMA=0.99, LAMBDA=0.65, NORM_TYPE="layer_norm",
                LR_LINEAR_DECAY=True, WANDB_MODE="disabled", TEST_DURING_TRAINING=False, CUDA_GRAPH=False)


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from oracle import jax_prng as jr
    from purejaxql_b200 import pqn_minatar
    train = pqn_minatar.make_train(_cfg())
    train.engine.env_shard = (rank, world)
    out = train(jr.split(jr.PRNGKey(5), 2))
    ts = out["runner_state"][0]
    np.save(os.path.join(out_dir, f"params{rank}.npy"), ts.params_flat.cpu().numpy())
    np.save(os.path.join(out_dir, f"loss{rank}.npy"), out["metrics"]["td_loss"].cpu().numpy())
    np.save(os.path.join(out_dir, f"ret{rank}.npy"), out["metrics"]["returned_episode_lengths"].cpu().numpy())
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_env_sharded_two_ranks_match_single_rank(tmp_path):
    import torch.multiprocessing as mp
    from oracle import jax_prng as jr
    from purejaxql_b200 import pqn_minatar
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    p0, p1 = np.load(tmp_path / "params0.npy"), np.load(tmp_path / "params1.npy")
    assert np.array_equal(p0, p1), "parameters must stay bit-identical across the env shards"
    torch.cuda.set_device(0)
    out = pqn_minatar.make_train(_cfg())(jr.split(jr.PRNGKey(5), 2))
    ref = out["runner_state"][0].params_flat.cpu().numpy()
    # same envs, same keys, same samples per gradient step; only the summation order of the batch mean differs
    assert np.abs(p0 - ref).max() < 2e-5, np.abs(p0 - ref).max()
    l0 = np.load(tmp_path / "loss0.npy")
    assert np.allclose(l0, out["metrics"]["td_loss"].cpu().numpy(), rtol=1e-4, atol=1e-6)
    # rollout bookkeeping is integer work on the union of the shards: exact
    assert np.array_equal(np.load(tmp_path / "ret0.npy"), out["metrics"]["returned_episode_lengths"].cpu().numpy())
