"""Recurrent (GRU) PQN on the float-observation gymnax envs — drop-in for purejaxql/pqn_rnn_gymnax.py.

    python -m purejaxql_b200.pqn_rnn_gymnax +alg=pqn_rnn_cartpole NUM_SEEDS=4
    python -m purejaxql_b200.pqn_rnn_gymnax +alg=pqn_rnn_memory_chain
    python -m purejaxql_b200.pqn_rnn_gymnax +alg=pqn_rnn_cartpole alg.ENV_NAME=MountainCar-v0
    python -m purejaxql_b200.pqn_rnn_gymnax +alg=pqn_rnn_cartpole alg.ENV_NAME=Catch-bsuite
    python -m purejaxql_b200.pqn_rnn_gymnax +alg=pqn_rnn_cartpole alg.ENV_NAME=UmbrellaChain-bsuite
    python -m purejaxql_b200.pqn_rnn_gymnax +alg=pqn_rnn_cartpole alg.ENV_NAME=MetaMaze-misc
    python -m purejaxql_b200.pqn_rnn_gymnax +alg=pqn_rnn_cartpole alg.ENV_NAME=GaussianBandit-misc
    python -m purejaxql_b200.pqn_rnn_gymnax +alg=pqn_rnn_cartpole "alg.ENV_NAME=[CartPole-v1,MemoryChain-bsuite,MetaMaze-misc]"

The envs are CartPole-v1, Acrobot-v1, MountainCar-v0, MemoryChain-bsuite, Catch-bsuite (50 inputs: every
NORM_TYPE / NORM_INPUT runs on it), DeepSea-bsuite (64 inputs), UmbrellaChain-bsuite, DiscountingChain-bsuite,
SimpleBandit-bsuite (11 actions: HIDDEN_SIZE 512 is refused), the meta-RL tasks BernoulliBandit-misc,
GaussianBandit-misc and MetaMaze-misc, and FourRooms-misc, each with gymnax's default ``EnvParams``.  The MinAtar games
are refused: the memory stores float observation rows.

``make_train(config)`` keeps the reference's contract (pqn_rnn_gymnax.py:117-560): config mutation (NUM_UPDATES,
NUM_UPDATES_DECAY, TEST_NUM_STEPS), ``RNNQNetwork`` (MLP trunk -> one-hot last action -> scanned GRU with done-resets ->
Q head), a memory of MEMORY_WINDOW + NUM_STEPS transitions warmed up with random actions, minibatches over ENVS (whole
trajectories) and the Q(lambda) targets computed inside the loss from the window's own q values.  As in the other
scripts ``train(rngs)`` takes the ``[NUM_SEEDS, 2]`` key array natively, and a list-valued ``ENV_NAME`` trains every
env of the list in one run (``env_list.py``; ``ENV_KWARGS.memory_length`` applies to the MemoryChain-bsuite entry).
"""
from __future__ import annotations

from . import _runner, env_list, envs, pbt, state, sweep
from .engine import prepare_config
from .engine_rnn import PQNRnnEngine, refuse_env


def _check_env(name):
    """The refusal a standalone run of `name` meets, without building the env."""
    envs.check_name(name)
    refuse_env(name)


def make_train(config):
    sweep.Grid(config)                       # refuses lists it cannot train before anything is built
    pbt.settings(config)                     # refuses bad PBT_* settings before anything is built
    if sweep.env_names(config) is not None:  # a list of envs: one engine per env on its own stream (env_list.py)
        return env_list.make_train(config, _make_train_one, _check_env, env_sharding=False)
    return _make_train_one(config)


def _make_train_one(config):
    env, env_params = envs.make(config["ENV_NAME"], flatten_obs=True)      # :134-139
    if config["ENV_NAME"] == "MemoryChain-bsuite":
        # :134-136 -- EnvParams(memory_length=ENV_KWARGS.get("memory_length", 10)): the script's default is 10, not
        # gymnax's 5; max_steps_in_episode keeps its default (1000), which is also TEST_NUM_STEPS's
        memory_length = (config.get("ENV_KWARGS") or {}).get("memory_length", 10)
        if isinstance(memory_length, bool) or not isinstance(memory_length, int) or memory_length < 1:
            raise ValueError(f"MemoryChain-bsuite needs ENV_KWARGS.memory_length to be a positive int, "
                             f"got {memory_length!r}")
        env_params = envs.EnvParams(env_params.max_steps_in_episode, memory_length=memory_length)
    # the window loss (pqn_rnn_loss_grad) takes at most 1024 trajectories per minibatch and needs two steps of window
    # (one loss step plus its bootstrap); refuse other shapes here rather than after the warm-up and the first rollout
    traj = config["NUM_ENVS"] // config["NUM_MINIBATCHES"]
    if traj > 1024:
        raise ValueError(f"NUM_ENVS / NUM_MINIBATCHES = {traj} trajectories per minibatch; the recurrent loss takes at "
                         f"most 1024")
    window = config.get("MEMORY_WINDOW", 0) + config["NUM_STEPS"]
    if window < 2:
        raise ValueError(f"MEMORY_WINDOW + NUM_STEPS = {window}; the recurrent loss needs a window of at least 2 steps")
    prepare_config(config, env_params.max_steps_in_episode, allow_test_steps_override=True)    # :119-132,140
    resume = state.load_for_resume(config, "pqn_rnn_gymnax")   # RESUME_FROM, checked before anything is built
    engine = PQNRnnEngine(config, env_params=env_params)
    engine.resume = resume

    def train(rngs):
        return engine.train(rngs)

    train.engine = engine
    return train


def single_run(config):
    # PQNRnnEngine has no env-sharded mode: under torchrun the ranks take seeds
    return _runner.single_run(config, make_train, alg_file_name="pqn_rnn", env_sharding=False)


def main(argv=None):
    return _runner.main(make_train, argv, env_sharding=False)


if __name__ == "__main__":
    main()
