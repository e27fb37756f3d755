"""PQN on the gymnax environments with the MLP Q-network — drop-in for
purejaxql/pqn_gymnax.py.

    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole NUM_SEEDS=8
    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole alg.ENV_NAME=Breakout-MinAtar
    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole alg.ENV_NAME=Seaquest-MinAtar
    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole alg.ENV_NAME=MountainCar-v0
    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole alg.ENV_NAME=Catch-bsuite
    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole alg.ENV_NAME=DeepSea-bsuite
    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole alg.ENV_NAME=FourRooms-misc
    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole alg.ENV_NAME=GaussianBandit-misc
    python -m purejaxql_b200.pqn_gymnax +alg=pqn_cartpole NUM_SEEDS=4 "alg.ENV_NAME=[CartPole-v1,Acrobot-v1,Catch-bsuite,DeepSea-bsuite]"

Every env of ``envs.ENV_IDS`` runs with its gymnax default ``EnvParams``: CartPole-v1, Acrobot-v1, MountainCar-v0
(200 steps), MemoryChain-bsuite, Catch-bsuite (its 10 x 5 board flattened to 50 inputs), DeepSea-bsuite (its 8 x 8
board flattened to 64 inputs), UmbrellaChain-bsuite, DiscountingChain-bsuite (5 actions), SimpleBandit-bsuite (one
constant input, 11 actions: HIDDEN_SIZE 512 is refused), BernoulliBandit-misc, GaussianBandit-misc, FourRooms-misc,
MetaMaze-misc and the MinAtar games (Seaquest-MinAtar included: restated from MinAtar, as gymnax 0.0.6 does not
register it; its board flattens to 1000 inputs).

On a MinAtar game the flattened (10,10,C) observation feeds the MLP as in the reference; the rollout keeps it as
packed bits and Dense_0 reads those directly (PQN_NET_MLP_BITS).

Differences from pqn_minatar (as in the reference, pqn_gymnax.py:29-58,92-97):
MLP ``QNetwork(HIDDEN_SIZE, NUM_LAYERS)`` without the /255, the observation is
flattened (``FlattenObservationWrapper``), ``TEST_NUM_STEPS`` may be overridden
from the config, and there is REW_SCALE.

A list-valued ``ENV_NAME`` trains every env of the list in one run (``env_list.py``): ``train(rngs)`` returns
``{env_name: <what a standalone train(rngs) of that env returns>}``.
"""
from __future__ import annotations

from . import _runner, env_list, envs, pbt, state, sweep
from .engine import PQNEngine, prepare_config


def make_train(config):
    sweep.Grid(config)                       # refuses lists it cannot train before anything is built
    pbt.settings(config)                     # refuses bad PBT_* settings before anything is built
    if sweep.env_names(config) is not None:  # a list of envs: one engine per env on its own stream (env_list.py)
        return env_list.make_train(config, _make_train_one, envs.check_name)
    return _make_train_one(config)


def _make_train_one(config):
    env, env_params = envs.make(config["ENV_NAME"], flatten_obs=True)      # :92-94
    prepare_config(config, env_params.max_steps_in_episode, allow_test_steps_override=True)    # :80-97
    resume = state.load_for_resume(config, "pqn_gymnax")   # RESUME_FROM, checked before anything is built
    engine = PQNEngine(config, network="mlp", flatten_obs=True)
    engine.resume = resume

    def train(rngs):
        return engine.train(rngs)

    train.engine = engine
    return train


def single_run(config):
    return _runner.single_run(config, make_train)


def tune(default_config):
    return _runner.tune(default_config, make_train)


def main(argv=None):
    return _runner.main(make_train, argv)


if __name__ == "__main__":
    main()
