"""PQN on MinAtar with the CNN Q-network — drop-in for purejaxql/pqn_minatar.py.

    python -m purejaxql_b200.pqn_minatar +alg=pqn_minatar alg.ENV_NAME=Breakout-MinAtar NUM_SEEDS=16
    python -m purejaxql_b200.pqn_minatar +alg=pqn_minatar alg.ENV_NAME=Seaquest-MinAtar NUM_SEEDS=4
    python -m purejaxql_b200.pqn_minatar +alg=pqn_minatar NUM_SEEDS=16 alg.NUM_ENVS=1024 \
        "alg.ENV_NAME=[Breakout-MinAtar,Asterix-MinAtar,SpaceInvaders-MinAtar,Freeway-MinAtar,Seaquest-MinAtar]"

Runs the four MinAtar games gymnax registers (``envs.MINATAR_GAMES``) and Seaquest-MinAtar, which gymnax 0.0.6 does
not register and which is restated here from MinAtar's own game (``envs.MINATAR_UNREGISTERED``; 10 channels, 6
actions).

``make_train(config)`` keeps the reference's contract (pqn_minatar.py:89-431):
it mutates ``config`` (NUM_UPDATES, NUM_UPDATES_DECAY, TEST_NUM_STEPS), asserts
the minibatch divisibility, and returns ``train``.  The reference wraps
``train`` in ``jax.jit(jax.vmap(...))`` over ``rngs``; here ``train(rngs)`` takes
the ``[NUM_SEEDS, 2]`` key array directly and returns the same dict with a
leading seed axis: ``{"runner_state": (train_state, (obs, env_state),
test_metrics, rng), "metrics": {name: [S, NUM_UPDATES]}}``.  A list-valued
``ENV_NAME`` returns ``{env_name: that dict}`` (``env_list.py``).
"""
from __future__ import annotations

from . import _runner, env_list, envs, pbt, state, sweep
from .engine import CNN_NEEDS_MINATAR, PQNEngine, prepare_config


def _check_env(name):
    """The refusal a standalone run of `name` meets, without building the env."""
    envs.check_name(name)
    if name not in envs.MINATAR_GAMES + envs.MINATAR_UNREGISTERED:
        raise ValueError(CNN_NEEDS_MINATAR)


def make_train(config):
    sweep.Grid(config)                       # refuses lists it cannot train before anything is built
    pbt.settings(config)                     # refuses bad PBT_* settings before anything is built
    if sweep.env_names(config) is not None:  # a list of envs: one engine per env on its own stream (env_list.py)
        return env_list.make_train(config, _make_train_one, _check_env)
    return _make_train_one(config)


def _make_train_one(config):
    env, env_params = envs.make(config["ENV_NAME"])                  # :103-104
    prepare_config(config, env_params.max_steps_in_episode, allow_test_steps_override=False)   # :91-105
    resume = state.load_for_resume(config, "pqn_minatar")   # RESUME_FROM, checked before anything is built
    engine = PQNEngine(config, network="cnn", flatten_obs=False)
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
