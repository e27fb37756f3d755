"""purejaxql_b200 — an H100-native (sm_90a) PQN rollout-and-update engine.

Host side: Python/PyTorch (device memory, streams, torch.distributed plumbing)
calling hand-written CUDA through the C ABI of ``libpqn_b200.so``
(``include/pqn_b200.h``).  Mirrors the ``make_train(config)`` / ``train()``
surface of mttga/purejaxql's ``pqn_minatar.py`` / ``pqn_gymnax.py``.

There is no CPU compute path: importing the kernels without the built library,
or running them without a CUDA device, raises.
"""
__version__ = "0.1.0"
