"""Device-side ``jax.random`` plumbing the training program needs on the host
side of the boundary: keys are int32/uint32 bit patterns in CUDA tensors and all
arithmetic runs in libpqn_b200 kernels (``pqn_rng_split`` / ``pqn_rng_bits`` /
``pqn_random_normal``).

Mirrors the calls in purejaxql/pqn_minatar.py: ``PRNGKey`` (:456), ``split``
(:108,112,172,183,213,309,...), ``permutation`` (:303); and ``normal``, which
gymnax's GaussianBandit-misc draws.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib


def PRNGKey(seed: int, device="cuda") -> torch.Tensor:
    """``jax.random.PRNGKey(seed)`` -> int32[2] tensor holding the uint32 words."""
    seed = int(seed)
    words = np.array([(seed >> 32) & 0xFFFFFFFF, seed & 0xFFFFFFFF], dtype=np.uint32)
    return torch.from_numpy(words.view(np.int32).copy()).to(device)


def as_key_tensor(rngs, device="cuda") -> torch.Tensor:
    """Accepts numpy uint32/int32 arrays or tensors of shape [..., 2]."""
    if isinstance(rngs, torch.Tensor):
        t = rngs
        if t.dtype != torch.int32:
            t = t.to(torch.int64).bitwise_and(0xFFFFFFFF)
            t = torch.where(t >= 2 ** 31, t - 2 ** 32, t).to(torch.int32)
        return t.to(device).contiguous()
    a = np.ascontiguousarray(np.asarray(rngs)).astype(np.uint32, copy=False)
    return torch.from_numpy(a.view(np.int32).copy()).to(device)


def to_numpy_u32(keys: torch.Tensor) -> np.ndarray:
    return keys.detach().cpu().numpy().view(np.uint32)


def split(keys: torch.Tensor, num: int = 2, rng_mode: int = 0) -> torch.Tensor:
    """``jax.random.split`` batched over leading axes: [..., 2] -> [..., num, 2]."""
    keys = keys.contiguous()
    lead = keys.shape[:-1]
    n = int(math.prod(lead)) if lead else 1
    out = torch.empty(lead + (num, 2), dtype=torch.int32, device=keys.device)
    _lib.check(_lib.lib().pqn_rng_split(_lib.p(keys), n, num, _lib.p(out), rng_mode, _lib.stream_ptr()),
               "pqn_rng_split")
    return out


def random_bits(keys: torch.Tensor, length: int, rng_mode: int = 0) -> torch.Tensor:
    """``jax.random.bits(key, (length,), uint32)`` for keys [n,2] -> int32[n,length] bit patterns."""
    keys = keys.contiguous()
    n = keys.shape[0]
    out = torch.empty((n, length), dtype=torch.int32, device=keys.device)
    _lib.check(_lib.lib().pqn_rng_bits(_lib.p(keys), n, length, _lib.p(out), rng_mode, _lib.stream_ptr()),
               "pqn_rng_bits")
    return out


def normal(key: torch.Tensor, n: int, rng_mode: int = 0) -> torch.Tensor:
    """``jax.random.normal(key, (n,))`` (float32) for one key [2] -> float32[n], in ``pqn_random_normal``."""
    key = key.contiguous()
    if key.shape != (2,):
        raise ValueError(f"normal takes one key of shape (2,), got {tuple(key.shape)}")
    out = torch.empty(int(n), dtype=torch.float32, device=key.device)
    _lib.check(_lib.lib().pqn_random_normal(_lib.p(key), _lib.p(out), int(n), rng_mode, _lib.stream_ptr()),
               "pqn_random_normal")
    return out


def permutation_workspace(n: int, S: int, device) -> torch.Tensor:
    """Scratch buffer of ``pqn_permutation`` for S keys and n elements (callers that permute every update keep one)."""
    nbytes = int(_lib.lib().pqn_permutation_workspace_bytes(int(n), int(S)))
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=device)


def permutation_indices(keys: torch.Tensor, n: int, rng_mode: int = 0, chunk: int = 0, workspace=None) -> torch.Tensor:
    """Index permutation of ``jax.random.permutation(key, x)`` for ``len(x)==n``, batched over keys [S,2] ->
    int32[S,n]: jax's ``_shuffle`` (ceil(3 ln n / ln(2^32-1)) rounds of a *stable* sort by fresh uint32 keys) in
    ``pqn_permutation`` (exact bucket + rank sort, csrc/pqn_perm.cu).  ``chunk > 0`` returns the minibatch layout
    int32[n // chunk, S, chunk] (minibatch i of seed s = positions [i*chunk, (i+1)*chunk) of its permutation)."""
    keys = keys.contiguous()
    S = keys.shape[0]
    ws = workspace if workspace is not None else permutation_workspace(n, S, keys.device)
    shape = (n // chunk, S, chunk) if chunk else (S, n)
    out = torch.empty(shape, dtype=torch.int32, device=keys.device)
    _lib.check(_lib.lib().pqn_permutation(_lib.p(keys), int(n), int(S), rng_mode, _lib.p(out), int(chunk), _lib.p(ws),
                                          _lib.stream_ptr()), "pqn_permutation")
    return out
