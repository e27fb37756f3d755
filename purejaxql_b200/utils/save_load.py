"""Checkpoint wire format of purejaxql/utils/save_load.py: safetensors whose
keys are the flax parameter paths joined with ",", one file per seed.

``save_state`` / ``load_state`` are this repo's own training-state file (``purejaxql_b200.state``): the flat device
buffers of a run between two updates, with a JSON metadata header, written atomically."""
from __future__ import annotations

import json
import os
import tempfile
from typing import Dict, Union

import torch
from safetensors import safe_open
from safetensors.torch import load_file, save_file


def _flatten(d: Dict, prefix=()):
    out = {}
    for k, v in d.items():
        if isinstance(v, dict):
            out.update(_flatten(v, prefix + (k,)))
        else:
            out[",".join(prefix + (k,))] = v
    return out


def _unflatten(flat: Dict):
    tree: Dict = {}
    for k, v in flat.items():
        d = tree
        parts = k.split(",")
        for p in parts[:-1]:
            d = d.setdefault(p, {})
        d[parts[-1]] = v
    return tree


def save_params(params: Dict, filename: Union[str, os.PathLike]) -> None:
    flat = {k: torch.as_tensor(v).detach().cpu().contiguous().clone() for k, v in _flatten(params).items()}
    save_file(flat, str(filename))


def load_params(filename: Union[str, os.PathLike]) -> Dict:
    return _unflatten(load_file(str(filename)))


def save_state(path: Union[str, os.PathLike], state: Dict) -> None:
    """Write ``state = {"tensors": {name: tensor}, "meta": JSON-able dict}`` as one safetensors file whose
    ``__metadata__`` holds the meta dict under "state".  The file is written to a temporary name in the same directory,
    fsynced and renamed over ``path``, so a write that is killed halfway leaves the previous file intact."""
    path = os.fspath(path)
    d = os.path.dirname(os.path.abspath(path))
    tensors = {k: torch.as_tensor(v).detach().cpu().contiguous() for k, v in state["tensors"].items()}
    fd, tmp = tempfile.mkstemp(dir=d, prefix=os.path.basename(path) + ".", suffix=".tmp")
    os.close(fd)
    try:
        save_file(tensors, tmp, metadata={"state": json.dumps(state["meta"])})
        with open(tmp, "rb+") as f:
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise
    dfd = os.open(d, os.O_RDONLY)
    try:
        os.fsync(dfd)                                             # the rename itself survives a crash
    finally:
        os.close(dfd)


def read_state_meta(path: Union[str, os.PathLike]) -> Dict:
    """The meta dict of a state file, without reading its tensors."""
    with safe_open(os.fspath(path), framework="pt") as f:
        md = f.metadata() or {}
    if "state" not in md:
        raise ValueError(f"{os.fspath(path)} is not a training-state file (its header has no 'state' metadata)")
    return json.loads(md["state"])


def load_state(path: Union[str, os.PathLike]) -> Dict:
    """``{"tensors": {name: CPU tensor}, "meta": dict}`` of a file written by save_state."""
    return {"tensors": load_file(os.fspath(path)), "meta": read_state_meta(path)}
