"""Q-network parameter blocks: flax-named views over the flat per-seed float32
block that libpqn_b200's kernels consume (``pqn_net_layout``).

Reference modules: ``QNetwork``/``CNN`` purejaxql/pqn_minatar.py:24-69 and MLP
``QNetwork`` purejaxql/pqn_gymnax.py:29-58; parameter tree names per SURVEY
Appendix C (flax auto-naming), e.g. ``params["CNN_0"]["Dense_0"]["kernel"]``.
``NORM_TYPE`` in {"layer_norm", "batch_norm", anything else = none} and
``NORM_INPUT`` follow pqn_minatar.py:31-36,61-66 / pqn_gymnax.py:38-51: with
batch_norm the two (or NUM_LAYERS) normalisations are ``BatchNorm`` modules —
flax auto-names them ``CNN_0/BatchNorm_0``, ``CNN_0/BatchNorm_1`` inside the CNN
and ``BatchNorm_1..L`` in the MLP (they share the module counter with the input
``BatchNorm_0``) — and own running statistics in ``batch_stats``; with "none"
the network has no normalisation parameters at all.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from . import _lib

NET_CNN = 0
NET_MLP = 1
NET_RNN = 2     # RNNQNetwork (GRU) of pqn_rnn_gymnax.py:57-105
NET_MLP_BITS = 3   # the MLP QNetwork fed a MinAtar env's packed {0,1} observation rows (D = 100 * C inputs)


class QNetworkSpec:
    def __init__(self, kind: int, in_c: int, num_actions: int, hidden: int = 128, layers: int = 2,
                 norm_type: str = "layer_norm", norm_input: bool = False):
        self.kind, self.in_c, self.num_actions, self.hidden, self.layers = kind, in_c, num_actions, hidden, layers
        self.norm_type = norm_type if norm_type in _lib.NORM_TYPES else "none"
        self.norm_input = bool(norm_input)
        self.desc = _lib.NetDesc(kind, in_c, hidden, layers, num_actions, _lib.NORM_TYPES.get(norm_type, 2),
                                 int(self.norm_input))
        self.stats_total = int(_lib.lib().pqn_net_stats_floats(self.desc))
        lay = _lib.NetLayout()
        _lib.check(_lib.lib().pqn_net_layout(self.desc, lay), "pqn_net_layout")
        self.layout = lay
        self.total = int(lay.total)
        self.entries = self._entries()

    # (flax path, offset, shape, fan_in for init or None, init kind)
    def _entries(self):
        L, A = self.layout, self.num_actions
        e = []

        def norm(prefix, idx, off_s, off_b, n):
            # flax auto-names: LayerNorm_i, or BatchNorm_i (CNN) / BatchNorm_{i+1} (MLP: the input one is BatchNorm_0)
            if self.norm_type == "layer_norm":
                name = f"LayerNorm_{idx}"
            elif self.norm_type == "batch_norm":
                name = f"BatchNorm_{idx if prefix else idx + 1}"
            else:
                return []
            return [(prefix + (name, "scale"), off_s, (n,), "ones"), (prefix + (name, "bias"), off_b, (n,), "zeros")]
        if self.kind == NET_CNN:
            C = self.in_c
            e += [(("BatchNorm_0", "scale"), L.bn_scale, (C,), "ones"),
                  (("BatchNorm_0", "bias"), L.bn_bias, (C,), "zeros"),
                  (("CNN_0", "Conv_0", "kernel"), L.conv_w, (3, 3, C, 16), "he"),
                  (("CNN_0", "Conv_0", "bias"), L.conv_b, (16,), "zeros")]
            e += norm(("CNN_0",), 0, L.ln0_scale, L.ln0_bias, 16)
            e += [(("CNN_0", "Dense_0", "kernel"), L.d0_w, (1024, 128), "he"),
                  (("CNN_0", "Dense_0", "bias"), L.d0_b, (128,), "zeros")]
            e += norm(("CNN_0",), 1, L.ln1_scale, L.ln1_bias, 128)
            e += [(("Dense_0", "kernel"), L.head_w, (128, A), "lecun"),
                  (("Dense_0", "bias"), L.head_b, (A,), "zeros")]
        else:
            D, H = self.in_c, self.hidden
            e += [(("BatchNorm_0", "scale"), L.bn_scale, (D,), "ones"),
                  (("BatchNorm_0", "bias"), L.bn_bias, (D,), "zeros")]
            for layer, (off_w, off_b, off_s, off_bi) in enumerate(self.dense_layers()):
                e += [((f"Dense_{layer}", "kernel"), off_w, (D if layer == 0 else H, H), "lecun"),
                      ((f"Dense_{layer}", "bias"), off_b, (H,), "zeros")]
                e += norm((), layer, off_s, off_bi, H)
            if self.kind == NET_RNN:
                # flax.linen.GRUCell: input denses ir/iz/in (bias, lecun_normal), recurrent hr/hz (no bias) and hn
                # (bias), orthogonal recurrent kernels
                g = ("ScannedRNN_0", "GRUCell_0")
                e += [(g + ("ir", "kernel"), L.gru_ir_w, (H + A, H), "lecun"), (g + ("ir", "bias"), L.gru_ir_b, (H,), "zeros"),
                      (g + ("iz", "kernel"), L.gru_iz_w, (H + A, H), "lecun"), (g + ("iz", "bias"), L.gru_iz_b, (H,), "zeros"),
                      (g + ("in", "kernel"), L.gru_in_w, (H + A, H), "lecun"), (g + ("in", "bias"), L.gru_in_b, (H,), "zeros"),
                      (g + ("hr", "kernel"), L.gru_hr_w, (H, H), "orthogonal"),
                      (g + ("hz", "kernel"), L.gru_hz_w, (H, H), "orthogonal"),
                      (g + ("hn", "kernel"), L.gru_hn_w, (H, H), "orthogonal"), (g + ("hn", "bias"), L.gru_hn_b, (H,), "zeros")]
            e += [((f"Dense_{self.layers}", "kernel"), L.head_w, (H, A), "lecun"),
                  ((f"Dense_{self.layers}", "bias"), L.head_b, (A,), "zeros")]
        return e

    def dense_layers(self):
        """(kernel, bias, norm scale, norm bias) offsets of every hidden layer (``pqn_net_dense_layer``; -1: none)."""
        out = []
        for layer in range(self.layers):
            off = (ctypes.c_int64 * 4)()
            _lib.check(_lib.lib().pqn_net_dense_layer(self.desc, layer, off), "pqn_net_dense_layer")
            out.append(tuple(int(v) for v in off))
        return out

    # ------------------------------------------------------------------ #
    def stats_entries(self):
        """(flax batch_stats path, offset of `mean` in the per-seed block, n); `var` follows at offset + n."""
        F = self.in_c
        out = [(("BatchNorm_0",), 0, F)]
        if self.norm_type == "batch_norm":
            if self.kind == NET_CNN:
                out += [(("CNN_0", "BatchNorm_0"), 2 * F, 16), (("CNN_0", "BatchNorm_1"), 2 * F + 32, 128)]
            else:
                out += [((f"BatchNorm_{l + 1}",), 2 * F + 2 * self.hidden * l, self.hidden) for l in range(self.layers)]
        return out

    def init_stats(self, S, device="cuda") -> torch.Tensor:
        """flax BatchNorm initial running statistics: mean 0, var 1 -> float32[S, stats_total]."""
        st = torch.zeros((S, self.stats_total), dtype=torch.float32)
        for _, off, n in self.stats_entries():
            st[:, off + n:off + 2 * n] = 1.0
        return st.to(device)

    def unflatten_stats(self, st: torch.Tensor) -> dict:
        tree: dict = {}
        for path, off, n in self.stats_entries():
            d = tree
            for k in path[:-1]:
                d = d.setdefault(k, {})
            d[path[-1]] = {"mean": st[:, off:off + n], "var": st[:, off + n:off + 2 * n]}
        return tree

    def flatten_stats(self, stats: dict, S: int = 1, device="cuda") -> torch.Tensor:
        """{"A/B": {"mean","var"}} (oracle) -> float32[S, stats_total]."""
        st = torch.zeros((S, self.stats_total), dtype=torch.float32)
        for path, off, n in self.stats_entries():
            d = stats["/".join(path)]
            st[:, off:off + n] = torch.as_tensor(np.asarray(d["mean"]), dtype=torch.float32).reshape(-1, n)
            st[:, off + n:off + 2 * n] = torch.as_tensor(np.asarray(d["var"]), dtype=torch.float32).reshape(-1, n)
        return st.to(device)

    # ------------------------------------------------------------------ #
    def unflatten(self, flat: torch.Tensor) -> dict:
        """float32[S, total] -> nested flax-style dict of [S, *shape] views."""
        tree: dict = {}
        for path, off, shape, _ in self.entries:
            n = int(np.prod(shape))
            v = flat[:, off:off + n].reshape((flat.shape[0],) + tuple(shape))
            d = tree
            for k in path[:-1]:
                d = d.setdefault(k, {})
            d[path[-1]] = v
        return tree

    def flatten(self, tree_or_flatdict: dict, S: int | None = None, device="cuda") -> torch.Tensor:
        """Nested dict, or flat dict keyed by "A/B/c" (oracle) or "A,B,c"
        (safetensors), of [S,*shape] (or unbatched [*shape]) arrays -> float32[S,total]."""
        def lookup(path):
            d = tree_or_flatdict
            for sep in ("/", ","):
                k = sep.join(path)
                if k in d:
                    return d[k]
            for k in path:
                d = d[k]
            return d
        first = torch.as_tensor(np.asarray(lookup(self.entries[0][0])))
        batched = first.dim() == 2
        if S is None:
            S = first.shape[0] if batched else 1
        flat = torch.zeros((S, self.total), dtype=torch.float32)
        for path, off, shape, _ in self.entries:
            v = torch.as_tensor(np.asarray(lookup(path)), dtype=torch.float32)
            n = int(np.prod(shape))
            flat[:, off:off + n] = v.reshape(S if batched else 1, n)
        return flat.to(device)

    def init(self, keys, device="cuda") -> torch.Tensor:
        """``network.init`` on the device (``pqn_net_init``): flax-default initialisers, deterministic in the
        per-seed key but not flax's draws (flax folds module paths into the key; see DESIGN.md).
        ``keys``: int32[S,2] CUDA tensor."""
        S = keys.shape[0]
        flat = torch.empty((S, self.total), dtype=torch.float32, device=keys.device)
        _lib.check(_lib.lib().pqn_net_init(self.desc, _lib.p(keys.contiguous()), _lib.p(flat), S, _lib.stream_ptr()),
                   "pqn_net_init")
        orth = [(off, shape) for _, off, shape, kind in self.entries if kind == "orthogonal"]
        if orth:   # flax recurrent_kernel_init = orthogonal(): QR of a normal matrix, per seed, on the host (tiny)
            ku = keys.detach().cpu().numpy().view(np.uint32)
            for s in range(S):
                gen = torch.Generator().manual_seed((int(ku[s, 0]) << 32 | int(ku[s, 1])) & (2 ** 63 - 1))
                for off, shape in orth:
                    m = torch.randn(shape, generator=gen, dtype=torch.float64)
                    qm, rm = torch.linalg.qr(m)
                    qm = qm * torch.sign(torch.diagonal(rm)).unsqueeze(0)
                    flat[s, off:off + qm.numel()] = qm.reshape(-1).to(torch.float32).to(flat.device)
        return flat

    def init_host(self, keys_u32: np.ndarray, device="cuda") -> torch.Tensor:
        """Host (torch CPU generator) variant of the same initialisers, kept for tests.  flax-default initialisers (he_normal for Conv/Dense_0 of the CNN,
        lecun_normal elsewhere — truncated normal at +-2 sigma, variance-scaled by
        fan_in; zeros biases; ones LayerNorm/BatchNorm scales).  Deterministic in
        the per-seed key but NOT bit-identical to flax's draws (flax folds module
        paths into the key; see DESIGN.md)."""
        S = keys_u32.shape[0]
        flat = torch.zeros((S, self.total), dtype=torch.float32)
        for s in range(S):
            g = torch.Generator().manual_seed(int(keys_u32[s, 0]) << 32 | int(keys_u32[s, 1]))
            for path, off, shape, kind in self.entries:
                n = int(np.prod(shape))
                if kind == "ones":
                    flat[s, off:off + n] = 1.0
                elif kind in ("he", "lecun"):
                    fan_in = int(np.prod(shape[:-1]))
                    var = (2.0 if kind == "he" else 1.0) / fan_in
                    std = math.sqrt(var) / 0.87962566103423978
                    w = torch.empty(n)
                    torch.nn.init.trunc_normal_(w, mean=0.0, std=1.0, a=-2.0, b=2.0, generator=g)
                    flat[s, off:off + n] = w * std
        return flat.to(device)

    def flat_names(self, sep=","):
        return [sep.join(p) for p, *_ in self.entries]
