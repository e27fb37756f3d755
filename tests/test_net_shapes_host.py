"""Parameter layout of the MLP and GRU Q-networks at every built shape (HIDDEN_SIZE 64..512, NUM_LAYERS 1..8), through
the C ABI (`pqn_net_layout`, `pqn_net_dense_layer`; host code, no kernel is launched), against the flax parameter
trees of the oracles; and the refusal of shapes that are not built."""
import ctypes

import numpy as np
import pytest

from oracle import pqn_ref_norm as RN
from oracle import pqn_rnn_ref as RR

WIDTHS = (64, 128, 256, 512)
MAX_LAYERS = 8


def _spec(kind, D, A, H, L, norm_type="layer_norm", norm_input=False):
    from purejaxql_b200.networks import QNetworkSpec
    return QNetworkSpec(kind, D, A, H, L, norm_type=norm_type, norm_input=norm_input)


def _dense_layer(spec, layer):
    from purejaxql_b200 import _lib
    off = (ctypes.c_int64 * 4)()
    _lib.check(_lib.lib().pqn_net_dense_layer(spec.desc, layer, off), "pqn_net_dense_layer")
    return tuple(int(v) for v in off)


CASES = [("mlp", nt, H, L) for nt in ("layer_norm", "batch_norm", "none") for H in WIDTHS for L in range(1, MAX_LAYERS + 1)]
CASES += [("rnn", "layer_norm", H, L) for H in WIDTHS for L in range(1, MAX_LAYERS + 1)]


@pytest.mark.parametrize("kind,norm_type,H,L", CASES)
def test_layout_blocks_match_flax_shapes(kind, norm_type, H, L):
    from purejaxql_b200.networks import NET_MLP, NET_RNN
    D, A = 6, 3
    spec = _spec(NET_MLP if kind == "mlp" else NET_RNN, D, A, H, L, norm_type)
    want = RN.mlp_param_shapes(D, A, H, L, norm_type) if kind == "mlp" else RR.rnn_param_shapes(D, A, H, L)
    got = {"/".join(p): tuple(shape) for p, _, shape, _ in spec.entries}
    assert got == {k: tuple(v) for k, v in want.items()}
    # disjoint, 4-float aligned blocks that cover the whole per-seed block
    spans = sorted((int(off), int(off) + int(np.prod(shape))) for _, off, shape, _ in spec.entries)
    assert all(a % 4 == 0 for a, _ in spans)
    assert all(spans[i][1] <= spans[i + 1][0] for i in range(len(spans) - 1))
    assert sum((b - a + 3) // 4 * 4 for a, b in spans) == spec.total
    # the per-layer call: layers 0 / 1 are the d0/ln0 and d1/ln1 fields; every layer's offsets are the entries'
    lay = spec.layout
    assert _dense_layer(spec, 0) == (lay.d0_w, lay.d0_b, lay.ln0_scale, lay.ln0_bias)
    if L >= 2:
        assert _dense_layer(spec, 1) == (lay.d1_w, lay.d1_b, lay.ln1_scale, lay.ln1_bias)
    else:
        assert (lay.d1_w, lay.d1_b, lay.ln1_scale, lay.ln1_bias) == (-1, -1, -1, -1)
    offs = {"/".join(p): off for p, off, *_ in spec.entries}
    norm = {"layer_norm": "LayerNorm_{}", "batch_norm": "BatchNorm_{}", "none": None}[norm_type]
    for layer in range(L):
        w, b, g, bi = _dense_layer(spec, layer)
        assert (w, b) == (offs[f"Dense_{layer}/kernel"], offs[f"Dense_{layer}/bias"])
        if norm is None:
            assert (g, bi) == (-1, -1)
        else:
            name = norm.format(layer + 1 if norm_type == "batch_norm" else layer)
            assert (g, bi) == (offs[f"{name}/scale"], offs[f"{name}/bias"])


def _layout_before_deep_layers(D, A, H, L, rnn, has_norm):
    """The layout formula of the networks with HIDDEN_SIZE in {128, 256} and NUM_LAYERS in {1, 2}, as it stood before
    deeper networks were built: the order is BatchNorm_0, Dense_0, norm 0, [Dense_1, norm 1], [GRU], head."""
    off = 0
    out = {}

    def take(name, n):
        nonlocal off
        out[name] = off
        off += (n + 3) // 4 * 4
    take("bn_scale", D); take("bn_bias", D)
    take("d0_w", D * H); take("d0_b", H)
    if has_norm:
        take("ln0_scale", H); take("ln0_bias", H)
    if L == 2:
        take("d1_w", H * H); take("d1_b", H)
        if has_norm:
            take("ln1_scale", H); take("ln1_bias", H)
    if rnn:
        for g in ("ir", "iz", "in"):
            take(f"gru_{g}_w", (H + A) * H); take(f"gru_{g}_b", H)
        take("gru_hr_w", H * H); take("gru_hz_w", H * H); take("gru_hn_w", H * H); take("gru_hn_b", H)
    take("head_w", H * A); take("head_b", A)
    out["total"] = off
    return out


@pytest.mark.parametrize("kind,norm_type", [("mlp", "layer_norm"), ("mlp", "batch_norm"), ("mlp", "none"),
                                            ("rnn", "layer_norm")])
@pytest.mark.parametrize("H,L", [(128, 1), (128, 2), (256, 1), (256, 2)])
def test_existing_shapes_keep_their_layout(kind, norm_type, H, L):
    from purejaxql_b200.networks import NET_MLP, NET_RNN
    D, A = 4, 2
    spec = _spec(NET_MLP if kind == "mlp" else NET_RNN, D, A, H, L, norm_type)
    want = _layout_before_deep_layers(D, A, H, L, kind == "rnn", norm_type != "none")
    lay = spec.layout
    for name, _ in lay._fields_:
        assert getattr(lay, name) == want.get(name, -1), name
    # the numbers for CartPole (D 4, A 2) at the shipped 256 x 2, written out
    if (kind, norm_type, H, L) == ("mlp", "layer_norm", 256, 2):
        assert (lay.d0_w, lay.d0_b, lay.ln0_scale, lay.ln0_bias) == (8, 1032, 1288, 1544)
        assert (lay.d1_w, lay.d1_b, lay.ln1_scale, lay.ln1_bias) == (1800, 67336, 67592, 67848)
        assert (lay.head_w, lay.head_b, lay.total) == (68104, 68616, 68620)
    if (kind, H, L) == ("rnn", 128, 1):
        assert (lay.gru_ir_w, lay.gru_hn_b, lay.head_w, lay.total) == (904, 100360, 100488, 100748)


def test_flat_names_of_deep_networks():
    from purejaxql_b200.networks import NET_MLP, NET_RNN
    mlp = _spec(NET_MLP, 4, 2, 64, 4)
    assert mlp.flat_names() == [
        "BatchNorm_0,scale", "BatchNorm_0,bias",
        "Dense_0,kernel", "Dense_0,bias", "LayerNorm_0,scale", "LayerNorm_0,bias",
        "Dense_1,kernel", "Dense_1,bias", "LayerNorm_1,scale", "LayerNorm_1,bias",
        "Dense_2,kernel", "Dense_2,bias", "LayerNorm_2,scale", "LayerNorm_2,bias",
        "Dense_3,kernel", "Dense_3,bias", "LayerNorm_3,scale", "LayerNorm_3,bias",
        "Dense_4,kernel", "Dense_4,bias"]
    bn = _spec(NET_MLP, 4, 2, 64, 3, norm_type="batch_norm")
    assert [n for n in bn.flat_names() if n.startswith("BatchNorm")] == [
        "BatchNorm_0,scale", "BatchNorm_0,bias", "BatchNorm_1,scale", "BatchNorm_1,bias",
        "BatchNorm_2,scale", "BatchNorm_2,bias", "BatchNorm_3,scale", "BatchNorm_3,bias"]
    assert [p for p, *_ in bn.stats_entries()] == [("BatchNorm_0",), ("BatchNorm_1",), ("BatchNorm_2",), ("BatchNorm_3",)]
    rnn = _spec(NET_RNN, 3, 2, 512, 3)
    g = "ScannedRNN_0,GRUCell_0,"
    assert rnn.flat_names() == [
        "BatchNorm_0,scale", "BatchNorm_0,bias",
        "Dense_0,kernel", "Dense_0,bias", "LayerNorm_0,scale", "LayerNorm_0,bias",
        "Dense_1,kernel", "Dense_1,bias", "LayerNorm_1,scale", "LayerNorm_1,bias",
        "Dense_2,kernel", "Dense_2,bias", "LayerNorm_2,scale", "LayerNorm_2,bias",
        g + "ir,kernel", g + "ir,bias", g + "iz,kernel", g + "iz,bias", g + "in,kernel", g + "in,bias",
        g + "hr,kernel", g + "hz,kernel", g + "hn,kernel", g + "hn,bias",
        "Dense_3,kernel", "Dense_3,bias"]


@pytest.mark.parametrize("kind", ["mlp", "rnn"])
@pytest.mark.parametrize("H,L,A,limit", [(128, 0, 2, "1 to 8"), (128, 9, 2, "1 to 8"), (96, 2, 2, "64, 128, 256 or 512"),
                                         (1024, 2, 2, "64, 128, 256 or 512"), (512, 2, 10, "limit 227 KB")])
def test_unbuilt_shapes_are_refused_with_the_limit(kind, H, L, A, limit):
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_MLP, NET_RNN
    with pytest.raises(_lib.PqnError) as e:
        _spec(NET_MLP if kind == "mlp" else NET_RNN, 4, A, H, L)
    assert limit in str(e.value)


def test_largest_head_at_512_is_built():
    from purejaxql_b200.networks import NET_MLP
    _spec(NET_MLP, 4, 9, 512, 4)          # 9 actions: the head backward's shared memory still fits at H = 512


def test_dense_layer_rejects_out_of_range_layers():
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_CNN, NET_MLP, QNetworkSpec
    spec = _spec(NET_MLP, 4, 2, 64, 3)
    off = (ctypes.c_int64 * 4)()
    for layer in (-1, 3):
        assert _lib.lib().pqn_net_dense_layer(spec.desc, layer, off) == -1
    assert _lib.lib().pqn_net_dense_layer(QNetworkSpec(NET_CNN, 4, 3).desc, 0, off) == -1
