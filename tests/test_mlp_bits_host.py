"""The MLP Q-network on packed MinAtar observations (PQN_NET_MLP_BITS) through the C ABI and the engine's network choice,
host code only: its parameter layout and flax names are the MLP's with D = 100 * C inputs at every built shape, other
input sizes are refused, pqn_gymnax builds it for every MinAtar game, and the recurrent script still refuses MinAtar."""
import ctypes

import pytest

from oracle import pqn_ref_norm as RN

GAMES = {"Breakout-MinAtar": (400, 3), "Asterix-MinAtar": (400, 5), "SpaceInvaders-MinAtar": (600, 4),
         "Freeway-MinAtar": (700, 3)}
WIDTHS = (64, 128, 256, 512)


def _spec(kind, D, A, H, L, norm_type="layer_norm", norm_input=False):
    from purejaxql_b200.networks import QNetworkSpec
    return QNetworkSpec(kind, D, A, H, L, norm_type=norm_type, norm_input=norm_input)


@pytest.mark.parametrize("D", [400, 600, 700])
@pytest.mark.parametrize("norm_type", ["layer_norm", "batch_norm", "none"])
def test_layout_equals_the_mlp_with_d_inputs(D, norm_type):
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_MLP, NET_MLP_BITS
    A = 3
    for H in WIDTHS:
        for L in range(1, 9):
            bits = _spec(NET_MLP_BITS, D, A, H, L, norm_type)
            mlp = _spec(NET_MLP, D, A, H, L, norm_type)
            for name, _ in bits.layout._fields_:
                assert getattr(bits.layout, name) == getattr(mlp.layout, name), (H, L, name)
            assert bits.entries == mlp.entries
            assert bits.stats_total == mlp.stats_total and bits.stats_entries() == mlp.stats_entries()
            want = RN.mlp_param_shapes(D, A, H, L, norm_type)
            assert {"/".join(p): tuple(s) for p, _, s, _ in bits.entries} == {k: tuple(v) for k, v in want.items()}
            assert bits.flat_names()[2] == "Dense_0,kernel"
            assert dict((",".join(p), s) for p, _, s, _ in bits.entries)["Dense_0,kernel"] == (D, H)
            for layer in range(L):
                ob, om = (ctypes.c_int64 * 4)(), (ctypes.c_int64 * 4)()
                _lib.check(_lib.lib().pqn_net_dense_layer(bits.desc, layer, ob))
                _lib.check(_lib.lib().pqn_net_dense_layer(mlp.desc, layer, om))
                assert tuple(ob) == tuple(om)
            assert _lib.lib().pqn_net_workspace_bytes(bits.desc, 2, 1000) > 0


@pytest.mark.parametrize("D", [4, 100, 399, 401, 500, 800, 1024])
def test_other_input_sizes_are_refused(D):
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_MLP_BITS
    with pytest.raises(_lib.PqnError) as e:
        _spec(NET_MLP_BITS, D, 3, 256, 2)
    assert "400, 600 or 700" in str(e.value)


@pytest.mark.parametrize("H,L,A,limit", [(96, 2, 3, "64, 128, 256 or 512"), (256, 9, 3, "1 to 8"),
                                         (512, 2, 10, "limit 227 KB")])
def test_mlp_limits_apply(H, L, A, limit):
    from purejaxql_b200 import _lib
    from purejaxql_b200.networks import NET_MLP_BITS
    with pytest.raises(_lib.PqnError) as e:
        _spec(NET_MLP_BITS, 400, A, H, L)
    assert limit in str(e.value)


@pytest.mark.parametrize("game", sorted(GAMES))
def test_pqn_gymnax_builds_the_packed_bits_mlp(game):
    from purejaxql_b200 import config_loader, envs
    from purejaxql_b200.engine import network_spec
    from purejaxql_b200.networks import NET_MLP_BITS
    c = config_loader.compose(["+alg=pqn_cartpole", f"alg.ENV_NAME={game}", "NUM_SEEDS=1", "SAVE_PATH=null"])
    c = {**c, **c["alg"]}
    env, _ = envs.make(game, flatten_obs=True)
    spec, row_words, dtype = network_spec(env, "mlp", c)
    D, A = GAMES[game]
    assert (spec.kind, spec.in_c, spec.num_actions, spec.hidden, spec.layers) == (NET_MLP_BITS, D, A, 256, 2)
    assert row_words == env.packed_obs_words == ((D + 31) // 32 + 3) // 4 * 4
    assert str(dtype) == "torch.int32"
    assert env.observation_space().shape == (D,)


def test_recurrent_script_still_refuses_minatar():
    from purejaxql_b200 import config_loader, pqn_rnn_gymnax
    c = config_loader.compose(["+alg=pqn_rnn_cartpole", "alg.ENV_NAME=Breakout-MinAtar", "NUM_SEEDS=1", "SAVE_PATH=null"])
    with pytest.raises(NotImplementedError, match="float-observation"):
        pqn_rnn_gymnax.make_train({**c, **c["alg"]})
