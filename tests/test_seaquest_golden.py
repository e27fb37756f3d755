"""Replays Seaquest trajectories recorded from MinAtar itself (and from gymnax, should a version register the game) by
tests/golden/make_seaquest_golden_from_ref.py; skipped until such files exist."""
import glob
import json
import os

import numpy as np
import pytest

import seaquest_oracle as SQ
from oracle import jax_prng as jr

HERE = os.path.dirname(os.path.abspath(__file__))
_MINATAR = os.path.join(HERE, "golden", "seaquest_minatar_ref.json")
_GYMNAX = sorted(glob.glob(os.path.join(HERE, "golden", "seaquest_gymnax_*_ref.npz")))


@pytest.mark.skipif(not os.path.exists(_MINATAR), reason="no Seaquest records from MinAtar yet "
                                                         "(tests/golden/make_seaquest_golden_from_ref.py)")
def test_oracle_step_matches_minatar():
    """every recorded MinAtar step, teacher-forced: the oracle's step from MinAtar's state, with MinAtar's draws,
    gives MinAtar's reward, terminal flag, next state and observation"""
    recs = json.load(open(_MINATAR))["records"]
    for t, rec in enumerate(recs):
        e = {k: (list(map(list, v)) if isinstance(v, list) else v) for k, v in rec["before"].items()}
        e["time"] = 0
        draws = [0 if d is None else int(d) for d in rec["draws"]]
        # MinAtar's choice([True, False]) / choice([True, False], p) return the value; the oracle takes lr and is_sub
        # as 0/1 and the rows as drawn
        r, term = SQ.Seaquest.act(e, rec["action"], *draws)
        assert (r, term) == (rec["reward"], rec["terminal"]), t
        after = dict(rec["after"])
        for k in SQ.SCALARS + SQ.FLAGS:
            if k in after and k != "terminal":
                assert e[k] == after[k], (t, k)
        for k in SQ.CAPS:
            assert [list(map(int, z)) for z in e[k]] == after[k], (t, k)
        if not term:
            e["time"] = 1
            o = SQ.Seaquest().get_obs(SQ._pack([e]))[0]
            assert sorted(map(tuple, np.argwhere(o > 0).tolist())) == sorted(map(tuple, rec["obs"])), t


@pytest.mark.skipif(not _GYMNAX, reason="no gymnax registers Seaquest-MinAtar yet")
@pytest.mark.parametrize("path", _GYMNAX or ["none"])
def test_oracle_matches_gymnax(path):
    g = dict(np.load(path))
    jr.DEFAULT_PARTITIONABLE = "partitionable" in os.path.basename(path)
    try:
        env = SQ.make(flatten=True)
        o_obs, o_st = env.reset(g["reset_keys"])
        assert np.array_equal(o_obs, g["obs0"])
        for t in range(g["action"].shape[0]):
            o_obs, o_st, o_r, o_d, _ = env.step(g["step_keys"][t], o_st, g["action"][t].astype(np.int32))
            assert np.array_equal(o_d, g["done"][t]) and np.array_equal(o_r, g["reward"][t].astype(np.float32)), t
            assert np.array_equal(o_obs, g["obs"][t]), t
    finally:
        jr.DEFAULT_PARTITIONABLE = False
