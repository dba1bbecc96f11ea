"""The adversarial scan-to-map worlds (tests/s2m_adversarial.py) checked on the CPU: each case's 5-NN set from the oracle's kd-tree
is the set built for it, each gate pair straddles its gate under the oracle, and the host build of dev_math.cuh::plane_fit_gate
decides every case as the oracle does, with the oracle's plane bits on every case it sends to the exact path (every degenerate set
and the gate cases the guard band catches)."""
import numpy as np
import pytest

import s2m_adversarial as S
from test_devmath_host import dm, fit_gate_device  # noqa: F401


def _corr(oracle, W):
    tree = oracle.KdTree(W["map"])
    cnt, valid, plane, idx, pw = oracle.find_surf_corr(tree, W["feats"], W["pose"])
    return tree, valid, plane, idx, pw


@pytest.mark.parametrize("world", S.WORLDS)
def test_world_sets_and_straddles(oracle, world):
    W = S.s2m_world(world)
    _, valid, _, idx, _ = _corr(oracle, W)
    for i, want in enumerate(W["sets"]):
        assert np.array_equal(np.sort(idx[i]), want), (world, i)
    N = W["notes"]
    for keep, refuse in (("plane_keep", "plane_refuse"), ("w_keep", "w_refuse")):
        if keep in N:
            assert valid[N[keep]].all() and not valid[N[refuse]].any(), keep
    if "origin_query" in N:
        assert not valid[N["origin_query"]].any()       # rng = 0: the weight is -inf
    assert valid[N["noisy_plane"]].any()


@pytest.mark.parametrize("world", S.WORLDS)
def test_plane_fit_gate_host_build_on_world(dm, oracle, world):  # noqa: F811
    W = S.s2m_world(world)
    _, valid, plane, idx, pw = _corr(oracle, W)
    m = W["map"][idx]
    ok, path, pl, _, _, _, _ = fit_gate_device(dm, m, pw[:, :3], 0.06, 0.4)
    assert np.array_equal(ok, valid)
    ex = np.concatenate([W["notes"][k] for k in S.EXACT if k in W["notes"]])
    assert (path[ex] == 1).all()                                 # the fast fit declines every degenerate set
    ex = path != 0
    assert pl[ex].tobytes() == plane[ex].tobytes()
    gate = np.concatenate([W["notes"][k] for k in ("plane_keep", "plane_refuse", "w_keep", "w_refuse") if k in W["notes"]])
    assert (path[gate] == 2).any()                               # and the guard band fires on gate cases
