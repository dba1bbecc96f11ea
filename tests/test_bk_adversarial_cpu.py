"""CPU tier of the backend's adversarial keyframe maps (tests/bk_adversarial.py): the oracle's 5-NN sets are the exhaustive
reference's at every gate, and every named case lands on the side of its threshold it was built for, at each variant."""
import numpy as np
import pytest

import bk_adversarial as BK
import knn_reference as KR


def _sel(oracle, q, pose):
    """the fp32 map-frame queries of the searches"""
    w = oracle.transform_cloud(q, pose)
    return np.stack([w["x"], w["y"], w["z"], np.ones(len(w), np.float32)], 1)


@pytest.mark.parametrize("world", BK.WORLDS)
def test_oracle_knn5_equals_exhaustive_reference_at_each_gate(oracle, world):
    W = BK.backend_world(world)
    for kind, m4, q, gates in (("edge", W["edge_map"], W["edge_q"], (1.0,)), ("surf", BK.f4(W["surf_map"]), W["surf_q"], BK.KD_RADII)):
        sel = _sel(oracle, q, W["pose"])
        idx, sqd = oracle.KdTree(m4).knn5(sel)
        okeys = (sqd.view(np.uint32).astype(np.uint64) << np.uint64(32)) | idx.astype(np.uint32).astype(np.uint64)
        for kd in gates:
            tau0 = KR.gate_tau(kd)
            _, _, rkeys = KR.reference_knn5(sel, m4, tau0)
            for i in range(len(sel)):
                inside = sqd[i] <= tau0
                k = int(inside.sum())
                assert inside[:k].all(), (kind, kd, i)             # ascending: the gate cuts a prefix
                assert (okeys[i, :k] == rkeys[i, :k]).all(), (kind, kd, i, okeys[i], rkeys[i])
                assert (rkeys[i, k:] == np.uint64(0xFFFFFFFFFFFFFFFF)).all(), (kind, kd, i)


# (case, variant, gate) -> the decisions the case must contain; None = both accepted and rejected
EDGE_EXPECT = {
    "gate_tau0": {1}, "gate_one": {0}, "gate_tau0_one": {1}, "gate_tie": {1}, "gate_three": {0}, "gate_below": {1},
    "duplicates": {0}, "collinear_axis": {1}, "ratio3_sweep": None, "symmetric": None,
}


@pytest.mark.parametrize("world", BK.WORLDS)
def test_every_case_hits_its_boundary_in_the_oracle(oracle, world):
    W = BK.backend_world(world)
    te = oracle.KdTree(W["edge_map"])
    for variant in (0, 1):
        v, pa, pb = oracle.correspond_edge(te, W["edge_q"], W["pose"], variant)
        for name, want in EDGE_EXPECT.items():
            got = set(v[W["edge_notes"][name]].tolist())
            assert got == (want if want is not None else {0, 1}), (world, variant, name, got)
        d = set(v[W["edge_notes"]["var1_dist"]].tolist())
        assert d == ({0, 1} if variant == 1 else {1}), (world, variant, d)
        # the exactly collinear query on its line: accepted with line ends on the line's axis
        ix = W["edge_notes"]["collinear_axis"]
        assert (v[ix] == 1).all() and ((pa[ix] == pb[ix]).sum(1) == 2).all()
    assert set(v[W["edge_notes"]["ratio3"]].tolist()) <= {0, 1}
    ts = oracle.KdTree(BK.f4(W["surf_map"]))
    n = W["surf_notes"]
    for variant in (0, 1):
        out = {}
        for kd in BK.KD_RADII:
            extra = dict(map_refl=W["surf_map"]["curvature"], feat_refl=W["surf_q"]["curvature"], reflect_thres=BK.REFLECT_THRES) \
                if variant == 0 else {}
            v, _, sc = oracle.correspond_surf_backend(ts, W["surf_q"], W["pose"], kd, BK.SURF_DIST_THRES, BK.W_GATE[variant],
                                                      BK.LIDAR_CONST[variant], **extra)
            out[kd] = v

            def got(name, v=v):
                return set(v[n[name]].tolist())
            assert got(f"gate_tau0_{kd}") == {1} and got(f"gate_above_{kd}") == {0}, (world, variant, kd)
        assert set(out[1.0][n["gate_above_0.49"]].tolist()) == {1}       # inside the default gate
        v = out[1.0]
        assert set(v[n[f"plane_thres_v{variant}"]].tolist()) == {0, 1}, (world, variant)
        assert set(v[n["coplanar_axis"]].tolist()) == {1} and set(v[n["collinear"]].tolist()) == {1}
        assert set(v[n["origin_plane"]].tolist()) == {0}
        if world == "near":
            ix = n["w_gate"][:2] if variant == 1 else n["w_gate"][2:]
            assert v[ix].tolist() == [1, 0], (variant, v[ix])
        if variant == 0:
            for name, want in (("refl_sum_eq", {1}), ("refl_sum_below", {1}), ("refl_sum_above", {0}), ("refl_tie_one", {0}),
                               ("refl_tie_all", {0}), ("refl_nan_query", {0}), ("refl_nan_map", {0})):
                assert set(v[n[name]].tolist()) == want, (world, name)
        else:
            for name in ("refl_sum_above", "refl_tie_all", "refl_nan_query"):        # the same planes, no reflectivity gate
                assert set(v[n[name]].tolist()) == {1}, (world, name)
