"""CPU tier of the ROT extractor's adversarial sweeps (tests/rot_adversarial.py): every named case is hit, read from the oracle's
outputs; oracle/oracle_rot.cpp equals the Python restatement (tests/rot_restate.py: ring, latch, relTime and intensity through
glibc; curvature; the sequential walk's labels and edge picks; the per-ring VoxelGrid) on every sweep; and the kernel's mask walk
equals the sequential walk on every processed ring of every sweep."""
import math

import numpy as np
import pytest

import rot_adversarial as A
import rot_oracle
import rot_restate as RS

F = np.float32


@pytest.fixture(scope="module")
def sweeps():
    return dict(A.all_sweeps())


@pytest.fixture(scope="module")
def outs(sweeps):
    return {nm: rot_oracle.extract_rot(s["pts"], s["q_imu"], s["q_lb"], s["line_num"], s["ds_rate"]) for nm, s in sweeps.items()}


@pytest.fixture(scope="module")
def assigned(sweeps):
    return {nm: RS.assign(s["pts"], s["line_num"]) for nm, s in sweeps.items()}


def _bits_equal_nan(a, b):
    a, b = np.asarray(a, F), np.asarray(b, F)
    return len(a) == len(b) and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


NAMES = [nm for nm, _ in A.all_sweeps()]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_equals_restatement(name, sweeps, outs, assigned):
    s, (rc, surf, edge, cut, lab, cur), a = sweeps[name], outs[name], assigned[name]
    assert rc == 0
    assert len(cut) == len(a["order"])
    assert cut["intensity"].tobytes() == a["intensity"].tobytes(), name
    if A.identity_q(s):       # identity de-skew: laserCloud is the input, bucketed by ring
        for f in ("x", "y", "z"):
            assert cut[f].tobytes() == s["pts"][f][a["order"]].tobytes(), (name, f)
    curv, label, edge_r, surf_r, _ = RS.restate_cloud(cut, a["ring"], s["line_num"], s["ds_rate"])
    assert _bits_equal_nan(curv, cur), name
    assert np.array_equal(label, lab), (name, np.nonzero(label != lab)[0][:10])
    assert edge_r.tobytes() == edge.tobytes(), name
    assert surf_r.tobytes() == surf.tobytes(), name


@pytest.mark.parametrize("name", NAMES)
def test_mask_walk_equals_sequential_walk(name, sweeps, outs, assigned):
    s, (_, _, _, cut, _, cur), a = sweeps[name], outs[name], assigned[name]
    P = np.stack([cut["x"], cut["y"], cut["z"]], 1).astype(F)
    rf, re = RS.ring_bounds(a["ring"], s["line_num"])
    n = 0
    for r in range(0, s["line_num"], s["ds_rate"]):
        if re[r] - rf[r] - 11 < 6:
            continue
        x = RS.walk_sequential(P, cur, int(rf[r]), int(re[r]))
        y = RS.walk_masks(P, cur, int(rf[r]), int(re[r]))
        assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) and x[2] == y[2], (name, r)
        n += 1
    assert n > 0 or name in ("single", "dropped")


def _ring_of_rows(a, rows):
    pos = {int(i): k for k, i in enumerate(a["order"])}
    return [a["ring"][pos[int(i)]] if int(i) in pos else -1 for i in rows]


def test_cases_are_hit(sweeps, outs, assigned):
    S, O, AS = sweeps, outs, assigned
    # tables: every verdict pair of a bin edge differs and its rows land in those rings (or are dropped)
    for ln in (16, 32, 64):
        nm = f"tables{ln}_ds1"
        edges = [c for c in S[nm]["cases"] if c.startswith("edge_")]
        assert len(edges) >= {16: 17, 32: 32, 64: 52}[ln], (ln, len(edges))
        for c in edges:
            vl, vh = map(int, c.split("_")[1:3])
            assert vl != vh
            rows = S[nm]["cases"][c]["rows"]
            got = _ring_of_rows(AS[nm], rows)
            assert sorted(got) == sorted([vl, vh]), (nm, c, got)
        if ln == 64:
            vs = {tuple(sorted(map(int, c.split("_")[1:3]))) for c in edges}
            assert (-1, 0) in vs and (-1, 50) in vs and (31, 32) in vs or (32, 32) in vs
        # r^2 around 9.0f: below removed, at and above kept; non-finite removed; an overflowing r^2 kept with curvature inf
        kept = set(AS[nm]["kept"])
        assert int(S[nm]["cases"]["r2_below9"]["rows"][0]) not in kept
        assert int(S[nm]["cases"]["r2_at9"]["rows"][0]) in kept and int(S[nm]["cases"]["r2_above9"]["rows"][0]) in kept
        assert not kept & set(S[nm]["cases"]["nonfinite_xyz"]["rows"].tolist())
        assert _ring_of_rows(AS[nm], S[nm]["cases"]["r2_overflow"]["rows"])[0] >= 0
        assert np.isinf(O[nm][5]).any()
        rf, re = RS.ring_bounds(AS[nm]["ring"], ln)
        extra = np.bincount(np.array([g for c in edges for g in _ring_of_rows(AS[nm], S[nm]["cases"][c]["rows"]) if g >= 0]), minlength=ln)
        assert re[2] - rf[2] == extra[2] and re[3] - rf[3] == 17 + extra[3] and re[4] - rf[4] == 16 + extra[4]   # rings of 0, 17, 16
    # azimuth: both endOri corrections, the latch at the first kept return, at the last and never, relTime outside [0, 1]
    assert AS["az_end_sub"]["start_branch"] == "sub" and AS["az_end_add"]["start_branch"] == "add"
    assert AS["tables16_ds1"]["start_branch"] is None
    assert AS["az_latch_never"]["latch"] is None
    lf = AS["az_latch_first"]
    assert lf["latch"] == int(S["az_latch_first"]["cases"]["latch_row"]["rows"][0]) and lf["kept"][0] == 0
    assert 0 not in lf["order"]                              # the table-dropped first return opened the sweep, never latched
    assert AS["az_latch_last"]["latch"] == AS["az_latch_last"]["kept"][-1]
    rel = AS["az_reltime_out"]["rel"]
    assert (rel < 0).any() and (rel > 1).any()
    ring0 = AS["az_reltime_out"]["ring"] == 0
    assert (AS["az_reltime_out"]["intensity"][ring0] < 0).any()
    lr = AS["latch_ring0"]
    row = int(S["latch_ring0"]["cases"]["latch_row"]["rows"][0])
    assert lr["latch"] == row and _ring_of_rows(lr, [row])[0] == 0
    # the latched branch's +2 pi round trip would change this return's azimuth and so its intensity
    p = S["latch_ring0"]["pts"][row]
    o = F(-RS.libm().atan2f(p["y"], p["x"]))
    assert F(float(F(float(o) + 2 * math.pi)) - 2 * math.pi) != o
    # curvature thresholds on the exact wall
    s, a, cur, lab = S["curv16"], AS["curv16"], O["curv16"][5], O["curv16"][4]
    pos = {int(i): k for k, i in enumerate(a["order"])}
    cv = lambda c: np.array([cur[pos[int(i)]] for i in s["cases"][c]["rows"]], F)
    lb = lambda c: np.array([lab[pos[int(i)]] for i in s["cases"][c]["rows"]])
    assert (cv("curv_eq2") == F(2.0)).all() and (lb("curv_eq2") == 0).all()
    assert cv("curv_2_up")[0] == np.nextafter(F(2), F(3)) and cv("curv_2_down")[0] == np.nextafter(F(2), F(0))
    assert cv("curv_01_up")[0] == np.nextafter(F(0.1), F(1)) and cv("curv_01_at")[0] == F(0.1)
    assert cv("curv_01_down")[0] == np.nextafter(F(0.1), F(0))
    wall = np.array([pos[int(i)] for i in s["cases"]["wall"]["rows"]])
    assert (cur[wall] == 0).sum() > 300                                  # zero-curvature runs
    assert (lb("gap_at") > 0).all() and (lb("gap_below") > 0).all()
    # the pick whose gaps are 0.05f marks no neighbour, so a sharp candidate after it is picked; the one a float below marks them all
    k = pos[int(s["cases"]["gap_at"]["rows"][0])]
    assert (cur[k + 1:k + 6] > 2.0).all() and (lab[k + 1:k + 6] > 0).any()
    k = pos[int(s["cases"]["gap_below"]["rows"][0])]
    assert (cur[k + 1:k + 6] > 2.0).all() and (lab[k + 1:k + 6] == 0).all()
    # more than 10 sharp candidates in one segment: the eleventh stays unlabelled
    picks = RS.restate_cloud(O["curv16"][3], a["ring"], 16, 1)[4]
    assert any(len(e) == 10 for e in picks[8])
    rf, re = RS.ring_bounds(a["ring"], 16)
    full = [(sp, ep) for sp, ep in RS.segments(int(rf[8]), int(re[8]))]
    assert any(((cur[sp:ep + 1] > 2.0) & (lab[sp:ep + 1] == 0)).any() for sp, ep in full)
    # shapes
    for nm, r, n in (("shapes64", 1, 1), ("shapes64", 2, 11), ("shapes64", 5, 12), ("shapes64", 9, 0), ("shapes64", 20, 6158),
                     ("ring16384", 8, 16384)):
        rf, re = RS.ring_bounds(AS[nm]["ring"], S[nm]["line_num"])
        assert re[r] - rf[r] == n, (nm, r)
    rf, re = RS.ring_bounds(AS["shapes64"]["ring"], 64)
    lens = [ep - sp + 1 for sp, ep in RS.segments(int(rf[20]), int(re[20]))]
    assert sorted(set(lens)) == [1024, 1025]
    assert len(O["dropped"][3]) == 0 and len(O["single"][3]) == 1
    # VoxelGrid: the overflow ring passes through in ring order, the ring just short of it is filtered (reversed: index order)
    for nm, through in (("vg_overflow", True), ("vg_short", False)):
        a = AS[nm]
        cut = O[nm][3]
        rf, re = RS.ring_bounds(a["ring"], 64)
        _, lf, _ = RS.walk_sequential(np.stack([cut["x"], cut["y"], cut["z"]], 1).astype(F), O[nm][5], int(rf[6]), int(re[6]))
        rows = cut[np.nonzero(lf)[0]]
        out = RS.restate_cloud(cut, a["ring"], 64, 1)[3]
        ring_out = out[np.isin(out["x"], rows["x"]) & (np.abs(out["x"]) > 1000)]
        assert len(rows) >= 30 and len(ring_out) == len(rows)
        assert np.array_equal(ring_out["x"], rows["x"]) == through, nm
    # the far cluster: PCL's indices merge returns that differ only in x
    a, cut = AS["vg_far"], O["vg_far"][3]
    surf = O["vg_far"][1]
    far_in = cut[(cut["x"] > 1e9)]
    far_out = surf[surf["x"] > 1e9]
    assert len(np.unique(far_in["x"])) == 3 and len(far_out) < len(np.unique(far_in["y"])) * 2
    # non-finite curvature: NaN in curv_nan, +inf in curv_inf
    assert np.isnan(O["curv_nan"][5]).sum() >= 1 and np.isposinf(O["curv_inf"][5]).sum() >= 1
    # full edge table: every segment of every ring picks 10
    assert len(O["edge_table"][2]) == 51 * 6 * 10
