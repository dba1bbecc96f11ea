"""The availability-mask walk of k_rot_ring (liliom_b200/csrc/extract_rot.cu, segments up to 1024 points) against the sequential
greedy walk it replaces (R/src/Preprocessing.cpp:401-500), both restated in Python for ONE ring (tests/rot_restate.py):

  * `walk_sequential` follows the reference loop line by line (it is also what oracle/oracle_rot.cpp does) and is pinned here
    against the oracle's labels on the synthetic HDL-64E sweep;
  * `walk_masks` follows the kernel's fast path: counting ranks instead of a sort, static candidate classes, one break flag per
    consecutive pair -> per-point suppression extents, availability masks in rank space, "next candidate" = highest / lowest set
    bit, a pick clears the bits of itself and of the neighbours it marks, marks beyond the segment's end carried to the next one.

The GPU tier proves the kernel bit-exact on sweeps; this tier proves the reformulation itself on adversarial rings the sweeps do not
contain: heavy curvature ties, values on the 0.1 / 2.0 thresholds, dense runs of sharp points (the eleventh-candidate break),
points within 0.5 m, gaps right at 0.05 m^2, picks next to segment boundaries."""
import numpy as np
import pytest

from rot_restate import F, walk_masks, walk_sequential


def _random_ring(rng, n):
    """A ring of n points: a polyline with mostly small steps, a few jumps around the 0.05 m^2 break, some points near the sensor;
    curvature drawn from a few discrete levels (ties) around both thresholds plus dense sharp runs."""
    steps = rng.choice([0.05, 0.1, 0.2, 0.2236, 0.2237, 0.23, 0.5], size=n, p=[0.25, 0.3, 0.2, 0.07, 0.06, 0.07, 0.05])
    ang = rng.uniform(0, 2 * np.pi, n) * 0.02
    x = 3.0 + np.cumsum(steps * np.cos(ang)); y = np.cumsum(steps * np.sin(ang)); z = rng.normal(0, 0.005, n)
    P = np.stack([x, y, z], 1).astype(F)
    near = rng.random(n) < 0.03
    P[near] = (rng.normal(0, 0.15, (near.sum(), 3))).astype(F)       # inside the 0.5 m ball: skipped by the flat walk and the flags
    levels = np.array([0.0, 0.01, 0.05, 0.0999, 0.1, 0.1001, 0.5, 1.9999, 2.0, 2.0001, 3.0, 3.0, 7.5, 40.0], F)
    curv = rng.choice(levels, size=n).astype(F)
    for _ in range(rng.integers(0, 4)):                               # dense sharp runs: the eleventh candidate must end the walk
        a = rng.integers(0, max(n - 40, 1)); curv[a:a + rng.integers(10, 40)] = F(rng.choice([2.5, 3.0, 9.0]))
    return P, curv


@pytest.mark.parametrize("seed", range(12))
def test_mask_walk_equals_sequential_walk_on_adversarial_rings(seed):
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.choice([24, 40, 97, 300, 777, 1500]))
    P, curv = _random_ring(rng, n)
    a = walk_sequential(P, curv, 0, n)
    b = walk_masks(P, curv, 0, n)
    assert np.array_equal(a[0], b[0])
    assert np.array_equal(a[1], b[1])
    assert a[2] == b[2]
    assert (a[0] != 0).sum() > 0 or n < 30


def test_sequential_restatement_matches_the_oracle_on_the_hdl_sweep():
    """Pins `walk_sequential` (and with it the equivalence above) to oracle/oracle_rot.cpp: same labels on every processed ring."""
    import oracle_lib as O
    from liliom_b200 import synth
    O.build()
    hdl, q = synth.make_hdl64_sweep(synth.default_true_pose())
    rc, surf, edge, cut, lab, cur = O.extract_rot(hdl, q, (1.0, 0, 0, 0), 64, 4)
    assert rc == 0
    ring = cut["intensity"].astype(np.int32)                           # intensity = scanID + 0.1 * relTime
    P = np.stack([cut["x"], cut["y"], cut["z"]], 1).astype(F)
    want = lab
    got = np.zeros(len(cut), np.int32)
    got_m = np.zeros(len(cut), np.int32)
    for r in range(0, 64, 4):
        idx = np.nonzero(ring == r)[0]
        if len(idx) == 0:
            continue
        rf, re = int(idx[0]), int(idx[-1]) + 1
        assert np.all(np.diff(idx) == 1)                               # ring-major cloud
        l, _, _ = walk_sequential(P, cur, rf, re)
        got[rf:re] = l[rf:re]
        l, _, _ = walk_masks(P, cur, rf, re)
        got_m[rf:re] = l[rf:re]
    assert np.array_equal(got, want)
    assert np.array_equal(got_m, want)
    assert (want == 2).sum() > 20 and (want == -1).sum() > 50
