"""The local map fed from the device (liliom_map_update_resident) and updated for many sessions in one call
(liliom_map_update_batch), against the existing calls, bit for bit.

Twin context sets get the same parameters and sweeps.  Set A runs the existing path (liliom_odometry_resident with ds_out, then
liliom_map_update of the downloaded cloud, or solo liliom_map_update_resident calls where the batch is under test), set B the new
one.  After every scan, per session: status, map size, the search index (liliom_map_download), the filtered cloud
(liliom_map_download_cloud), the pose, stats and DS bytes of the step, and (batch against solo) the launch counters."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ITERS = 4
IDENT = np.array([1.0, 0, 0, 0, 0, 0, 0])
ENVS = ("LILIOM_TEST_SHRINK_BOX", "LILIOM_HZ_CHAIN")


@pytest.fixture(scope="module")
def world():
    """Five Horizon sweeps and three 64-line sweeps along a short path, each with its true pose and a perturbed guess."""
    from liliom_b200 import synth
    T0 = synth.default_true_pose()
    hz, rot = [], []
    for k in range(5):
        T = np.array(T0); T[4] += 0.6 * k; T[5] += 0.12 * k
        pts, q = synth.make_horizon_sweep(T, seed=1 + k, dropout=0.02 + 0.05 * k)      # different sweep sizes
        hz.append(dict(T=T, guess=synth.perturbed_pose(T), pts=pts, q=q))
    for k in range(3):
        T = np.array(T0); T[4] += 0.5 * k; T[5] -= 0.1 * k
        pts, q = synth.make_hdl64_sweep(T, seed=2 + k, steps=1200 + 300 * k)
        rot.append(dict(T=T, guess=synth.perturbed_pose(T), pts=pts, q=q))
    return {0: hz, 1: rot}


def _ctx(variant, max_map_frames=None, env=()):
    import liliom_b200 as L
    p = L.default_params(variant)
    if max_map_frames is not None:
        p.max_map_frames = max_map_frames
    old = {k: os.environ.get(k) for k in ENVS}
    for k in old:
        os.environ.pop(k, None)
    os.environ.update(dict(env))                           # read at liliom_create
    try:
        return L.Context(p)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


class Spec:
    """One session: its layout, its FIFO length, its environment, and where in the sweep list it starts."""

    def __init__(self, variant=0, frames=None, env=(), start=0):
        self.variant, self.frames, self.env, self.start = variant, frames, env, start

    def make(self):
        return _ctx(self.variant, self.frames, self.env)

    def sweep(self, world, k):
        sws = world[self.variant]
        return sws[(self.start + k) % len(sws)]


def _odo(c, guess, mode=None):
    """liliom_odometry_resident with ds_out, whatever it returns: (rc, pose bytes, stats bytes, DS cloud)."""
    import liliom_b200 as L
    lib = L._binding.lib()
    mode = L.MODE_GN if mode is None else mode
    pose = np.array(guess, dtype=np.float64)
    st = (L._binding.IterStats * ITERS)()
    ds = np.zeros(65536, c.dtype)
    nds = C.c_int()
    rc = lib.liliom_odometry_resident(c._h, pose.ctypes.data_as(C.POINTER(C.c_double)), ITERS, 15, mode, st, ds.ctypes.data_as(C.c_void_p),
                                      len(ds), C.byref(nds))
    return rc, pose, bytes(memoryview(st)) if rc == 0 else b"", ds[:nds.value].copy()


def _scan(c, sw):
    c.upload_scan(sw["pts"])
    c.extract_resident(sw["q"])


def _map_state(c):
    import liliom_b200 as L
    try:
        cloud = c.map_download_cloud().tobytes()
    except L.LiliomError as e:
        cloud = e.code
    return c.map_size(), c.map_download().tobytes(), cloud


def _last_error(c):
    import liliom_b200 as L
    return L._binding.lib().liliom_last_error(c._h).decode()


def _counters(c):
    k = c.counters()
    return (k.launches, k.lib_launches)


def _try(f):
    import liliom_b200 as L
    try:
        return 0, f()
    except L.LiliomError as e:
        return e.code, 0


def _same_step(a, b, what):
    assert a[0] == b[0], (what, "status", a[0], b[0])
    assert a[1].tobytes() == b[1].tobytes(), (what, "pose")
    assert a[2] == b[2], (what, "stats")
    assert len(a[3]) == len(b[3]) and a[3].tobytes() == b[3].tobytes(), (what, "DS")


def _same_map(a, b, what):
    sa, sb = _map_state(a), _map_state(b)
    assert sa[0] == sb[0], (what, "map size", sa[0], sb[0])
    assert sa[1] == sb[1], (what, "search index")
    assert sa[2] == sb[2], (what, "filtered cloud")


def _close(*sets):
    for s in sets:
        for c in s:
            c.close()


def _pose_for(step, sw):
    """The pose a frame is saved with: the solved pose of a step that ran, the sweep's true pose otherwise (no map yet)."""
    return step[1] if step[0] == 0 and np.all(np.isfinite(step[1])) else sw["T"]


# ---------------------------------------------------------------- resident equals host
@pytest.mark.parametrize("variant", [0, 1])
def test_resident_update_equals_update_through_the_host(world, variant):
    """26 scans (the 20-frame FIFO fills and pops): odometry_resident with ds_out + liliom_map_update(ds_out) against
    liliom_map_update_resident."""
    spec = Spec(variant)
    a, b = spec.make(), spec.make()
    for k in range(26):
        sw = spec.sweep(world, k)
        _scan(a, sw); _scan(b, sw)
        ra, rb = _odo(a, sw["guess"]), _odo(b, sw["guess"])
        _same_step(ra, rb, (variant, k))
        assert ra[0] == (-8 if k == 0 else 0), (k, ra[0])           # LILIOM_E_NOMAP on the first scan: the frame is still resident
        pose = _pose_for(ra, sw)
        ma = a.map_update(ra[3], pose)
        mb = b.map_update_resident(pose)
        assert ma == mb and ma > 0, (k, ma, mb)
        _same_map(a, b, (variant, k))
    mb = b.map_update_resident(pose)                                 # the update only reads the scan: it can be pushed again
    assert mb == a.map_update(ra[3], pose)
    _same_map(a, b, (variant, "pushed twice"))
    _close([a, b])


# ---------------------------------------------------------------- batch equals solo
def _prefill(world, specs, sets, counts):
    """counts[i] solo steps on session i of every set: different FIFO fill levels at the first batched call."""
    for i, s in enumerate(specs):
        for k in range(counts[i]):
            sw = s.sweep(world, 100 + k)
            for cs in sets:
                _scan(cs[i], sw)
                r = _odo(cs[i], sw["guess"])
                cs[i].map_update_resident(_pose_for(r, sw))


def _batched_steps(world, specs, A_, B_, steps, what):
    """Per step: scan + odometry solo on both sets, then solo liliom_map_update_resident on A and ONE liliom_map_update_batch on B."""
    import liliom_b200 as L
    for k in range(steps):
        poses = []
        for i, s in enumerate(specs):
            sw = s.sweep(world, k)
            _scan(A_[i], sw); _scan(B_[i], sw)
            ra, rb = _odo(A_[i], sw["guess"]), _odo(B_[i], sw["guess"])
            _same_step(ra, rb, (what, k, i))
            poses.append(_pose_for(ra, sw))
        solo = [_try(lambda: A_[i].map_update_resident(poses[i])) for i in range(len(specs))]
        n_map, status = L.map_update_batch(B_, poses)
        for i in range(len(specs)):
            assert (int(status[i]), int(n_map[i])) == solo[i], (what, k, i, solo[i], status[i], n_map[i])
            _same_map(A_[i], B_[i], (what, k, i))
            assert _counters(A_[i]) == _counters(B_[i]), (what, k, i, _counters(A_[i]), _counters(B_[i]))


def _solo_after(world, specs, A_, B_, what):
    """One more solo step on both sets: the batch left every context (FIFO, entry array, index) in the solo state."""
    for i, s in enumerate(specs):
        sw = s.sweep(world, 50)
        _scan(A_[i], sw); _scan(B_[i], sw)
        ra, rb = _odo(A_[i], sw["guess"]), _odo(B_[i], sw["guess"])
        _same_step(ra, rb, (what, "solo after", i))
        pose = _pose_for(ra, sw)
        assert _try(lambda: A_[i].map_update_resident(pose)) == _try(lambda: B_[i].map_update_resident(pose)), (what, i)
        _same_map(A_[i], B_[i], (what, "solo after", i))
        assert _counters(A_[i]) == _counters(B_[i]), (what, "solo after", i)


@pytest.mark.parametrize("B", [1, 2, 8, 32, 34])
def test_map_update_batch_matches_solo(world, B):
    """Horizon and 64-line sessions mixed, different sweeps, FIFO lengths 3 / 5 / 20 at different fill levels (so some sessions
    pop a frame in the call and others do not); 34 sessions take two launches per stage."""
    specs = [Spec(variant=1 if i % 3 == 2 else 0, frames=(3, 5, 20)[(i // 2) % 3], start=i) for i in range(B)]
    A_, B_ = [s.make() for s in specs], [s.make() for s in specs]
    _prefill(world, specs, (A_, B_), [(i * 2) % 5 + 1 for i in range(B)])
    _batched_steps(world, specs, A_, B_, 5, f"B={B}")
    _solo_after(world, specs, A_, B_, f"B={B}")
    _close(A_, B_)


# ---------------------------------------------------------------- every fall-back inside a batch
def _strip_step(c, surf, k, shifted):
    """A thin strip of surf features through liliom_odometry (host input), stretched past 2^20 voxels in x when `shifted`: the frame
    liliom_map_update_resident then takes has keys that do not fit 21 bits, while the 1 m cell grid still holds the extent."""
    f = surf.copy(); f["x"] += np.float32(0.37 * k)
    if shifted:
        f["x"][:5] += np.float32(600000.0)
    return _try(lambda: len(c.odometry(f, IDENT, 1)[2]))


def test_every_fallback_inside_a_batch(world):
    """Sessions that leave the shared path at each of its exits, each next to ordinary sessions, over six steps: the first update
    (0), an update after liliom_map_push_frame (1) and after liliom_map_clear (2), keys that do not fit 21 bits (3, its strip
    frames saved under the identity pose), an escaped cell-grid box (4, LILIOM_TEST_SHRINK_BOX), an empty resident cloud (5, at
    steps 1 and 4), a FIFO longer than the entry array's 64 slots (6); 7 and 8 are ordinary."""
    import liliom_b200 as L
    specs = [Spec(0, 5), Spec(0, 5, start=1), Spec(1, 5), Spec(0, 3), Spec(0, 5, env={"LILIOM_TEST_SHRINK_BOX": "1"}, start=2), Spec(0, 5, start=3),
             Spec(0, 70, start=4), Spec(1, 5, start=1), Spec(0, 20)]
    n = len(specs)
    A_, B_ = [s.make() for s in specs], [s.make() for s in specs]
    _prefill(world, specs, (A_, B_), [0, 2, 2, 0, 2, 2, 2, 2, 2])
    strip = None
    for k in range(6):
        poses = []
        for i, s in enumerate(specs):
            sw = s.sweep(world, k)
            for c in (A_[i], B_[i]):
                if i == 5 and k in (1, 4):
                    c.upload_scan(sw["pts"][:0])
                    c.extract_resident(sw["q"])
                else:
                    _scan(c, sw)
            if i == 3:
                if strip is None:
                    surf = A_[i].features_download()[0]
                    strip = surf[(np.abs(surf["y"]) < 3.0) & (np.abs(surf["z"]) < 3.0)][:2000].copy()
                    assert len(strip) > 100
                ra, rb = _strip_step(A_[i], strip, k, k == 2), _strip_step(B_[i], strip, k, k == 2)
                assert ra == rb, (k, ra, rb)
                poses.append(IDENT)
                continue
            ra, rb = _odo(A_[i], sw["guess"]), _odo(B_[i], sw["guess"])
            _same_step(ra, rb, ("fallbacks", k, i))
            if i == 5 and k in (1, 4):
                assert len(ra[3]) == 0
            poses.append(_pose_for(ra, sw))
            if i == 1 and k == 2:                           # a plain push between two updates: the entry array is rebuilt
                for c in (A_[i], B_[i]):
                    c.map_push_frame(ra[3], poses[-1])
            if i == 2 and k == 3:
                for c in (A_[i], B_[i]):
                    c.map_clear()
        before = [_counters(c) for c in A_]
        solo = [_try(lambda: A_[i].map_update_resident(poses[i])) for i in range(n)]
        spent = [tuple(x - y for x, y in zip(_counters(c), b)) for c, b in zip(A_, before)]    # (kernels, library calls) of each update
        # the steady-state update launches the same kernels whatever the sizes: sessions 7 and 8 pin that count, and a session
        # that left the shared path at this step must show another one
        assert spent[7] == spent[8], (k, spent)
        off = {0: [0], 1: [2], 2: [3], 3: [0, 2, 3, 4, 5], 4: range(6), 5: [1, 4], 6: range(6)}
        for i, steps in off.items():
            assert (spent[i] != spent[8]) == (k in steps), ("exit not taken as planned", k, i, spent[i], spent[8])
        n_map, status = L.map_update_batch(B_, poses)
        for i in range(n):
            assert (int(status[i]), int(n_map[i])) == solo[i], ("fallbacks", k, i, solo[i], status[i], n_map[i])
            assert solo[i][0] == 0, (k, i, solo[i])
            _same_map(A_[i], B_[i], ("fallbacks", k, i))
            assert _counters(A_[i]) == _counters(B_[i]), ("fallbacks", k, i, _counters(A_[i]), _counters(B_[i]))
    _solo_after(world, [s for i, s in enumerate(specs) if i != 3], [c for i, c in enumerate(A_) if i != 3],
                [c for i, c in enumerate(B_) if i != 3], "fallbacks")
    _close(A_, B_)


# ---------------------------------------------------------------- errors
def test_nothing_resident_is_that_sessions_error_only(world):
    """A fresh context, one whose buffer liliom_voxelgrid rewrote and one whose buffer liliom_kf_add rewrote have no scan to push:
    LILIOM_E_ARG with a text, solo and as their status in a batch, their maps untouched; the other sessions are updated.  Two
    sessions run on a caller's stream."""
    import liliom_b200 as L
    import torch
    specs = [Spec(0, 5), Spec(0, 5, start=1), Spec(0, 5, start=2), Spec(1, 5), Spec(0, 5, start=3), Spec(1, 5, start=1)]
    A_, B_ = [s.make() for s in specs], [s.make() for s in specs]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    B_[3].set_stream(streams[0].cuda_stream); B_[4].set_stream(streams[1].cuda_stream)
    _prefill(world, specs[1:], (A_[1:], B_[1:]), [2] * 5)
    poses = []
    for i, s in enumerate(specs):
        sw = s.sweep(world, 0)
        if i == 0:
            poses.append(sw["T"])
            continue
        for c in (A_[i], B_[i]):
            _scan(c, sw)
        ra, rb = _odo(A_[i], sw["guess"]), _odo(B_[i], sw["guess"])
        _same_step(ra, rb, ("errors", i))
        poses.append(_pose_for(ra, sw))
        if i == 1:
            for c in (A_[i], B_[i]):
                c.voxelgrid(ra[3], 0.8)
        if i == 2:
            surf, edge, _ = A_[i].features_download()
            for c in (A_[i], B_[i]):
                c.kf_add(L.backend_default_params(0), edge, surf, download=False)
    before = [_map_state(c) for c in B_]
    solo = [_try(lambda: A_[i].map_update_resident(poses[i])) for i in range(len(specs))]
    assert [r[0] for r in solo] == [L._binding.E_ARG] * 3 + [0] * 3
    assert "resident" in _last_error(A_[0])
    n_map, status = L.map_update_batch(B_, poses)
    for i in range(len(specs)):
        assert (int(status[i]), int(n_map[i])) == solo[i], (i, solo[i], status[i], n_map[i])
        _same_map(A_[i], B_[i], ("errors", i))
        if i < 3:
            assert _map_state(B_[i]) == before[i], i
            assert "resident" in _last_error(B_[i])
    _close(A_, B_)


@pytest.mark.parametrize("variant", [0, 1])
def test_a_search_with_other_features_leaves_the_resident_scan_alone(world, variant):
    """liliom_scan_to_map and liliom_find_surf_corr with a different feature count (fewer, and more than the scan's buffer was sized
    for) between the odometry call and the map update: the update still pushes the scan the odometry call left, all of it, solo
    and in a batch, as the twin that pushes ds_out does."""
    import liliom_b200 as L
    spec = Spec(variant, 5)
    a, b, c2 = spec.make(), spec.make(), spec.make()
    other = spec.make()                                     # a second session of the batch, undisturbed
    for k in range(6):
        sw = spec.sweep(world, k)
        rs = []
        for c in (a, b, c2, other):
            _scan(c, sw)
            rs.append(_odo(c, sw["guess"]))
        ra = rs[0]
        # the searches move the next step's launch-shape predictor, and with the grid the order of its fp64 sums: the disturbed
        # sessions' poses may differ from A's in their last bits.  The scan does not depend on the pose; every frame is saved under A's.
        for r in rs[1:]:
            assert r[0] == ra[0] and len(r[3]) == len(ra[3]) and r[3].tobytes() == ra[3].tobytes(), (variant, k)
        pose = _pose_for(ra, sw)
        ma = a.map_update(ra[3], pose)
        if k >= 1 and len(ra[3]) > 20:                      # a map exists: searches with 7 features, then with 3x the scan's
            few = ra[3][:7]
            many = np.concatenate([ra[3]] * 3)
            for c in (b, c2):
                _try(lambda: c.scan_to_map(few, pose, 1))
                _try(lambda: c.find_surf_corr(many, pose))
                _try(lambda: c.scan_to_map(many, pose, 1))
        assert b.map_update_resident(pose) == ma, (k, ma)
        n_map, status = L.map_update_batch([other, c2], [pose, pose])
        assert list(status) == [0, 0] and list(n_map) == [ma, ma], (k, status, n_map, ma)
        for c in (b, c2, other):
            _same_map(a, c, (variant, k))
    _close([a, b, c2, other])


def test_whole_call_refusals_change_nothing(world):
    import liliom_b200 as L
    lib = L._binding.lib()
    specs = [Spec(0, 5), Spec(1, 5)]
    cs = [s.make() for s in specs]
    _prefill(world, specs, (cs,), [2, 2])
    for c, s in zip(cs, specs):
        _scan(c, s.sweep(world, 0))
        _odo(c, s.sweep(world, 0)["guess"])
    before = [(_map_state(c), _counters(c)) for c in cs]
    dp, ip, vp = C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_void_p
    poses = np.tile(IDENT, (2, 1)).copy()
    n_map, status = np.zeros(2, np.int32), np.full(2, 77, np.int32)
    P, N, S = poses.ctypes.data_as(dp), n_map.ctypes.data_as(ip), status.ctypes.data_as(ip)

    def arr(*h):
        return (vp * len(h))(*h)
    h = [c._h for c in cs]
    calls = [lib.liliom_map_update_batch(arr(*h), 0, P, N, S), lib.liliom_map_update_batch(arr(*h), -1, P, N, S),
             lib.liliom_map_update_batch(None, 2, P, N, S), lib.liliom_map_update_batch(arr(*h), 2, None, N, S),
             lib.liliom_map_update_batch(arr(*h), 2, P, N, None), lib.liliom_map_update_batch(arr(h[0], None), 2, P, N, S),
             lib.liliom_map_update_batch(arr(h[0], h[0]), 2, P, N, S)]
    assert calls == [L._binding.E_ARG] * len(calls), calls
    assert list(status) == [77, 77]
    assert [(_map_state(c), _counters(c)) for c in cs] == before
    with pytest.raises(ValueError):
        L.map_update_batch(cs, np.zeros((1, 7)))
    n_map, status = L.map_update_batch(cs, [s.sweep(world, 0)["T"] for s in specs])     # NULL n_map is allowed, and the call still works
    assert list(status) == [0, 0] and all(n_map > 0)
    assert lib.liliom_map_update_batch(arr(*h), 2, P, None, S) == 0
    _close(cs)


# ---------------------------------------------------------------- the whole fleet loop
@pytest.mark.parametrize("mode_name", ["gn", "ceres"])
def test_fleet_loop_equals_solo_loop_with_host_round_trips(world, mode_name):
    """25 scans of four sessions.  Set B: extract batch -> map update batch (the previous scan's frame and its solved pose) ->
    odometry batch, no cloud crossing PCIe.  Set A: the same loop with solo calls, the frame downloaded through ds_out and
    uploaded again through liliom_map_update."""
    import liliom_b200 as L
    mode = L.MODE_GN if mode_name == "gn" else L.MODE_CERES
    specs = [Spec(0, 20), Spec(1, 20), Spec(0, 6, start=2), Spec(1, 4, start=1)]
    n = len(specs)
    A_, B_ = [s.make() for s in specs], [s.make() for s in specs]
    prev = None                                             # per session: (DS cloud, pose) of the previous scan
    for k in range(25):
        sws = [s.sweep(world, k) for s in specs]
        for i in range(n):
            A_[i].upload_scan(sws[i]["pts"]); B_[i].upload_scan(sws[i]["pts"])
            A_[i].extract_resident(sws[i]["q"])
        _, st_x = L.extract_resident_batch(B_, np.stack([sw["q"] for sw in sws]))
        assert not st_x.any()
        if prev is not None:
            ma = [A_[i].map_update(prev[i][0], prev[i][1]) for i in range(n)]
            mb, st_m = L.map_update_batch(B_, [p[1] for p in prev])
            assert not st_m.any() and list(mb) == ma, (k, ma, mb, st_m)
            for i in range(n):
                _same_map(A_[i], B_[i], ("fleet", mode_name, k, i))
        guesses = np.array([sw["guess"] for sw in sws])
        ra = [_odo(A_[i], guesses[i], mode) for i in range(n)]
        P, st_o, stats, ds = L.odometry_resident_batch_ex(B_, guesses, ITERS, 15, mode, want_stats=True, want_ds=True)
        for i in range(n):
            rb = (int(st_o[i]), P[i], b"".join(bytes(memoryview(s)) for s in stats[i]) if st_o[i] == 0 else b"", ds[i])
            _same_step(ra[i], rb, ("fleet", mode_name, k, i))
        prev = [(ra[i][3], _pose_for(ra[i], sws[i])) for i in range(n)]
    _close(A_, B_)
