"""No call's bytes depend on what its context did before: interleaved call histories against fresh contexts.

A context keeps about sixty grow-only device buffers between calls, many shared across call families, and a set of
read-before-write contracts (scan sentinels, control words that rotate with the call count, device-side counts, per-call state
such as the GN partials and qstate).  A call that reads what an earlier call left shows up only after a particular history, and
memory from a fresh cudaMalloc is usually zero, so fresh-context tests hide it.  Every operation of tests/history_ops.py runs here
after other calls, and its outputs (and those of the call that follows it) must equal the same operation's on a fresh context,
byte for byte.

Comparator rule: the reference for a call T is a fresh context.  Only when T's query count is known only on the device (the
odometry calls, Op.dev_count) does that fresh context first replay the history's last scan-to-map call that ran its step, with
the same inputs (a following scan is replayed with the operation input that installed its map):
s2m_plan sizes such a call from the previous scan's query count (n_last), and the launch shape sets the fold order of the GN sums
(DESIGN.md §6).  No other replay is made."""
import numpy as np
import pytest

import history_ops as H

pytestmark = pytest.mark.gpu


class Hist:
    """A context and the calls it has served; remembers the last scan-to-map input for the comparator rule"""

    def __init__(self, kind, **params):
        self.kind, self.params = kind, params
        self.c = H.make_ctx(kind, **params)
        self.last_s2m = None           # (op, the input names that replay it)
        self.last_input = None

    def run(self, op, name):
        out = op.inputs[name](self.c) if name != "nxt" else op.nxt(self.c)
        if name == "nxt":
            # the next scan runs on the map the operation's input installed: its replay is that input, then the next scan
            if op.nxt is H.nxt_s2m and ran(out):
                self.last_s2m = (op, [self.last_input, "nxt"])
        else:
            self.last_input = name
            if op.s2m and ran(out):
                self.last_s2m = (op, [name])
        return out

    def nxt(self, op):
        return self.run(op, "nxt")

    def close(self):
        self.c.close()


def ran(out):
    """the call ran its scan-to-map step: a refused one (E_ARG, E_NOMAP, E_FEWMAP, or this session's status in a batch) never
    reaches s2m_finish, so it leaves the previous step's query count in place"""
    return out.get("rc", 0) == 0 and ("st" not in out or np.frombuffer(out["st"], np.int32)[0] == 0)


def reference(kind, op, name, last_s2m, params=None, then_nxt=True):
    """(outputs of op's input `name`, outputs of op.nxt) on a fresh context, by the comparator rule"""
    B = Hist(kind, **(params or {}))
    try:
        if op.dev_count and last_s2m is not None:
            for x in last_s2m[1]:
                B.run(last_s2m[0], x)
        out = B.run(op, name)
        return out, (B.nxt(op) if then_nxt else None)
    finally:
        B.close()


def diff(a, b):
    """the keys whose values differ"""
    return sorted(k for k in set(a) | set(b) if a.get(k) != b.get(k))


def case_ids():
    return [(kind, op.name) for kind in H.KINDS for op in H.ops_of(kind)]


# ------------------------------------------------------------------------------------------ (a) shrink after grow
@pytest.mark.parametrize("kind,name", case_ids())
def test_shrink_after_grow(kind, name):
    """A runs the operation's large input, then a smaller one, then the following call; a fresh context runs the smaller one and
    the following call.  Every input other than large: small, empty, the block edges, refused."""
    op = H.by_name(name)
    assert "large" in op.inputs
    bad = []
    for inp in op.inputs:
        if inp == "large":
            continue
        A = Hist(kind)
        try:
            before = A.run(op, "large")
            last = A.last_s2m
            got = A.run(op, inp)
            got_next = A.nxt(op)
        finally:
            A.close()
        if inp == "refused":
            bad += refused_check(kind, op, before, got, got_next)
            continue
        want, want_next = reference(kind, op, inp, last)
        if got != want:
            bad.append((inp, diff(got, want)))
        if got_next != want_next:
            bad.append((inp, "next", diff(got_next, want_next)))
    assert not bad, bad


def refused_check(kind, op, before, got, got_next):
    """A refused call returns its code, the same as on a fresh context, and changes nothing: the state it reports is what the large
    input left, and (when the refused input installs nothing of its own) the next call gives what it gives right after the large
    input, on a context that never saw the refusal"""
    bad = []
    codes = {k: got[k] for k in ("rc", "st") if k in got}
    want, _ = reference(kind, op, "refused", None, then_nxt=False)
    if not codes or any(want.get(k) != v for k, v in codes.items()):
        bad.append(("refused", "code", codes, {k: want.get(k) for k in codes}))
    if "rc" in codes and codes["rc"] == 0 or "st" in codes and not np.frombuffer(codes["st"], np.int32).any():
        bad.append(("refused", "not refused", codes))
    state = [k for k in got if k not in ("rc", "st")]
    if any(got[k] != before.get(k) for k in state):
        bad.append(("refused", "state", [k for k in state if got[k] != before.get(k)]))
    if op.refused_pure:
        C = Hist(kind)
        try:
            C.run(op, "large")
            if C.nxt(op) != got_next:
                bad.append(("refused", "next"))
        finally:
            C.close()
    return bad


# ------------------------------------------------------------------------------------------ (b) foreign history
COOP = (("voxelgrid", "coop"), ("extract_horizon", "small"), ("scan_to_map_gn", "mid"), ("icp_align", "small"))


def history_of(kind):
    """Every operation the kind's context accepts, on its large input, one refused and one empty call of each operation that
    has them, and five calls of each cooperative kernel (k_vg_coop, k_hz_coop, k_gn_persistent, k_icp_persistent), so that every
    rotating control slot is used and reused."""
    ops = H.ops_of("48" if kind == "48chain" else kind)
    names = {op.name for op in ops}
    seq = [(op, "large") for op in ops]
    seq += [(op, x) for op in ops for x in ("refused", "empty") if x in op.inputs]
    seq += [(H.by_name(n), x) for n, x in COOP if n in names] * 5
    return seq


def _foreign(kind, order, targets):
    """One context serves the whole history in a seeded order (or its reverse); then every operation of the kind in turn, on its
    small input, then the call that follows it, each against a fresh context; between two operations, the large inputs of the
    next three in the history refill the scratch with other families' data.  Where the oracle has the input, the operation on the
    long-lived context must also give the oracle's bytes."""
    seq = history_of(kind)
    perm = np.random.default_rng(20261018 + len(kind)).permutation(len(seq))
    if order == "reversed":
        perm = perm[::-1]
    seq = [seq[i] for i in perm]
    A = Hist(kind)
    bad = []
    try:
        for op, x in seq:
            A.run(op, x)
        for t, op in enumerate(targets):
            inp = "small" if "small" in op.inputs else "large"
            last = A.last_s2m
            got = A.run(op, inp)
            got_next = A.nxt(op)
            want, want_next = reference(kind, op, inp, last)
            if got != want:
                bad.append((op.name, inp, diff(got, want)))
            if got_next != want_next:
                bad.append((op.name, "next", diff(got_next, want_next)))
            if inp in op.oracle:
                ref = op.oracle[inp]()
                if any(got[k] != v for k, v in ref.items()):
                    bad.append((op.name, inp, "oracle", [k for k, v in ref.items() if got[k] != v]))
            for k in range(3):
                A.run(*seq[(3 * t + k) % len(seq)])
    finally:
        A.close()
    assert not bad, bad


@pytest.mark.parametrize("order", ["seeded", "reversed"])
@pytest.mark.parametrize("kind", list(H.KINDS))
def test_foreign_history(kind, order, oracle):
    _foreign(kind, order, H.ops_of(kind))


# ------------------------------------------------------------------------------------------ (c) named cases
def _same(a_fn, b_fn, what):
    ga, gb = a_fn(), b_fn()
    assert ga == gb, (what, diff(ga, gb) if isinstance(ga, dict) else None)


def test_map_update_entry_count_equals_last_removal_index():
    """k_inc_mark's sentinel removed[E] = 0: a stream that removed entries with E = 1500 entries before the update (three
    500-point frames, one popped per update), map_clear, then a stream whose third update sees E = 1500 without a pop (two
    750-point frames).  Every map on both contexts also equals the map the full rebuild makes of the same frames."""
    w = H.world()
    prm = dict(max_map_frames=3)
    A, B, R = (H.make_ctx(k, **prm) for k in ("48", "48", "48"))
    try:
        def stream(c, n, k, base):
            out = []
            for i in range(k):
                p = np.array(w["T"]); p[4] += 0.3 * i
                pts = w["hz"][base + i * n:base + (i + 1) * n]
                assert np.isfinite(pts["x"]).all()
                out.append((c.map_update(pts, p), H.b(c.map_download_cloud()), H.b(c.map_download())))
            return out

        stream(A, 500, 6, 0)
        A.map_clear()
        got, want = stream(A, 750, 5, 4000), stream(B, 750, 5, 4000)
        assert got == want
        for i in range(5):                                       # the rebuild of the FIFO's last frames
            R.map_clear()
            for j in range(max(0, i - 2), i + 1):
                p = np.array(w["T"]); p[4] += 0.3 * j
                R.map_push_frame(w["hz"][4000 + j * 750:4000 + (j + 1) * 750], p)
            R.map_rebuild()
            assert H.b(R.map_download_cloud()) == got[i][1], i
    finally:
        for c in (A, B, R):
            c.close()


def test_rot_hdl64_then_16_line_sweep(oracle):
    """The lessflat sentinel and the ring scratch: a 130k-point HDL-64E extraction, then a 16-line sweep, on the same context.
    Elevation rings (a 16-line context: the HDL-64E returns outside its table are dropped) against a fresh context and the oracle,
    and PointCloud2 `ring` fields (a 64-line context fed a 16-ring message) against a fresh context."""
    import liliom_b200 as L
    import rot_adversarial as RA
    from liliom_b200 import synth
    w = H.world()
    sw16 = RA.tables_sweep(16, 1)
    s16 = dict(sw16); s16["ds_rate"] = 4

    def run16(c):
        r = c.extract_rot(s16["pts"], s16["q_imu"], s16["q_lb"])
        return {**H._extract_out(r), **H.feats_state(c), "lab": H.b(c.extract_rot_labels(len(s16["pts"])))}
    A, B = H.make_ctx("32", line_num=16, ds_rate=4), H.make_ctx("32", line_num=16, ds_rate=4)
    try:
        A.extract_rot(w["hdl"], w["q_hdl"])
        got = run16(A)
        assert got == run16(B)
        _rc, s, e, k, _lab, _cur = oracle.extract_rot(s16["pts"], s16["q_imu"], s16["q_lb"], 16, 4)
        assert (got["surf"], got["edge"], got["cut"]) == (H.b(s), H.b(e), H.b(k))
    finally:
        A.close(); B.close()
    pts, q, ring, step = synth.make_spinning_sweep(w["T"], synth.uniform_elevations(16, 15.0, -15.0), 900, seed=3)
    msg16 = synth.encode_pc2(pts, ring, step, "pcl32", steps=900, lines=16)
    A, B = H.make_ctx("32"), H.make_ctx("32")
    try:
        for c in (A, B):
            c.set_ring_source(L.RING_FIELD)
        A.extract_rot_pc2(H.pc2("pcl32", True), w["q_hdl"])
        _same(lambda: {**H._extract_out(A.extract_rot_pc2(msg16, q)), **H.feats_state(A)},
              lambda: {**H._extract_out(B.extract_rot_pc2(msg16, q)), **H.feats_state(B)}, "ring field")
    finally:
        A.close(); B.close()


@pytest.mark.parametrize("first", ["resident", "host"])
def test_resident_horizon_then_host_extraction(first):
    """A resident Horizon extraction (sizes only on the device) and a host one (sizes on the host) on one context, in either order,
    a refused ROT extraction between them; then the de-skew, the download and the keyframe hand-off read the last extraction's
    sizes.  Against a fresh context that ran only the last extraction."""
    import liliom_b200 as L
    w = H.world()
    pts, q = w["hz"], w["q_hz"]
    bp = L.backend_default_params(0)

    def last(c):
        if first == "resident":
            r = H._extract_out(c.extract_horizon(pts[:3000], q))
        else:
            c.upload_scan(pts[:3000])
            r = {"n": repr(c.extract_resident(q))}
        out = {**r, **H.feats_state(c)}
        c.undistort_resident((0.3, -0.1, 0.05), (0.9999, 0.01, -0.005, 0.002))
        out.update({f"u_{k}": v for k, v in H.feats_state(c).items()})
        c.kf_clear()
        out["kf"] = repr(c.kf_add_resident(bp, c))
        out["full"] = H.b(c.global_map(L.KF_FULL, [0], [H.IDENT7], H.TINY_LEAF))
        out["surf"] = H.b(c.global_map(L.KF_SURF, [0], [H.IDENT7], H.TINY_LEAF))
        return out

    A, B = H.make_ctx("48"), H.make_ctx("48")
    try:
        if first == "resident":
            A.upload_scan(pts); A.extract_resident(q)
        else:
            A.extract_horizon(pts, q)
        assert H.code(lambda: A.extract_rot(w["hdl"][:100], w["q_hdl"])) == L._binding.E_ARG
        _same(lambda: last(A), lambda: last(B), first)
    finally:
        A.close(); B.close()


@pytest.mark.parametrize("modes", ["gn_gn", "ceres_gn", "gn_ceres"])
def test_s2m_large_grid_then_small(modes):
    """A scan-to-map of 3000 and of 24000 queries (more blocks than SMs), then one of 200 (16 lanes, a small grid): the stale
    partials columns, qstate / use_state, lm_state; solo and batched calls alternate on the same context so that the barrier
    count advances through both paths.  Every call against a fresh context (the batch beside a fresh second session)."""
    import liliom_b200 as L
    w = H.world()
    mode = {"gn": L.MODE_GN, "ceres": L.MODE_CERES}
    m1, m2 = (mode[x] for x in modes.split("_"))

    def solo(c, n, m):
        c.map_set_points(w["map"])
        pose, st = c.scan_to_map(H.s2m_feats(n), w["guess"], 4 if m == L.MODE_GN else 2, 6, m)
        return {"pose": H.b(pose), "stats": H.b(st)}

    def batch(c, n, m):
        h = H.make_ctx("48")
        try:
            for x, k in ((c, n), (h, 300)):
                x.map_set_points(w["map"])
                x.upload_feats(H.s2m_feats(k))
            r = L.scan_to_map_resident_batch_ex([c, h], [w["guess"]] * 2, 4 if m == L.MODE_GN else 2, 6, m, want_stats=True)
            return {"pose": H.b(r[0]), "st": H.b(r[1]), "stats": H.b(r[2][0]) + H.b(r[2][1])}
        finally:
            h.close()

    plan = [(solo, 3000, m1), (solo, 24000, m1), (solo, 200, m2), (batch, 3000, m1), (batch, 200, m2), (solo, 200, m2),
            (batch, 24000, m1), (solo, 200, m2), (batch, 200, m2)]
    A = H.make_ctx("48")
    try:
        for i, (f, n, m) in enumerate(plan):
            B = H.make_ctx("48")
            try:
                _same(lambda: f(A, n, m), lambda: f(B, n, m), (i, f.__name__, n, m))
            finally:
                B.close()
    finally:
        A.close()


def test_s2m_after_a_denser_map():
    """qstate / use_state: the first GN pass of a call must not start from the previous call's per-query state.  A step on a
    denser map of the same world leaves each query a fifth distance that is too small for the sparser map the next step runs on;
    a pass that trusted it would cut the search short.  Against a fresh context."""
    import liliom_b200 as L
    from liliom_b200 import synth
    w = H.world()
    dense, _ = synth.make_map(400_000)

    def step(c, m):
        c.map_set_points(m)
        pose, st = c.scan_to_map(H.s2m_feats(2000), w["guess"], H.ITERS, 6, L.MODE_GN)
        return {"pose": H.b(pose), "stats": H.b(st)}

    A, B = H.make_ctx("48"), H.make_ctx("48")
    try:
        step(A, dense)
        _same(lambda: step(A, w["map"]), lambda: step(B, w["map"]), "sparse after dense")
    finally:
        A.close(); B.close()


def test_backend_41_keyframes_then_2():
    """kf_tab and the block segments: a 41-keyframe store, local map and loop closure with a window of its last kWinMax = 16
    keyframes, then a 2-keyframe one on the same backend context, against a fresh context."""
    import liliom_b200 as L
    from liliom_b200 import synth
    seq41 = synth.make_keyframe_sequence(41, 48)
    bp = L.backend_default_params(0)

    def run(c, k):
        c.kf_clear()
        out = {}
        for e, s, _p in seq41[:k]:
            kid, eds, sds = c.kf_add(bp, e, s)
            out[f"kf{kid}"] = H.b(eds) + H.b(sds)
        poses = [p for _e, _s, p in seq41[:k]]
        out["bmap"] = repr(c.bmap_build(bp, list(range(k)), poses))
        out["l0"], out["l1"] = H.b(c.bmap_download(0)), H.b(c.bmap_download(1))
        win = list(range(max(0, k - 16), k))
        ne, ns = c.backend_window_correspond(bp, win, [poses[i] for i in win])
        out["ne"], out["ns"] = H.b(ne), H.b(ns)
        out["blocks"] = H.b(c.backend_window_blocks([poses[i] for i in win]))
        out["corr"] = H.b([H.b(x) for s in range(len(win)) for kind in (0, 1) for x in c.backend_window_corr(s, kind)])
        r = c.loop_align([k - 1], [poses[-1]], list(range(k - 1)), poses[:-1], 0.4, max_iter=20)
        out["loop"] = H.b(r[0]) + repr(r[1:]).encode()
        return out

    A, B = H.make_ctx("48"), H.make_ctx("48")
    try:
        run(A, 41)
        _same(lambda: run(A, 2), lambda: run(B, 2), "2 after 41")
    finally:
        A.close(); B.close()


def test_pc2_full_sweep_then_one_row_then_refused_batch():
    """wire_in grown by a full HDL-64E PointCloud2, then a one-row message, then a batch whose first session is refused, then a
    valid message; every step's decode and the extraction of the resident sweep against a fresh context."""
    import liliom_b200 as L
    from liliom_b200 import synth
    w = H.world()
    one_row = synth.encode_pc2(w["hdl"][:37], w["ring"][:37], w["step"][:37], "velodyne22")
    bad = L.PC2(b"", 1, 5, 16, 80, [])

    def step(c, what):
        if what == "batch":
            h = H.make_ctx("32")
            try:
                clouds, st = L.convert_batch([c, h], [bad, H.pc2_first(300)], download=True)
                out = {"clouds": H.b([x for x in clouds if x is not None]), "st": H.b(st)}
            finally:
                h.close()
        else:
            out = {"cloud": H.b(c.convert_pc2(one_row if what == "one_row" else H.pc2("ouster48", False)))}
        if what == "batch":           # the refused session keeps its resident sweep: checked against one_row_only below
            return out
        return {**out, **H.nxt_resident_sweep(c)}

    def one_row_only():
        R = H.make_ctx("32")
        try:
            R.convert_pc2(one_row)
            return H.nxt_resident_sweep(R)
        finally:
            R.close()

    A = H.make_ctx("32")
    try:
        A.convert_pc2(H.pc2("hesai26", True))
        for what in ("one_row", "batch", "valid"):
            B = H.make_ctx("32")
            try:
                _same(lambda: step(A, what), lambda: step(B, what), what)
                if what == "batch":
                    _same(lambda: H.nxt_resident_sweep(A), one_row_only, "refused session keeps the one-row sweep")
            finally:
                B.close()
    finally:
        A.close()


def _spec_clouds():
    """surf clouds of the odometry: 'fits' (the cooperative filter takes it), 'missed' (300 copies of one point make the
    cooperative filter decline, and two far points give the scan's voxel box more than 2^24 cells: the speculative 24-bit keys
    miss and the step is redone with 32-bit keys)"""
    hz = H.world()["hz"]
    fits = hz[:20_000].copy()
    heavy = np.repeat(hz[:1], 300)
    far = hz[:2].copy()
    far["x"], far["y"], far["z"] = (300.0, -300.0), (300.0, -300.0), (25.0, -25.0)
    return {"fits": fits, "missed": np.concatenate([hz[:20_000], heavy, far])}


@pytest.mark.parametrize("order", ["missed_fits", "fits_missed"])
def test_odometry_spec_missed_then_fits(order, oracle):
    """odo_spec_missed: an odometry call whose scan VoxelGrid missed the speculative key width, then one that fits, and the
    reverse.  The second call's down-sampled scan is the oracle's VoxelGrid, and its pose, stats and scan equal a fresh context's
    (which replays the first call: the query count is only on the device)."""
    import liliom_b200 as L
    w = H.world()
    clouds = _spec_clouds()
    a, b = order.split("_")

    def odo(c, name):
        c.map_set_points(w["map"])
        pose, st, ds = c.odometry(clouds[name], w["guess"], H.ITERS, 6, L.MODE_GN)
        return {"pose": H.b(pose), "stats": H.b(st), "ds": H.b(ds)}

    import vg_adversarial as VG
    leaf = L.default_params(0).leaf_scan
    for name, c in clouds.items():     # what odo_filter decides from: the cooperative filter's member cap and the 24-bit key box
        _ov, _mb, div_b, _n, _d = VG.params(c, leaf)
        cells = int(np.prod(np.array(div_b, np.int64)))
        keys = np.floor(np.stack([c["x"], c["y"], c["z"]], 1).astype(np.float32) * np.float32(1 / np.float32(leaf))).astype(np.int64)
        heavy = np.unique(keys, axis=0, return_counts=True)[1].max() > VG.VGC_VCAP
        assert (heavy and cells >= (1 << 24) - 1) == (name == "missed"), (name, heavy, cells)
    A, B = H.make_ctx("48"), H.make_ctx("48")
    try:
        odo(A, a)
        got = odo(A, b)
        odo(B, a)
        assert got == odo(B, b)
        assert got["ds"] == H.b(oracle.voxelgrid(clouds[b], A.params.leaf_scan))
    finally:
        A.close(); B.close()


def test_batched_ceres_odometry_with_an_empty_scan():
    """A session of the batched Ceres odometry whose sweep leaves no surf feature (700 returns of the HDL-64E sweep) runs: its
    scan filter wrote no VgParams, so the step has none of this call to read back.  The other session's results are its solo
    call's, and a call on either context afterwards succeeds."""
    import liliom_b200 as L
    w = H.world()
    pts, q = w["hdl"], w["q_hdl"]
    c, h, solo = H.make_ctx("32"), H.make_ctx("32"), H.make_ctx("32")
    try:
        for x, n in ((c, 24000), (h, 700), (solo, 24000)):
            x.map_set_points(w["map"])
            x.upload_scan(pts[:n])
            n_surf = x.extract_resident(q)[0]
            assert (n_surf == 0) == (x is h), n_surf
        poses, status, _st, ds = L.odometry_resident_batch_ex([c, h], [w["guess"]] * 2, 2, 6, L.MODE_CERES, want_ds=True)
        assert list(status) == [0, 0] and len(ds[1]) == 0
        pose, _s, ds0 = solo.odometry_resident(w["guess"], 2, 6, L.MODE_CERES, want_ds=True, cap=65536)
        assert H.b(poses[0]) == H.b(pose) and H.b(ds[0]) == H.b(ds0)
        for x in (c, h):
            x.map_set_points(w["map"][:1000])
    finally:
        for x in (c, h, solo):
            x.close()
