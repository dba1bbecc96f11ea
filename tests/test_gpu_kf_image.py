"""GPU tests of the keyframe image (liliom_kf_export / liliom_kf_import).  Its contract is the one the multi-store calls use: a
context D that imports an image of store C's keyframes L holds the same clouds, so every call that reads keyframes gives on D,
with the mapped ids, the bytes it gives on C with L, and D's export is the image again.  Also: the image's contents against what
the store received (tests/kf_image_reference.py decodes it), subsets, repeats and images without full clouds, a restart across
two processes, every malformed image refused with nothing changed, a store at size and an image past 2^31 bytes, and seeded call
histories before and after."""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import kf_image_reference as R

pytestmark = pytest.mark.gpu

IDENT = np.array([1.0, 0, 0, 0, 0, 0, 0])
TINY_LEAF = 1e-4          # PCL declines every keyframe-sized cloud at this leaf: global_map gives the stored clouds back
LOOP = dict(max_corr_dist=2.0, max_iter=60, trans_eps=1e-8, fit_eps=1e-8)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _L():
    import liliom_b200 as L
    return L


def _b(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _err(c):
    return _L()._binding.lib().liliom_last_error(c._h).decode()


def _nudge(pose, k):
    from liliom_b200 import synth
    dq = synth.q_from_axis_angle([1, -1, 2], np.deg2rad(0.15 * k))
    return np.concatenate([synth.qmul(pose[:4], dq), pose[4:] + 0.01 * k * np.array([1.0, -0.5, 0.25])])


class Store:
    """A store built from a seeded keyframe sequence with kf_add + kf_add_full, and what it received and returned: the
    down-sampled edge and surf outputs and the received full clouds.  Two more keyframes: one with empty edge, surf and full
    clouds, and one without a full cloud."""

    def __init__(self, stride, n_kf=6, seed=3):
        L = _L()
        from liliom_b200 import synth
        self.variant = 0 if stride == 48 else 1
        self.stride = stride
        self.bp = L.backend_default_params(self.variant)
        self.c = L.Context(variant=self.variant)
        self.seq = synth.make_keyframe_sequence(n_kf, stride=stride, seed=seed, full=True)
        self.edge, self.surf, self.full, self.poses = [], [], [], []
        empty = np.zeros(0, self.c.dtype)
        for e, s, p, f in self.seq:
            self.add(e, s, f, p)
        self.add(empty, empty, empty, self.seq[0][2])
        e, s, p, _ = self.seq[1]
        self.add(e, s, None, _nudge(p, 3))

    def add(self, e, s, f, p):
        kid, eds, sds = self.c.kf_add(self.bp, e, s)
        self.edge.append(eds); self.surf.append(sds); self.poses.append(p)
        self.full.append(f)
        if f is not None:
            self.c.kf_add_full(self.bp, kid, f)

    def close(self):
        self.c.close()


@pytest.fixture(scope="module", params=[48, 32], ids=["horizon_v0", "rot_v1"])
def store(request):
    s = Store(request.param)
    yield s
    s.close()


def _layers(c):
    out = []
    for layer in (0, 1):
        try:
            out.append(_b(c.bmap_download(layer)))
        except _L().LiliomError as e:
            out.append(e.code)
    return out


def _searches(c, bp, ids, poses):
    L = _L()
    try:
        ne, ns = c.backend_window_correspond(bp, ids, poses)
    except L.LiliomError as e:
        return [e.code]
    out = [ne.tolist(), ns.tolist()]
    for slot in range(len(ids)):
        out += [_b(x) for kind in (0, 1) for x in c.backend_window_corr(slot, kind)]
    out.append(_b(c.backend_window_blocks(np.array([_nudge(p, 2) for p in poses]))))
    return out


def _readers(c, bp, ids, poses, full=True):
    """every single-store reader of the listed keyframes on c: the local map and the window calls, kf_cloud, loop_align, both
    global maps with and without Tbl"""
    L = _L()
    tbl = np.concatenate([np.array(bp.q_lb[:]), np.array(bp.t_lb[:])])
    out = dict(bmap=c.bmap_build(bp, ids, poses))
    out["layers"] = _layers(c)
    out["win"] = _searches(c, bp, ids[:3], poses[:3])
    out["cloud"] = _b(c.kf_cloud(ids, poses, 0.4))
    T, fit, conv, it, ns, nt = c.loop_align(ids[:2], [_nudge(p, 1) for p in poses[:2]], ids, poses, 0.4, **LOOP)
    out["loop"] = (_b(T), fit, conv, it, ns, nt)
    for kind in ((L.KF_FULL, L.KF_SURF) if full else (L.KF_SURF,)):
        for pre in (None, tbl):
            for leaf in (0.3, TINY_LEAF):
                out[(kind, pre is None, leaf)] = _b(c.global_map(kind, ids, poses, leaf, pre7=pre))
    return out


# ---------------------------------------------------------------- 1. the contents
def test_the_image_holds_what_the_store_received(store, oracle):
    s = store
    img = s.c.kf_export()
    d = R.decode(img)
    h = d["header"]
    assert bytes(h["magic"]) == R.MAGIC and h["stride"] == s.stride and h["k"] == len(s.edge) and h["flags"] == R.FLAG_FULL
    assert len(img) == R.size(s.stride, [(int(r["n_edge"]), int(r["n_surf"]), int(r["n_full"])) for r in d["records"]])
    assert int(h["points_sum"]) == R.checksum(d["a"] + d["f"])
    assert int(h["table_sum"]) == R.table_sum(img[:64], img[64:64 + 16 * len(s.edge)])
    for i, (e, su, f) in enumerate(d["kfs"]):
        assert e == _b(s.edge[i]) and su == _b(s.surf[i]), i
        if s.full[i] is None:
            assert f is None, i
        elif s.variant == 0:
            assert f == _b(s.full[i]), i                                    # as received
        else:
            assert f == _b(oracle.voxelgrid(s.full[i], s.bp.surf_leaf)), i  # VoxelGrid(surf_leaf) of it
    assert d["kfs"][-2] == (b"", b"", b"") and d["kfs"][-1][2] is None
    assert len(s.c.kf_export([])) == 64


# ---------------------------------------------------------------- 2. the round trip
def test_round_trip_gives_every_reader_the_source_bytes(store):
    L = _L()
    s = store
    img = s.c.kf_export()
    D = L.Context(variant=s.variant)
    try:
        assert D.kf_import(img) == (0, len(s.edge)) and D.kf_count() == len(s.edge)
        assert D.kf_export() == img
        n = len(s.edge) - 1                                    # the last keyframe has no full cloud: FULL maps list the others
        for ids in ([0, 1, 2, 3, 4, 5, 6], [5, 2, 2, 6, 0], [3]):
            poses = [_nudge(s.poses[i], j) for j, i in enumerate(ids)]
            assert all(i < n for i in ids)
            assert _readers(D, s.bp, ids, poses) == _readers(s.c, s.bp, ids, poses), ids
    finally:
        D.close()


def test_imported_store_beside_live_ones(store):
    L = _L()
    s = store
    other = Store(s.stride, n_kf=4, seed=9)
    D = L.Context(variant=s.variant)
    try:
        D.kf_import(s.c.kf_export())
        entries = [(0, 1), (1, 0), (0, 3), (1, 2), (0, 1), (0, 6)]
        ids = [i for _, i in entries]
        poses = [_nudge((s.poses if k == 0 else other.poses)[i], j) for j, (k, i) in enumerate(entries)]
        live = [s.c if k == 0 else other.c for k, _ in entries]
        imp = [D if k == 0 else other.c for k, _ in entries]
        caller = other.c
        for kind in (L.KF_FULL, L.KF_SURF):
            for leaf in (0.3, TINY_LEAF):
                assert _b(caller.global_map_multi(kind, imp, ids, poses, leaf)) == _b(caller.global_map_multi(kind, live, ids, poses, leaf))
        a = caller.loop_align_multi(imp[:2], ids[:2], poses[:2], imp, ids, poses, 0.4, **LOOP)
        b = caller.loop_align_multi(live[:2], ids[:2], poses[:2], live, ids, poses, 0.4, **LOOP)
        assert _b(a[0]) == _b(b[0]) and a[1:] == b[1:]
        want = caller.bmap_build_multi(s.bp, live, ids, poses), _layers(caller)
        assert (caller.bmap_build_multi(s.bp, imp, ids, poses), _layers(caller)) == want
    finally:
        D.close()
        other.close()


@pytest.mark.parametrize("B", [1, 5, 33])
def test_imported_prior_shared_by_a_fleet_batch(store, B):
    L = _L()
    s = store
    D = L.Context(variant=s.variant)
    sess = [L.Context(variant=s.variant) for _ in range(B)]
    try:
        D.kf_import(s.c.kf_export(full=False))
        rng = np.random.default_rng(B)
        lists = [[int(x) for x in rng.integers(0, len(s.edge), int(rng.integers(1, 6)))] for _ in range(B)]
        poses = [[_nudge(s.poses[i], j + b) for j, i in enumerate(l)] for b, l in enumerate(lists)]

        def run(prior):
            cnt, st = L.bmap_build_batch_multi(sess, [s.bp] * B, [[prior] * len(l) for l in lists], lists, poses)
            assert (st == 0).all()
            out = [cnt.tobytes()] + [_layers(c) for c in sess]
            out += [_searches(c, s.bp, l[:2], p[:2]) for c, l, p in zip(sess[:3], lists, poses)]
            return out
        assert run(D) == run(s.c)
    finally:
        for c in sess + [D]:
            c.close()


# ---------------------------------------------------------------- 3. lists
def test_subsets_repeats_no_full_and_appending(store):
    L = _L()
    s = store
    whole = R.decode(s.c.kf_export())["kfs"]
    ids = [6, 2, 2, 0, 7, 3]
    d = R.decode(s.c.kf_export(ids))
    assert d["kfs"] == [whole[i] for i in ids]
    nf = R.decode(s.c.kf_export(ids, full=False))
    assert nf["header"]["flags"] == 0 and nf["f"] == b"" and [x[:2] for x in nf["kfs"]] == [whole[i][:2] for i in ids]
    assert all(int(r["n_full"]) == -1 for r in nf["records"])
    # appended onto a non-empty store: ids first_id + j hold entry j
    D = L.Context(variant=s.variant)
    try:
        for e, su, _, _ in s.seq[:3]:
            D.kf_add(s.bp, e, su, download=False)
        first, k = D.kf_import(s.c.kf_export(ids, full=False))
        assert (first, k) == (3, len(ids)) and D.kf_count() == 3 + len(ids)
        mapped = [first + j for j in range(k)]
        poses = [_nudge(s.poses[i], j) for j, i in enumerate(ids)]
        assert D.kf_export(mapped, full=False) == s.c.kf_export(ids, full=False)
        assert _readers(D, s.bp, mapped, poses, full=False) == _readers(s.c, s.bp, ids, poses, full=False)
        with pytest.raises(L.LiliomError) as e:                   # no full clouds were imported
            D.global_map(L.KF_FULL, mapped[:1], poses[:1], 0.3)
        assert e.value.code == L._binding.E_ARG
        # ... and kf_add_full may attach one later: the same bytes as the source's keyframe 0's
        j0 = ids.index(0)
        D.kf_add_full(s.bp, mapped[j0], s.seq[0][3])
        assert _b(D.global_map(L.KF_FULL, [mapped[j0]], [IDENT], 0.3)) == _b(s.c.global_map(L.KF_FULL, [0], [IDENT], 0.3))
    finally:
        D.close()


# ---------------------------------------------------------------- 4. across processes
_RECIPE = r'''
import os, sys
import numpy as np
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import liliom_b200 as L
from liliom_b200 import synth

mode, out = sys.argv[1], sys.argv[2]
old = synth.make_keyframe_sequence(8, stride=48, seed=21)
new = synth.make_keyframe_sequence(8, stride=48, seed=22)
bp = L.backend_default_params(0)
bp.q_lb[:] = [1.0, 0.0, 0.0, 0.0]
bp.t_lb[:] = [0.0, 0.0, 0.0]
T_off = np.concatenate([synth.q_from_axis_angle([0.2, -0.1, 1.0], np.deg2rad(2.0)), [0.35, -0.35, 0.1]])
q_inv = T_off[:4] * np.array([1.0, -1.0, -1.0, -1.0])
compose = lambda q, t, p: np.concatenate([synth.qmul(q, p[:4]), synth.qrot(q, p[4:]) + t])
in_new = lambda p: compose(q_inv, -synth.qrot(q_inv, T_off[4:]), p)
P, B = L.Context(variant=0), L.Context(variant=0)
if mode == "first":                      # the previous run: its store, saved with its poses
    for e, s, _ in old:
        P.kf_add(bp, e, s, download=False)
    open(os.path.join(out, "prior.kfimg"), "wb").write(P.kf_export())
    np.save(os.path.join(out, "prior_poses.npy"), np.array([p for _, _, p in old]))
    ids = list(range(8))
else:                                    # the restarted process: the saved store imported
    first, k = P.kf_import(open(os.path.join(out, "prior.kfimg"), "rb").read())
    ids = list(range(first, first + k))
poses = np.load(os.path.join(out, "prior_poses.npy"))
for e, s, _ in new:
    B.kf_add(bp, e, s, download=False)
tgt = [3, 4, 5, 6, 7]
T, fit, conv, it, ns, nt = B.loop_align_multi([B], [5], [in_new(new[5][2])], [P] * 5, [ids[i] for i in tgt], [poses[i] for i in tgt], 0.4,
                                              max_corr_dist=2.0, max_iter=100)
R_ = T[:3, :3]
w = np.sqrt(max(1e-30, 1.0 + R_[0, 0] + R_[1, 1] + R_[2, 2])) / 2
qT = np.array([w, (R_[2, 1] - R_[1, 2]) / (4 * w), (R_[0, 2] - R_[2, 0]) / (4 * w), (R_[1, 0] - R_[0, 1]) / (4 * w)])
qTi = qT * np.array([1.0, -1.0, -1.0, -1.0])
placed = [compose(qTi, -synth.qrot(qTi, T[:3, 3]), poses[i]) for i in range(8)]
ne_map, ns_map = B.bmap_build_multi(bp, [P] * 8, ids, placed)
win = [4, 5, 6]
here = np.array([in_new(new[i][2]) for i in win])
ne, ns_ = B.backend_window_correspond(bp, win, here)
np.savez(os.path.join(out, mode + ".npz"), T=T, fit=np.array([fit, conv, it, ns, nt]), counts=np.array([ne_map, ns_map]),
         edge=B.bmap_download(0).view(np.uint8), surf=B.bmap_download(1).view(np.uint8), ne=ne, ns=ns_,
         blocks=B.backend_window_blocks(here))
P.close(); B.close()
'''


def test_a_restart_across_processes(tmp_path):
    script = tmp_path / "recipe.py"
    script.write_text(f"ROOT = {ROOT!r}\n" + textwrap.dedent(_RECIPE))
    for mode in ("first", "restarted"):
        r = subprocess.run([sys.executable, str(script), mode, str(tmp_path)], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
    a, b = np.load(tmp_path / "first.npz"), np.load(tmp_path / "restarted.npz")
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        assert a[k].tobytes() == b[k].tobytes(), k
    assert a["fit"][1] == 1 and a["counts"][1] > 50 and (a["ns"] > 0).all()


# ---------------------------------------------------------------- 5. refusals
def _raw_import(c, img):
    L = _L()
    a = np.frombuffer(img, np.uint8)
    first, k = C.c_int(-7), C.c_int(-7)
    rc = L._binding.lib().liliom_kf_import(c._h, a.ctypes.data_as(C.c_void_p) if a.size else None, a.size, C.byref(first), C.byref(k))
    return rc, first.value, k.value


def _resident(c):
    """a resident scan (an odometry call) on a Horizon context"""
    from liliom_b200 import synth
    m, _ = synth.make_map(30_000, seed=1)
    c.map_set_points(m)
    T = synth.default_true_pose()
    pts, q = synth.make_horizon_sweep(T, seed=41)
    surf, _, _ = c.extract_horizon(pts, q)
    c.odometry(surf, synth.perturbed_pose(T), 4)


MESSAGE = dict(magic="bad magic", version="unknown version", stride="point_stride", flags="unknown flags", counts="bad counts",
               totals="totals", length="length", table="table checksum", points="points checksum")


def test_malformed_images_change_nothing(store):
    L = _L()
    s = store
    img = s.c.kf_export([0, 1, 7, 2])             # keyframe 7 has no full cloud
    cases = R.malformed(img, s.stride)
    assert {w for _, _, w in cases} == set(R.CHECKS)
    T = L.Context(variant=s.variant)
    try:
        for e, su, _, f in s.seq[:2]:
            kid, _, _ = T.kf_add(s.bp, e, su, download=False)
            T.kf_add_full(s.bp, kid, f)
        T.bmap_build(s.bp, [0, 1], s.poses[:2])
        if s.stride == 48:
            _resident(T)
        before = (T.kf_count(), T.kf_export(), _layers(T))
        for name, bad, want in cases:
            rc, first, k = _raw_import(T, bad)
            assert rc == L._binding.E_ARG, name
            assert _err(T).startswith("keyframe image: " + MESSAGE[want]), (name, _err(T))
            assert (first, k) == (-7, -7)
            assert (T.kf_count(), T.kf_export(), _layers(T)) == before, name
        if s.stride == 48:
            T.map_update_resident(IDENT)              # the scan is still resident
        assert _raw_import(T, img)[0] == 0 and T.kf_export([2, 3, 4, 5]) == img
    finally:
        T.close()


def test_export_refusals(store):
    L = _L()
    s = store
    lib = L._binding.lib()
    n = C.c_longlong(-1)
    ids = (C.c_int * 2)(0, len(s.edge))
    assert lib.liliom_kf_export(s.c._h, ids, 2, 1, None, 0, C.byref(n)) == L._binding.E_ARG and "unknown keyframe id" in _err(s.c)
    assert lib.liliom_kf_export(s.c._h, ids, -1, 1, None, 0, C.byref(n)) == L._binding.E_ARG
    assert lib.liliom_kf_export(s.c._h, None, 0, 2, None, 0, C.byref(n)) == L._binding.E_ARG
    img = s.c.kf_export()
    buf = (C.c_char * len(img))()
    assert lib.liliom_kf_export(s.c._h, None, 0, 1, buf, len(img) - 1, C.byref(n)) == L._binding.E_CAPACITY
    assert n.value == len(img) and bytes(buf) == b"\0" * len(img)
    os.environ["LILIOM_TEST_LOOPBACK"] = "kfimg:0/2"
    try:
        lb = L.Context(L.default_params(s.variant))
    finally:
        os.environ.pop("LILIOM_TEST_LOOPBACK", None)
    try:
        assert lib.liliom_kf_export(lb._h, None, 0, 1, None, 0, C.byref(n)) == L._binding.E_ARG
        assert _raw_import(lb, img)[0] == L._binding.E_ARG
    finally:
        lb.close()


# ---------------------------------------------------------------- 6. at size
def test_a_300_keyframe_store_round_trips():
    L = _L()
    from liliom_b200 import synth
    bp = L.backend_default_params(0)
    A, D = L.Context(variant=0), L.Context(variant=0)
    try:
        seq = synth.make_keyframe_sequence(300, stride=48, seed=5, full=True)
        for e, s, _, f in seq:
            kid, _, _ = A.kf_add(bp, e, s, download=False)
            A.kf_add_full(bp, kid, f)
        img = A.kf_export()
        assert len(img) > 300 * 20_000 * 48
        assert D.kf_import(img) == (0, 300) and D.kf_export() == img
        ids = list(range(0, 300, 7))
        poses = [p for _, _, p, _ in seq[::7]]
        for kind in (L.KF_FULL, L.KF_SURF):
            assert _b(D.global_map(kind, ids, poses, 0.4)) == _b(A.global_map(kind, ids, poses, 0.4))
        assert D.bmap_build(bp, ids[-5:], poses[-5:]) == A.bmap_build(bp, ids[-5:], poses[-5:]) and _layers(D) == _layers(A)
    finally:
        A.close(); D.close()


def test_an_image_past_2_31_bytes():
    L = _L()
    bp = L.backend_default_params(0)
    rng = np.random.default_rng(11)
    n = 4_000_000
    A, D = L.Context(variant=0), L.Context(variant=0)
    try:
        cloud = np.zeros(n, L.PT48)
        cloud.view(np.uint8)[:] = rng.integers(0, 256, n * 48, dtype=np.uint8)     # any bytes: a plain copy keeps them
        for i in range(12):
            e = np.zeros(0, L.PT48)
            kid, _, _ = A.kf_add(bp, e, e, download=False)
            cloud.view(np.uint8)[:8] = i                                          # every keyframe's full cloud differs
            A.kf_add_full(bp, kid, cloud)
        img = A.kf_export()
        assert len(img) > 2**31 and len(img) == R.HEADER + 12 * R.RECORD + 12 * n * 48
        assert int(np.frombuffer(img[:64], R.HDR)[0]["points_sum"]) == R.checksum(memoryview(img)[64 + 12 * 16:])
        assert D.kf_import(img) == (0, 12)
        assert D.kf_export() == img
        del img
        last = R.decode(D.kf_export([11]))["kfs"][0][2]
        cloud.view(np.uint8)[:8] = 11
        assert last == _b(cloud)
    finally:
        A.close(); D.close()


# ---------------------------------------------------------------- 7. histories
def _fresh(kind, op, name):
    import history_ops as H
    c = H.make_ctx(kind)
    try:
        return op.inputs[name](c)
    finally:
        c.close()


@pytest.mark.parametrize("kind", ["48", "32"])
def test_export_and_import_around_call_histories(kind):
    """a store's image imported before a seeded history of the catalogue's operations (those whose launch shape does not follow
    the previous scan), each operation's outputs equal to a fresh context's; then, after the history, the image imported and
    exported again and its keyframes read as on a fresh context that imported it"""
    import history_ops as H
    L = _L()
    s = Store(H.stride(kind), n_kf=4, seed=13)
    img = s.c.kf_export()
    rng = np.random.default_rng(17 if kind == "48" else 19)
    ops = [op for op in H.ops_of(kind) if not op.dev_count and not op.s2m]
    X = H.make_ctx(kind)
    F = H.make_ctx(kind)
    try:
        assert X.kf_import(img) == (0, len(s.edge))
        for _ in range(10):
            op = ops[int(rng.integers(len(ops)))]
            name = sorted(op.inputs)[int(rng.integers(len(op.inputs)))]
            assert op.inputs[name](X) == _fresh(kind, op, name), (op.name, name)
        first, k = X.kf_import(img)
        mapped = list(range(first, first + k))
        assert X.kf_export(mapped) == img
        assert F.kf_import(img) == (0, k) and F.kf_export() == img
        ids = [0, 2, 4, 1]
        poses = [_nudge(s.poses[i], j) for j, i in enumerate(ids)]
        assert _readers(X, s.bp, [mapped[i] for i in ids], poses) == _readers(F, s.bp, ids, poses)
    finally:
        X.close(); F.close(); s.close()
