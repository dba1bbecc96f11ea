"""The streamed workload at its size (BASELINE config 5), driven through the calls bench.py drives it with: a 130k-point HDL-64E
sweep against a 10 M-point local map held as a FIFO of 20 world-frame clouds, with the map maintenance inside the step.

At this size the map's VoxelGrid box is about 1.2 km across (far more than 2^24 cells at leaf 0.4), voxels span the boundaries
between the frames' slabs, and every step rotates the FIFO, so the concatenation the filter sees changes order.  Checked:
  - installing the map (map_clear, 20 x map_push_frame_device from torch tensors, map_rebuild) on a context bound to a torch
    stream with set_stream: map_download_cloud equals the oracle's VoxelGrid(0.4) of the concatenation bit for bit, and
    map_download gives those xyz with w = the point's index;
  - upload_scan + extract_resident + odometry_resident (GN and Ceres-faithful) on that map, every pass re-anchored against an
    oracle kd-tree over the oracle's filtered map (tests/reanchor.py), and want_stats=False returning the same pose bits;
  - the dense probe's shape (every return of the sweep a query, upload_feats + scan_to_map_resident), all 10 passes re-anchored;
  - three streamed steps by the bench's rule (re-push the frame the FIFO is about to drop): context A by map_push_frame_device +
    map_rebuild, context B by map_update_device.  After each, both clouds equal the oracle's VoxelGrid of the rotated
    concatenation bit for bit, A's and B's map_download are identical, and the next scan's pose has the same bits on A and B.

Runtime: 20 to 40 s on one H100 80GB HBM3 host with 8 oracle threads, 8 to 15 s of it the module's world (10 M-point map, its
frames on the device, the oracle's VoxelGrid and kd-tree), built once per module."""
import json

import numpy as np
import pytest

import reanchor as RA
from test_devmath_host import dm  # noqa: F401  (the host build of dev_math.cuh, a fixture)

pytestmark = pytest.mark.gpu

ITERS = 10
NTHREADS = 8
FIELDS = ("x", "y", "z", "intensity")      # PointXYZI; the scan's surf_last_ds is compared on these
IDENT = np.array([1.0, 0, 0, 0, 0, 0, 0])


def _same_cloud(got, want, what, whole=True):
    """Bit for bit: every byte of every record (x, y, z, w, intensity and the padding words) when `whole`, else the fields of
    PointXYZI (x, y, z, intensity).  A failure names the fields that differ."""
    assert len(got) == len(want), (what, len(got), len(want))
    if whole and got.view(np.uint8).tobytes() == want.view(np.uint8).tobytes():
        return
    names = got.dtype.names if whole else FIELDS
    bad = {f: int(np.count_nonzero(got[f].view(np.uint32) != want[f].view(np.uint32))) for f in names}
    assert not any(bad.values()), (what, bad)


def _xyzw(cloud):
    out = np.ones((len(cloud), 4), np.float32)
    out[:, 0] = cloud["x"]; out[:, 1] = cloud["y"]; out[:, 2] = cloud["z"]
    return out


def _say(what, rep):
    print(f"reanchor {what} " + json.dumps({k: float(v) for k, v in rep.items() if k not in ("branches", "n_corr", "lm_iters")}
                                          | ({"branches": sorted(set(rep["branches"]))} if "branches" in rep else {})))


@pytest.fixture(scope="module")
def stream(oracle):
    """The bench's streamed world: bench.make_workload's map and first sweep, bench.make_frames' 20 slabs as device tensors, the
    oracle's filtered map and its kd-tree, the oracle's ROT features of the sweep, and the torch stream the contexts run on."""
    import torch
    import bench
    import liliom_b200 as L
    m, sweeps = bench.make_workload("stream", 10_000_000, 1)
    frames = bench.make_frames(m, L.PT32)
    del m
    assert len(frames) == 20
    frames_dev = [torch.from_numpy(f.view(np.uint8).reshape(-1)).to("cuda") for f in frames]
    torch.cuda.synchronize()
    want = oracle.voxelgrid(np.concatenate(frames), 0.4)
    sw = sweeps[0]
    _, surf_o, _, _, _, _ = oracle.extract_rot(sw["pts"], sw["q"], (1.0, 0, 0, 0), 64, 4)
    prm = L.default_params(1)
    s = torch.cuda.Stream()
    w = dict(frames=frames, frames_dev=frames_dev, want=want, tree=oracle.KdTree(_xyzw(want)), sw=sw, surf_o=surf_o,
             ds_o=oracle.voxelgrid(surf_o, 0.4), prm=prm, torch_stream=s, ctxs=[])
    yield w
    for c in w["ctxs"]:
        c.close()
    torch.cuda.synchronize()


def _close(w, *cs):
    """Give a context's 10 M-point map back as soon as its test is done with it."""
    for c in cs:
        c.close()
        w["ctxs"].remove(c)


def _install(w):
    import liliom_b200 as L
    c = L.Context(w["prm"])
    w["ctxs"].append(c)
    c.set_stream(w["torch_stream"].cuda_stream)
    c.map_clear()
    for fd in w["frames_dev"]:
        c.map_push_frame_device(fd.data_ptr(), fd.numel() // L.PT32.itemsize, IDENT)
    return c, c.map_rebuild()


def _scan(c, sw, want_stats=True, mode=None, iters=ITERS, cap=0):
    import liliom_b200 as L
    c.upload_scan(sw["pts"])
    c.extract_resident(sw["q"])
    return c.odometry_resident(sw["guess"], iters, mode=L.MODE_GN if mode is None else mode, want_stats=want_stats,
                               want_ds=cap > 0, cap=cap)


def test_install_and_scan_to_map_at_size(oracle, dm, stream):  # noqa: F811
    import liliom_b200 as L
    w = stream
    c, n = _install(w)
    want = w["want"]
    print(f"stream map: {sum(len(f) for f in w['frames'])} points in 20 frames -> {n} after VoxelGrid(0.4)")
    assert n == len(want) and 9_000_000 < n < 10_000_000
    x, y = want["x"], want["y"]
    cells = (np.ptp(x) / 0.4) * (np.ptp(y) / 0.4) * (np.ptp(want["z"]) / 0.4)
    assert np.ptp(x) > 1000 and cells > 2 ** 24          # the box the issue's size reaches
    _same_cloud(c.map_download_cloud(), want, "install")                          # every byte of every record
    xyzw = c.map_download()
    assert len(xyzw) == n
    assert np.array_equal(xyzw[:, :3].view(np.uint32), _xyzw(want)[:, :3].view(np.uint32))
    assert np.array_equal(xyzw[:, 3].view(np.int32), np.arange(n, dtype=np.int32))
    sw, ds_o, tree = w["sw"], w["ds_o"], w["tree"]
    pc, _ = _install(w)                       # the device's own correspondences come from a second context with the same map
    pr = lambda pose: pc.find_surf_corr(ds_o, pose)[:2]  # noqa: E731
    # the resident leg's call, twice (the first sizes its launches from the upper bound, the second is one persistent launch)
    for call in range(2):
        pose, st, ds = _scan(c, sw, cap=len(sw["pts"]))
        _same_cloud(ds, ds_o, f"surf_last_ds call {call}", whole=False)
        rep = RA.check_gn(oracle, tree, ds_o, sw["guess"], st, dm, NTHREADS, f"stream/odometry_resident/call{call}", pr)
        _say(f"stream/odometry_resident/call{call}", rep)
        assert st[0].n_corr > 0.5 * len(ds_o)
    pose_n, none, nds = _scan(c, sw, want_stats=False)
    assert none is None and nds == len(ds_o) and pose_n.tobytes() == pose.tobytes()
    _, st, _ = _scan(c, sw, mode=L.MODE_CERES, iters=2)
    _say("stream/odometry_resident/ceres", RA.check_ceres(oracle, tree, ds_o, sw["guess"], st, 15, NTHREADS, "stream/ceres", pr))
    # the dense probe's shape: every return of the sweep a query
    feats = _xyzw(sw["pts"])
    c.upload_feats(feats)
    pose_d, st = c.scan_to_map_resident(sw["guess"], ITERS, mode=L.MODE_GN, want_stats=True)
    pose_dn, _ = c.scan_to_map_resident(sw["guess"], ITERS, mode=L.MODE_GN, want_stats=False)
    assert pose_dn.tobytes() == pose_d.tobytes()
    rep = RA.check_gn(oracle, tree, feats, sw["guess"], st, dm, NTHREADS, "stream/dense", lambda pose: pc.find_surf_corr(feats, pose)[:2])
    _say("stream/dense", rep)
    assert st[0].n_corr > 0.3 * len(feats)
    _close(w, c, pc)


def test_streamed_steps_rebuild_and_incremental(oracle, dm, stream):  # noqa: F811
    """Three steps by the bench's rule: push number p re-pushes frame p % 20, the one the FIFO is about to drop."""
    import liliom_b200 as L
    w = stream
    a, na = _install(w)
    b, nb = _install(w)
    assert na == nb == len(w["want"])
    sw = w["sw"]
    for c in (a, b):                          # both contexts make the same calls from here on: the same launch shapes
        _scan(c, sw, want_stats=False)
    order = list(range(20))
    for p in range(3):
        j = p % 20
        fd = w["frames_dev"][j]
        n = fd.numel() // L.PT32.itemsize
        a.map_push_frame_device(fd.data_ptr(), n, IDENT)
        ma = a.map_rebuild()
        mb = b.map_update_device(fd.data_ptr(), n, IDENT)
        order = order[1:] + [j]
        want = oracle.voxelgrid(np.concatenate([w["frames"][k] for k in order]), 0.4)
        assert ma == mb == len(want), (p, ma, mb, len(want))
        _same_cloud(a.map_download_cloud(), want, f"rebuild step {p}")
        _same_cloud(b.map_download_cloud(), want, f"incremental step {p}")
        da, db = a.map_download(), b.map_download()
        assert da.tobytes() == db.tobytes(), p
        pa, _, _ = _scan(a, sw, want_stats=False)
        pb, _, _ = _scan(b, sw, want_stats=False)
        assert pa.tobytes() == pb.tobytes(), (p, pa, pb)
    # the last step's map (the FIFO rotated by three frames) through the checker
    tree = oracle.KdTree(_xyzw(want))
    _, st, _ = _scan(a, sw)
    rep = RA.check_gn(oracle, tree, w["ds_o"], sw["guess"], st, dm, NTHREADS, "stream/after 3 steps",
                      lambda pose: b.find_surf_corr(w["ds_o"], pose)[:2])
    _say("stream/after 3 steps", rep)
    _close(w, a, b)
