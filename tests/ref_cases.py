"""The inputs on which the reference's own front-end and odometry code (oracle/_ref/libref_*.so, tests/ref_lib.py) is compared with
the oracle (test_ref_pinned_cpu.py) and with the device (test_gpu_ref_pinned.py), and the reference's outputs on them.

Every case has an id, its inputs (built here from seeded generators) and a `reference()` that runs the compiled reference on them.
tests/golden/ref_pinned.json holds, per case, the SHA-256 of the inputs and of every cloud the reference published, and the q it
published with (`python tests/make_golden_ref.py` writes it where the libraries are built).  So the device is checked against
the reference's own outputs on machines where the reference tree, and so oracle/_ref/, is absent."""
from __future__ import annotations

import hashlib
import json
import os

import numpy as np

import ref_lib as R

F = np.float32
DBL_EPS = np.finfo(np.float64).eps
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pinned.json")
Q_LB = np.array([0.9238795325112867, 0.0, 0.0, 0.3826834323650898]) * 1.0000001


# ------------------------------------------------------------------------------------------------------------ digests
def canon(a) -> bytes:
    """the bytes of an array with every NaN made the one quiet NaN (a NaN's sign and payload follow the compiler's operand order,
    not the arithmetic); point clouds of both layouts are float32 throughout"""
    a = np.ascontiguousarray(a)
    if a.dtype.fields is not None or a.dtype == np.float32:
        f = a.view(np.float32).reshape(-1).copy()
        f[np.isnan(f)] = np.float32("nan")
        return f.tobytes()
    if a.dtype == np.float64:
        f = a.reshape(-1).copy()
        f[np.isnan(f)] = np.nan
        return f.tobytes()
    return a.tobytes()


def digest(a) -> list:
    """[count, sha256 of canon(a)]"""
    return [int(len(a)) if np.ndim(a) else 1, hashlib.sha256(canon(a)).hexdigest()]


def q_hex(q) -> list:
    return [float(v).hex() for v in np.asarray(q, np.float64)]


def q_of(hexes) -> np.ndarray:
    return np.array([float.fromhex(h) for h in hexes], np.float64)


def record(inputs, outputs: dict) -> dict:
    """the fixture entry of one case: input digest, output digests, and q (hex) when the case publishes one"""
    e = {"in": digest(inputs)}
    for k, v in outputs.items():
        e[k] = q_hex(v) if k == "q" else digest(v)
    return e


def load_golden() -> dict:
    with open(GOLDEN) as fh:
        return json.load(fh)["cases"]


# ------------------------------------------------------------------------------------------------------------ inputs
def make_world_small():
    """the conftest world_small fixture, rebuilt for the fixture writer"""
    from liliom_b200 import synth
    m, _ = synth.make_map(100_000)
    T = synth.default_true_pose()
    hz, q_hz = synth.make_horizon_sweep(T)
    hdl, q_hdl = synth.make_hdl64_sweep(T)
    return dict(map=m, T=T, guess=synth.perturbed_pose(T), hz=hz, q_hz=q_hz, hdl=hdl, q_hdl=q_hdl)


def hz_safe(pts):
    """The Horizon node indexes mat[scan_id] without a bound (L/src/Preprocessing.cpp:265-267): a point of line >= 6 that passes
    the depth and reflectivity gates would be written past the array.  Such points are left out; lines >= 6 that fail the
    reflectivity gate (decided on the stored float alone) stay in and reach the cutted cloud."""
    inten = pts["intensity"].astype(np.float64)
    curv = pts["curvature"].astype(np.float64)
    hi_line = np.isfinite(inten) & (inten >= 6.0) & (inten < 2.0 ** 31)
    gate_open = (curv >= 0.05) & (curv <= 25.45)
    return pts[~(hi_line & gate_open)]


def hz_sweeps(world_small):
    import hz_adversarial as H
    return [("world_small", dict(pts=world_small["hz"], q=world_small["q_hz"]))] + list(H.all_sweeps())


def imu_streams():
    rng = np.random.default_rng(17)
    t0, t_cur = 10.0, 10.1
    g = lambda n: rng.normal(0.0, 0.4, (n, 3))
    out = {}
    st = np.sort(t0 - 0.02 + rng.uniform(0, 0.15, 40)); out["irregular"] = list(zip(st, g(40)))
    st = np.concatenate([t0 + 0.005 * np.arange(20), [t_cur], t_cur + 0.005 * np.arange(1, 5)])
    out["stamp_at_scan_time"] = list(zip(st, g(len(st))))
    out["single"] = [(t0 + 0.03, g(1)[0])]
    st = t0 - 0.0025 + 0.005 * np.arange(30); out["interpolated"] = list(zip(st, g(30)))
    return t0, t_cur, out


def rot_cut_nonempty(pts):
    """at least one finite point at 3 m or more: the ROT node reads points[0] of the cut cloud (R/src/Preprocessing.cpp:285)"""
    fin = np.isfinite(pts["x"]) & np.isfinite(pts["y"]) & np.isfinite(pts["z"])
    with np.errstate(over="ignore", invalid="ignore"):
        r2 = (pts["x"] * pts["x"] + pts["y"] * pts["y"]) + pts["z"] * pts["z"]
    return bool((fin & (r2 >= F(9.0))).any())


def rot_tied(cut, curv, line_num):
    """True when some sort range of the classifier (R/src/Preprocessing.cpp:405-410: six per ring) holds two candidates (curvature
    > 2.0 or < 0.1) of equal curvature.  The reference sorts with std::sort, which is not stable; the oracle DEFINES the order of
    equal curvatures as ascending index, so the features of such a sweep are the oracle's definition, not the reference's."""
    ring = np.array([int(v) for v in cut["intensity"]])
    start = 0
    for r in range(line_num):
        cnt = int((ring == r).sum())
        sp0, ep0 = start + 5, start + cnt - 6
        start += cnt
        if ep0 - sp0 < 6:
            continue
        for j in range(6):
            sp = sp0 + (ep0 - sp0) * j // 6; ep = sp0 + (ep0 - sp0) * (j + 1) // 6 - 1
            c = curv[sp:ep + 1]
            c = c[(c > 2.0) | (c < 0.1)]
            if len(np.unique(c)) != len(c):
                return True
    return False


INTENSITIES = [-0.3, -1.05, -2147483904.0, 0.0, 3.0, 5.0, F(0.1), F(2.1), F(1.0999999), F(0.05), 16777217.0, 16777216.0 + 0.5,
               2147483648.0, 3.0e9, 1e38, np.nan, np.inf, -np.inf, F(0.0999999), F(4.0999999)]


def quats():
    e = DBL_EPS
    return {"identity": (1.0, 0.0, 0.0, 0.0), "negative_w": (-0.8, 0.1, -0.5, 0.3), "half_turn": (0.0, 0.0, 0.0, 1.0),
            "non_unit": (1.7, 0.2, -0.4, 0.9), "at_one_minus_eps": (1.0 - e, 0.0, 0.0, 0.0),
            "below_one_minus_eps": (1.0 - 2 * e, 1e-8, 0.0, 0.0), "above_one_minus_eps": (np.nextafter(1.0 - e, 2.0), 1e-8, 0.0, 0.0)}


def dtype_of(variant):
    return R.PT48 if variant == 0 else R.PT32


def points(dtype, xyz):
    """PointType cloud (default-constructed fields) with the given x, y, z"""
    xyz = np.asarray(xyz, np.float32).reshape(len(xyz), -1)
    p = np.zeros(len(xyz), dtype)
    p["x"] = xyz[:, 0]; p["y"] = xyz[:, 1]; p["z"] = xyz[:, 2]; p["w"] = 1.0
    return p


def lo_cloud(dtype, n, seed):
    """a cloud for undistortion and transformCloud: every edge intensity, random normals and reflectivity"""
    rng = np.random.default_rng(seed)
    p = points(dtype, rng.uniform(-30, 30, (n, 3)))
    p["intensity"] = np.resize(np.asarray(INTENSITIES, F), n)
    if "nx" in p.dtype.names:
        p["nx"], p["ny"], p["nz"] = rng.normal(size=(3, n)).astype(F); p["curvature"] = rng.uniform(0, 25, n).astype(F)
    return p


def velodyne_msg(pts):
    """the cloud as a Velodyne driver publishes it: x, y, z, intensity (FLOAT32), ring (UINT16), 20-byte points"""
    import liliom_b200 as L
    rec = np.zeros(len(pts), [("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4"), ("ring", "<u2"), ("pad", "<u2")])
    for f in ("x", "y", "z", "intensity"):
        rec[f] = pts[f]
    fields = [("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("intensity", 12, 7, 1), ("ring", 16, 4, 1)]
    return L.PC2(rec.view(np.uint8).reshape(-1).copy(), 1, len(pts), 20, 20 * len(pts), fields)


# ------------------------------------------------------------------------------------------------------------ cases
class Case:
    def __init__(self, cid, inputs, reference, **kw):
        self.id, self.inputs, self._ref = cid, inputs, reference
        self.__dict__.update(kw)

    def reference(self) -> dict:
        return self._ref()


def _node_out(out):
    surf, edge, cut, q = out
    return dict(surf=surf, edge=edge, cut=cut, q=q)


def hz_cases(world_small):
    """the Horizon node (L/src/Preprocessing.cpp) on world_small and every hz_adversarial sweep, q_iMU = the sweep's q"""
    out = []
    for name, sw in hz_sweeps(world_small):
        pts = hz_safe(np.ascontiguousarray(sw["pts"], R.PT48))
        out.append(Case(f"hz/{name}", pts, lambda pts=pts, q=sw["q"]: _node_out(R.node_run(R.HorizonNode(), pts, q)), pts=pts))
    return out


def livox_cases():
    """FormatConvert on every hz_adversarial Livox message but the lines >= 6 (which the Horizon node would write outside its
    cell array), and its cloud through the Horizon node at q = identity"""
    import hz_adversarial as H
    out = []
    for name, recs, stride in H.livox_messages():
        if name == "line_6_255":
            continue

        def ref(recs=recs, stride=stride):
            conv = R.convert_livox(recs, stride)
            d = _node_out(R.node_run(R.HorizonNode(), conv, (1.0, 0.0, 0.0, 0.0)))
            d["conv"] = conv
            return d
        out.append(Case(f"livox/{name}", np.ascontiguousarray(recs).view(np.uint8), ref, recs=recs, stride=stride))
    return out


def rot_world_cases(world_small):
    """the ROT node on world_small's HDL-64 sweep at 16 / 32 / 64 lines, ds_rate 1 and 2, both q_lb, as a typed cloud and as the
    driver's PointCloud2"""
    pts = np.ascontiguousarray(world_small["hdl"], R.PT32)
    out = []
    for ln in (16, 32, 64):
        for ds in (1, 2):
            for k, qlb in enumerate(((1.0, 0.0, 0.0, 0.0), Q_LB)):
                out.append(Case(f"rot/{ln}/{ds}/{k}", pts, lambda ln=ln, ds=ds, qlb=qlb: _node_out(
                    R.node_run(R.RotNode(ln, ds, qlb), pts, world_small["q_hdl"])), pts=pts, ln=ln, ds=ds, qlb=qlb, pc2=False))

                def ref_pc2(ln=ln, ds=ds, qlb=qlb):
                    node = R.RotNode(ln, ds, qlb)
                    return _node_out(R.node_run(node, velodyne_msg(pts), world_small["q_hdl"], cloud=node.cloud_pc2))
                out.append(Case(f"rot_pc2/{ln}/{ds}/{k}", pts, ref_pc2, pts=pts, ln=ln, ds=ds, qlb=qlb, pc2=True))
    return out


def rot_adv_cases():
    """the ROT node on every rot_adversarial sweep with a point past the 3 m cut, at its own settings"""
    import rot_adversarial as RA
    out = []
    for name, sw in RA.all_sweeps():
        if not rot_cut_nonempty(sw["pts"]):
            continue
        pts = np.ascontiguousarray(sw["pts"], R.PT32)
        out.append(Case(f"rot_adv/{name}", pts, lambda pts=pts, sw=sw: _node_out(
            R.node_run(R.RotNode(sw["line_num"], sw["ds_rate"], sw["q_lb"]), pts, sw["q_imu"])), pts=pts, sw=sw))
    return out


def undist_cases(variant):
    """LidarOdometry::undistortion on every edge intensity and quaternion, with and without a translation"""
    pts = lo_cloud(dtype_of(variant), 200, 3 + variant)
    out = []
    for name, q in quats().items():
        for k, trans in enumerate(((0.0, 0.0, 0.0), (0.31, -1.7, 0.05))):
            out.append(Case(f"undist/{variant}/{name}/{k}", pts, lambda q=q, trans=trans: dict(
                out=R.Odometry(variant).undistort(pts, trans, q)), pts=pts, q=q, trans=trans))
    return out


def surf_worlds(world_small):
    """(name, map n x 4, queries n x 4, pose): world_small's down-sampled Horizon features against its map, and every
    s2m_adversarial world"""
    import oracle_lib as O
    import s2m_adversarial as S
    surf, _, _ = O.extract_horizon(world_small["hz"], world_small["q_hz"])
    ds = O.voxelgrid(surf, 0.4)
    f4 = np.ones((len(ds), 4), F); f4[:, 0], f4[:, 1], f4[:, 2] = ds["x"], ds["y"], ds["z"]
    out = [("world_small", np.ascontiguousarray(world_small["map"], F).reshape(-1, 4), f4, np.asarray(world_small["guess"], np.float64))]
    for w in S.WORLDS:
        W = S.s2m_world(w)
        out.append((w, np.ascontiguousarray(W["map"], F), np.ascontiguousarray(W["feats"], F), np.asarray(W["pose"], np.float64)))
    return out


def surf_cases(variant, world_small):
    """findCorrespondingSurfFeatures: the accepted points in order and their planes (x, y, z, intensity of the `normal` point)"""
    dt = dtype_of(variant)
    out = []
    for name, m4, q4, pose in surf_worlds(world_small):
        feats = points(dt, q4[:, :3])

        def ref(m4=m4, feats=feats, pose=pose):
            cnt, pts, nrm = R.Odometry(variant).find_surf_corr(points(dt, m4[:, :3]), feats, pose)
            return dict(pts=pts, plane=np.stack([nrm["x"], nrm["y"], nrm["z"], nrm["intensity"]], 1))
        out.append(Case(f"surf/{variant}/{name}", np.concatenate([m4.reshape(-1), q4.reshape(-1)]), ref, m4=m4, feats=feats, pose=pose))
    return out


def map_steps(variant, world_small):
    """26 scans of the odometry's map maintenance: random thirds of the extracted features, scan 7 empty, a moving pose"""
    import oracle_lib as O
    if variant == 0:
        surf, _, _ = O.extract_horizon(world_small["hz"], world_small["q_hz"])
    else:
        _, surf, _, _, _, _ = O.extract_rot(world_small["hdl"], world_small["q_hdl"])
    surf = np.ascontiguousarray(surf, dtype_of(variant))
    rng = np.random.default_rng(21)
    steps = []
    for k in range(26):
        s = surf[np.sort(rng.permutation(len(surf))[: len(surf) // 3])] if k != 7 else surf[:0]
        pose = np.array(world_small["T"], np.float64); pose[4] += 0.3 * k; pose[5] -= 0.07 * k
        steps.append((s, pose))
    return steps, 21 * len(surf) + 1


def map_case(variant, world_small):
    """buildLocalMap + downSampleCloud over the 26 scans: map<k> the local map scan k was matched against (k >= 1), ds<k> its own
    down-sampled cloud"""
    steps, cap = map_steps(variant, world_small)

    def ref():
        od = R.Odometry(variant)
        d = {}
        for k, (s, pose) in enumerate(steps):
            m, ds = od.map_step(s, pose, cap)
            if m is not None:
                d[f"map{k}"] = m; d[f"ds{k}"] = ds
        return d
    return Case(f"map/{variant}", np.concatenate([s for s, _ in steps]), ref, steps=steps)


def node_cases(variant, world_small):
    """the Preprocessing node (Horizon or ROT at 64 lines, ds_rate 4) over one IMU stream and three clouds"""
    t0, t_cur, streams = imu_streams()
    pts = world_small["hz"] if variant == 0 else world_small["hdl"]
    seq = ((t0, pts), (t_cur, pts[:0]), (t_cur + 0.1, pts[:0]))
    out = []
    for name, stream in streams.items():
        def ref(stream=stream):
            node = R.HorizonNode() if variant == 0 else R.RotNode(64, 4)
            for st, gy in stream:
                node.imu(st, gy)
            res = [node.cloud(stamp, cl) for stamp, cl in seq]
            assert res[0] is None and res[1] is None and res[2] is not None
            return _node_out(res[2])
        gyro = np.array([[st, *gy] for st, gy in stream], np.float64)
        out.append(Case(f"node/{variant}/{name}", gyro, ref, stream=stream, seq=seq))
    return out


def all_cases(world_small):
    cases = hz_cases(world_small) + livox_cases() + rot_world_cases(world_small) + rot_adv_cases()
    for v in (0, 1):
        cases += undist_cases(v) + surf_cases(v, world_small) + [map_case(v, world_small)] + node_cases(v, world_small)
    return cases
