"""ctypes loader for oracle/_ref/libref_*.so: the reference's own front-end and odometry translation units compiled against the
shim headers of oracle/ref/ (`make -C oracle ref`, run by build() where the reference tree is present) — TEST INFRASTRUCTURE.
Only oracle/_ref/ is opened, never the reference tree."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
NAMES = ("fc", "hz", "rot", "lo", "lo_rot")

PT48 = np.dtype([("x", "f4"), ("y", "f4"), ("z", "f4"), ("w", "f4"), ("nx", "f4"), ("ny", "f4"), ("nz", "f4"), ("nw", "f4"),
                 ("intensity", "f4"), ("curvature", "f4"), ("p0", "f4"), ("p1", "f4")])
PT32 = np.dtype([("x", "f4"), ("y", "f4"), ("z", "f4"), ("w", "f4"), ("intensity", "f4"), ("p0", "f4"), ("p1", "f4"), ("p2", "f4")])


class Pc2Field(C.Structure):
    _fields_ = [("name", C.c_char * 16), ("offset", C.c_uint), ("datatype", C.c_ubyte), ("count", C.c_uint)]


def path(name: str) -> str:
    return os.path.join(REF_DIR, f"libref_{name}.so")


def available() -> bool:
    return all(os.path.exists(path(n)) for n in NAMES)


_libs: dict = {}


def lib(name: str):
    if name not in _libs:
        p = path(name)
        if not os.path.exists(p):
            raise FileNotFoundError(f"{p} is missing: build() compiles it from the reference tree (make -C oracle ref)")
        L = C.CDLL(p)
        vp, dp = C.c_void_p, C.POINTER(C.c_double)
        if name == "fc":
            L.ref_fc_convert.argtypes = [vp, C.c_int, C.c_int, C.c_double, vp, C.c_int]
        elif name == "hz":
            L.ref_hz_create.argtypes = [C.c_double, C.c_double]; L.ref_hz_create.restype = None
            L.ref_hz_imu.argtypes = [C.c_double, dp]; L.ref_hz_imu.restype = None
            L.ref_hz_cloud.argtypes = [C.c_double, vp, C.c_int, C.c_int]
            L.ref_hz_set_q.argtypes = [dp]; L.ref_hz_set_q.restype = None
            L.ref_hz_q_published.argtypes = [dp]; L.ref_hz_q_published.restype = None
            L.ref_hz_take.argtypes = [C.c_int, vp, C.c_int]
        elif name == "rot":
            L.ref_rot_create.argtypes = [C.c_int, C.c_int, dp]; L.ref_rot_create.restype = None
            L.ref_rot_imu.argtypes = [C.c_double, dp]; L.ref_rot_imu.restype = None
            L.ref_rot_cloud.argtypes = [C.c_double, vp, C.c_int, C.c_int]
            L.ref_rot_cloud_pc2.argtypes = [C.c_double, vp, C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.POINTER(Pc2Field), C.c_int, C.c_int]
            L.ref_rot_set_q.argtypes = [dp]; L.ref_rot_set_q.restype = None
            L.ref_rot_q_published.argtypes = [dp]; L.ref_rot_q_published.restype = None
            L.ref_rot_take.argtypes = [C.c_int, vp, C.c_int]
        else:
            L.ref_lo_create.argtypes = []; L.ref_lo_create.restype = None
            L.ref_lo_undistort.argtypes = [vp, C.c_int, dp, dp]; L.ref_lo_undistort.restype = None
            L.ref_lo_transform_cloud.argtypes = [vp, C.c_int, dp, vp]; L.ref_lo_transform_cloud.restype = None
            L.ref_lo_transform_point.argtypes = [vp, C.c_int, dp, vp]; L.ref_lo_transform_point.restype = None
            L.ref_lo_find_surf_corr.argtypes = [vp, C.c_int, vp, C.c_int, dp, vp, vp]
            L.ref_lo_pose_init.argtypes = [dp, dp, dp]; L.ref_lo_pose_init.restype = None
            L.ref_lo_compute_relative.argtypes = [dp, dp, dp]; L.ref_lo_compute_relative.restype = None
            L.ref_lo_map_step.argtypes = [vp, C.c_int, dp, vp, C.c_int, vp, C.POINTER(C.c_int)]
        _libs[name] = L
    return _libs[name]


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _d(a):
    return None if a is None else np.ascontiguousarray(a, np.float64).ctypes.data_as(C.POINTER(C.c_double))


def _vec(a):
    return np.ascontiguousarray(a, np.float64)


# ---------------------------------------------------------------- FormatConvert
def convert_livox(records, stride=None, stamp=0.0):
    """livoxLidarHandler on one CustomMsg (LIVOX20 records, or raw bytes + stride); returns the published PointXYZINormal cloud"""
    a = np.ascontiguousarray(records)
    if stride is None:
        stride = a.dtype.itemsize
    a = a.view(np.uint8).reshape(-1)
    n = a.size // stride
    out = np.zeros(max(n, 1), PT48)
    got = lib("fc").ref_fc_convert(_p(a), n, stride, stamp, _p(out), len(out))
    assert got == n, got
    return out[:n]


# ---------------------------------------------------------------- Preprocessing nodes
class _Node:
    kind = ""
    dtype = PT48

    def imu(self, stamp, gyro):
        getattr(self.L, f"ref_{self.kind}_imu")(float(stamp), _d(_vec(gyro)))

    def set_q(self, q):
        getattr(self.L, f"ref_{self.kind}_set_q")(_d(_vec(q)))

    def cloud(self, stamp, pts, is_dense=False):
        """cloudHandler; returns None while the node queues or waits for IMU, else (surf, edge, cutted, q_iMU at publish)"""
        pts = np.ascontiguousarray(pts, self.dtype)
        before = self.published
        self.published = getattr(self.L, f"ref_{self.kind}_cloud")(float(stamp), _p(pts), len(pts), int(is_dense))
        return self._result(before)

    def _result(self, before):
        if self.published == before:
            return None
        take = getattr(self.L, f"ref_{self.kind}_take")
        outs = []
        for k in range(3):
            n = take(k, None, 0)
            o = np.zeros(max(n, 1), self.dtype)
            take(k, _p(o), len(o))
            outs.append(o[:n])
        q = np.zeros(4)
        getattr(self.L, f"ref_{self.kind}_q_published")(q.ctypes.data_as(C.POINTER(C.c_double)))
        return outs[0], outs[1], outs[2], q


class HorizonNode(_Node):
    """LiLi-OM/src/Preprocessing.cpp's node (one per process at a time: creating another replaces it)"""
    kind, dtype = "hz", PT48

    def __init__(self, surf_thres=0.2, edge_thres=4.0):
        self.L = lib("hz"); self.published = 0
        self.L.ref_hz_create(surf_thres, edge_thres)


class RotNode(_Node):
    """LiLi-OM-ROT/src/Preprocessing.cpp's node (one per process at a time)"""
    kind, dtype = "rot", PT32

    def __init__(self, line_num=64, ds_rate=1, q_lb=(1.0, 0.0, 0.0, 0.0)):
        self.L = lib("rot"); self.published = 0
        self.L.ref_rot_create(int(line_num), int(ds_rate), _d(_vec(q_lb)))

    def cloud_pc2(self, stamp, msg, is_dense=False):
        """cloudHandler on a driver's PointCloud2 (liliom_b200.PC2: payload, geometry, field tuples)"""
        f = (Pc2Field * max(len(msg.fields), 1))()
        for i, (name, off, dt, cnt) in enumerate(msg.fields):
            f[i].name = name.encode()[:15]; f[i].offset = off; f[i].datatype = dt; f[i].count = cnt
        data = np.ascontiguousarray(msg.data)
        before = self.published
        self.published = self.L.ref_rot_cloud_pc2(float(stamp), _p(data), msg.height, msg.width, msg.point_step, msg.row_step, f,
                                                  len(msg.fields), int(is_dense))
        return self._result(before)


def node_run(node, pts, q, t0=0.0, cloud=None):
    """One sweep through a fresh node with q_iMU = q: three clouds queue (the node processes the first when the third arrives),
    one IMU message with zero rate before the scan end makes processIMU multiply q_iMU by deltaQ(0) = identity.  `cloud` is the
    node's handler to call for the processed sweep (default node.cloud)."""
    send = cloud or node.cloud
    empty = np.zeros(0, node.dtype)
    node.imu(t0 + 0.09, (0.0, 0.0, 0.0))
    assert send(t0, pts) is None
    assert node.cloud(t0 + 0.1, empty) is None
    node.set_q(q)
    out = node.cloud(t0 + 0.2, empty)
    assert out is not None
    return out


# ---------------------------------------------------------------- LidarOdometry
class Odometry:
    """LidarOdometry.cpp at member level (variant 0: LiLi-OM, PointXYZINormal; 1: LiLi-OM-ROT, PointXYZI)"""

    def __init__(self, variant=0):
        self.L = lib("lo" if variant == 0 else "lo_rot")
        self.dtype = PT48 if variant == 0 else PT32
        assert self.L.ref_lo_point_size() == self.dtype.itemsize
        self.L.ref_lo_create()

    def points(self, xyz):
        """PointType cloud (default-constructed fields) with the given x, y, z"""
        xyz = np.asarray(xyz, np.float32).reshape(-1, xyz.shape[-1])
        p = np.zeros(len(xyz), self.dtype)
        p["x"] = xyz[:, 0]; p["y"] = xyz[:, 1]; p["z"] = xyz[:, 2]; p["w"] = 1.0
        return p

    def undistort(self, pts, trans, quat=(1.0, 0.0, 0.0, 0.0)):
        out = np.ascontiguousarray(pts, self.dtype).copy()
        self.L.ref_lo_undistort(_p(out), len(out), _d(_vec(trans)), _d(_vec(quat)))
        return out

    def transform_cloud(self, pts, pose7):
        pts = np.ascontiguousarray(pts, self.dtype)
        out = np.zeros(max(len(pts), 1), self.dtype)
        self.L.ref_lo_transform_cloud(_p(pts), len(pts), _d(_vec(pose7)), _p(out))
        return out[:len(pts)]

    def transform_point(self, pts, pose7):
        pts = np.ascontiguousarray(pts, self.dtype)
        out = np.zeros(max(len(pts), 1), self.dtype)
        self.L.ref_lo_transform_point(_p(pts), len(pts), _d(_vec(pose7)), _p(out))
        return out[:len(pts)]

    def find_surf_corr(self, map_pts, feats, pose7):
        """(surf_res_cnt, accepted points, their `normal` points) in the node's order"""
        m = np.ascontiguousarray(map_pts, self.dtype); f = np.ascontiguousarray(feats, self.dtype)
        pts = np.zeros(max(len(f), 1), self.dtype); nrm = np.zeros(max(len(f), 1), self.dtype)
        cnt = self.L.ref_lo_find_surf_corr(_p(m), len(m), _p(f), len(f), _d(_vec(pose7)), _p(pts), _p(nrm))
        return cnt, pts[:cnt], nrm[:cnt]

    def pose_init(self, abs7, rel7):
        out = np.zeros(7)
        self.L.ref_lo_pose_init(_d(_vec(abs7)), _d(_vec(rel7)), out.ctypes.data_as(C.POINTER(C.c_double)))
        return out

    def compute_relative(self, prev7, cur7):
        out = np.zeros(7)
        self.L.ref_lo_compute_relative(None if prev7 is None else _d(_vec(prev7)), _d(_vec(cur7)),
                                       out.ctypes.data_as(C.POINTER(C.c_double)))
        return out

    def map_step(self, surf, pose7, cap):
        """(local map the scan was matched against or None on the initialising scan, the scan's down-sampled cloud)"""
        s = np.ascontiguousarray(surf, self.dtype)
        out = np.zeros(max(cap, 1), self.dtype); ds = np.zeros(max(len(s), 1), self.dtype); nds = C.c_int()
        m = self.L.ref_lo_map_step(_p(s), len(s), _d(_vec(pose7)), _p(out), len(out), _p(ds), C.byref(nds))
        assert m <= cap, (m, cap)
        return (None if m < 0 else out[:m]), ds[:nds.value]
