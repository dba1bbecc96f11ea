"""ctypes loader for oracle/liboracle.so — TEST INFRASTRUCTURE (the product never imports this)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
SO = os.path.join(ORACLE_DIR, "liboracle.so")

PT48 = np.dtype([("x", "f4"), ("y", "f4"), ("z", "f4"), ("w", "f4"), ("nx", "f4"), ("ny", "f4"), ("nz", "f4"), ("nw", "f4"),
                 ("intensity", "f4"), ("curvature", "f4"), ("p0", "f4"), ("p1", "f4")])
PT32 = np.dtype([("x", "f4"), ("y", "f4"), ("z", "f4"), ("w", "f4"), ("intensity", "f4"), ("p0", "f4"), ("p1", "f4"), ("p2", "f4")])


class IterStats(C.Structure):
    _fields_ = [("n_corr", C.c_int), ("lm_iters", C.c_int), ("cost", C.c_double), ("jtj_jtr", C.c_double * 27), ("pose7", C.c_double * 7)]


def build():
    srcs = [os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.endswith((".cpp", ".h")) or f == "Makefile"]
    if os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(s) for s in srcs):
        return
    subprocess.run(["make", "-C", ORACLE_DIR], check=True, capture_output=True)


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(SO)
        vp, dp, ip = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)
        L.orc_voxelgrid.argtypes = [vp, C.c_int, C.c_int, C.c_float, vp, C.c_int]
        L.orc_kdtree_build.argtypes = [vp, C.c_int]; L.orc_kdtree_build.restype = vp
        L.orc_kdtree_free.argtypes = [vp]; L.orc_kdtree_free.restype = None
        L.orc_knn5.argtypes = [vp, vp, C.c_int, vp, vp, C.c_int]; L.orc_knn5.restype = None
        L.orc_knn5_brute.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp]; L.orc_knn5_brute.restype = None
        L.orc_find_surf_corr.argtypes = [vp, vp, C.c_int, vp, C.c_int, dp, vp, vp, vp, vp, C.c_int]
        L.orc_normal_equations.argtypes = [vp, C.c_int, vp, vp, dp, C.c_double, dp]; L.orc_normal_equations.restype = None
        L.orc_scan_to_map_gn.argtypes = [vp, vp, C.c_int, vp, C.c_int, dp, C.c_int, C.POINTER(IterStats), C.c_int]
        L.orc_scan_to_map_ceres.argtypes = [vp, vp, C.c_int, vp, C.c_int, dp, C.c_int, C.c_int, C.POINTER(IterStats), C.c_int]
        L.orc_ceres_solve.argtypes = [vp, C.c_int, vp, vp, dp, C.c_int, dp]
        L.orc_extract_horizon.argtypes = [vp, C.c_int, dp, C.c_double, C.c_double, vp, ip, vp, ip, vp, ip]
        L.orc_extract_rot.argtypes = [vp, C.c_int, dp, dp, C.c_int, C.c_int, vp, ip, vp, ip, vp, ip, vp, vp]
        L.orc_correspond_edge.argtypes = [vp, vp, C.c_int, vp, C.c_int, dp, C.c_int, vp, vp, vp]
        L.orc_correspond_surf_backend.argtypes = [vp, vp, C.c_int, vp, C.c_int, dp, C.c_double, C.c_double, C.c_double, C.c_double,
                                                  vp, vp, C.c_double, vp, vp, vp]
        L.orc_backend_edge_block.argtypes = [vp, C.c_int, vp, vp, vp, C.c_double, dp, C.c_double, dp]; L.orc_backend_edge_block.restype = None
        L.orc_backend_surf_block.argtypes = [vp, C.c_int, vp, vp, vp, dp, dp, dp, C.c_double, dp]; L.orc_backend_surf_block.restype = None
        L.orc_convert_livox.argtypes = [vp, C.c_int, C.c_int, vp]; L.orc_convert_livox.restype = None
        L.orc_solve_rotation.argtypes = [dp, dp, dp, C.c_double]; L.orc_solve_rotation.restype = None
        L.orc_pose_compose.argtypes = [dp, dp, dp]; L.orc_pose_compose.restype = None
        L.orc_pose_relative.argtypes = [dp, dp, dp]; L.orc_pose_relative.restype = None
        L.orc_transform_cloud.argtypes = [vp, C.c_int, C.c_int, dp, vp]; L.orc_transform_cloud.restype = None
        L.orc_undistort.argtypes = [vp, C.c_int, C.c_int, dp, dp]; L.orc_undistort.restype = None
        L.orc_eigen_sym3.argtypes = [dp, dp, dp]; L.orc_eigen_sym3.restype = None
        L.orc_colpiv_qr_solve.argtypes = [C.c_int, dp, dp, dp]; L.orc_colpiv_qr_solve.restype = None
        L.orc_slerp_identity.argtypes = [dp, C.c_double, dp]; L.orc_slerp_identity.restype = None
        L.orc_fit_gate_batch.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp, vp]; L.orc_fit_gate_batch.restype = None
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def voxelgrid(pts, leaf):
    pts = np.ascontiguousarray(pts)
    out = np.zeros(max(len(pts), 1), pts.dtype)
    m = lib().orc_voxelgrid(_p(pts), len(pts), pts.dtype.itemsize, leaf, _p(out), len(out))
    return out[:m]


class KdTree:
    def __init__(self, map_xyzw):
        self.map = np.ascontiguousarray(map_xyzw, dtype=np.float32).reshape(-1, 4)
        self.h = lib().orc_kdtree_build(_p(self.map), len(self.map))

    def __del__(self):
        try:
            lib().orc_kdtree_free(self.h)
        except Exception:
            pass

    def knn5(self, q, nthreads=1):
        q = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, 4)
        idx = np.zeros((len(q), 5), np.int32); sqd = np.zeros((len(q), 5), np.float32)
        lib().orc_knn5(self.h, _p(q), len(q), _p(idx), _p(sqd), nthreads)
        return idx, sqd


def knn5_brute(map_xyzw, q):
    m = np.ascontiguousarray(map_xyzw, dtype=np.float32).reshape(-1, 4)
    q = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, 4)
    idx = np.zeros((len(q), 5), np.int32); sqd = np.zeros((len(q), 5), np.float32)
    lib().orc_knn5_brute(_p(m), len(m), _p(q), len(q), _p(idx), _p(sqd))
    return idx, sqd


def _f4(feats):
    feats = np.ascontiguousarray(feats)
    if feats.dtype.fields is not None:
        out = np.ones((len(feats), 4), np.float32)
        out[:, 0] = feats["x"]; out[:, 1] = feats["y"]; out[:, 2] = feats["z"]
        return out
    return np.ascontiguousarray(feats, dtype=np.float32).reshape(-1, 4)


def find_surf_corr(tree: KdTree, feats, pose7, nthreads=1):
    f = _f4(feats); n = len(f)
    pose = np.asarray(pose7, np.float64)
    valid = np.zeros(max(n, 1), np.uint8); plane = np.zeros((max(n, 1), 4), np.float32)
    idx = np.zeros((max(n, 1), 5), np.int32); pw = np.zeros((max(n, 1), 4), np.float32)
    cnt = lib().orc_find_surf_corr(tree.h, _p(tree.map), len(tree.map), _p(f), n, _d(pose), _p(valid), _p(plane), _p(idx), _p(pw), nthreads)
    return cnt, valid[:n], plane[:n], idx[:n], pw[:n]


def normal_equations(feats, valid, plane, pose7, a=0.1):
    f = _f4(feats)
    out = np.zeros(29)
    lib().orc_normal_equations(_p(f), len(f), _p(np.ascontiguousarray(valid)), _p(np.ascontiguousarray(plane)), _d(np.asarray(pose7, np.float64)), a, _d(out))
    return out


def scan_to_map_gn(tree: KdTree, feats, pose7, iters, nthreads=1):
    f = _f4(feats)
    pose = np.array(pose7, np.float64)
    st = (IterStats * max(iters, 1))()
    rc = lib().orc_scan_to_map_gn(tree.h, _p(tree.map), len(tree.map), _p(f), len(f), _d(pose), iters, st, nthreads)
    return rc, pose, [st[i] for i in range(iters)]


def scan_to_map_ceres(tree: KdTree, feats, pose7, match_cnt, max_num_iter, nthreads=1):
    f = _f4(feats)
    pose = np.array(pose7, np.float64)
    st = (IterStats * max(match_cnt, 1))()
    rc = lib().orc_scan_to_map_ceres(tree.h, _p(tree.map), len(tree.map), _p(f), len(f), _d(pose), match_cnt, max_num_iter, st, nthreads)
    return rc, pose, [st[i] for i in range(match_cnt)]


def extract_horizon(pts, q_imu, surf_thres=0.2, edge_thres=4.0):
    pts = np.ascontiguousarray(pts, dtype=PT48); n = len(pts)
    surf = np.zeros(max(n, 1), PT48); edge = np.zeros(max(n, 1), PT48); cut = np.zeros(max(n, 1), PT48)
    ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
    lib().orc_extract_horizon(_p(pts), n, _d(np.asarray(q_imu, np.float64)), surf_thres, edge_thres, _p(surf), C.byref(ns), _p(edge), C.byref(ne), _p(cut), C.byref(nc))
    return surf[:ns.value], edge[:ne.value], cut[:nc.value]


def extract_rot(pts, q_imu, q_lb=(1.0, 0, 0, 0), line_num=64, ds_rate=4):
    pts = np.ascontiguousarray(pts, dtype=PT32); n = len(pts)
    surf = np.zeros(max(n, 1), PT32); edge = np.zeros(max(n, 1), PT32); cut = np.zeros(max(n, 1), PT32)
    lab = np.zeros(max(n, 1), np.int32); cur = np.zeros(max(n, 1), np.float32)
    ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
    rc = lib().orc_extract_rot(_p(pts), n, _d(np.asarray(q_imu, np.float64)), _d(np.asarray(q_lb, np.float64)), line_num, ds_rate,
                               _p(surf), C.byref(ns), _p(edge), C.byref(ne), _p(cut), C.byref(nc), _p(lab), _p(cur))
    return rc, surf[:ns.value], edge[:ne.value], cut[:nc.value], lab[:nc.value], cur[:nc.value]


def correspond_edge(tree: KdTree, feats, pose7, variant=0):
    f = _f4(feats); n = len(f)
    valid = np.zeros(max(n, 1), np.uint8); pa = np.zeros((max(n, 1), 3), np.float32); pb = np.zeros((max(n, 1), 3), np.float32)
    lib().orc_correspond_edge(tree.h, _p(tree.map), len(tree.map), _p(f), n, _d(np.asarray(pose7, np.float64)), variant, _p(valid), _p(pa), _p(pb))
    return valid[:n], pa[:n], pb[:n]


def correspond_surf_backend(tree: KdTree, feats, pose7, kd_max_radius=1.0, surf_dist_thres=0.06, w_gate=0.3, lidar_const=1.0,
                            map_refl=None, feat_refl=None, reflect_thres=0.0):
    f = _f4(feats); n = len(f)
    valid = np.zeros(max(n, 1), np.uint8); plane = np.zeros((max(n, 1), 4), np.float32); score = np.zeros(max(n, 1), np.float64)
    mr = None if map_refl is None else np.ascontiguousarray(map_refl, np.float32)
    fr = None if feat_refl is None else np.ascontiguousarray(feat_refl, np.float32)
    lib().orc_correspond_surf_backend(tree.h, _p(tree.map), len(tree.map), _p(f), n, _d(np.asarray(pose7, np.float64)), kd_max_radius,
                                      surf_dist_thres, w_gate, lidar_const, _p(mr), _p(fr), reflect_thres, _p(valid), _p(plane), _p(score))
    return valid[:n], plane[:n], score[:n]


def transform_cloud(pts, pose7):
    pts = np.ascontiguousarray(pts)
    out = np.zeros_like(pts)
    lib().orc_transform_cloud(_p(pts), len(pts), pts.dtype.itemsize, _d(np.asarray(pose7, np.float64)), _p(out))
    return out


def undistort(pts, trans, quat=(1.0, 0.0, 0.0, 0.0)):
    out = np.ascontiguousarray(pts).copy()
    t = np.asarray(trans, np.float64); q = np.asarray(quat, np.float64)
    lib().orc_undistort(_p(out), len(out), out.dtype.itemsize, _d(t), _d(q))
    return out


def eigen_sym3(a):
    a = np.ascontiguousarray(a, np.float64).reshape(9)
    ev = np.zeros(3); vec = np.zeros(9)
    lib().orc_eigen_sym3(_d(a), _d(ev), _d(vec))
    return ev, vec.reshape(3, 3)


def colpiv_qr_solve(A, b):
    A = np.ascontiguousarray(A, np.float64); b = np.ascontiguousarray(b, np.float64)
    x = np.zeros(3)
    lib().orc_colpiv_qr_solve(len(A), _d(A.reshape(-1)), _d(b), _d(x))
    return x


def fit_gate(m, s, plane_thres=0.06, w_gate=0.4):
    """L/src/LidarOdometry.cpp:369-405 on n neighbourhoods m (n x 5 x 4 fp32) and transformed queries s (n x 3 fp32): the QR
    plane fit and both gates at the thresholds (scalars or one per neighbourhood).  Returns (ok, plane, weight, the QR's un-normalised normal)."""
    m = np.ascontiguousarray(m, np.float32).reshape(-1, 5, 4); s = np.ascontiguousarray(s, np.float32).reshape(-1, 3)
    n = len(m)
    ok = np.zeros(max(n, 1), np.uint8); plane = np.zeros((max(n, 1), 4), np.float32)
    w = np.zeros(max(n, 1), np.float32); nv = np.zeros((max(n, 1), 3))
    thr = np.ascontiguousarray(np.broadcast_to(np.asarray(plane_thres, np.float64), (n,)))
    wg = np.ascontiguousarray(np.broadcast_to(np.asarray(w_gate, np.float64), (n,)))
    lib().orc_fit_gate_batch(_p(m), _p(s), n, _p(thr), _p(wg), _p(ok), _p(plane), _p(w), _p(nv))
    return ok[:n], plane[:n], w[:n], nv[:n]


def slerp_identity(q, t):
    out = np.zeros(4)
    lib().orc_slerp_identity(_d(np.asarray(q, np.float64)), float(t), _d(out))
    return out


def ceres_solve(feats, valid, plane, pose7, max_num_iter=15):
    f = _f4(feats)
    pose = np.array(pose7, np.float64)
    cost = C.c_double()
    it = lib().orc_ceres_solve(_p(f), len(f), _p(np.ascontiguousarray(valid)), _p(np.ascontiguousarray(plane)), _d(pose), max_num_iter, C.byref(cost))
    return it, pose, cost.value


def backend_edge_block(feats, valid, pa, pb, s_weight, pose7_body, cauchy_b=1.0):
    """(f1) LidarEdgeFactor rows of one keyframe reduced to [21 | 6 | cost | count], tangent order [t, rot]."""
    f = _f4(feats)
    out = np.zeros(29)
    lib().orc_backend_edge_block(_p(f), len(f), _p(np.ascontiguousarray(valid, np.uint8)), _p(np.ascontiguousarray(pa, np.float32)),
                                 _p(np.ascontiguousarray(pb, np.float32)), float(s_weight), _d(np.asarray(pose7_body, np.float64)), float(cauchy_b), _d(out))
    return out


def backend_surf_block(feats, valid, plane, score, pose7_body, q_lb=(1.0, 0, 0, 0), t_lb=(0.0, 0, 0), cauchy_b=1.0):
    """(f1) LidarPlaneNormFactor rows of one keyframe reduced to [21 | 6 | cost | count], tangent order [t, rot]."""
    f = _f4(feats)
    out = np.zeros(29)
    lib().orc_backend_surf_block(_p(f), len(f), _p(np.ascontiguousarray(valid, np.uint8)), _p(np.ascontiguousarray(plane, np.float32)),
                                 _p(np.ascontiguousarray(score, np.float64)), _d(np.asarray(pose7_body, np.float64)),
                                 _d(np.asarray(q_lb, np.float64)), _d(np.asarray(t_lb, np.float64)), float(cauchy_b), _d(out))
    return out


LIVOX20 = np.dtype([("offset_time", "<u4"), ("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("reflectivity", "u1"), ("tag", "u1"), ("line", "u1"), ("pad", "u1")])


def convert_livox(custom_pts, stride=None):
    """(f3) FormatConvert::livoxLidarHandler on an array of livox CustomPoint (LIVOX20 records or raw bytes + stride)."""
    a = np.ascontiguousarray(custom_pts)
    if stride is None:
        stride = a.dtype.itemsize
        n = len(a)
    else:
        n = a.size // stride
    out = np.zeros(max(n, 1), PT48)
    lib().orc_convert_livox(_p(a), n, stride, _p(out))
    return out[:n]
