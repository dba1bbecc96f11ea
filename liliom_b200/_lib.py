"""ctypes binding of libliliom_b200.so (the C ABI declared in include/liliom.h).

The product path has NO CPU fallback: if the CUDA library has not been built this module raises
on import of the library handle, and `liliom_create` fails with LILIOM_E_CUDA without a GPU.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# LILIOM_LIB: tuning builds of the same CUDA library (tools/ab_variants.py); the product is libliliom_b200.so
LIB_PATH = os.environ.get("LILIOM_LIB") or os.path.join(_HERE, "libliliom_b200.so")

# numpy mirrors of the PCL layouts (include/liliom.h)
PT48 = np.dtype([("x", "f4"), ("y", "f4"), ("z", "f4"), ("w", "f4"),
                 ("nx", "f4"), ("ny", "f4"), ("nz", "f4"), ("nw", "f4"),
                 ("intensity", "f4"), ("curvature", "f4"), ("p0", "f4"), ("p1", "f4")])
PT32 = np.dtype([("x", "f4"), ("y", "f4"), ("z", "f4"), ("w", "f4"),
                 ("intensity", "f4"), ("p0", "f4"), ("p1", "f4"), ("p2", "f4")])
# livox_ros_driver::CustomPoint as laid out in the C++ message struct (20 bytes; the wire layout is the first 19)
LIVOX20 = np.dtype([("offset_time", "<u4"), ("x", "<f4"), ("y", "<f4"), ("z", "<f4"),
                    ("reflectivity", "u1"), ("tag", "u1"), ("line", "u1"), ("pad", "u1")])
assert PT48.itemsize == 48 and PT32.itemsize == 32 and LIVOX20.itemsize == 20

OK, E_ARG, E_CUDA, E_FEWMAP, E_CAPACITY, E_GRID, E_LINES, E_NCCL, E_NOMAP = 0, -1, -2, -3, -4, -5, -6, -7, -8
MODE_CERES, MODE_GN = 0, 1
KF_FULL, KF_SURF = 0, 1      # liliom_global_map: which stored cloud of each keyframe
RING_ELEVATION, RING_FIELD = 0, 1   # liliom_set_ring_source: ROT scanID from the elevation tables / the PointCloud2 `ring` field
TIME_AZIMUTH, TIME_FIELD = 0, 1     # liliom_set_time_source: ROT relTime from the azimuth rule / a PointCloud2 per-point time field


class Params(C.Structure):
    _fields_ = [("abi_version", C.c_int), ("point_stride", C.c_int),
                ("surf_thres", C.c_double), ("edge_thres", C.c_double),
                ("line_num", C.c_int), ("ds_rate", C.c_int), ("rot_ds_leaf", C.c_float),
                ("leaf_scan", C.c_float), ("leaf_map", C.c_float),
                ("knn_max_sqdist", C.c_double), ("plane_thres", C.c_double), ("weight_gate", C.c_double),
                ("huber_a", C.c_double), ("max_map_frames", C.c_int),
                ("max_scan_points", C.c_int), ("max_map_points", C.c_int)]


class IterStats(C.Structure):
    _fields_ = [("n_corr", C.c_int), ("lm_iters", C.c_int), ("cost", C.c_double),
                ("jtj_jtr", C.c_double * 27), ("pose7", C.c_double * 7)]


class BackendParams(C.Structure):
    """liliom_backend_params (include/liliom.h): the BackendFusion settings the keyframe store, local map and window use."""
    _fields_ = [("variant", C.c_int), ("edge_leaf", C.c_float), ("surf_leaf", C.c_float),
                ("kd_max_radius", C.c_double), ("surf_dist_thres", C.c_double), ("w_gate", C.c_double), ("lidar_const", C.c_double),
                ("reflect_thres", C.c_double), ("cauchy_b", C.c_double), ("q_lb", C.c_double * 4), ("t_lb", C.c_double * 3)]


class Counters(C.Structure):
    _fields_ = [("launches", C.c_ulonglong), ("lib_launches", C.c_ulonglong), ("knn_ms", C.c_double),
                ("knn_launches", C.c_ulonglong), ("knn_queries", C.c_ulonglong), ("knn_candidates", C.c_ulonglong)]


EXPORTS = [
    "liliom_default_params", "liliom_create", "liliom_destroy", "liliom_strerror", "liliom_last_error",
    "liliom_extract_horizon", "liliom_extract_rot", "liliom_extract_rot_labels", "liliom_voxelgrid",
    "liliom_map_push_frame", "liliom_map_rebuild", "liliom_map_clear", "liliom_map_set_points", "liliom_map_size",
    "liliom_map_download", "liliom_scan_to_map", "liliom_odometry_resident", "liliom_find_surf_corr",
    "liliom_correspond_edge", "liliom_correspond_surf", "liliom_comm_get_unique_id", "liliom_comm_init",
    "liliom_get_counters", "liliom_set_kernel_timing", "liliom_upload_feats", "liliom_scan_to_map_resident",
    "liliom_odometry", "liliom_set_stream", "liliom_upload_scan", "liliom_extract_resident", "liliom_point_stride",
    "liliom_map_set_cloud", "liliom_correspond_surf_refl",
    "liliom_backend_edge_block", "liliom_backend_surf_block", "liliom_convert_livox", "liliom_extract_horizon_livox",
    "liliom_pc2_layout", "liliom_comm_peer_export", "liliom_comm_peer_attach",
    "liliom_map_push_frame_device", "liliom_knn_block_stats", "liliom_comm_set_shard_block", "liliom_undistort",
    "liliom_map_update", "liliom_map_update_device", "liliom_map_download_cloud", "liliom_icp_align",
    "liliom_comm_peer_epoch", "liliom_comm_peer_set_epoch",
    "liliom_backend_default_params", "liliom_kf_add", "liliom_kf_count", "liliom_kf_clear", "liliom_bmap_build",
    "liliom_bmap_download", "liliom_backend_window_correspond", "liliom_backend_window_blocks", "liliom_backend_window_corr",
    "liliom_kf_cloud", "liliom_kf_add_full", "liliom_global_map", "liliom_loop_align",
    "liliom_convert_pc2", "liliom_extract_rot_pc2", "liliom_set_ring_source", "liliom_set_time_source",
]
NODE_EXPORTS = ["liliom_pre_create", "liliom_pre_destroy", "liliom_pre_imu", "liliom_pre_cloud", "liliom_pre_cloud_pc2",
                "liliom_lo_create", "liliom_lo_destroy", "liliom_lo_edge", "liliom_lo_surf", "liliom_lo_full", "liliom_lo_run"]


class Pc2Field(C.Structure):
    _fields_ = [("name", C.c_char * 16), ("offset", C.c_uint), ("datatype", C.c_ubyte), ("count", C.c_uint)]


def pc2_layout(point_stride: int):
    """(fields, point_step) of the sensor_msgs/PointCloud2 pcl::toROSMsg builds for the 48 / 32-byte clouds."""
    f = (Pc2Field * 8)()
    step = C.c_int()
    n = lib().liliom_pc2_layout(point_stride, f, 8, C.byref(step))
    if n < 0:
        raise LiliomError(n)
    return [(f[i].name.decode(), f[i].offset, f[i].datatype, f[i].count) for i in range(n)], step.value


class Pc2Msg(C.Structure):
    """liliom_pc2_msg (include/liliom.h)."""
    _fields_ = [("data", C.c_void_p), ("height", C.c_uint), ("width", C.c_uint), ("point_step", C.c_uint), ("row_step", C.c_uint),
                ("fields", C.POINTER(Pc2Field)), ("n_fields", C.c_int), ("is_bigendian", C.c_int)]


class PC2:
    """A sensor_msgs/PointCloud2 as a driver publishes it: the payload bytes (height * row_step, little-endian), the header
    fields the decode reads and the field list as (name, offset, datatype, count) tuples."""

    def __init__(self, data, height: int, width: int, point_step: int, row_step: int, fields, is_bigendian: bool = False):
        self.data = np.ascontiguousarray(np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else data).view(np.uint8).reshape(-1)
        self.height, self.width, self.point_step, self.row_step = int(height), int(width), int(point_step), int(row_step)
        self.fields = [(str(n), int(o), int(d), int(c)) for n, o, d, c in fields]
        self.is_bigendian = bool(is_bigendian)

    def c_msg(self):
        """(Pc2Msg, field array): the field array must stay alive as long as the Pc2Msg is used."""
        f = (Pc2Field * max(len(self.fields), 1))()
        for i, (n, o, d, c) in enumerate(self.fields):
            f[i].name = n.encode()[:15]; f[i].offset = o; f[i].datatype = d; f[i].count = c
        m = Pc2Msg(self.data.ctypes.data_as(C.c_void_p) if self.data.size else None, self.height, self.width, self.point_step,
                   self.row_step, f, len(self.fields), 1 if self.is_bigendian else 0)
        return m, f


class LoOutput(C.Structure):
    _fields_ = [("ran", C.c_int), ("initialized", C.c_int), ("kf", C.c_int), ("n_map", C.c_int), ("n_surf_ds", C.c_int),
                ("status", C.c_int), ("abs_pose", C.c_double * 7), ("rel_pose", C.c_double * 7), ("stamp", C.c_double)]


_lib = None


def lib() -> C.CDLL:
    """Load the CUDA library (raises if it has not been built — there is no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  liliom_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    vp, ip, dp, fp = C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_float)
    L.liliom_default_params.argtypes = [C.POINTER(Params), C.c_int]
    L.liliom_default_params.restype = None
    L.liliom_create.argtypes = [C.POINTER(vp), C.POINTER(Params), C.c_int]
    L.liliom_destroy.argtypes = [vp]
    L.liliom_destroy.restype = None
    L.liliom_strerror.argtypes = [C.c_int]
    L.liliom_strerror.restype = C.c_char_p
    L.liliom_last_error.argtypes = [vp]
    L.liliom_last_error.restype = C.c_char_p
    L.liliom_extract_horizon.argtypes = [vp, vp, C.c_int, dp, vp, C.c_int, ip, vp, C.c_int, ip, vp, C.c_int, ip]
    L.liliom_extract_rot.argtypes = [vp, vp, C.c_int, dp, dp, vp, C.c_int, ip, vp, C.c_int, ip, vp, C.c_int, ip]
    L.liliom_extract_rot_labels.argtypes = [vp, vp, vp, C.c_int]
    L.liliom_voxelgrid.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, vp, C.c_int, ip]
    L.liliom_map_push_frame.argtypes = [vp, vp, C.c_int, dp]
    L.liliom_map_rebuild.argtypes = [vp, ip]
    L.liliom_map_clear.argtypes = [vp]
    L.liliom_map_set_points.argtypes = [vp, vp, C.c_int]
    L.liliom_map_size.argtypes = [vp]
    L.liliom_map_download.argtypes = [vp, vp, C.c_int, ip]
    L.liliom_scan_to_map.argtypes = [vp, vp, C.c_int, C.c_int, dp, C.c_int, C.c_int, C.c_int, C.POINTER(IterStats)]
    L.liliom_odometry_resident.argtypes = [vp, dp, C.c_int, C.c_int, C.c_int, C.POINTER(IterStats), vp, C.c_int, ip]
    L.liliom_find_surf_corr.argtypes = [vp, vp, C.c_int, C.c_int, dp, vp, vp, vp, vp, dp]
    L.liliom_correspond_edge.argtypes = [vp, vp, C.c_int, C.c_int, dp, C.c_int, vp, vp, vp]
    L.liliom_correspond_surf.argtypes = [vp, vp, C.c_int, C.c_int, dp, C.c_double, C.c_double, C.c_double, C.c_double, vp, vp, vp]
    L.liliom_comm_get_unique_id.argtypes = [vp]
    L.liliom_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liliom_get_counters.argtypes = [vp, C.POINTER(Counters), C.c_int]
    L.liliom_set_kernel_timing.argtypes = [vp, C.c_int]
    L.liliom_upload_feats.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liliom_scan_to_map_resident.argtypes = [vp, dp, C.c_int, C.c_int, C.c_int, C.POINTER(IterStats)]
    L.liliom_odometry.argtypes = [vp, vp, C.c_int, dp, C.c_int, C.c_int, C.c_int, C.POINTER(IterStats), vp, C.c_int, ip]
    L.liliom_set_stream.argtypes = [vp, vp]
    L.liliom_upload_scan.argtypes = [vp, vp, C.c_int]
    L.liliom_extract_resident.argtypes = [vp, dp, dp, ip, ip, ip]
    L.liliom_point_stride.argtypes = [vp]
    L.liliom_map_set_cloud.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liliom_correspond_surf_refl.argtypes = [vp, vp, C.c_int, dp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, vp, vp, vp]
    L.liliom_backend_edge_block.argtypes = [vp, dp, C.c_double, C.c_double, dp]
    L.liliom_backend_surf_block.argtypes = [vp, dp, dp, dp, C.c_double, dp]
    L.liliom_convert_livox.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_int]
    L.liliom_extract_horizon_livox.argtypes = [vp, vp, C.c_int, C.c_int, dp, vp, C.c_int, ip, vp, C.c_int, ip, vp, C.c_int, ip]
    L.liliom_pc2_layout.argtypes = [C.c_int, vp, C.c_int, ip]
    L.liliom_convert_pc2.argtypes = [vp, C.POINTER(Pc2Msg), vp, C.c_int, ip]
    L.liliom_extract_rot_pc2.argtypes = [vp, C.POINTER(Pc2Msg), dp, dp, vp, C.c_int, ip, vp, C.c_int, ip, vp, C.c_int, ip]
    L.liliom_set_ring_source.argtypes = [vp, C.c_int]
    L.liliom_set_time_source.argtypes = [vp, C.c_int, C.c_char_p]
    L.liliom_comm_peer_export.argtypes = [vp, vp]
    L.liliom_comm_peer_attach.argtypes = [vp, vp, C.c_int, C.c_int]
    L.liliom_comm_peer_epoch.argtypes = [vp, C.POINTER(C.c_uint)]
    L.liliom_comm_peer_set_epoch.argtypes = [vp, C.c_uint]
    L.liliom_map_push_frame_device.argtypes = [vp, vp, C.c_int, dp]
    L.liliom_comm_set_shard_block.argtypes = [vp, C.c_int]
    L.liliom_undistort.argtypes = [vp, vp, C.c_int, dp, dp]
    L.liliom_map_update.argtypes = [vp, vp, C.c_int, dp, ip]
    L.liliom_map_update_device.argtypes = [vp, vp, C.c_int, dp, ip]
    L.liliom_map_download_cloud.argtypes = [vp, vp, C.c_int, ip]
    L.liliom_icp_align.argtypes = [vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_double, C.c_int, C.c_double, C.c_double, dp, dp, ip, ip]
    L.liliom_knn_block_stats.argtypes = [vp, dp, C.POINTER(C.c_ulonglong)]
    bpp = C.POINTER(BackendParams)
    L.liliom_backend_default_params.argtypes = [bpp, C.c_int]; L.liliom_backend_default_params.restype = None
    L.liliom_kf_add.argtypes = [vp, bpp, vp, C.c_int, vp, C.c_int, ip, vp, C.c_int, ip, vp, C.c_int, ip]
    L.liliom_kf_count.argtypes = [vp]
    L.liliom_kf_clear.argtypes = [vp]
    L.liliom_bmap_build.argtypes = [vp, bpp, ip, dp, C.c_int, ip, ip]
    L.liliom_bmap_download.argtypes = [vp, C.c_int, vp, C.c_int, ip]
    L.liliom_backend_window_correspond.argtypes = [vp, bpp, ip, dp, C.c_int, ip, ip]
    L.liliom_backend_window_blocks.argtypes = [vp, dp, C.c_int, dp]
    L.liliom_backend_window_corr.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, ip]
    L.liliom_kf_cloud.argtypes = [vp, ip, dp, C.c_int, C.c_float, vp, C.c_int, ip]
    L.liliom_kf_add_full.argtypes = [vp, bpp, C.c_int, vp, C.c_int, ip]
    L.liliom_global_map.argtypes = [vp, C.c_int, ip, dp, C.c_int, dp, C.c_float, vp, C.c_int, ip]
    L.liliom_loop_align.argtypes = [vp, ip, dp, C.c_int, ip, dp, C.c_int, C.c_float, C.c_double, C.c_int, C.c_double, C.c_double,
                                    dp, dp, ip, ip, ip, ip]
    L.liliom_pre_create.argtypes = [vp, C.c_int, dp]; L.liliom_pre_create.restype = vp
    L.liliom_pre_destroy.argtypes = [vp]; L.liliom_pre_destroy.restype = None
    L.liliom_pre_imu.argtypes = [vp, C.c_double, dp]; L.liliom_pre_imu.restype = None
    L.liliom_pre_cloud.argtypes = [vp, C.c_double, vp, C.c_int, vp, C.c_int, ip, vp, C.c_int, ip, vp, C.c_int, ip, dp, dp]
    L.liliom_pre_cloud_pc2.argtypes = [vp, C.c_double, C.POINTER(Pc2Msg), vp, C.c_int, ip, vp, C.c_int, ip, vp, C.c_int, ip, dp, dp]
    L.liliom_lo_create.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int]; L.liliom_lo_create.restype = vp
    L.liliom_lo_destroy.argtypes = [vp]; L.liliom_lo_destroy.restype = None
    for f in (L.liliom_lo_edge, L.liliom_lo_surf, L.liliom_lo_full):
        f.argtypes = [vp, C.c_double, vp, C.c_int]; f.restype = None
    L.liliom_lo_run.argtypes = [vp, C.POINTER(LoOutput), vp, C.c_int, ip, vp, C.c_int, ip, vp, C.c_int, ip]
    _lib = L
    return L


class LiliomError(RuntimeError):
    def __init__(self, code: int, detail: str = ""):
        self.code = code
        msg = lib().liliom_strerror(code).decode()
        super().__init__(f"liliom error {code}: {msg}" + (f" ({detail})" if detail else ""))


def _ptr(a: np.ndarray | None):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _dptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def backend_default_params(variant: int = 0) -> BackendParams:
    p = BackendParams()
    lib().liliom_backend_default_params(C.byref(p), variant)
    return p


def _ids(ids):
    return np.ascontiguousarray(ids, dtype=np.int32).reshape(-1)


def _poses(poses7, k):
    p = np.ascontiguousarray(poses7, dtype=np.float64).reshape(-1, 7) if k else np.zeros((1, 7))
    assert len(p) >= k
    return p


def default_params(variant: int = 0) -> Params:
    p = Params()
    lib().liliom_default_params(C.byref(p), variant)
    return p


class Context:
    """One liliom_ctx (one per ROS node in the reference; not thread-safe)."""

    def __init__(self, params: Params | None = None, device: int = 0, variant: int = 0):
        self.params = params if params is not None else default_params(variant)
        self._h = C.c_void_p()
        rc = lib().liliom_create(C.byref(self._h), C.byref(self.params), device)
        if rc != OK:
            self._h = None
            raise LiliomError(rc, "liliom_create: no CUDA device / bad params (no CPU fallback)")
        self.stride = self.params.point_stride
        self.dtype = PT48 if self.stride == 48 else PT32

    def close(self):
        if getattr(self, "_h", None):
            lib().liliom_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != OK:
            raise LiliomError(rc, lib().liliom_last_error(self._h).decode())

    # ---- L1 ----
    def extract_horizon(self, pts: np.ndarray, q_imu, out=None):
        """out = optional (surf, edge, cut) caller-owned PT48 arrays (e.g. pinned) to receive the clouds."""
        pts = np.ascontiguousarray(pts, dtype=PT48)
        n = len(pts)
        q = np.asarray(q_imu, dtype=np.float64)
        if out is None:
            surf = np.empty(max(n, 1), PT48); edge = np.empty(max(n, 1), PT48); cut = np.empty(max(n, 1), PT48)
        else:
            surf, edge, cut = out
        ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
        self._check(lib().liliom_extract_horizon(self._h, _ptr(pts), n, _dptr(q), _ptr(surf), len(surf), C.byref(ns),
                                                 _ptr(edge), len(edge), C.byref(ne), _ptr(cut), len(cut), C.byref(nc)))
        return surf[:ns.value], edge[:ne.value], cut[:nc.value]

    def extract_rot(self, pts: np.ndarray, q_imu, q_lb=(1.0, 0.0, 0.0, 0.0), out=None):
        pts = np.ascontiguousarray(pts, dtype=PT32)
        n = len(pts)
        q = np.asarray(q_imu, dtype=np.float64); ql = np.asarray(q_lb, dtype=np.float64)
        if out is None:
            surf = np.empty(max(n, 1), PT32); edge = np.empty(max(n, 1), PT32); cut = np.empty(max(n, 1), PT32)
        else:
            surf, edge, cut = out
        ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
        self._check(lib().liliom_extract_rot(self._h, _ptr(pts), n, _dptr(q), _dptr(ql), _ptr(surf), len(surf), C.byref(ns),
                                             _ptr(edge), len(edge), C.byref(ne), _ptr(cut), len(cut), C.byref(nc)))
        return surf[:ns.value], edge[:ne.value], cut[:nc.value]

    def extract_rot_labels(self, n: int):
        lab = np.zeros(max(n, 1), np.int32); cur = np.zeros(max(n, 1), np.float32)
        self._check(lib().liliom_extract_rot_labels(self._h, _ptr(lab), _ptr(cur), len(lab)))
        return lab[:n], cur[:n]

    def voxelgrid(self, pts: np.ndarray, leaf: float):
        pts = np.ascontiguousarray(pts)
        stride = pts.dtype.itemsize
        out = np.zeros(max(len(pts), 1), pts.dtype)
        m = C.c_int()
        self._check(lib().liliom_voxelgrid(self._h, _ptr(pts), len(pts), stride, leaf, _ptr(out), len(out), C.byref(m)))
        return out[:m.value]

    # ---- L2 ----
    def map_set_points(self, xyzw: np.ndarray):
        xyzw = np.ascontiguousarray(xyzw, dtype=np.float32).reshape(-1, 4)
        self._check(lib().liliom_map_set_points(self._h, _ptr(xyzw), len(xyzw)))

    def map_push_frame(self, pts: np.ndarray, pose7):
        pts = np.ascontiguousarray(pts, dtype=self.dtype)
        p = np.asarray(pose7, dtype=np.float64)
        self._check(lib().liliom_map_push_frame(self._h, _ptr(pts), len(pts), _dptr(p)))

    def map_push_frame_device(self, dev_ptr: int, n: int, pose7):
        """push_frame from a DEVICE buffer of n points (point_stride bytes each), e.g. a torch CUDA tensor's data_ptr()."""
        p = np.asarray(pose7, dtype=np.float64)
        self._check(lib().liliom_map_push_frame_device(self._h, C.c_void_p(dev_ptr), n, _dptr(p)))

    def undistort(self, pts: np.ndarray, trans, quat=(1.0, 0.0, 0.0, 0.0)) -> np.ndarray:
        """LidarOdometry::undistortion on the device; returns the moved copy."""
        out = np.ascontiguousarray(pts, dtype=self.dtype).copy()
        t = np.asarray(trans, dtype=np.float64); q = np.asarray(quat, dtype=np.float64)
        self._check(lib().liliom_undistort(self._h, _ptr(out), len(out), _dptr(t), _dptr(q)))
        return out

    def map_update(self, pts: np.ndarray, pose7) -> int:
        """push_frame + incremental refresh of the filtered map (SURVEY §8 f2); returns the map size."""
        pts = np.ascontiguousarray(pts, dtype=self.dtype)
        p = np.asarray(pose7, dtype=np.float64)
        m = C.c_int()
        self._check(lib().liliom_map_update(self._h, _ptr(pts), len(pts), _dptr(p), C.byref(m)))
        return m.value

    def map_update_device(self, dev_ptr: int, n: int, pose7) -> int:
        p = np.asarray(pose7, dtype=np.float64)
        m = C.c_int()
        self._check(lib().liliom_map_update_device(self._h, C.c_void_p(dev_ptr), n, _dptr(p), C.byref(m)))
        return m.value

    def map_download_cloud(self) -> np.ndarray:
        m = C.c_int()
        self._check(lib().liliom_map_download_cloud(self._h, None, 0, C.byref(m)))
        out = np.zeros(max(m.value, 1), self.dtype)
        self._check(lib().liliom_map_download_cloud(self._h, _ptr(out), len(out), C.byref(m)))
        return out[:m.value]

    def icp_align(self, src: np.ndarray, tgt: np.ndarray, max_corr_dist=30.0, max_iter=100, trans_eps=1e-6, fit_eps=1e-6):
        """Loop-closure ICP (SURVEY §8 f4): returns (T 4x4, fitness, converged, iterations)."""
        s, stride = self._feats(src)
        t, stride_t = self._feats(tgt)
        assert stride == stride_t
        T = np.zeros(16, np.float64); fit = C.c_double(); conv = C.c_int(); it = C.c_int()
        self._check(lib().liliom_icp_align(self._h, _ptr(s), len(s), _ptr(t), len(t), stride, max_corr_dist, max_iter, trans_eps, fit_eps,
                                           _dptr(T), C.byref(fit), C.byref(conv), C.byref(it)))
        return T.reshape(4, 4), fit.value, bool(conv.value), it.value

    def map_rebuild(self) -> int:
        m = C.c_int()
        self._check(lib().liliom_map_rebuild(self._h, C.byref(m)))
        return m.value

    def map_clear(self):
        self._check(lib().liliom_map_clear(self._h))

    def map_size(self) -> int:
        return lib().liliom_map_size(self._h)

    def map_download(self) -> np.ndarray:
        m = self.map_size()
        out = np.zeros((max(m, 1), 4), np.float32)
        mo = C.c_int()
        self._check(lib().liliom_map_download(self._h, _ptr(out), len(out), C.byref(mo)))
        return out[:mo.value]

    @staticmethod
    def _feats(feats: np.ndarray):
        feats = np.ascontiguousarray(feats)
        if feats.dtype.fields is None:
            feats = np.ascontiguousarray(feats, dtype=np.float32).reshape(-1, 4)
            return feats, 16
        return feats, feats.dtype.itemsize

    def scan_to_map(self, feats: np.ndarray, pose7, match_cnt: int, max_num_iter: int = 15, mode: int = MODE_GN):
        f, stride = self._feats(feats)
        pose = np.array(pose7, dtype=np.float64)
        st = (IterStats * max(match_cnt, 1))()
        self._check(lib().liliom_scan_to_map(self._h, _ptr(f), len(f), stride, _dptr(pose), match_cnt, max_num_iter, mode, st))
        return pose, [st[i] for i in range(match_cnt)]

    def upload_feats(self, feats: np.ndarray):
        f, stride = self._feats(feats)
        self._check(lib().liliom_upload_feats(self._h, _ptr(f), len(f), stride))

    def scan_to_map_resident(self, pose7, match_cnt: int, max_num_iter: int = 15, mode: int = MODE_GN, want_stats: bool = False):
        pose = np.array(pose7, dtype=np.float64)
        st = (IterStats * max(match_cnt, 1))() if want_stats else None
        self._check(lib().liliom_scan_to_map_resident(self._h, _dptr(pose), match_cnt, max_num_iter, mode, st))
        return pose, ([st[i] for i in range(match_cnt)] if want_stats else None)

    def odometry_resident(self, pose7, match_cnt: int, max_num_iter: int = 15, mode: int = MODE_GN, want_ds: bool = False, cap: int = 0,
                          want_stats: bool = True):
        pose = np.array(pose7, dtype=np.float64)
        st = (IterStats * max(match_cnt, 1))() if want_stats else None
        nds = C.c_int()
        ds = np.zeros(max(cap, 1), self.dtype) if want_ds else None
        self._check(lib().liliom_odometry_resident(self._h, _dptr(pose), match_cnt, max_num_iter, mode, st, _ptr(ds), cap if want_ds else 0, C.byref(nds)))
        return pose, ([st[i] for i in range(match_cnt)] if want_stats else None), (ds[:nds.value] if want_ds else nds.value)

    def odometry(self, surf_feats: np.ndarray, pose7, match_cnt: int, max_num_iter: int = 15, mode: int = MODE_GN,
                 ds_out: np.ndarray | None = None, pose_out: np.ndarray | None = None, want_stats: bool = True):
        """LidarOdometry node view: un-down-sampled surf cloud in (host), pose + surf_last_ds out."""
        f = surf_feats
        if f.dtype != self.dtype or not f.flags.c_contiguous:
            f = np.ascontiguousarray(f, dtype=self.dtype)
        pose = pose_out if pose_out is not None else np.empty(7, np.float64)
        pose[:] = pose7
        st = (IterStats * max(match_cnt, 1))() if want_stats else None
        nds = C.c_int()
        if ds_out is None:
            ds_out = np.empty(max(len(f), 1), self.dtype)
        self._check(lib().liliom_odometry(self._h, _ptr(f), len(f), _dptr(pose), match_cnt, max_num_iter, mode, st, _ptr(ds_out), len(ds_out), C.byref(nds)))
        return pose, ([st[i] for i in range(match_cnt)] if want_stats else None), ds_out[:nds.value]

    def set_stream(self, cuda_stream: int | None):
        self._check(lib().liliom_set_stream(self._h, C.c_void_p(cuda_stream) if cuda_stream else None))

    def upload_scan(self, pts: np.ndarray):
        pts = np.ascontiguousarray(pts, dtype=self.dtype)
        self._check(lib().liliom_upload_scan(self._h, _ptr(pts), len(pts)))

    def extract_resident(self, q_imu, q_lb=(1.0, 0.0, 0.0, 0.0)):
        q = np.asarray(q_imu, dtype=np.float64); ql = np.asarray(q_lb, dtype=np.float64)
        ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
        self._check(lib().liliom_extract_resident(self._h, _dptr(q), _dptr(ql), C.byref(ns), C.byref(ne), C.byref(nc)))
        return ns.value, ne.value, nc.value

    def find_surf_corr(self, feats: np.ndarray, pose7):
        f, stride = self._feats(feats)
        n = len(f)
        pose = np.array(pose7, dtype=np.float64)
        valid = np.zeros(max(n, 1), np.uint8); plane = np.zeros((max(n, 1), 4), np.float32)
        idx = np.zeros((max(n, 1), 5), np.int32); sqd = np.zeros((max(n, 1), 5), np.float32)
        s29 = np.zeros(29, np.float64)
        self._check(lib().liliom_find_surf_corr(self._h, _ptr(f), n, stride, _dptr(pose), _ptr(valid), _ptr(plane), _ptr(idx), _ptr(sqd), _dptr(s29)))
        return valid[:n], plane[:n], idx[:n], sqd[:n], s29

    def correspond_edge(self, feats: np.ndarray, pose7, variant: int = 0):
        f, stride = self._feats(feats)
        n = len(f)
        pose = np.array(pose7, dtype=np.float64)
        valid = np.zeros(max(n, 1), np.uint8); pa = np.zeros((max(n, 1), 3), np.float32); pb = np.zeros((max(n, 1), 3), np.float32)
        self._check(lib().liliom_correspond_edge(self._h, _ptr(f), n, stride, _dptr(pose), variant, _ptr(valid), _ptr(pa), _ptr(pb)))
        return valid[:n], pa[:n], pb[:n]

    def correspond_surf(self, feats: np.ndarray, pose7, kd_max_radius=1.0, surf_dist_thres=0.06, w_gate=0.3, lidar_const=1.0):
        f, stride = self._feats(feats)
        n = len(f)
        pose = np.array(pose7, dtype=np.float64)
        valid = np.zeros(max(n, 1), np.uint8); plane = np.zeros((max(n, 1), 4), np.float32); score = np.zeros(max(n, 1), np.float64)
        self._check(lib().liliom_correspond_surf(self._h, _ptr(f), n, stride, _dptr(pose), kd_max_radius, surf_dist_thres, w_gate,
                                                 lidar_const, _ptr(valid), _ptr(plane), _ptr(score)))
        return valid[:n], plane[:n], score[:n]

    def map_set_cloud(self, pts: np.ndarray):
        pts = np.ascontiguousarray(pts)
        self._check(lib().liliom_map_set_cloud(self._h, _ptr(pts), len(pts), pts.dtype.itemsize))

    def correspond_surf_refl(self, feats: np.ndarray, pose7, kd_max_radius=1.0, surf_dist_thres=0.1, w_gate=0.2, lidar_const=1.0, reflect_thres=10.0):
        f = np.ascontiguousarray(feats, dtype=PT48)
        n = len(f)
        pose = np.array(pose7, dtype=np.float64)
        valid = np.zeros(max(n, 1), np.uint8); plane = np.zeros((max(n, 1), 4), np.float32); score = np.zeros(max(n, 1), np.float64)
        self._check(lib().liliom_correspond_surf_refl(self._h, _ptr(f), n, _dptr(pose), kd_max_radius, surf_dist_thres, w_gate, lidar_const,
                                                      reflect_thres, _ptr(valid), _ptr(plane), _ptr(score)))
        return valid[:n], plane[:n], score[:n]

    def backend_edge_block(self, pose7_body, s_weight: float, cauchy_b: float = 1.0):
        """(f1) 29 scalars of the LidarEdgeFactor rows on the correspondences of the last correspond_edge call."""
        out = np.zeros(29)
        self._check(lib().liliom_backend_edge_block(self._h, _dptr(np.asarray(pose7_body, np.float64)), float(s_weight), float(cauchy_b), _dptr(out)))
        return out

    def backend_surf_block(self, pose7_body, q_lb=(1.0, 0.0, 0.0, 0.0), t_lb=(0.0, 0.0, 0.0), cauchy_b: float = 1.0):
        """(f1) 29 scalars of the LidarPlaneNormFactor rows on the correspondences of the last correspond_surf* call."""
        out = np.zeros(29)
        self._check(lib().liliom_backend_surf_block(self._h, _dptr(np.asarray(pose7_body, np.float64)), _dptr(np.asarray(q_lb, np.float64)),
                                                    _dptr(np.asarray(t_lb, np.float64)), float(cauchy_b), _dptr(out)))
        return out

    # ---- backend keyframe store, local map and window (f5) ----
    def kf_add(self, bp: BackendParams, edge_last: np.ndarray, surf_last: np.ndarray, download: bool = True):
        """downSampleCloud (scan half) + store: returns (kf_id, edge_ds, surf_ds); the clouds are None when download=False."""
        e = np.ascontiguousarray(edge_last, dtype=self.dtype); s = np.ascontiguousarray(surf_last, dtype=self.dtype)
        kid, ne, ns = C.c_int(), C.c_int(), C.c_int()
        eo = np.zeros(max(len(e), 1), self.dtype) if download else None
        so = np.zeros(max(len(s), 1), self.dtype) if download else None
        self._check(lib().liliom_kf_add(self._h, C.byref(bp), _ptr(e), len(e), _ptr(s), len(s), C.byref(kid),
                                        _ptr(eo), len(eo) if download else 0, C.byref(ne), _ptr(so), len(so) if download else 0, C.byref(ns)))
        if not download:
            return kid.value, None, None
        return kid.value, eo[:ne.value], so[:ns.value]

    def kf_count(self) -> int:
        return lib().liliom_kf_count(self._h)

    def kf_clear(self):
        self._check(lib().liliom_kf_clear(self._h))

    def bmap_build(self, bp: BackendParams, kf_ids, poses7):
        """buildLocalMapWithLandMark + downSampleCloud (map half) on the device: returns (edge layer size, surf layer size)."""
        ids = _ids(kf_ids); p = _poses(poses7, len(ids))
        ne, ns = C.c_int(), C.c_int()
        self._check(lib().liliom_bmap_build(self._h, C.byref(bp), ids.ctypes.data_as(C.POINTER(C.c_int)), _dptr(p), len(ids),
                                            C.byref(ne), C.byref(ns)))
        return ne.value, ns.value

    def bmap_download(self, layer: int) -> np.ndarray:
        """edge_local_map_ds (layer 0) or surf_local_map_ds (layer 1), all fields."""
        m = C.c_int()
        self._check(lib().liliom_bmap_download(self._h, layer, None, 0, C.byref(m)))
        out = np.zeros(max(m.value, 1), self.dtype)
        self._check(lib().liliom_bmap_download(self._h, layer, _ptr(out), len(out), C.byref(m)))
        return out[:m.value]

    def backend_window_correspond(self, bp: BackendParams, kf_ids, poses7_lidar):
        """Edge and surf searches of the window keyframes against the local map: returns (n_edge_corr, n_surf_corr) per keyframe."""
        ids = _ids(kf_ids); k = len(ids); p = _poses(poses7_lidar, k)
        ne = np.zeros(max(k, 1), np.int32); ns = np.zeros(max(k, 1), np.int32)
        ipp = C.POINTER(C.c_int)
        self._check(lib().liliom_backend_window_correspond(self._h, C.byref(bp), ids.ctypes.data_as(ipp), _dptr(p), k,
                                                           ne.ctypes.data_as(ipp), ns.ctypes.data_as(ipp)))
        return ne[:k], ns[:k]

    def backend_window_blocks(self, poses7_body) -> np.ndarray:
        """(k, 2, 29): the edge and surf normal-equation blocks of every window keyframe at its body pose."""
        p = np.ascontiguousarray(poses7_body, dtype=np.float64).reshape(-1, 7)
        out = np.zeros((len(p), 2, 29))
        self._check(lib().liliom_backend_window_blocks(self._h, _dptr(p), len(p), _dptr(out)))
        return out

    def backend_window_corr(self, slot: int, kind: int):
        """Test hook: (valid, pa, pb) of window keyframe `slot` for kind 0, (valid, plane, score) for kind 1."""
        n = C.c_int()
        self._check(lib().liliom_backend_window_corr(self._h, slot, kind, None, None, None, 0, C.byref(n)))
        m = max(n.value, 1)
        valid = np.zeros(m, np.uint8)
        if kind == 0:
            a = np.zeros((m, 3), np.float32); b = np.zeros((m, 3), np.float32)
        else:
            a = np.zeros((m, 4), np.float32); b = np.zeros(m, np.float64)
        self._check(lib().liliom_backend_window_corr(self._h, slot, kind, _ptr(valid), _ptr(a), _ptr(b), m, C.byref(n)))
        return valid[:n.value], a[:n.value], b[:n.value]

    def kf_cloud(self, kf_ids, poses7, leaf: float) -> np.ndarray:
        """detectLoopClosure's clouds: edge then surf of every listed keyframe, transformed, VoxelGrid(leaf)."""
        ids = _ids(kf_ids); p = _poses(poses7, len(ids))
        ipp = C.POINTER(C.c_int)
        n = C.c_int()
        self._check(lib().liliom_kf_cloud(self._h, ids.ctypes.data_as(ipp), _dptr(p), len(ids), leaf, None, 0, C.byref(n)))
        out = np.zeros(max(n.value, 1), self.dtype)
        self._check(lib().liliom_kf_cloud(self._h, ids.ctypes.data_as(ipp), _dptr(p), len(ids), leaf, _ptr(out), len(out), C.byref(n)))
        return out[:n.value]

    def loop_align(self, src_ids, src_poses, tgt_ids, tgt_poses, leaf: float, max_corr_dist=30.0, max_iter=100, trans_eps=1e-6,
                   fit_eps=1e-6):
        """Loop closure from the store: kf_cloud of both lists and icp_align of the first onto the second, on the device.
        Returns (T 4x4, fitness, converged, iterations, n_src, n_tgt)."""
        si = _ids(src_ids); sp = _poses(src_poses, len(si))
        ti = _ids(tgt_ids); tp = _poses(tgt_poses, len(ti))
        ipp = C.POINTER(C.c_int)
        T = np.zeros(16, np.float64); fit = C.c_double(); conv = C.c_int(); it = C.c_int(); ns = C.c_int(); nt = C.c_int()
        self._check(lib().liliom_loop_align(self._h, si.ctypes.data_as(ipp), _dptr(sp), len(si), ti.ctypes.data_as(ipp), _dptr(tp), len(ti),
                                            leaf, max_corr_dist, max_iter, trans_eps, fit_eps, _dptr(T), C.byref(fit), C.byref(conv),
                                            C.byref(it), C.byref(ns), C.byref(nt)))
        return T.reshape(4, 4), fit.value, bool(conv.value), it.value, ns.value, nt.value

    def kf_add_full(self, bp: BackendParams, kf_id: int, full: np.ndarray) -> int:
        """downSampleCloud (full-cloud half): attach keyframe kf_id's full body-frame cloud, stored as received (variant 0) or
        VoxelGrid(surf_leaf) of it (variant 1).  Returns the points stored."""
        f = np.ascontiguousarray(full, dtype=self.dtype)
        m = C.c_int()
        self._check(lib().liliom_kf_add_full(self._h, C.byref(bp), int(kf_id), _ptr(f), len(f), C.byref(m)))
        return m.value

    def global_map(self, kind: int, kf_ids, poses7, leaf: float, pre7=None) -> np.ndarray:
        """publishCompleteMap / save_pcd's map: the stored cloud of `kind` (KF_FULL or KF_SURF) of every listed keyframe,
        transformed by pre7 (optional) and then by its pose, concatenated, VoxelGrid(leaf); the transformed concatenation itself
        when PCL declines the filter (index overflow)."""
        ids = _ids(kf_ids); p = _poses(poses7, len(ids))
        pre = None if pre7 is None else np.ascontiguousarray(pre7, dtype=np.float64).reshape(7)
        ipp = C.POINTER(C.c_int)
        args = (self._h, int(kind), ids.ctypes.data_as(ipp), _dptr(p), len(ids), None if pre is None else _dptr(pre), leaf)
        n = C.c_int()
        self._check(lib().liliom_global_map(*args, None, 0, C.byref(n)))
        out = np.zeros(max(n.value, 1), self.dtype)
        self._check(lib().liliom_global_map(*args, _ptr(out), len(out), C.byref(n)))
        return out[:n.value]

    # ---- wire formats (f3) ----
    @staticmethod
    def _livox(custom_pts, stride):
        a = np.ascontiguousarray(custom_pts)
        if stride is None:
            stride = a.dtype.itemsize
            return a, len(a), stride
        return a, a.size * a.dtype.itemsize // stride, stride

    def convert_livox(self, custom_pts: np.ndarray, stride: int | None = None, download: bool = True):
        a, n, stride = self._livox(custom_pts, stride)
        out = np.zeros(max(n, 1), PT48) if download else None
        self._check(lib().liliom_convert_livox(self._h, _ptr(a), n, stride, _ptr(out), len(out) if download else 0))
        return out[:n] if download else n

    def extract_horizon_livox(self, custom_pts: np.ndarray, q_imu, stride: int | None = None, out=None):
        a, n, stride = self._livox(custom_pts, stride)
        q = np.asarray(q_imu, dtype=np.float64)
        if out is None:
            surf = np.empty(max(n, 1), PT48); edge = np.empty(max(n, 1), PT48); cut = np.empty(max(n, 1), PT48)
        else:
            surf, edge, cut = out
        ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
        self._check(lib().liliom_extract_horizon_livox(self._h, _ptr(a), n, stride, _dptr(q), _ptr(surf), len(surf), C.byref(ns),
                                                       _ptr(edge), len(edge), C.byref(ne), _ptr(cut), len(cut), C.byref(nc)))
        return surf[:ns.value], edge[:ne.value], cut[:nc.value]

    def convert_pc2(self, msg: PC2, download: bool = True):
        """pcl::fromROSMsg(msg, PointXYZI) on the device; the sweep stays resident (extract_resident).  Returns the PT32 cloud,
        or its size when download=False."""
        m, _f = msg.c_msg()
        n = msg.width * msg.height
        out = np.zeros(max(n, 1), PT32) if download else None
        got = C.c_int()
        self._check(lib().liliom_convert_pc2(self._h, C.byref(m), _ptr(out), len(out) if download else 0, C.byref(got)))
        return out[:got.value] if download else got.value

    def set_ring_source(self, source: int):
        """RING_ELEVATION (default): the ROT extractor takes each return's ring from its elevation (line_num 16/32/64 tables);
        RING_FIELD: from the PointCloud2's `ring` field (convert_pc2 / extract_rot_pc2 / extract_resident, line_num 1..128)."""
        self._check(lib().liliom_set_ring_source(self._h, int(source)))

    def set_time_source(self, source: int, name=None):
        """TIME_AZIMUTH (default): the ROT extractor takes each return's relTime from the reference's azimuth rule;
        TIME_FIELD: from the PointCloud2's per-point time field `name` (e.g. "time", "t", "timestamp"), normalised over the
        surviving returns (convert_pc2 / extract_rot_pc2 / extract_resident)."""
        nm = name.encode() if isinstance(name, str) else name
        self._check(lib().liliom_set_time_source(self._h, int(source), nm))

    def extract_rot_pc2(self, msg: PC2, q_imu, q_lb=(1.0, 0.0, 0.0, 0.0), out=None):
        """extract_rot on the decoded PointCloud2 without a host cloud in between; out = optional (surf, edge, cut) PT32 arrays."""
        m, _f = msg.c_msg()
        n = msg.width * msg.height
        q = np.asarray(q_imu, dtype=np.float64); ql = np.asarray(q_lb, dtype=np.float64)
        if out is None:
            surf = np.empty(max(n, 1), PT32); edge = np.empty(max(n, 1), PT32); cut = np.empty(max(n, 1), PT32)
        else:
            surf, edge, cut = out
        ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
        self._check(lib().liliom_extract_rot_pc2(self._h, C.byref(m), _dptr(q), _dptr(ql), _ptr(surf), len(surf), C.byref(ns),
                                                 _ptr(edge), len(edge), C.byref(ne), _ptr(cut), len(cut), C.byref(nc)))
        return surf[:ns.value], edge[:ne.value], cut[:nc.value]

    # ---- multi-GPU / instrumentation ----
    def comm_init(self, unique_id: bytes, nranks: int, rank: int):
        buf = C.create_string_buffer(unique_id, 128)
        self._check(lib().liliom_comm_init(self._h, buf, nranks, rank))

    def comm_set_shard_block(self, metres: int):
        self._check(lib().liliom_comm_set_shard_block(self._h, metres))

    def comm_peer_export(self) -> bytes:
        """64-byte IPC handle of this rank's exchange buffer (fused multi-GPU exchange, include/liliom.h)."""
        buf = C.create_string_buffer(64)
        self._check(lib().liliom_comm_peer_export(self._h, buf))
        return buf.raw

    def comm_peer_attach(self, handles, rank: int):
        """handles: the exported handles of all ranks in rank order (e.g. from dist.all_gather_object)."""
        blob = b"".join(handles)
        buf = C.create_string_buffer(blob, len(blob))
        self._check(lib().liliom_comm_peer_attach(self._h, buf, len(handles), rank))

    def comm_peer_epoch(self) -> int:
        e = C.c_uint()
        self._check(lib().liliom_comm_peer_epoch(self._h, C.byref(e)))
        return e.value

    def comm_peer_set_epoch(self, epoch: int):
        """Recovery after a lost exchange: every rank sets max-over-ranks(comm_peer_epoch()) + 2 (include/liliom.h)."""
        self._check(lib().liliom_comm_peer_set_epoch(self._h, epoch))

    def counters(self, reset: bool = False) -> Counters:
        c = Counters()
        self._check(lib().liliom_get_counters(self._h, C.byref(c), 1 if reset else 0))
        return c

    def knn_block_stats(self, pose7):
        """(queries, points in their full 27-cell blocks) for the resident queries at pose7: the C-bar of SURVEY.md §8(d)."""
        p = np.asarray(pose7, dtype=np.float64)
        out = (C.c_ulonglong * 2)()
        self._check(lib().liliom_knn_block_stats(self._h, _dptr(p), out))
        return int(out[0]), int(out[1])

    def set_kernel_timing(self, on):
        """True / 1: time every kNN+Jacobian launch; N > 1: every N-th scan-to-map call; False / 0: off."""
        self._check(lib().liliom_set_kernel_timing(self._h, int(on)))


def comm_get_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    rc = lib().liliom_comm_get_unique_id(buf)
    if rc != OK:
        raise LiliomError(rc)
    return buf.raw


class PreprocessingNode:
    """Host-side mirror of the reference's Preprocessing node (csrc/host/nodes.cpp) on a Context."""

    def __init__(self, ctx: Context, q_lb=(1.0, 0.0, 0.0, 0.0)):
        self.ctx = ctx
        variant = 1 if ctx.stride == 32 else 0
        self._cap = 0
        self._bufs = None
        self._h = lib().liliom_pre_create(ctx._h, variant, _dptr(np.asarray(q_lb, np.float64)))

    def close(self):
        if self._h:
            lib().liliom_pre_destroy(self._h); self._h = None

    def imu(self, stamp: float, gyro):
        lib().liliom_pre_imu(self._h, float(stamp), _dptr(np.asarray(gyro, np.float64)))

    def _out_bufs(self, n: int):
        cap = max(self._cap, n)
        if cap > self._cap or self._bufs is None:
            self._cap = cap
            self._bufs = [np.empty(max(cap, 1), self.ctx.dtype) for _ in range(3)]
        return self._bufs, max(cap, 1)

    def cloud(self, stamp: float, pts: np.ndarray):
        """Returns None while queueing / waiting for IMU, else (stamp, surf, edge, cutted, q_imu)."""
        pts = np.ascontiguousarray(pts, dtype=self.ctx.dtype)
        (surf, edge, cut), cap = self._out_bufs(len(pts))
        ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
        st = C.c_double(); q = np.zeros(4)
        rc = lib().liliom_pre_cloud(self._h, float(stamp), _ptr(pts), len(pts), _ptr(surf), cap, C.byref(ns), _ptr(edge), cap, C.byref(ne),
                                    _ptr(cut), cap, C.byref(nc), C.byref(st), _dptr(q))
        return self._result(rc, st, surf, edge, cut, ns, ne, nc, q)

    def cloud_pc2(self, stamp: float, msg: PC2):
        """The ROT node's cloudHandler on the driver's PointCloud2 (liliom_pre_cloud_pc2); same results as cloud()."""
        m, _f = msg.c_msg()
        (surf, edge, cut), cap = self._out_bufs(msg.width * msg.height)
        ns, ne, nc = C.c_int(), C.c_int(), C.c_int()
        st = C.c_double(); q = np.zeros(4)
        rc = lib().liliom_pre_cloud_pc2(self._h, float(stamp), C.byref(m), _ptr(surf), cap, C.byref(ns), _ptr(edge), cap, C.byref(ne),
                                        _ptr(cut), cap, C.byref(nc), C.byref(st), _dptr(q))
        return self._result(rc, st, surf, edge, cut, ns, ne, nc, q)

    def _result(self, rc, st, surf, edge, cut, ns, ne, nc, q):
        if rc < 0:
            raise LiliomError(rc, lib().liliom_last_error(self.ctx._h).decode())
        if rc == 0:
            return None
        return st.value, surf[:ns.value].copy(), edge[:ne.value].copy(), cut[:nc.value].copy(), q


class LidarOdometryNode:
    """Host-side mirror of the reference's LidarOdometry node (csrc/host/nodes.cpp) on a Context."""

    def __init__(self, ctx: Context, max_num_iter=15, scan_match_cnt=1, if_to_deskew=False, mode=MODE_CERES):
        self.ctx = ctx
        self._cap = 0
        self._bufs = None
        self._h = lib().liliom_lo_create(ctx._h, max_num_iter, scan_match_cnt, 1 if if_to_deskew else 0, mode)

    def close(self):
        if self._h:
            lib().liliom_lo_destroy(self._h); self._h = None

    def feed(self, stamp: float, edge: np.ndarray, surf: np.ndarray, full: np.ndarray):
        for fn, a in ((lib().liliom_lo_edge, edge), (lib().liliom_lo_surf, surf), (lib().liliom_lo_full, full)):
            a = np.ascontiguousarray(a, dtype=self.ctx.dtype)
            self._cap = max(self._cap, len(a))
            fn(self._h, float(stamp), _ptr(a), len(a))

    def run(self, want_clouds: bool = True):
        out = LoOutput()
        ne, ns, nf = C.c_int(), C.c_int(), C.c_int()
        if not want_clouds:
            rc = lib().liliom_lo_run(self._h, C.byref(out), None, 0, C.byref(ne), None, 0, C.byref(ns), None, 0, C.byref(nf))
            if rc != OK:
                raise LiliomError(rc, lib().liliom_last_error(self.ctx._h).decode())
            return out, None, None, None
        cap = max(self._cap, 1)
        if self._bufs is None or len(self._bufs[0]) < cap:
            self._bufs = [np.empty(cap, self.ctx.dtype) for _ in range(3)]
        e, s, f = self._bufs
        rc = lib().liliom_lo_run(self._h, C.byref(out), _ptr(e), len(e), C.byref(ne), _ptr(s), len(s), C.byref(ns), _ptr(f), len(f), C.byref(nf))
        if rc != OK:
            raise LiliomError(rc, lib().liliom_last_error(self.ctx._h).decode())
        return out, e[:ne.value].copy(), s[:ns.value].copy(), f[:nf.value].copy()
