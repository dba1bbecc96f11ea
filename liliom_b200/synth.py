"""Deterministic synthetic inputs for the LiLi-OM hot path (SURVEY.md §8 d): no dataset ships with
the reference and there is no network, so tests and bench.py use a seeded planar world.

World: ground z = 0; a lattice of 40 m city blocks with 8 m high walls
  X-walls: planes y = 20 + 40k, spanning x in [40j + 4, 40j + 36]
  Y-walls: planes x = 20 + 40k, spanning y in [40j + 4, 40j + 36]
  poles  : vertical cylinders r = 0.15 m at (10 + 20a, 6 + 20b) (edge features)
Map    : ~one point per occupied 0.4 m voxel of those surfaces (jittered lattice, sigma 1 cm normal
         noise) = what pcl::VoxelGrid(0.4) leaves of a dense local map (L/src/LidarOdometry.cpp:316).
Sweeps : Livox-Horizon-like (6 lines x 4000 time columns, FormatConvert encoding,
         L/src/FormatConvert.cpp:14-22) and HDL-64E-like (64 rings x 2031 azimuth steps, ring
         elevations = inverse of R/src/Preprocessing.cpp:332-337), ray-cast from a given pose with
         the sensor rotating at a constant gyro rate so that the reference's de-skew is consistent.
"""
from __future__ import annotations

import numpy as np

from ._lib import PC2, PT32, PT48

BLOCK = 40.0
WALL_H = 8.0
WALL_LO, WALL_HI = 4.0, 36.0
POLE_R = 0.15


# ------------------------------------------------------------------ quaternion helpers (w,x,y,z)
def qmul(a, b):
    aw, ax, ay, az = a; bw, bx, by, bz = b
    return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx])


def qrot(q, v):
    q = np.asarray(q, float); v = np.asarray(v, float)
    qv = q[1:]
    uv = 2.0 * np.cross(qv, v)
    return v + q[0] * uv + np.cross(qv, uv)


def q_from_axis_angle(axis, angle):
    axis = np.asarray(axis, float); axis = axis / np.linalg.norm(axis)
    return np.concatenate([[np.cos(angle / 2)], np.sin(angle / 2) * axis])


def pose_compose(a7, b7):
    """a ∘ b (apply b in a's frame) — L/src/LidarOdometry.cpp:415-442."""
    a7 = np.asarray(a7, float); b7 = np.asarray(b7, float)
    return np.concatenate([qmul(a7[:4], b7[:4]), qrot(a7[:4], b7[4:]) + a7[4:]])


def perturbed_pose(true7, dt=(0.10, -0.05, 0.02), ddeg=1.0):
    """Initial guess = T* ∘ (δt, δθ about (1,1,1)/√3) (SURVEY.md §8 d)."""
    dq = q_from_axis_angle([1, 1, 1], np.deg2rad(ddeg))
    return pose_compose(true7, np.concatenate([dq, dt]))


def integrate_gyro(omega, sweep=0.1, rate=200.0):
    """q_iMU as the reference builds it: product of un-normalised deltaQ(0.5(g0+g1)dt)
    (L/include/utils/math_tools.h:125-138, L/src/Preprocessing.cpp:129-133), constant rate."""
    q = np.array([1.0, 0, 0, 0])
    dt = 1.0 / rate
    for _ in range(int(round(sweep * rate))):
        th = np.asarray(omega, float) * dt
        q = qmul(q, np.array([1.0, th[0] / 2, th[1] / 2, th[2] / 2]))
    return q


# ------------------------------------------------------------------ map
def _surface_lattice(rng, u0, u1, v0, v1, step=0.4):
    nu = max(int(np.floor((u1 - u0) / step)), 1); nv = max(int(np.floor((v1 - v0) / step)), 1)
    u = u0 + (np.arange(nu) + 0.5) * step; v = v0 + (np.arange(nv) + 0.5) * step
    uu, vv = np.meshgrid(u, v, indexing="ij")
    uu = uu + rng.uniform(-0.15, 0.15, uu.shape); vv = vv + rng.uniform(-0.15, 0.15, vv.shape)
    nn = rng.normal(0.0, 0.01, uu.shape)
    return uu.ravel(), vv.ravel(), nn.ravel()


def make_map(m_target: int, seed: int = 20260923):
    """Returns float32 [M,4] (x,y,z,1) with M == m_target exactly (nearest-to-origin subset of a
    slightly larger world) and the half-extent S of the world that was generated."""
    rng = np.random.default_rng(seed)
    per_block = (BLOCK * BLOCK + 2 * (WALL_HI - WALL_LO) * WALL_H) / 0.16
    nb = int(np.ceil(np.sqrt(m_target * 1.35 / per_block)))
    nb += nb % 2   # even number of blocks per side, world centred on the origin
    S = nb * BLOCK / 2.0
    parts = []
    u, v, n = _surface_lattice(rng, -S, S, -S, S)
    parts.append(np.stack([u, v, n], 1))                                    # ground
    ks = np.arange(-nb // 2, nb // 2)
    for k in ks:
        for j in ks:
            yk = 20.0 + BLOCK * k; x0 = BLOCK * j + WALL_LO; x1 = BLOCK * j + WALL_HI
            u, v, n = _surface_lattice(rng, x0, x1, 0.0, WALL_H)
            parts.append(np.stack([u, yk + n, v], 1))                       # X-wall (plane y = yk)
            xk = 20.0 + BLOCK * k; y0 = BLOCK * j + WALL_LO; y1 = BLOCK * j + WALL_HI
            u, v, n = _surface_lattice(rng, y0, y1, 0.0, WALL_H)
            parts.append(np.stack([xk + n, u, v], 1))                       # Y-wall (plane x = xk)
    pts = np.concatenate(parts, 0)
    if len(pts) < m_target:
        raise RuntimeError("world too small for the requested map size")
    r2 = pts[:, 0] ** 2 + pts[:, 1] ** 2
    keep = np.argpartition(r2, m_target - 1)[:m_target]
    keep.sort()
    out = np.ones((m_target, 4), np.float32)
    out[:, :3] = pts[keep].astype(np.float32)
    return out, S


# ------------------------------------------------------------------ ray casting
def _raycast(o, d, max_range=190.0):
    """o [3], d [N,3] unit directions (world). Returns range [N] (inf = no hit)."""
    n = len(d)
    best = np.full(n, np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        # ground
        t = -o[2] / d[:, 2]
        ok = (t > 0.05) & (t < max_range)
        best = np.where(ok & (t < best), t, best)
        kmax = int(np.ceil(max_range / BLOCK)) + 1
        for axis in (0, 1):        # axis 1: X-walls (y = const), axis 0: Y-walls (x = const)
            other = 1 - axis
            base = np.floor((o[axis] - 20.0) / BLOCK)
            for k in range(-kmax, kmax + 1):
                c = 20.0 + BLOCK * (base + k)
                t = (c - o[axis]) / d[:, axis]
                ok = (t > 0.05) & (t < max_range)
                h = o[2] + t * d[:, 2]
                w = o[other] + t * d[:, other]
                wm = np.mod(w, BLOCK)
                ok &= (h >= 0.0) & (h <= WALL_H) & (wm >= WALL_LO) & (wm <= WALL_HI)
                best = np.where(ok & (t < best), t, best)
        # poles: circles in xy at (10 + 20a, 6 + 20b), height WALL_H
        dxy2 = d[:, 0] ** 2 + d[:, 1] ** 2
        a0 = np.floor((o[0] - 10.0) / 20.0); b0 = np.floor((o[1] - 6.0) / 20.0)
        for a in range(-3, 5):
            for b in range(-3, 5):
                cx = 10.0 + 20.0 * (a0 + a); cy = 6.0 + 20.0 * (b0 + b)
                ox = o[0] - cx; oy = o[1] - cy
                bb = ox * d[:, 0] + oy * d[:, 1]
                cc = ox * ox + oy * oy - POLE_R ** 2
                disc = bb * bb - dxy2 * cc
                t = (-bb - np.sqrt(np.where(disc > 0, disc, np.nan))) / dxy2
                h = o[2] + t * d[:, 2]
                ok = (disc > 0) & (t > 0.05) & (t < max_range) & (h >= 0) & (h <= WALL_H)
                best = np.where(ok & (t < best), t, best)
    return best


def _slerp_from_identity(q, s):
    """Eigen slerp(I -> q) for an array of fractions s (numpy, used only to generate sweeps)."""
    qn = q / np.linalg.norm(q)
    ang = 2.0 * np.arccos(np.clip(qn[0], -1, 1))
    axis = qn[1:]
    na = np.linalg.norm(axis)
    axis = axis / na if na > 0 else np.array([0.0, 0, 1.0])
    half = 0.5 * ang * s
    return np.concatenate([np.cos(half)[:, None], np.sin(half)[:, None] * axis[None, :]], 1)


def _rotate_many(qs, v):
    qv = qs[:, 1:]
    uv = 2.0 * np.cross(qv, v)
    return v + qs[:, :1] * uv + np.cross(qv, uv)


def make_horizon_sweep(true_pose7, seed: int = 1, omega=(0.0, 0.0, 0.2), dropout=0.02, noise=0.02):
    """24,000-point Livox-Horizon-like sweep (time order). Returns (pts PT48[n], q_imu[4])."""
    rng = np.random.default_rng(seed)
    lines, cols = 6, 4000
    elev = np.deg2rad(np.linspace(-12.55, 12.55, lines))
    s = np.arange(cols) / (cols - 1.0)                       # fraction of the sweep
    tri = 2.0 * np.abs(2.0 * ((s * 2.0) % 1.0) - 1.0) - 1.0   # two back-and-forth passes
    az = np.deg2rad(40.85) * tri
    L, Cc = np.meshgrid(np.arange(lines), np.arange(cols), indexing="xy")   # time-major: col outer, line inner
    L = L.ravel(); Cc = Cc.ravel()
    a = az[Cc]; frac = s[Cc]
    # each laser wobbles +-2.5 deg in elevation (13 periods per sweep) like the Horizon's rosette, so the
    # six lines cover the field of view instead of tracing six thin arcs
    e = elev[L] + np.deg2rad(2.5) * np.sin(2.0 * np.pi * 13.0 * frac + 1.3 * L)
    d_s = np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], 1)
    q_imu = integrate_gyro(omega)
    q_t = _slerp_from_identity(q_imu, frac)
    d_start = _rotate_many(q_t, d_s)                          # direction in the sweep-start frame
    T = np.asarray(true_pose7, float)
    qT = np.broadcast_to(T[:4], (len(d_start), 4))
    d_w = _rotate_many(qT, d_start)
    rng_m = _raycast(T[4:], d_w)
    hit = np.isfinite(rng_m) & (rng.uniform(size=len(rng_m)) >= dropout)
    r = np.where(hit, rng_m, 0.0) + rng.normal(0.0, noise, len(rng_m))
    p = d_s * r[:, None]                                      # raw (distorted) point in the sensor frame at its own time
    out = np.zeros(int(hit.sum()), PT48)
    out["x"] = p[hit, 0]; out["y"] = p[hit, 1]; out["z"] = p[hit, 2]; out["w"] = 1.0
    fs = (frac[hit]).astype(np.float32)
    out["intensity"] = (L[hit].astype(np.float32) + fs * np.float32(0.1)).astype(np.float32)   # FormatConvert.cpp:19-20
    refl = rng.integers(10, 201, size=len(out))
    out["curvature"] = (0.1 * refl).astype(np.float32)                                          # FormatConvert.cpp:21
    return out, q_imu


def hdl64_elevations():
    """Ring elevations (deg) mapped to scanID 0..63 by R/src/Preprocessing.cpp:332-337."""
    up = 2.0 - np.arange(32) / 3.0
    lo = -8.83 - np.arange(32) / 2.0
    return np.concatenate([up, lo])


def make_hdl64_sweep(true_pose7, seed: int = 2, omega=(0.0, 0.0, 0.2), steps: int = 2031, noise=0.02, dropout=0.01, grid: bool = False):
    """~130k-point HDL-64E-like sweep in firing order (azimuth-major, clockwise). Returns (PT32[n], q_imu); grid=True appends
    each return's ring (0..63, the row of hdl64_elevations) and azimuth step (0..steps-1), which organised layouts need."""
    pts, q_imu, ring, step = make_spinning_sweep(true_pose7, hdl64_elevations(), steps, seed=seed, omega=omega, noise=noise,
                                                 dropout=dropout)
    if grid:
        return pts, q_imu, ring, step
    return pts, q_imu


def uniform_elevations(lines: int = 128, top_deg: float = 22.5, bottom_deg: float = -22.5):
    """Ring elevations (deg) of a uniform spinning LiDAR numbered from the top, as Ouster numbers its beams: ring 0 at top_deg,
    ring lines-1 at bottom_deg (an OS-1-128-like fan by default)."""
    return np.linspace(top_deg, bottom_deg, lines)


def make_spinning_sweep(true_pose7, elevations_deg, steps: int, seed: int = 2, omega=(0.0, 0.0, 0.2), noise=0.02, dropout=0.01,
                        max_range=120.0):
    """One sweep of a spinning LiDAR with any beam layout: ring r fires at elevations_deg[r], `steps` azimuth columns per turn,
    in firing order (azimuth-major, clockwise), ray-cast from true_pose7 while the sensor turns at the gyro rate omega.
    Returns (PT32[n], q_imu, ring[n], step[n]): each return's ring (the index into elevations_deg) and azimuth step, which the
    driver publishes in its `ring` field and organised layouts need."""
    rng = np.random.default_rng(seed)
    elev = np.deg2rad(np.asarray(elevations_deg, float))
    k = np.arange(steps)
    frac = k / float(steps)
    az = -(2.0 * np.pi * frac) - 0.3        # clockwise: -atan2(y,x) increases with time
    K, R = np.meshgrid(k, np.arange(len(elev)), indexing="ij")
    K = K.ravel(); R = R.ravel()
    e = elev[R]; a = az[K]; f = frac[K]
    d_s = np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], 1)
    q_imu = integrate_gyro(omega)
    q_t = _slerp_from_identity(q_imu, f)
    d_start = _rotate_many(q_t, d_s)
    T = np.asarray(true_pose7, float)
    d_w = _rotate_many(np.broadcast_to(T[:4], (len(d_start), 4)), d_start)
    rng_m = _raycast(T[4:], d_w, max_range=max_range)
    hit = np.isfinite(rng_m) & (rng.uniform(size=len(rng_m)) >= dropout)
    r = np.where(hit, rng_m, 0.0) + rng.normal(0.0, noise, len(rng_m))
    p = d_s * r[:, None]
    out = np.zeros(int(hit.sum()), PT32)
    out["x"] = p[hit, 0]; out["y"] = p[hit, 1]; out["z"] = p[hit, 2]; out["w"] = 1.0
    out["intensity"] = rng.integers(0, 256, size=len(out)).astype(np.float32)
    return out, q_imu, R[hit].astype(np.int32), K[hit].astype(np.int32)


# ------------------------------------------------------------------ PointCloud2 as spinning-LiDAR drivers publish it
PC2_F32, PC2_F64, PC2_U8, PC2_U16, PC2_U32 = 7, 8, 2, 4, 6      # sensor_msgs::PointField datatypes
_PC2_NP = {PC2_F32: "<f4", PC2_F64: "<f8", PC2_U8: "u1", PC2_U16: "<u2", PC2_U32: "<u4"}
# Representative driver layouts, described from knowledge of the drivers' published point types (not from their sources):
#   velodyne22    packed x, y, z, intensity (f32), ring (u16), time (f32): 22 B per point, one row in firing order
#   pcl32         PCL-aligned 32 B: x, y, z at 0-11, intensity at 16, ring (u16) at 20, the rest padding; one row
#   ouster48      organised rings x columns (64 x steps), 48 B: x, y, z, intensity (f32) at 16, t (u32), reflectivity (u16),
#                 ring (u8), ambient (u16), range (u32); (0, 0, 0) for a missing return
#   organised_nan organised 64 x steps, 16 B points listed intensity first, NaN for a missing return, rows padded by 40 bytes
#   hesai26       packed x, y, z, intensity (f32), timestamp (f64, absolute seconds) at 16, ring (u16) at 24: 26 B per point,
#                 one row in firing order
PC2_LAYOUTS = ("velodyne22", "pcl32", "ouster48", "organised_nan")
# the per-point time field of the layouts that carry one (LILIOM_TIME_FIELD): a step-k return fires k * 0.1 / steps s into the sweep
PC2_TIME_FIELDS = {"velodyne22": "time", "ouster48": "t", "hesai26": "timestamp"}
HESAI_EPOCH = 1.7e9                   # hesai26: absolute stamp of the sweep start, s


def encode_pc2(pts, ring, step, layout: str, steps: int = 2031, lines: int = 64, t0: float = 0.0) -> PC2:
    """The sweep pts (PT32, with make_hdl64_sweep(grid=True)'s or make_spinning_sweep's ring and step per return) as the
    PointCloud2 a driver of the given layout would publish; organised layouts are lines x steps.  Bytes that no field covers
    are filled with a non-zero pattern.  t0: seconds added to every return's time (velodyne22 `time`, ouster48 `t` in whole
    ns, hesai26 `timestamp`), so that the first return need not be at 0; t0 = 0 leaves the existing layouts as they were."""
    F, U8, U16, U32 = PC2_F32, PC2_U8, PC2_U16, PC2_U32
    xyz = [("x", 0, F, 1), ("y", 4, F, 1), ("z", 8, F, 1)]
    organised, pad, missing = False, 0, 0.0
    if layout == "velodyne22":
        fields, point_step = xyz + [("intensity", 12, F, 1), ("ring", 16, U16, 1), ("time", 18, F, 1)], 22
    elif layout == "pcl32":
        fields, point_step = xyz + [("intensity", 16, F, 1), ("ring", 20, U16, 1)], 32
    elif layout == "ouster48":
        fields = xyz + [("intensity", 16, F, 1), ("t", 20, U32, 1), ("reflectivity", 24, U16, 1), ("ring", 26, U8, 1),
                        ("ambient", 28, U16, 1), ("range", 32, U32, 1)]
        point_step, organised = 48, True
    elif layout == "organised_nan":
        fields = [("intensity", 12, F, 1)] + xyz
        point_step, organised, pad, missing = 16, True, 40, np.nan
    elif layout == "hesai26":
        fields, point_step = xyz + [("intensity", 12, F, 1), ("timestamp", 16, PC2_F64, 1), ("ring", 24, U16, 1)], 26
    else:
        raise ValueError(f"unknown PointCloud2 layout {layout!r}")
    dt = np.dtype({"names": [f[0] for f in fields], "formats": [_PC2_NP[f[2]] for f in fields],
                   "offsets": [f[1] for f in fields], "itemsize": point_step})
    height, width = (lines, steps) if organised else (1, len(pts))
    rec = np.full(height * width * point_step, 0xA5, np.uint8).view(dt)
    ring = np.asarray(ring, np.int64); step = np.asarray(step, np.int64)
    if organised:
        for f in fields:
            rec[f[0]] = missing if f[0] in ("x", "y", "z") else 0
        idx = ring * width + step
    else:
        idx = np.arange(len(pts))
    for f in ("x", "y", "z", "intensity"):
        rec[f][idx] = pts[f]
    if "ring" in dt.names:
        rec["ring"][idx] = ring
    if layout == "velodyne22":
        rec["time"][idx] = (step * (0.1 / steps) + t0).astype(np.float32)
    if layout == "hesai26":
        rec["timestamp"][idx] = HESAI_EPOCH + t0 + step * (0.1 / steps)
    if layout == "ouster48":
        r = np.sqrt(pts["x"].astype(np.float64) ** 2 + pts["y"].astype(np.float64) ** 2 + pts["z"].astype(np.float64) ** 2)
        rec["t"][idx] = step * (100_000_000 // steps) + int(round(t0 * 1e9))
        rec["reflectivity"][idx] = pts["intensity"].astype(np.uint16)
        rec["ambient"][idx] = 100
        rec["range"][idx] = np.round(r * 1000.0).astype(np.uint32)
    row_step = width * point_step + pad
    data = np.full((height, row_step), 0xA5, np.uint8)
    data[:, :width * point_step] = rec.view(np.uint8).reshape(height, width * point_step)
    return PC2(data.reshape(-1), height, width, point_step, row_step, fields)


def default_true_pose():
    """Sensor 1.8 m above ground inside a block, yawed 8 deg, slightly pitched."""
    q = qmul(q_from_axis_angle([0, 0, 1], np.deg2rad(8.0)), q_from_axis_angle([0, 1, 0], np.deg2rad(-1.5)))
    return np.concatenate([q, [2.0, 3.0, 1.8]])


def make_keyframe_sequence(n: int, stride: int = 48, seed: int = 7, step=1.5, yaw_deg=2.0, surf_every: int = 8, full: bool = False,
                           revisit: int = 0):
    """A seeded keyframe stream for the backend (SURVEY.md §8 f5): n Horizon sweeps (no rotation inside a sweep, i.e. the
    clouds the backend receives after de-skew) taken every `step` metres along a gently turning path through the world.
    Each keyframe is split the way the extractors split a sweep: edge = returns from poles and wall tops (line-like
    neighbourhoods), surf = every `surf_every`-th other return.  Reflectivity (the `curvature` field, FormatConvert.cpp:21)
    is per surface kind plus a little noise, so the reflectivity-weighted plane fit of the Horizon backend sees real planes.
    Returns a list of (edge, surf, pose7) with clouds in the body frame, PT48 (stride 48) or PT32 (stride 32); full=True appends
    each keyframe's whole sweep (the /full_point_cloud the edge and surf clouds were split from): (edge, surf, pose7, full).
    revisit > 0 appends that many keyframes that come back to the poses of keyframes 0, 1, ... with new sweeps (a loop closure)."""
    rng = np.random.default_rng(seed)
    T0 = default_true_pose()
    out = []
    for i in range(n + revisit):
        j = i if i < n else i - n
        yaw = np.deg2rad(yaw_deg * j)
        q = qmul(q_from_axis_angle([0, 0, 1], yaw), T0[:4])
        t = T0[4:] + np.array([step * j, 0.35 * np.sin(0.4 * j), 0.0])
        pose = np.concatenate([q, t])
        pts, _ = make_horizon_sweep(pose, seed=seed * 1000 + i, omega=(0.0, 0.0, 0.0))
        p = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(np.float64)
        w = _rotate_many(np.broadcast_to(q, (len(p), 4)), p) + t
        px = (w[:, 0] - 10.0) - 20.0 * np.round((w[:, 0] - 10.0) / 20.0)
        py = (w[:, 1] - 6.0) - 20.0 * np.round((w[:, 1] - 6.0) / 20.0)
        pole = np.hypot(px, py) < 0.4
        top = w[:, 2] > WALL_H - 0.6
        ground = w[:, 2] < 0.2
        edge_m = pole | top
        base = np.where(pole, 12.0, np.where(top, 8.0, np.where(ground, 2.0, 6.0)))
        pts["curvature"] = (base + rng.normal(0.0, 0.05, len(pts))).astype(np.float32)
        surf_idx = np.flatnonzero(~edge_m)[::surf_every]
        edge, surf = pts[edge_m], pts[surf_idx]
        if stride == 32:
            def to32(a):
                b = np.zeros(len(a), PT32)
                for f in ("x", "y", "z", "w", "intensity"):
                    b[f] = a[f]
                return b
            edge, surf, pts = to32(edge), to32(surf), to32(pts)
        out.append((edge, surf, pose, pts) if full else (edge, surf, pose))
    return out
