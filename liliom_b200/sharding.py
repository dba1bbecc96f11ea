"""Host-side statement of the multi-GPU partition rule implemented in csrc/ (knn_core.cuh
`owner_of` and `shard_keep`): space is cut into 16 m blocks (shifted by half a block in z), a block belongs to rank
(bx + 3 by + 5 bz) mod nranks, a query is processed by the owner of the block its transformed position
falls in, and a rank's map shard holds every point whose +-halo box touches a block it owns (so the
query's whole 1 m search ball is local).  Used by bench.py to report shard sizes and by the gloo tests."""
from __future__ import annotations

import numpy as np


def owner_of(xyz: np.ndarray, nranks: int, block: int = 16) -> np.ndarray:
    """knn_core.cuh::owner_of: cube coordinates (z shifted by half an edge), linear hash bx + 3 by + 5 bz mod nranks."""
    xyz = np.asarray(xyz, np.float32)
    inv = np.float32(1.0 / block)
    bx = np.floor(xyz[..., 0] * inv).astype(np.int64)
    by = np.floor(xyz[..., 1] * inv).astype(np.int64)
    bz = np.floor(xyz[..., 2] * inv + np.float32(0.5)).astype(np.int64)
    return np.mod(bx + 3 * by + 5 * bz, nranks).astype(np.int32)


def shard_mask(xyz: np.ndarray, nranks: int, rank: int, halo: float = 1.0, block: int = 16) -> np.ndarray:
    xyz = np.asarray(xyz, np.float32)
    keep = np.zeros(len(xyz), bool)
    h = np.float32(halo)
    for c in range(8):
        off = np.array([h if c & 1 else -h, h if c & 2 else -h, h if c & 4 else -h], np.float32)
        keep |= owner_of(xyz + off, nranks, block) == rank
    return keep


def transform_f32(p_xyz: np.ndarray, pose7) -> np.ndarray:
    """q * p + t in fp64 (Eigen's expression), narrowed to fp32 (L/src/LidarOdometry.cpp:221-238)."""
    q = np.asarray(pose7[:4], np.float64); t = np.asarray(pose7[4:], np.float64)
    p = np.asarray(p_xyz, np.float64)
    uv = 2.0 * np.cross(q[1:], p)
    return (p + q[0] * uv + np.cross(q[1:], uv) + t).astype(np.float32)
