"""liliom_b200 — H100-native (sm_90a) implementation of the per-scan hot path of KIT-ISAS/lili-om.

Layout (SURVEY.md §8): `csrc/` hand-written CUDA kernels + the C ABI (include/liliom.h),
`_lib.py` ctypes binding, `synth.py` seeded synthetic worlds and sweeps.
There is no CPU fallback: every compute entry point runs the CUDA library or raises.
"""
from . import _lib as _binding
from ._lib import (Context, Params, IterStats, Counters, LiliomError, default_params, comm_get_unique_id,  # noqa: F401
                   PT48, PT32, LIVOX20, MODE_CERES, MODE_GN, LIB_PATH, EXPORTS, NODE_EXPORTS, PreprocessingNode, LidarOdometryNode, LoOutput, pc2_layout, PC2,
                   BackendParams, backend_default_params, KF_FULL, KF_SURF, KF_IMAGE_FULL, RING_ELEVATION, RING_FIELD,
                   TIME_AZIMUTH, TIME_FIELD, scan_to_map_resident_batch, odometry_resident_batch,
                   scan_to_map_resident_batch_ex, odometry_resident_batch_ex, extract_resident_batch, map_update_batch,
                   backend_window_correspond_batch, backend_window_blocks_batch, loop_align_batch, LoopParams, LoopResult,
                   convert_batch, WireMsg, WIRE_LIVOX, WIRE_PC2, undistort_resident_batch, kf_add_resident_batch,
                   bmap_build_batch, bmap_build_batch_multi, loop_align_batch_multi)

__all__ = ["Context", "Params", "IterStats", "Counters", "LiliomError", "default_params", "comm_get_unique_id",
           "PT48", "PT32", "MODE_CERES", "MODE_GN", "LIB_PATH", "EXPORTS",
           "BackendParams", "backend_default_params", "KF_FULL", "KF_SURF", "KF_IMAGE_FULL", "PC2", "RING_ELEVATION", "RING_FIELD",
           "TIME_AZIMUTH", "TIME_FIELD", "scan_to_map_resident_batch", "odometry_resident_batch",
           "scan_to_map_resident_batch_ex", "odometry_resident_batch_ex", "extract_resident_batch", "map_update_batch",
           "backend_window_correspond_batch", "backend_window_blocks_batch", "loop_align_batch", "LoopParams", "LoopResult",
           "convert_batch", "WireMsg", "WIRE_LIVOX", "WIRE_PC2", "undistort_resident_batch", "kf_add_resident_batch",
           "bmap_build_batch", "bmap_build_batch_multi", "loop_align_batch_multi"]
