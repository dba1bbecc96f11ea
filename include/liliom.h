/* liliom.h — C ABI of libliliom_b200.so: an H100-native (sm_90a) drop-in for the per-scan hot
 * path of KIT-ISAS/lili-om.  The reference has no FFI/plugin interface for this path (it is
 * private member functions of two ROS node classes), so each entry point cites the reference
 * code it replaces; INTEGRATION.md shows the call a maintainer adds inside the node.
 * Citations are relative to the reference repository root
 * (L/ = LiLi-OM/, R/ = LiLi-OM-ROT/).
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is caller-owned HOST memory unless a
 *    function says "_dev"; the library never retains a host pointer after returning;
 *  - every call is synchronous from the caller's view (the context's stream is drained before
 *    return), matching the single-threaded ROS spinner the reference runs on
 *    (L/src/Preprocessing.cpp:417, L/src/LidarOdometry.cpp:697-703);
 *  - a context is NOT thread-safe and not re-entrant: one per node, one caller thread;
 *  - return value 0 = OK, <0 = LILIOM_E_* ; on error outputs and the pose are left untouched,
 *    mirroring the reference's "ROS_WARN + early return" (L/src/LidarOdometry.cpp:485-488);
 *  - pose layout [qw,qx,qy,qz,tx,ty,tz] fp64 = abs_pose (L/src/LidarOdometry.cpp:34-36);
 *  - point layouts are PCL's: 48-byte pcl::PointXYZINormal (L/include/utils/common.h:72-73)
 *    and 32-byte pcl::PointXYZI (R/include/utils/common.h:73), i.e. the bytes
 *    pcl::fromROSMsg / toROSMsg produce and consume.
 *  - there is NO CPU fallback: without a CUDA device liliom_create fails with LILIOM_E_CUDA.
 */
#ifndef LILIOM_H
#define LILIOM_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

#define LILIOM_ABI_VERSION 1

enum {
    LILIOM_OK          = 0,
    LILIOM_E_ARG       = -1,  /* null pointer, negative size, bad stride/mode */
    LILIOM_E_CUDA      = -2,  /* CUDA runtime error / no device (see liliom_last_error) */
    LILIOM_E_FEWMAP    = -3,  /* map has < 10 points: pose untouched (L/src/LidarOdometry.cpp:485-488) */
    LILIOM_E_CAPACITY  = -4,  /* caller buffer or configured capacity too small */
    LILIOM_E_GRID      = -5,  /* map extent too large for the dense 1 m cell table */
    LILIOM_E_LINES     = -6,  /* line_num not in {16,32,64} (R/src/Preprocessing.cpp:344-347), or not in 1..128 with
                                 LILIOM_RING_FIELD (liliom_set_ring_source) */
    LILIOM_E_NCCL      = -7,  /* NCCL unavailable or failed */
    LILIOM_E_NOMAP     = -8   /* scan_to_map called before any map was set */
};

typedef struct liliom_ctx liliom_ctx;

typedef struct { float x, y, z, w; } liliom_f4;
typedef struct { float x, y, z, w; float nx, ny, nz, nw; float intensity, curvature, p0, p1; } liliom_pt48; /* pcl::PointXYZINormal */
typedef struct { float x, y, z, w; float intensity, p0, p1, p2; } liliom_pt32;                             /* pcl::PointXYZI */

/* Every tunable the reference reads from the ROS parameter server or hard-codes on this path. */
typedef struct {
    int    abi_version;        /* = LILIOM_ABI_VERSION */
    int    point_stride;       /* 48 (Horizon package) or 32 (ROT package) */
    /* Preprocessing — Horizon: /preprocessing/{surf_thres,edge_thres}, L/src/Preprocessing.cpp:44-54 */
    double surf_thres;         /* default 0.2 */
    double edge_thres;         /* default 4.0 */
    /* Preprocessing — ROT: /preprocessing/{line_num,ds_rate}, R/src/Preprocessing.cpp:67-75; ds_v :14 */
    int    line_num;           /* 16 | 32 | 64 (elevation tables); 1..128 with LILIOM_RING_FIELD */
    int    ds_rate;            /* ring decimation */
    float  rot_ds_leaf;        /* 0.6 */
    /* LidarOdometry: leaf sizes L/src/LidarOdometry.cpp:155-156; gates :365,:389,:400; Huber :507; FIFO :290 */
    float  leaf_scan;          /* 0.4 */
    float  leaf_map;           /* 0.4 */
    double knn_max_sqdist;     /* 1.0  — 5th-neighbour squared distance gate (<= 4.0 supported) */
    double plane_thres;        /* 0.06 */
    double weight_gate;        /* 0.4  */
    double huber_a;            /* 0.1  */
    int    max_map_frames;     /* 20   */
    /* capacities (device buffers are sized from these at create time and grown on demand) */
    int    max_scan_points;    /* raw points per sweep, default 400000 (R/src/Preprocessing.cpp:9-12) */
    int    max_map_points;     /* default 2,000,000 */
} liliom_params;

/* variant 0 = Horizon package defaults (config L/config/config_fr_iosb.yaml),
 * variant 1 = ROT package defaults (R/config/config_fr_iosb.yaml). */
void liliom_default_params(liliom_params* p, int variant);

int  liliom_create(liliom_ctx** out, const liliom_params* p, int device);
int  liliom_point_stride(const liliom_ctx* c);          /* 48 or 32, as configured at creation */
void liliom_destroy(liliom_ctx* c);
const char* liliom_strerror(int code);
const char* liliom_last_error(const liliom_ctx* c);   /* detail of the last LILIOM_E_CUDA/NCCL */

/* ===================== L1: feature extraction ===================== */

/* Replaces the body of Preprocessing::cloudHandler between pcl::fromROSMsg and pcl::toROSMsg,
 * L/src/Preprocessing.cpp:219-383 (removeNaN, removeClosedPointCloud 0.1 m, gyro de-skew,
 * 6x4000 binning, 664-patch PCA labelling).  pts = n points as published by FormatConvert
 * (L/src/FormatConvert.cpp:14-22: intensity = line + 0.1*t/t_end, curvature = 0.1*reflectivity).
 * q_imu_wxyz = the un-normalised q_iMU produced by processIMU (:135-171), which stays host-side.
 * Outputs (capacities in points) = the three clouds published at :385-401.
 * The surf features stay resident on the device for liliom_odometry_resident(). */
int liliom_extract_horizon(liliom_ctx* c, const liliom_pt48* pts, int n, const double q_imu_wxyz[4],
                           liliom_pt48* surf_out, int surf_cap, int* n_surf,
                           liliom_pt48* edge_out, int edge_cap, int* n_edge,
                           liliom_pt48* cutted_out, int cut_cap, int* n_cut);

/* Replaces R/src/Preprocessing.cpp:276-509 (removeNaN, removeClosedPointCloud 3.0 m, ring id,
 * azimuth/relTime, de-skew with q_lb*q*q_lb^-1, 11-point curvature, per-segment sort + greedy
 * labelling, per-ring VoxelGrid 0.6 of the less-flat points).
 * edge_out = cornerPointsLessSharp, surf_out = surfPointsLessFlat, cutted_out = laserCloud (:511-527). */
int liliom_extract_rot(liliom_ctx* c, const liliom_pt32* pts, int n, const double q_imu_wxyz[4],
                       const double q_lb_wxyz[4],
                       liliom_pt32* surf_out, int surf_cap, int* n_surf,
                       liliom_pt32* edge_out, int edge_cap, int* n_edge,
                       liliom_pt32* cutted_out, int cut_cap, int* n_cut);
/* Test hook: per-point cloudLabel / cloudCurvature (R/src/Preprocessing.cpp:9-12) of the last
 * liliom_extract_rot call, in laserCloud order; either pointer may be NULL. */
int liliom_extract_rot_labels(liliom_ctx* c, int* label_out, float* curv_out, int cap);

/* pcl::VoxelGrid::filter (L/src/LidarOdometry.cpp:315-323; R/src/Preprocessing.cpp:502-508):
 * centroid of all fields per occupied voxel, output in ascending voxel index. stride = 48|32. */
int liliom_voxelgrid(liliom_ctx* c, const void* pts, int n, int stride, float leaf,
                     void* out, int cap, int* n_out);

/* ===================== L2: scan-to-map ===================== */

/* Local-map lifecycle, replaces buildLocalMap + downSampleCloud(map) + kd-tree build
 * (L/src/LidarOdometry.cpp:280-303, 316-317, 490).
 * push_frame: transformCloud (:246-278) of one frame's down-sampled surf cloud by its saved pose,
 *   appended to the FIFO of the last `max_map_frames` frames (:290-299);
 * rebuild: concatenation (:301-302) -> VoxelGrid(leaf_map) -> 1 m cell grid (the kd-tree's stand-in).
 * n_map_out (optional) = surf_from_map_ds size. */
int liliom_map_push_frame(liliom_ctx* c, const void* surf_ds_body, int n, const double pose7[7]);
int liliom_map_rebuild(liliom_ctx* c, int* n_map_out);
/* SURVEY §8 (f2): the same two steps as ONE incremental call — liliom_map_update == liliom_map_push_frame followed by
 * liliom_map_rebuild, bit for bit (same FIFO, same filtered cloud in the same order, same cell grid), but the VoxelGrid state
 * lives on the device across scans: the new frame's voxel keys are sorted on their own and merged into the resident sorted entry
 * array while the dropped frame's entries leave it, instead of re-sorting the whole concatenation (liliom_b200/csrc/map.cu).
 * Mixing it with the two separate calls is allowed (the entry array is rebuilt once after them).  Sharded contexts and clouds
 * whose voxel coordinates do not fit 21 bits take the two-step path internally.  _device: d_surf_ds_body is a DEVICE pointer. */
int liliom_map_update(liliom_ctx* c, const void* surf_ds_body, int n, const double pose7[7], int* n_map_out);
int liliom_map_update_device(liliom_ctx* c, const void* d_surf_ds_body, int n, const double pose7[7], int* n_map_out);
/* liliom_map_update with the frame taken from the context itself: surf_last_ds of the context's last liliom_odometry /
 * liliom_odometry_resident (or its batch forms), as left on the device.  pose7: the pose to save the frame with.  Bit for bit
 * liliom_map_update(c, <that cloud downloaded through ds_out>, n_ds, pose7, n_map_out), without the cloud crossing PCIe.
 * The scan is resident from the end of an odometry call (one that returned LILIOM_E_NOMAP / LILIOM_E_FEWMAP included) until
 * another call rewrites the buffer it lies in: liliom_voxelgrid, liliom_kf_add, liliom_kf_add_resident, liliom_kf_cloud, liliom_loop_align,
 * liliom_global_map, or an odometry call that fails.  Calls that only search (liliom_scan_to_map and its resident and
 * batch forms, liliom_find_surf_corr) leave it alone, whatever their feature count: the scan keeps its own count.  With no scan resident: LILIOM_E_ARG (see liliom_last_error), nothing
 * changed.  The map update itself only reads the scan, so it stays resident across this call (and may be pushed again). */
int liliom_map_update_resident(liliom_ctx* c, const double pose7[7], int* n_map_out);
/* surf_from_map_ds with all its fields (point_stride bytes per point), in liliom_map_download order (single GPU): the
 * filtered cloud of the last liliom_map_rebuild or liliom_map_update (empty after liliom_map_clear).  A map installed with
 * liliom_map_set_points, liliom_map_set_cloud or liliom_icp_align has no filtered cloud behind it: LILIOM_E_NOMAP (see
 * liliom_last_error) until the next rebuild or update. */
int liliom_map_download_cloud(liliom_ctx* c, void* out, int cap, int* m_out);

/* push_frame for pipelines that keep surf_last_ds on the device (both nodes in one process): d_surf_ds_body is a DEVICE
 * pointer to n points of point_stride bytes, valid until the call returns.  Same semantics otherwise. */
int liliom_map_push_frame_device(liliom_ctx* c, const void* d_surf_ds_body, int n, const double pose7[7]);
int liliom_map_clear(liliom_ctx* c);
/* Install an already down-sampled world-frame map (float4 xyz*, w ignored) — the synthetic
 * 1 M..10 M-point maps of the benchmark configs.  With a communicator (liliom_comm_init) each
 * rank keeps only the 16 m blocks it owns plus a halo. */
int liliom_map_set_points(liliom_ctx* c, const liliom_f4* xyzw, int m);
int liliom_map_size(const liliom_ctx* c);        /* points resident on this rank */
int liliom_map_download(liliom_ctx* c, liliom_f4* xyzw_out, int cap, int* m_out);  /* surf_from_map_ds */

enum { LILIOM_MODE_CERES = 0, LILIOM_MODE_GN = 1 };

typedef struct {
    int    n_corr;       /* surf_res_cnt at the linearisation pose (L/src/LidarOdometry.cpp:408) */
    int    lm_iters;     /* LM iterations run by this outer iteration (1 in GN mode) */
    double cost;         /* 1/2 sum rho(r^2) at the linearisation pose */
    double jtj_jtr[27];  /* upper triangle of J^T J (21, row-major) + J^T r (6); tangent = [rot, trans] */
    double pose7[7];     /* pose after this outer iteration */
} liliom_iter_stats;

/* Replaces downSampleCloud(scan) + updateTransformationWithCeres up to :561
 * (L/src/LidarOdometry.cpp:319-322, 483-561; R/src/LidarOdometry.cpp:469-547).
 * feats = surf_last_ds (already down-sampled, body frame; stride 48|32|16 — only xyz is read).
 * mode CERES: match_cnt outer iterations of [findCorrespondingSurfFeatures (:352-413) + a
 *   Ceres-2.0-default LM of <= max_num_iter iterations, Huber(0.1), 15 ms cap disabled];
 * mode GN   : match_cnt iterations of [re-associate + one Gauss-Newton step] (max_num_iter ignored).
 * stats: NULL or match_cnt entries.
 * On a context with a communicator mode CERES is refused with LILIOM_E_ARG unless liliom_comm_set_ceres(c, 1): then every
 * LM evaluation of an outer iteration is one all-reduce of the 29 sums over the ranks' own correspondences, and every rank
 * takes the same trust-region decisions and returns the same pose bits.  That pose is not bit-identical to one GPU's (the
 * sums are added in another order); it agrees with it within the LM's rounding bounds. */
int liliom_scan_to_map(liliom_ctx* c, const void* feats_body, int n, int stride, double pose7_inout[7],
                       int match_cnt, int max_num_iter, int mode, liliom_iter_stats* stats);

/* Same, on the surf features left on the device by the last liliom_extract_* call:
 * VoxelGrid(leaf_scan) then scan-to-map, no host round trip (both nodes in one process).
 * ds_out (optional, capacity ds_cap) receives surf_last_ds for savePoses (:345-349). */
int liliom_odometry_resident(liliom_ctx* c, double pose7_inout[7], int match_cnt, int max_num_iter, int mode,
                             liliom_iter_stats* stats, void* ds_out, int ds_cap, int* n_ds);

/* The LidarOdometry node's view of the same step: surf_feats = the /surf_features cloud as received
 * (host, point_stride bytes per point, NOT yet down-sampled; L/src/LidarOdometry.cpp:165-169).
 * Runs downSampleCloud(scan) (:319-322) and the scan-to-map solve on the device; ds_out receives
 * surf_last_ds (what savePoses stores, :345-349, and what liliom_map_push_frame later takes). */
int liliom_odometry(liliom_ctx* c, const void* surf_feats, int n, double pose7_inout[7], int match_cnt, int max_num_iter,
                    int mode, liliom_iter_stats* stats, void* ds_out, int ds_cap, int* n_ds);

/* Test hook: one pass of findCorrespondingSurfFeatures at pose7 (no pose update).
 * valid: n bytes; plane: n*4 floats {w*nx,w*ny,w*nz,w*d} (:401-405); nn_idx: n*5 indices into
 * the map in the order returned by liliom_map_download; sqd: n*5. Any output may be NULL. */
int liliom_find_surf_corr(liliom_ctx* c, const void* feats_body, int n, int stride, const double pose7[7],
                          unsigned char* valid, float* plane, int* nn_idx, float* sqd, double out29[29]);

/* ===================== backend kernel reuse (SURVEY §8 a16/a18) ===================== */
/* findCorrespondingCornerFeatures, L/src/BackendFusion.cpp:1531-1599 (variant 0) /
 * R/src/BackendFusion.cpp:1394-1462 (variant 1).  Uses the map installed in `c` as the edge map. */
int liliom_correspond_edge(liliom_ctx* c, const void* feats_body, int n, int stride, const double pose7[7],
                           int variant, unsigned char* valid, float* pa, float* pb);
/* findCorrespondingSurfFeatures of the backend, R/src/BackendFusion.cpp:1464-1520
 * (kd_max_radius, surf_dist_thres, weight gate, score = lidar_const*w). */
int liliom_correspond_surf(liliom_ctx* c, const void* feats_body, int n, int stride, const double pose7[7],
                           double kd_max_radius, double surf_dist_thres, double w_gate, double lidar_const,
                           unsigned char* valid, float* plane, double* score);

/* Horizon backend variant, L/src/BackendFusion.cpp:1601-1681: rows of the plane fit weighted by
 * 1/|reflectivity difference| (the `curvature` channel, L/src/FormatConvert.cpp:21), candidates rejected when the summed
 * difference exceeds reflect_thres (:1628), score = lidar_const*(w + exp(-sum)) (:1676).  The map must have been installed
 * with liliom_map_set_cloud (keeps the reflectivity channel); feats are 48-byte points. */
int liliom_map_set_cloud(liliom_ctx* c, const void* pts, int m, int stride);
int liliom_correspond_surf_refl(liliom_ctx* c, const void* feats48, int n, const double pose7[7], double kd_max_radius,
                                double surf_dist_thres, double w_gate, double lidar_const, double reflect_thres,
                                unsigned char* valid, float* plane, double* score);

/* ---- SURVEY §8 (f1): the LiDAR residual blocks of ONE window keyframe, reduced on the device ----
 * L/src/BackendFusion.cpp:919-979 adds, per keyframe of the sliding window, one LidarEdgeFactor
 * (L/include/factors/LidarKeyframeFactor.h:12-62) per edge correspondence and one LidarPlaneNormFactor (:65-108) per
 * surf correspondence on the parameter blocks (tmpTrans, tmpQuat) under ceres::CauchyLoss(1.0) (:845) and
 * QuaternionParameterization; the same factors are evaluated again for the marginalisation (:1087-1148).
 * These calls evaluate those rows at pose7_body = [qw,qx,qy,qz,tx,ty,tz] of the keyframe on the correspondences the
 * preceding liliom_correspond_edge / liliom_correspond_surf(_refl) call left resident in `c`, and return the keyframe's
 * normal-equation block: out29 = upper triangle of J^T J (21, row-major) | J^T r (6) | cost = 1/2 sum rho | count, with
 * the robustified rows sqrt(rho')[dr/dt, dr/dq * PlusJacobian] — tangent order [t(3), rot(3)] (the parameter-block order).
 * They can be called repeatedly at different poses (LM iterations on frozen correspondences).
 * edge: s_weight = the factor's `s` (pt.intensity = lidar_const, :1581); the extrinsics are not applied (:38).
 * surf: point_w = q * (q_lb^-1 * (p - t_lb)) + t (:87-88), residual score*(n~.point_w + d~). */
int liliom_backend_edge_block(liliom_ctx* c, const double pose7_body[7], double s_weight, double cauchy_b, double out29[29]);
int liliom_backend_surf_block(liliom_ctx* c, const double pose7_body[7], const double q_lb_wxyz[4], const double t_lb[3],
                              double cauchy_b, double out29[29]);

/* ---- SURVEY §8 (f5): the backend's keyframe clouds and local map on the device, a whole window's LiDAR rows per call ----
 * Single-GPU (LILIOM_E_ARG on a sharded context), point_stride bytes per point.  None of these calls touches the odometry map
 * (liliom_map_*, scan-to-map, ICP target); a dedicated backend context is still the recommended set-up (INTEGRATION.md §3). */
typedef struct {
    int    variant;             /* 0 = L/ (Horizon): reflectivity-weighted planes, edge s = (float)lidar_const;
                                   1 = R/ (ROT): dist < 0.1 edge gate (R:1443), 200/N_edge and 1000/N_surf weights (R:843, :861) */
    float  edge_leaf, surf_leaf;            /* /backend_fusion/edge_ds, surf_ds (L:229-230, :339-348, :563-566) */
    double kd_max_radius;                   /* squared-distance gate of the surf search (L:1615, R:1476) */
    double surf_dist_thres;                 /* plane gate (L:1651) */
    double w_gate;                          /* weight gate (L:1665 0.2, R:1504 0.3) */
    double lidar_const;                     /* L:1581 / :1676, R:843 */
    double reflect_thres;                   /* L:1628 (variant 0 only) */
    double cauchy_b;                        /* ceres::CauchyLoss(1.0), L:845 */
    double q_lb[4], t_lb[3];                /* lidar -> body extrinsics of LidarPlaneNormFactor (wxyz, metres) */
} liliom_backend_params;
/* The values of L/config/config_fr_iosb.yaml (variant 0) and R/config/config_fr_iosb.yaml (variant 1). */
void liliom_backend_default_params(liliom_backend_params* p, int variant);

/* Keyframe store: BackendFusion::downSampleCloud, scan half (L:1502-1514) + saveKeyFramesAndFactors' clouds (:1688-1695).
 * VoxelGrid(edge_leaf) / VoxelGrid(surf_leaf) of the received body-frame clouds on the device, appended to a device arena.
 * *kf_id = 0, 1, 2, ... in call order.  Host outputs are optional (NULL: no download; LILIOM_E_CAPACITY when too small).
 * The arena grows geometrically (copying); steady state allocates nothing. */
int liliom_kf_add(liliom_ctx* c, const liliom_backend_params* bp, const void* edge_last, int n_edge, const void* surf_last, int n_surf,
                  int* kf_id, void* edge_ds_out, int edge_cap, int* n_edge_ds, void* surf_ds_out, int surf_cap, int* n_surf_ds);
int liliom_kf_count(const liliom_ctx* c);
int liliom_kf_clear(liliom_ctx* c);      /* drops every keyframe, the local map and the window correspondences */

/* A keyframe store across restarts: the stored clouds of listed keyframes as one checked byte image, and that image appended to
 * any context's store, bit for bit.  Layout (liliom_b200/csrc/kf_image.h), little-endian: a 64-byte header (magic "LILIKF01",
 * version 1, point_stride, k, flags, edge+surf points, full points, table checksum, points checksum), k 16-byte records
 * (n_edge, n_surf, n_full with -1 = no full cloud, a reserved zero), section A (each keyframe's edge then surf points, in table
 * order), section F (the full clouds); size = 64 + 16 k + point_stride * (points).  Only the point layout is recorded: the
 * backend parameters stay per call, the poses stay the caller's.  Importing an image of store C's keyframes L into D gives every
 * call that reads keyframes (bmap_build and the window calls, kf_cloud, loop_align, global_map, every _multi and _batch_multi
 * form with D as a store) on D with the mapped ids the bytes it gives on C with L, and liliom_kf_export(D) gives the image back. */
enum { LILIOM_KF_IMAGE_FULL = 1 };   /* export flag: include the full clouds */
/* The listed keyframes of c's store as one byte image, in list order.  kf_ids == NULL: every keyframe, in id order (k ignored).
 * Repeated ids give repeated keyframes.  Without LILIOM_KF_IMAGE_FULL every record has n_full = -1 and F is empty.
 * image == NULL: *bytes = the image size only.  cap < size: LILIOM_E_CAPACITY, *bytes = the size, nothing written.
 * LILIOM_E_ARG: unknown id, k < 0, unknown flag bits, a sharded context.
 * Writes no state that another call reads: the store, the local map layers, the resident window, the odometry map and a resident
 * scan (liliom_map_update_resident) stay as they were.  One launch gathers and checksums the points on the device. */
int liliom_kf_export(liliom_ctx* c, const int* kf_ids, int k, int flags, void* image, long long cap, long long* bytes);
/* Appends the image's keyframes to c's store: their ids are *first_id .. *first_id + *k - 1, in image order.  All or nothing.
 * A malformed image gives LILIOM_E_ARG with liliom_last_error naming the first failed check (in order: magic and version,
 * point_stride equal to c's, flags, counts, totals, exact length, table checksum, points checksum; the last on the device after
 * the upload), and then liliom_kf_count and every stored byte are unchanged (an arena may have grown).  A sharded context:
 * LILIOM_E_ARG.  Leaves the same state alone as liliom_kf_export. */
int liliom_kf_import(liliom_ctx* c, const void* image, long long bytes, int* first_id, int* k);

/* Backend local map: buildLocalMapWithLandMark (L:1387-1484) + downSampleCloud, map half (:1486-1492).  For each listed keyframe,
 * in list order, its stored clouds transformed by poses7[i] (transformCloud, :730-767; the caller composes q_po*q_bl,
 * q_po*t_bl + t_po as at :1425-1426), edge and surf concatenated separately (:1479-1483), VoxelGrid(edge_leaf) /
 * VoxelGrid(surf_leaf), a cell grid per layer (edge: the 1.0 gate of :1543; surf: kd_max_radius).  Stateless: the reference's
 * deque policy (:1407-1477) stays with the caller, who passes each deque entry's cached pose.  An unknown id: LILIOM_E_ARG,
 * the previous layers stay.  k = 0 builds empty layers. */
int liliom_bmap_build(liliom_ctx* c, const liliom_backend_params* bp, const int* kf_ids, const double* poses7, int k,
                      int* n_edge_map, int* n_surf_map);
/* liliom_bmap_build of B independent sessions in one call.  bps, k, status: B entries; kf_ids, poses7: B per-session pointers;
 * n_edge_map, n_surf_map: B ints each, or NULL.  Session i gets exactly what
 * liliom_bmap_build(ctxs[i], &bps[i], kf_ids[i], poses7[i], k[i], &n_edge_map[i], &n_surf_map[i]) would give it, bit for bit:
 * status, liliom_last_error, both counts, both layers (liliom_bmap_download), both cell grids and the surf layer's reflectivity as
 * every later window search sees them, launches and lib_launches, and everything else on ctxs[i] left alone (the keyframe store,
 * the resident window, the odometry map and a resident scan for liliom_map_update_resident), so that solo and batched calls mix
 * freely.  Horizon (48-byte, variant 0) and ROT (32-byte, variant 1) sessions may be mixed, each with its own list and parameters.
 * Every kernel of the keyframe gather, both layers' VoxelGrid chains (edge, then surf), both layers' box passes and cell grids and
 * the reflectivity runs once for up to 32 sessions on ctxs[0]'s stream (other sessions' streams are joined with events); the
 * library sorts and scans stay per session, in order on the same stream.  The call waits three times for all sessions together
 * (the layers' counts, the cell grids' boxes, the end) where a solo call waits five times when both layers hold points.  A
 * session whose voxel index wraps (wide keys) finishes on its solo path inside the call.
 * A session's own error (every error its solo call returns: an unknown id, the previous layers staying downloadable; k < 0; a
 * NULL list with k > 0; an invalid bp; LILIOM_E_GRID; a non-finite layer point) is its status; the others run.
 * LILIOM_E_ARG for the whole call, nothing changed: B < 1, a NULL array (ctxs, bps, kf_ids, poses7, k, status), a NULL or
 * repeated context, contexts on different devices, a context with a communicator. */
int liliom_bmap_build_batch(liliom_ctx* const* ctxs, int B, const liliom_backend_params* bps, const int* const* kf_ids,
                            const double* const* poses7, const int* k, int* n_edge_map, int* n_surf_map, int* status);
/* liliom_bmap_build_multi of B independent sessions in one call (a fleet tracking in a shared prior map).  stores: B per-session
 * arrays, stores[i][e] the store of session i's entry e (liliom_bmap_build_multi's stores); the other arguments as
 * liliom_bmap_build_batch.  Session i gets exactly what liliom_bmap_build_multi(ctxs[i], &bps[i], stores[i], kf_ids[i], poses7[i],
 * k[i], &n_edge_map[i], &n_surf_map[i]) would give it, bit for bit, with everything liliom_bmap_build_batch promises (status,
 * liliom_last_error, counts, layers, cell grids, reflectivity, launches and lib_launches, everything else on ctxs[i] left alone),
 * so that solo and batched calls mix freely.  Launches and waits as liliom_bmap_build_batch; the gather of every session reads the
 * stores' arenas where they lie.  A session whose voxel index wraps finishes on its solo multi-store path inside the call.
 * Stores: a store may be any backend context on the device: a session's own caller, another session's caller in the same batch, or
 * one store shared by every session.  They are only read.  The streams of every caller and of every distinct store of a running
 * session are joined into ctxs[0]'s stream with events before the first read; the call returns with every read done.  No other
 * host thread may call into a store during the call.
 * A session's own error (every error its solo call returns: a NULL stores[i] or store, a store on another device, of another
 * point_stride or with a communicator, an id unknown to its store, and every liliom_bmap_build_batch session error) is its status;
 * the others run.  LILIOM_E_ARG for the whole call, nothing changed: as liliom_bmap_build_batch, and a NULL stores. */
int liliom_bmap_build_batch_multi(liliom_ctx* const* ctxs, int B, const liliom_backend_params* bps, liliom_ctx* const* const* stores,
                                  const int* const* kf_ids, const double* const* poses7, const int* k, int* n_edge_map, int* n_surf_map,
                                  int* status);
/* edge_local_map_ds (layer 0) / surf_local_map_ds (layer 1) with all fields (published on every run, :1516-1526).
 * out = NULL: *m = size only. */
int liliom_bmap_download(liliom_ctx* c, int layer, void* out, int cap, int* m);

/* optimizeSlidingWindowWithLandMark, LiDAR rows (L:919-979, again at :1087-1148).  The caller passes the lidar poses
 * Q2 = Q * q_lb^-1, T2 = T - Q2 * t_lb (:929-930) and the keyframe ids (the reference's idx-1, :935-936), k <= 16.  Runs the
 * edge search (L:1531-1599 / R:1394-1462) and the surf search (L:1601-1681 / R:1464-1520) of every window keyframe against the
 * two layers (one launch per kind); the correspondences stay on the device.  n_*_corr[i] = found correspondences of keyframe i.
 * The gate of :933 (surf layer > 50 && edge layer > 0) failing: LILIOM_E_FEWMAP, counts 0, nothing resident. */
int liliom_backend_window_correspond(liliom_ctx* c, const liliom_backend_params* bp, const int* kf_ids, const double* poses7_lidar,
                                     int k, int* n_edge_corr, int* n_surf_corr);
/* Every LidarEdgeFactor / LidarPlaneNormFactor row of every window keyframe at its body pose poses7_body[i] under
 * CauchyLoss(cauchy_b), reduced per keyframe and kind as liliom_backend_edge_block / _surf_block do (same partition, same
 * fixed-order sums): out29[i][0] = edge block, out29[i][1] = surf block of keyframe i (k * 2 * 29 doubles).  The variant's weights
 * are applied on the device: variant 1 s = fl(fl(fl(lidar_const)*200)/N_edge) (R:843), score*1000/N_surf in double (R:861);
 * variant 0 s = (double)(float)lidar_const (L:1581).  k must be the k of the resident window; may be called repeatedly. */
int liliom_backend_window_blocks(liliom_ctx* c, const double* poses7_body, int k, double* out29);
/* Test hook: one window keyframe's resident correspondences.  kind 0: valid, a (3 floats), b (3 floats) per edge query;
 * kind 1: valid, plane (4 floats), score (1 double) per surf query.  *n = that keyframe's query count. */
int liliom_backend_window_corr(liliom_ctx* c, int slot, int kind, unsigned char* valid, void* a, void* b, int cap, int* n);

/* Loop-closure clouds from the store, detectLoopClosure (L:2473-2547): per keyframe, edge THEN surf (:2492-2493, :2519-2520)
 * transformed by poses7[i], concatenated, VoxelGrid(leaf), downloaded (out = NULL: *n only).  The result feeds liliom_icp_align
 * (callers that bring their own clouds); liliom_loop_align composes both loop-closure clouds and aligns them on the device. */
int liliom_kf_cloud(liliom_ctx* c, const int* kf_ids, const double* poses7, int k, float leaf, void* out, int cap, int* n);

/* Loop closure from the store in one call, detectLoopClosure's clouds + performLoopClosure's alignment (L:2473-2582):
 * source = liliom_kf_cloud(src_ids, src_poses7, k_src, leaf) (latest_key_frames_ds), target = liliom_kf_cloud(tgt_ids,
 * tgt_poses7, k_tgt, leaf) (his_key_frames_ds), both kept on the device, then liliom_icp_align's ICP on them.  The result is
 * bit-identical to those three calls (the ICP on a second context of the same point layout); *n_src / *n_tgt (optional) = the
 * two cloud sizes.  The target gets a search index of its own: the odometry map, the local map, the resident correspondences
 * (single keyframe and window) and the keyframe store are left as they were.  An empty source or target: LILIOM_OK, identity,
 * *converged = 0, *iters = 0.  LILIOM_E_ARG (nothing changes): an unknown id, leaf <= 0, max_corr_dist <= 0, max_iter < 1, a
 * sharded context. */
int liliom_loop_align(liliom_ctx* c, const int* src_ids, const double* src_poses7, int k_src, const int* tgt_ids,
                      const double* tgt_poses7, int k_tgt, float leaf, double max_corr_dist, int max_iter, double trans_eps,
                      double fit_eps, double T16[16], double* fitness, int* converged, int* iters, int* n_src, int* n_tgt);

/* downSampleCloud, full-cloud half (L:1494-1500, R:1373-1376): attach the keyframe's /full_point_cloud (body frame,
 * point_stride bytes per point) to keyframe kf_id.  variant 0 stores it as received (full_clouds); variant 1 stores
 * VoxelGrid(surf_leaf) of it (full_clouds_ds).  Once per keyframe (a second call: LILIOM_E_ARG, nothing changes).
 * *n_stored (optional) = points stored.  The full clouds have a device arena of their own (geometric growth, copying). */
int liliom_kf_add_full(liliom_ctx* c, const liliom_backend_params* bp, int kf_id, const void* full, int n, int* n_stored);
/* The backend's keyframe from the clouds an extraction left resident on src (BackendFusion's edge_last / surf_last / full_cloud):
 * bit for bit what
 *   liliom_features_download(src, S, .., &ns, E, .., &ne, F, .., &nf);
 *   liliom_kf_add(c, bp, E, ne, S, ns, kf_id, NULL, 0, n_edge_ds, NULL, 0, n_surf_ds);
 *   liliom_kf_add_full(c, bp, *kf_id, F, nf, n_full_stored);
 * does to c: the same id, counts, stored clouds (edge/surf arena and full arena) and state (vg_out rewritten: no scan for
 * liliom_map_update_resident on c).  src is not changed.  src == c is allowed.  All or nothing: on any error nothing is stored and
 * liliom_kf_count(c) is unchanged.  n_edge_ds / n_surf_ds / n_full_stored are optional.
 * Streams: c's work is ordered after src's work so far (an event when their streams differ); the call is synchronous, so src
 * may be reused as soon as it returns.
 * LILIOM_E_ARG, nothing changed: NULL c / bp / src / kf_id, an invalid bp (as liliom_kf_add), no clouds resident on src,
 * different point strides or devices, a communicator on either context. */
int liliom_kf_add_resident(liliom_ctx* c, const liliom_backend_params* bp, liliom_ctx* src,
                           int* kf_id, int* n_edge_ds, int* n_surf_ds, int* n_full_stored);
/* liliom_kf_add_resident of B independent sessions in one call: session i stores into ctxs[i] the clouds left resident on srcs[i].
 * bps: B structs; srcs: B contexts; kf_id, status: B ints; n_edge_ds, n_surf_ds, n_full_stored: B ints each, or NULL.  Session i
 * gets exactly what liliom_kf_add_resident(ctxs[i], &bps[i], srcs[i], &kf_id[i], &n_edge_ds[i], &n_surf_ds[i], &n_full_stored[i])
 * would give it, bit for bit: status, liliom_last_error, id and counts, the stored edge/surf and full clouds and their places in
 * both arenas, launches and lib_launches, and the state left in both contexts (no resident scan for liliom_map_update_resident on
 * ctxs[i]; srcs[i] unchanged), so that solo and batched calls mix freely.  A session with no keyframe this tick is simply left
 * out.  Horizon (48-byte, usually variant 0) and ROT (32-byte, usually variant 1) sessions may be mixed, each with its own
 * parameters.
 * Sources: srcs[i] may be ctxs[i] itself, another session's backend, or the source of several sessions.  The store never writes a
 * source's resident clouds, and every source's sizes are read before any session writes, so the result is that of the solo calls
 * run in any order.
 * Every kernel of the VoxelGrid chains runs once for up to 32 sessions on ctxs[0]'s stream (the edge chains of every session, then
 * the surf chains, then variant 1's full chains); the library sorts and scans stay per session, in order on the same stream, and
 * variant 0's full clouds are device-to-device copies.  The streams of every backend and of every running session's source are
 * joined in before the shared launches with events, and every backend's stream is joined out after them.  The call waits three
 * times for all sessions together (the sizes of the sources whose sizes are only on the device, every cloud's count, the stored
 * clouds) where B solo calls wait four times each (Horizon with variant 0, ROT with variant 1); a batch without device-only sizes
 * waits twice.  A session whose voxel index wraps (wide keys) finishes on its solo path inside the call.  An arena's growth copy
 * is queued on ctxs[0]'s stream and waits once more.  The call is synchronous: a source may be reused as soon as it returns.
 * A session's own error (every error its solo call returns: no clouds resident on the source, an invalid bp, different strides
 * or devices, a source with a communicator, a NULL srcs[i]) is its status, and that session is left unchanged; the others run.
 * LILIOM_E_ARG for the whole call, nothing changed: B < 1, a NULL array (ctxs, bps, srcs, kf_id, status), a NULL or repeated
 * backend context, backend contexts on different devices, a backend context with a communicator. */
int liliom_kf_add_resident_batch(liliom_ctx* const* ctxs, int B, const liliom_backend_params* bps, liliom_ctx* const* srcs,
                                 int* kf_id, int* n_edge_ds, int* n_surf_ds, int* n_full_stored, int* status);

enum { LILIOM_KF_FULL = 0, LILIOM_KF_SURF = 1 };
/* publishCompleteMap (L:2644-2685, R:2409-2447) / the save_pcd map of mapVisualizationThread (L:2703-2718, R:2463-2477).
 * For each listed keyframe, in list order: its stored cloud of `kind`, transformed by pre7 (optional, NULL = skip; the
 * intermediate cloud rounded to fp32 as PCL stores it) and then by poses7[i]; all of them concatenated; VoxelGrid(leaf).
 * The caller selects the keyframes (every mapping_interval-th, the > 10 gate of :2646) and composes the poses
 * (q_po*q_bl, q_po*t_bl + t_po, :2659-2660); stateless, like liliom_bmap_build.  PCL's index overflow: the output is the
 * transformed concatenation itself, as PCL publishes it.  out = NULL: *n only.  Listed points >= 2^31: LILIOM_E_CAPACITY.
 * A listed keyframe without a full cloud (kind FULL) or an unknown id: LILIOM_E_ARG, nothing changes.
 * The filter reads the stored clouds where they lie (no concatenation buffer outside PCL's declined case). */
int liliom_global_map(liliom_ctx* c, int kind, const int* kf_ids, const double* poses7, int k, const double pre7[7],
                      float leaf, void* out, int cap, int* n);

/* ---- the keyframes of several stores (a fleet's sessions, or a restarted session and its previous run's context) ----
 * A store is any backend context (liliom_kf_add*); the calls below read the listed keyframes where they lie in each store's
 * arenas and run everything else on c, into c's buffers, exactly as the single-store call on c: the result is bit for bit that
 * of liliom_global_map / liliom_loop_align on a context D whose store holds the same clouds (e.g. the same kf_add / kf_add_full
 * calls replayed), called with the mapped list; with every entry naming c, that of the single-store call on c.
 * They write what that call writes on c (the keyframe table, VoxelGrid scratch, vg_out: no resident scan for
 * liliom_map_update_resident afterwards; liliom_loop_align_multi also the loop index and source) and never write a store.
 * Each distinct store stream is joined into c's stream with an event before the first read; the call returns with every read
 * done.  No other host thread may call into a store during the call (growing an arena frees the old one).
 * LILIOM_E_ARG, nothing changed: a NULL array or store, a store on another device, of another point_stride or with a
 * communicator, an id unknown to its store, KF_FULL on a keyframe without a full cloud, and whatever the single-store call
 * refuses.  LILIOM_E_CAPACITY, nothing changed: 2^31 listed points or more (per cloud for the loop closure). */
/* publishCompleteMap / save_pcd over keyframes of several stores.  Entry i = keyframe kf_ids[i] of stores[i], placed by
 * poses7[7i..] (after pre7s[7i..] when pre7s is not NULL: each robot's own Tbl).  The result runs on c, into c's buffers. */
int liliom_global_map_multi(liliom_ctx* c, int kind, liliom_ctx* const* stores, const int* kf_ids, const double* poses7, int k,
                            const double* pre7s, float leaf, void* out, int cap, int* n);
/* liliom_loop_align with each cloud's keyframes drawn from any stores; the ICP and its index on c. */
int liliom_loop_align_multi(liliom_ctx* c, liliom_ctx* const* src_stores, const int* src_ids, const double* src_poses7, int k_src,
                            liliom_ctx* const* tgt_stores, const int* tgt_ids, const double* tgt_poses7, int k_tgt, float leaf,
                            double max_corr_dist, int max_iter, double trans_eps, double fit_eps,
                            double T16[16], double* fitness, int* converged, int* iters, int* n_src, int* n_tgt);
/* liliom_bmap_build over keyframes of several stores: entry i = keyframe kf_ids[i] of stores[i], placed by poses7[7i..].  The
 * result is bit for bit liliom_bmap_build on a context D whose store holds the same clouds, called with the mapped list: status,
 * both counts, both layers (liliom_bmap_download), both cell grids and the Horizon layer's reflectivity as every later
 * liliom_backend_window_correspond / _blocks on c sees them; with every entry naming c, liliom_bmap_build on c.  A store may be any
 * backend context on c's device: c itself, another session's, or a prior run's store that several sessions share (a fleet tracking
 * in a prior map).  The stores are only read; each distinct store stream is joined into c's stream with an event before the first
 * read, and the call returns with every read done.  No other host thread may call into a store during the call.
 * LILIOM_E_ARG, nothing changed (the previous layers stay downloadable): a NULL array or store (k > 0), a store on another device,
 * of another point_stride or with a communicator, an id unknown to its store, and whatever liliom_bmap_build refuses. */
int liliom_bmap_build_multi(liliom_ctx* c, const liliom_backend_params* bp, liliom_ctx* const* stores, const int* kf_ids,
                            const double* poses7, int k, int* n_edge_map, int* n_surf_map);

/* ---- SURVEY §8 (f3): wire format on the sensor side — FormatConvert's livoxLidarHandler on the device ----
 * L/src/FormatConvert.cpp:11-24: livox_ros_driver::CustomPoint {uint32 offset_time; float x,y,z; uint8 reflectivity,
 * tag, line} -> pcl::PointXYZINormal with intensity = line + 0.1*float(offset_time/(float)time_end) (:19-20),
 * curvature = 0.1*reflectivity (:21), time_end = points.back().offset_time (:13).
 * stride = 20 (the C++ message struct in memory) or 19 (serialised wire bytes).
 * liliom_convert_livox leaves the converted sweep resident (as liliom_upload_scan does) and optionally downloads it;
 * liliom_extract_horizon_livox = convert + liliom_extract_horizon without the 48-byte host cloud in between
 * (H2D traffic 19-20 B/point instead of 48). */
int liliom_convert_livox(liliom_ctx* c, const void* custom_pts, int n, int stride, liliom_pt48* out, int cap);
int liliom_extract_horizon_livox(liliom_ctx* c, const void* custom_pts, int n, int stride, const double q_imu_wxyz[4],
                                 liliom_pt48* surf_out, int surf_cap, int* n_surf,
                                 liliom_pt48* edge_out, int edge_cap, int* n_edge,
                                 liliom_pt48* cutted_out, int cut_cap, int* n_cut);

/* ---- SURVEY §8 (f4): the loop-closure alignment, BackendFusion::performLoopClosure (L/src/BackendFusion.cpp:2552-2582) ----
 * pcl::IterativeClosestPoint with the reference's settings (:2566-2570: max correspondence distance 30, 100 iterations,
 * transformation epsilon 1e-6, euclidean fitness epsilon 1e-6) on src = latest_key_frames_ds against tgt = his_key_frames_ds
 * (host clouds, stride 48|32|16): per iteration the nearest target point of every transformed source point (kept within
 * max_corr_dist), the rigid transform by the SVD closed form, PCL's default convergence criteria.  T16 = getFinalTransformation()
 * (row-major 4x4, target <- source), *fitness = getFitnessScore(), *converged = hasConverged(), *iters = iterations run.
 * The target is installed as the context's map (the backend aligns its own keyframes with liliom_loop_align instead, which
 * leaves the map alone).  The whole loop, the fitness pass included, is one cooperative launch with one stream synchronise.
 * fp64 where PCL is fp32; PCL's setRANSACIterations is a no-op for this class (no rejector installed), so the alignment is
 * deterministic. */
int liliom_icp_align(liliom_ctx* c, const void* src, int n_src, const void* tgt, int n_tgt, int stride, double max_corr_dist,
                     int max_iter, double trans_eps, double fit_eps, double T16[16], double* fitness, int* converged, int* iters);

/* ---- SURVEY §8 (f3): LidarOdometry::undistortion on the device (L/src/LidarOdometry.cpp:178-199) ----
 * Moves every point of a keyframe cloud (point_stride bytes per point, in place) to the end of the sweep:
 * p' = slerp(I, quat; ratio) * p + ratio * trans, ratio = min(frac(intensity) / 0.1, 1).  publishCloudLast (:624-632) calls it
 * on the three keyframe clouds with quat = identity and trans = the relative translation of the scan. */
int liliom_undistort(liliom_ctx* c, void* pts_inout, int n, const double trans[3], const double quat_wxyz[4]);
/* publishCloudLast's undistortion (L/src/LidarOdometry.cpp:178-199, :624-632) on the three clouds the last extraction on c left
 * resident (surf, edge, cut / laserCloud), in place, in one launch, with no host traffic.  Afterwards liliom_features_download(c)
 * returns, bit for bit, what liliom_undistort(c, cloud, n, trans, quat) returns on each cloud it returned before the call (the
 * payload publishCloudLast publishes).  Counts, the odometry's down-sampled scan (liliom_map_update_resident), the queries, the map
 * and everything else on c are left alone.  Calling it twice de-skews twice, as calling undistortion twice does.
 * LILIOM_E_ARG, nothing changed: no clouds resident (as liliom_features_download), NULL trans / quat. */
int liliom_undistort_resident(liliom_ctx* c, const double trans[3], const double quat_wxyz[4]);
/* liliom_undistort_resident of B independent sessions in one call.  trans: 3*B doubles, quat_wxyz: 4*B doubles, status: B ints.
 * Session i gets exactly what liliom_undistort_resident(ctxs[i], trans + 3*i, quat_wxyz + 4*i) would give it, bit for bit: status,
 * liliom_last_error, the de-skewed clouds (liliom_features_download), launches, and everything else on ctxs[i] left alone, so that
 * solo and batched calls mix freely.  A session without a keyframe this tick is simply left out of ctxs.  Horizon (48-byte) and
 * ROT (32-byte) sessions may be mixed, each with its own motion.
 * The three clouds of up to 32 sessions share one k_undistort_batch launch on ctxs[0]'s stream (other sessions' streams are
 * joined with events), each cloud with its solo launch's blocks; a resident Horizon extraction's sizes are read on the device; a
 * session whose clouds have no points takes part in no launch, as in its solo call.  The call waits once for all sessions.
 * A session's own error (LILIOM_E_ARG: no clouds resident) is its status; the others run.
 * LILIOM_E_ARG for the whole call, nothing changed: B < 1, a NULL array (ctxs, trans, quat_wxyz, status), a NULL or repeated
 * context, contexts on different devices, a context with a communicator. */
int liliom_undistort_resident_batch(liliom_ctx* const* ctxs, int B, const double* trans, const double* quat_wxyz, int* status);

/* ---- SURVEY §8 (f3), publishing side: the PointCloud2 layout pcl::toROSMsg gives these clouds ----
 * L/src/Preprocessing.cpp:385-401, L/src/LidarOdometry.cpp:634-649: pcl::toROSMsg copies the point array verbatim into
 * sensor_msgs::PointCloud2::data (point_step = sizeof(PointT), is_dense as in the cloud, height 1) and lists the fields
 * PCL registers for the point type.  The buffers this library returns ARE that payload: a node can pass msg.data.data()
 * (resized to n * point_step) as the output pointer and fill the header from this table — no intermediate PCL cloud.
 * datatype follows sensor_msgs::PointField (7 = FLOAT32).  Returns the number of fields (8 for stride 48, 4 for 32),
 * or LILIOM_E_ARG / LILIOM_E_CAPACITY. */
typedef struct { char name[16]; unsigned int offset; unsigned char datatype; unsigned int count; } liliom_pc2_field;
int liliom_pc2_layout(int point_stride, liliom_pc2_field* fields, int cap, int* point_step);

/* ---- SURVEY §8 (f3), sensor side of the ROT package: the driver's sensor_msgs::PointCloud2 as received ----
 * R/src/Preprocessing.cpp:248-281 receives the spinning LiDAR's PointCloud2 (Velodyne, Ouster, ...) and runs
 * pcl::fromROSMsg(msg, pcl::PointXYZI) (:277) before removeNaNFromPointCloud / removeClosedPointCloud (:280-281).  These calls
 * take the message's fields and payload as they are: only height * row_step bytes cross PCIe (22 B per point for a packed
 * Velodyne XYZIRT layout instead of 32), and the decode runs on the device.
 * Decode (pcl::fromROSMsg): each of x, y, z, intensity is read from the FIRST message field with that name, datatype FLOAT32 (7)
 * and count 1 or 0 (a FLOAT64 "x" before a FLOAT32 "x" is skipped); a field without such a match keeps PCL's default value 0;
 * w = 1 and the padding floats are 0.  Point (r, c) is read at r * row_step + c * point_step (organised clouds, padded rows):
 * n = width * height points in row-major order, read byte by byte (any point_step and offset alignment).
 * The decoded sweep then goes through liliom_extract_rot unchanged.  is_dense is not an input: non-finite x/y/z are always
 * dropped, as liliom_extract_rot does.  (PCL's removeNaNFromPointCloud skips that check for is_dense = true; a driver that sets
 * is_dense and still emits NaN leaves the reference undefined — its start / end azimuth at :285-288 can become NaN.)
 * LILIOM_E_ARG, nothing changed: a null msg, a null data with a non-empty payload, null fields with n_fields > 0, n_fields < 0,
 * point_step 0, row_step < width * point_step, width * height > INT_MAX, a mapped field with offset + 4 > point_step,
 * is_bigendian != 0, or a context that is not 32-byte (ROT). */
typedef struct {
    const void* data;                          /* msg.data.data(): height * row_step bytes, little-endian */
    unsigned int height, width, point_step, row_step;
    const liliom_pc2_field* fields; int n_fields;   /* msg.fields; names NUL-terminated (longer names truncated to 15 chars) */
    int is_bigendian;                          /* msg.is_bigendian; nonzero is rejected */
} liliom_pc2_msg;

/* pcl::fromROSMsg(msg, pcl::PointXYZI) on the device (R/src/Preprocessing.cpp:277).  The decoded sweep stays resident like
 * liliom_upload_scan's (liliom_extract_resident can run on it).  *n = width * height; out = NULL: no download; out with
 * cap < *n: LILIOM_E_CAPACITY (*n reported, nothing converted). */
int liliom_convert_pc2(liliom_ctx* c, const liliom_pc2_msg* msg, liliom_pt32* out, int cap, int* n);
/* = liliom_convert_pc2 + liliom_extract_rot without the 32-byte host cloud in between (R/src/Preprocessing.cpp:277-509). */
int liliom_extract_rot_pc2(liliom_ctx* c, const liliom_pc2_msg* msg, const double q_imu_wxyz[4], const double q_lb_wxyz[4],
                           liliom_pt32* surf_out, int surf_cap, int* n_surf, liliom_pt32* edge_out, int edge_cap, int* n_edge,
                           liliom_pt32* cutted_out, int cut_cap, int* n_cut);

/* Where the ROT extractor takes each return's ring (scanID) from; a setting of the context, like liliom_set_stream.
 * LILIOM_RING_ELEVATION (the default): from the point's elevation through the reference's three tables
 *   (R/src/Preprocessing.cpp:315-347: line_num 16 = VLP-16, 32 = HDL-32E, 64 = HDL-64E, which keeps -24.33..+2 deg only).
 * LILIOM_RING_FIELD: from the driver's per-point `ring` field of the PointCloud2, for sensors of any beam layout (Ouster
 *   OS-0/1/2, VLS-128, Pandar, RS-Ruby, ...).  The extraction is the reference's with exactly one substitution: scanID = ring.
 *   A point is kept iff 0 <= ring < line_num; a point outside that range is dropped like a table miss.  Everything else (NaN /
 *   3 m removal, start / end azimuth from the first / last surviving point, the halfPassed latch, relTime, intensity =
 *   ring + 0.1 * relTime, de-skew, ring concatenation, curvature, picks, VoxelGrid 0.6) is unchanged.
 *   - the ring field: the FIRST field named "ring" with datatype UINT8 (2) or UINT16 (4) and count 1 or 0, read byte by byte;
 *     a message without one, or with one that does not fit in point_step, is refused with LILIOM_E_ARG and changes nothing;
 *   - line_num may be 1..128 (one CTA per ring: 128 rings are one wave on a 132-SM H100); outside: LILIOM_E_LINES;
 *   - liliom_convert_pc2 and liliom_extract_rot_pc2 decode the ring with the sweep; liliom_extract_resident uses the rings
 *     decoded with the resident sweep.  After liliom_upload_scan, liliom_convert_livox or a change of the ring source no ring
 *     ids are resident and liliom_extract_resident returns LILIOM_E_ARG;
 *   - liliom_extract_rot (host 32-byte points carry no ring) returns LILIOM_E_ARG.
 * Returns LILIOM_E_ARG for another source, or LILIOM_RING_FIELD on a context that is not 32-byte (ROT). */
enum { LILIOM_RING_ELEVATION = 0, LILIOM_RING_FIELD = 1 };
int liliom_set_ring_source(liliom_ctx* c, int source);

/* Where the ROT extractor takes each return's relTime from; a second setting of the context beside the ring source (the two
 * are independent: all four combinations are valid).
 * LILIOM_TIME_AZIMUTH (the default): the reference's azimuth rule (R/src/Preprocessing.cpp:285-294, 349-367): start / end
 *   azimuth from the first / last surviving point and the halfPassed latch, which assume the points arrive in firing order.
 *   On ring-major organised clouds (Ouster, organised Velodyne) the latch fires inside the first ring and relTime is wrong.
 * LILIOM_TIME_FIELD: from the driver's per-point time field of the PointCloud2, named by field_name (Velodyne "time",
 *   Ouster "t", Hesai / Robosense "timestamp").  The extraction is the reference's with exactly one substitution:
 *     relTime = (float)((t_i - t_min) / (t_max - t_min))   (in double; 0 for every point when t_max == t_min)
 *   where t_min / t_max are the smallest / largest time over the points that survive the NaN / 3 m removal (the set the
 *   reference takes startOri / endOri from, before the ring filter): the reference's own normalisation, first return 0 and
 *   last 1, with the time in place of the azimuth, so any unit and any origin work (seconds, nanoseconds, absolute stamps).
 *   A point whose FLOAT32 / FLOAT64 time is not finite is dropped with the NaN points and does not enter t_min / t_max.
 *   Everything else (the NaN / 3 m removal, the ring source, intensity = ring + 0.1 * relTime, the de-skew
 *   q_lb * slerp(I, qIMU, ratio) * q_lb^-1, ring concatenation, curvature, picks, VoxelGrid 0.6) is unchanged.
 *   - the time field: the FIRST field named field_name (at most 15 characters, matched like the other names) with datatype
 *     FLOAT32 (7), FLOAT64 (8) or UINT32 (6) and count 1 or 0, read byte by byte and converted exactly to double; a message
 *     without one, or with one that does not fit in point_step, is refused with LILIOM_E_ARG and changes nothing;
 *   - liliom_convert_pc2 and liliom_extract_rot_pc2 decode the time with the sweep; liliom_extract_resident uses the times
 *     decoded with the resident sweep.  After liliom_upload_scan, liliom_convert_livox or any liliom_set_time_source call no
 *     times are resident and liliom_extract_resident returns LILIOM_E_ARG;
 *   - liliom_extract_rot (host 32-byte points carry no time) returns LILIOM_E_ARG.
 * field_name is ignored for LILIOM_TIME_AZIMUTH.  Returns LILIOM_E_ARG for another source, for LILIOM_TIME_FIELD with a NULL
 * or longer name, or for LILIOM_TIME_FIELD on a context that is not 32-byte (ROT). */
enum { LILIOM_TIME_AZIMUTH = 0, LILIOM_TIME_FIELD = 1 };
int liliom_set_time_source(liliom_ctx* c, int source, const char* field_name);

/* ===================== multi-GPU (one context per rank) ===================== */
/* 128-byte NCCL unique id: rank 0 calls get, the launcher broadcasts it, every rank calls init.
 * After init, liliom_map_set_points shards the map by 16 m block hash (+halo) and every
 * liliom_scan_to_map / liliom_odometry_resident is COLLECTIVE: per iteration one all-reduce of
 * the 27 J^T J|J^T r scalars (+cost,count) then an identical 6x6 solve on every rank.
 * In mode CERES (after liliom_comm_set_ceres(c, 1)) each outer iteration all-reduces the linearisation sums once and then
 * runs the LM in exactly 1 + max(0, max_num_iter) rounds of [the 29 sums over this rank's correspondences, their all-reduce,
 * the same trust-region step on every rank]; rounds after the LM stopped still all-reduce (zeros), so every rank issues the
 * same collectives.  Its pose bits depend on nranks and the shard block.  An all-reduce failure returns LILIOM_E_NCCL with
 * the pose untouched.  The batch calls (liliom_*_batch*) still refuse communicator contexts. */
int liliom_comm_get_unique_id(void* id128);
int liliom_comm_init(liliom_ctx* c, const void* id128, int nranks, int rank);
/* Edge of the cubes the map is sharded by (metres, a power of two in [8, 256]; default 16).  Larger cubes replicate less
 * halo (a 64 m cube with its 1 m + voxel-diagonal rim holds ~1.1x its own points, a 16 m cube ~1.45x) at a coarser load
 * balance.  Must be the same on every rank and set before the map is installed / the first frame is pushed. */
int liliom_comm_set_shard_block(liliom_ctx* c, int metres);
/* Ceres mode on a context with a communicator.  0 (the default): LILIOM_E_ARG, as without this call.  1: the collective LM
 * above.  Any other value: LILIOM_E_ARG.  Accepted on any context, at any time (before or after liliom_comm_init); only calls
 * on a context with a communicator read it.  Must be the same on every rank, like liliom_comm_set_shard_block. */
int liliom_comm_set_ceres(liliom_ctx* c, int on);

/* Fused exchange over peer memory (single node, NVLink / NVSwitch; optional, after liliom_comm_init): every rank exports the
 * 64-byte cudaIpcMemHandle of its exchange buffer, the launcher all-gathers them, every rank attaches all of them in rank
 * order.  From then on a GN-mode scan-to-map runs all its iterations in ONE cooperative launch per rank: after the local
 * reduction each rank stores its 29 sums directly into every peer's buffer (flag-in-data words) and reads the others' from
 * its own — no ncclAllReduce, no per-iteration launches.  Sums are added in rank order on every rank: identical poses.
 * nranks == 1 is accepted (self-exchange; exercises the protocol on one GPU). */
int liliom_comm_peer_export(liliom_ctx* c, void* handle64);
int liliom_comm_peer_attach(liliom_ctx* c, const void* handles /* nranks * 64 bytes, rank order */, int nranks, int rank);
/* Recovery after a LILIOM_E_NCCL from the fused exchange (a rank did not publish within the wait bound): the ranks that ran
 * the scan advanced their exchange epoch, a rank that never entered it did not, and every later scan would time out as well.
 * Every rank reads its epoch, the application agrees on the maximum over the ranks (its own all-reduce — the ranks must meet
 * anyway before they continue), and every rank sets maximum + 2: words left in the exchange buffers carry smaller epochs and
 * never match a later one.  Host-side bookkeeping only; nothing is launched. */
int liliom_comm_peer_epoch(liliom_ctx* c, unsigned int* epoch);
int liliom_comm_peer_set_epoch(liliom_ctx* c, unsigned int epoch);

/* ===================== instrumentation ===================== */
typedef struct {
    unsigned long long launches;      /* kernels of this library launched since create/reset */
    unsigned long long lib_launches;  /* CUB sort/scan calls issued (library plumbing) */
    double knn_ms;                    /* sum of CUDA-event durations of the kNN+Jacobian kernel */
    unsigned long long knn_launches;  /* number of timed launches in knn_ms */
    unsigned long long knn_queries;   /* queries searched by those launches, summed over passes (counted on the device) */
    unsigned long long knn_candidates;/* map points examined by those launches after pruning (counted on the device) */
} liliom_counters;
int liliom_get_counters(liliom_ctx* c, liliom_counters* out, int reset);
/* The C-bar of the algorithmic-bytes figure (SURVEY.md §8 d: B_q = 16 + 27*8 + 16*C-bar per query and pass): for the
 * queries resident after the last scan-to-map / odometry call, transformed by pose7, out2[0] = queries (owned by this
 * rank when the map is sharded), out2[1] = map points in their full 3x3x3 cell blocks.  The search itself examines fewer
 * (pruning; knn_candidates above counts those).  Not on the hot path. */
int liliom_knn_block_stats(liliom_ctx* c, const double pose7[7], unsigned long long out2[2]);
/* on = 1: bracket every kNN+Jacobian launch with a CUDA-event pair on the context stream and count its queries /
 * candidates on the device; on = N > 1: do so on every N-th scan-to-map call only (each event of the pair adds dependent
 * stream latency to the step); 0 (default): off. */
int liliom_set_kernel_timing(liliom_ctx* c, int on);
/* Run all library work on a caller-owned CUDA stream (cudaStream_t passed as void*; NULL restores the
 * context's own stream).  Calls stay synchronous; this only lets the caller bracket them with events. */
int liliom_set_stream(liliom_ctx* c, void* cuda_stream);
/* Device-resident benchmark hooks.  upload_scan: copy a raw sweep (point_stride bytes per point) into
 * HBM; extract_resident: run the extractor of the context's variant on it without downloading the
 * clouds (q_lb ignored for the Horizon variant); the surf features stay resident for
 * liliom_odometry_resident(). */
int liliom_upload_scan(liliom_ctx* c, const void* pts, int n);
int liliom_extract_resident(liliom_ctx* c, const double q_imu_wxyz[4], const double q_lb_wxyz[4],
                            int* n_surf, int* n_edge, int* n_cut);
/* The three clouds the last extraction on this context left resident (liliom_extract_*, liliom_extract_resident or
 * liliom_extract_resident_batch), as liliom_extract_horizon / liliom_extract_rot would have returned them: surf, edge and
 * cutted (ROT: laserCloud), point_stride bytes per point.  The counts are always written; any cloud pointer may be NULL (count
 * only).  A cloud larger than its capacity: LILIOM_E_CAPACITY, nothing written.  Nothing resident (no extraction yet, the last
 * one failed, or liliom_odometry replaced the surf features): LILIOM_E_ARG. */
int liliom_features_download(liliom_ctx* c, void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap, int* n_edge,
                             void* cut, int cut_cap, int* n_cut);
/* keep `n` feature points resident (feats stride 16/32/48) */
int liliom_upload_feats(liliom_ctx* c, const void* feats_body, int n, int stride);
/* run scan-to-map on the resident features; pose in/out on host but no other traffic */
int liliom_scan_to_map_resident(liliom_ctx* c, double pose7_inout[7], int match_cnt, int max_num_iter, int mode,
                                liliom_iter_stats* stats);

/* ===================== several sessions in one call ===================== */
/* One GN-mode scan-to-map step of B independent sessions (contexts) in as few launches as fit on the device.
 * Session i gets exactly what liliom_scan_to_map_resident(ctxs[i], poses7 + 7*i, match_cnt, 0, LILIOM_MODE_GN,
 * stats ? stats + i*match_cnt : NULL) would give it, bit for bit, including the state it leaves in ctxs[i].
 * status[i] = that call's return value; a session with LILIOM_E_NOMAP / LILIOM_E_FEWMAP keeps its pose, the others run.
 * Sessions whose solo call runs all iterations in one cooperative launch share cooperative launches (each with its own grid
 * barrier, so no session waits for another); the others take their solo path inside the same call.
 * LILIOM_E_ARG for the whole call, nothing changed: B < 1, a NULL array (ctxs, poses7_inout, status), match_cnt < 0, a NULL
 * or repeated context, contexts on different devices, a context with a communicator (liliom_comm_init; sharded or fused).
 * Streams: the shared launches run on ctxs[0]'s stream; every other session's stream (liliom_set_stream) is ordered before
 * and after them with events, and the call is synchronous like every other call.
 * Counters: launches advances on every session that took part in a launch; knn_queries / knn_candidates are counted per
 * session on the device; the event timing of the shared launches (knn_ms, knn_launches) goes to ctxs[0] only. */
int liliom_scan_to_map_resident_batch(liliom_ctx* const* ctxs, int B, double* poses7_inout, int match_cnt,
                                      liliom_iter_stats* stats, int* status);
/* Same, with the semantics of liliom_odometry_resident per session: VoxelGrid(leaf_scan) of the surf features that the
 * session's last liliom_extract_* / liliom_extract_resident left resident, then the step.  ds_out[i] / ds_cap[i] / n_ds[i]
 * are optional per session (NULL arrays or NULL entries: no download). */
int liliom_odometry_resident_batch(liliom_ctx* const* ctxs, int B, double* poses7_inout, int match_cnt,
                                   liliom_iter_stats* stats, void* const* ds_out, const int* ds_cap, int* n_ds, int* status);
/* The batched step in either mode, with per-session counts.  Session i gets exactly what
 * liliom_scan_to_map_resident(ctxs[i], poses7 + 7*i, match_cnt[i], max_num_iter[i], mode, stats ? stats[i] : NULL) would give
 * it, bit for bit: pose, status, every liliom_iter_stats entry (lm_iters included), the device-side counts, launches and the
 * state left in ctxs[i].  match_cnt: B entries >= 0 (0: the session runs no scan-to-map kernel, as its solo call).
 * max_num_iter: B entries, passed on as the solo call takes them; may be NULL in LILIOM_MODE_GN, where it is ignored.
 * stats: NULL, or B pointers, each NULL (no stats for that session) or match_cnt[i] records.
 * LILIOM_MODE_CERES: per outer iteration, the sessions still iterating share one per-pass search launch per lane count
 * (k_knn_plane_batch, up to 32 sessions each), then one LM launch with one 512-thread block per session (k_lm_solve_batch),
 * so B LM solves run side by side on B SMs.  LILIOM_MODE_GN: as liliom_scan_to_map_resident_batch, sessions of equal
 * match_cnt share cooperative launches.
 * LILIOM_E_ARG for the whole call, nothing changed: every refusal of liliom_scan_to_map_resident_batch, a NULL match_cnt, a
 * negative match_cnt[i], a mode other than LILIOM_MODE_CERES / LILIOM_MODE_GN, LILIOM_MODE_CERES with a NULL max_num_iter.
 * Per-session errors, streams and counters as liliom_scan_to_map_resident_batch.  liliom_scan_to_map_resident_batch is
 * this call with match_cnt[i] = match_cnt, LILIOM_MODE_GN and stats[i] = stats + i*match_cnt. */
int liliom_scan_to_map_resident_batch_ex(liliom_ctx* const* ctxs, int B, double* poses7_inout, const int* match_cnt,
                                         const int* max_num_iter, int mode, liliom_iter_stats* const* stats, int* status);
/* Same, with the semantics of liliom_odometry_resident per session (as liliom_odometry_resident_batch).  A session whose
 * VoxelGrid speculation misses is redone by its own solo path, in `mode` with its own max_num_iter[i]. */
int liliom_odometry_resident_batch_ex(liliom_ctx* const* ctxs, int B, double* poses7_inout, const int* match_cnt,
                                      const int* max_num_iter, int mode, liliom_iter_stats* const* stats, void* const* ds_out,
                                      const int* ds_cap, int* n_ds, int* status);
/* One driver message of a session of liliom_convert_batch: kind LILIOM_WIRE_LIVOX with liliom_convert_livox's custom_pts, n
 * and stride (19 or 20), or LILIOM_WIRE_PC2 with liliom_convert_pc2's msg.  The fields of the other kind are not read. */
enum { LILIOM_WIRE_LIVOX = 0, LILIOM_WIRE_PC2 = 1 };
typedef struct {
    int kind;
    const void* custom_pts; int n; int stride;
    const liliom_pc2_msg* pc2;
} liliom_wire_msg;
/* liliom_convert_livox / liliom_convert_pc2 of B independent sessions in one call: the fleet's front door, in front of
 * liliom_extract_resident_batch.  msgs: B messages; out, cap: NULL, or B entries (a NULL out[i]: no download for session i);
 * n, status: B ints.  Session i gets exactly what its solo call would give it, bit for bit:
 *   LIVOX: liliom_convert_livox(ctxs[i], m.custom_pts, m.n, m.stride, out ? out[i] : NULL, cap ? cap[i] : 0), and n[i] = m.n
 *          on success;
 *   PC2:   liliom_convert_pc2(ctxs[i], m.pc2, out ? out[i] : NULL, cap ? cap[i] : 0, &n[i]).
 * That covers the status, n[i] (written where the solo call writes it), the downloaded bytes, the resident sweep and its ring /
 * time side channels (decoded under the session's own liliom_set_ring_source / liliom_set_time_source), liliom_last_error and
 * the launch counters, so a later liliom_extract_resident or liliom_extract_resident_batch behaves as after the solo call.
 * A session's own refusal is its status and leaves that session unchanged; the others run.  The refusals are those of the solo
 * call (a bad stride, a NULL payload, a malformed PointCloud2, a missing ring or time field under the field sources,
 * LILIOM_E_CAPACITY), and LILIOM_E_ARG for a kind that does not fit the context: LIVOX on a 32-byte context, PC2 on a 48-byte
 * one, or an unknown kind.  Horizon (48-byte) and ROT (32-byte) sessions may be mixed.
 * Each accepted session's payload is copied into its own staging buffer, the copies queued back to back on ctxs[0]'s stream;
 * then one decode launch per kind for up to 32 sessions (each session's points start on a block boundary), the downloads and
 * one stream synchronise for the whole call, where B solo calls wait B times.  Sessions with 0 points take part in no launch.
 * The library does not pin the payloads: page-locked payloads are copied by asynchronous DMA, pageable ones as the solo call
 * copies them.  Other sessions' streams are joined to ctxs[0]'s with events.
 * LILIOM_E_ARG for the whole call, nothing changed: B < 1, a NULL array (ctxs, msgs, n, status), a NULL or repeated context,
 * contexts on different devices, a context with a communicator.
 * For a single session the solo call is faster (no event joins, no session table). */
int liliom_convert_batch(liliom_ctx* const* ctxs, int B, const liliom_wire_msg* msgs, void* const* out, const int* cap, int* n,
                         int* status);
/* liliom_extract_resident of B independent sessions in one call.  q_imu: 4*B doubles; q_lb: 4*B doubles or NULL (identity,
 * as the solo call's NULL).  n_surf / n_edge / n_cut / status: B ints each.  Horizon (48-byte) and ROT (32-byte) contexts
 * may be mixed.  Session i gets exactly what liliom_extract_resident(ctxs[i], q_imu + 4*i, q_lb ? q_lb + 4*i : NULL, ...)
 * would give it, bit for bit: status and counts (-1 for Horizon sessions, whose counts stay on the device), the resident
 * clouds, the labels and curvatures of liliom_extract_rot_labels, and the state left in ctxs[i].  Each session reads its
 * own ring / time sources and side channels.  A session's own error (LILIOM_E_LINES, LILIOM_E_ARG for a missing side
 * channel or ds_rate < 1, LILIOM_E_CAPACITY for a ring above 16384 or a segment above 4096 points) is its status; the
 * others run.
 * ROT sessions run every stage of the chain in shared launches of up to 32 sessions on ctxs[0]'s stream (the rings: one block
 * per ring of every session); the library sorts and scans stay per session, in order on the same stream.  Horizon sessions whose solo call
 * is one cooperative launch share cooperative launches (83 blocks and one barrier word per session, as many sessions per
 * launch as are co-resident) on ctxs[0]'s stream; the others (LILIOM_HZ_CHAIN, empty sweeps) take their solo path.  Other
 * sessions' streams are joined to ctxs[0]'s with events.  The call is synchronous, with one stream synchronise for all
 * sessions (the solo ROT call has one per call).
 * LILIOM_E_ARG for the whole call, nothing changed: B < 1, a NULL array (ctxs, q_imu, n_surf, n_edge, n_cut, status), a NULL
 * or repeated context, contexts on different devices, a context with a communicator.
 * Counters: every session's launches and lib_launches advance as in its solo call.  For a single session the solo call is
 * faster (no event joins). */
int liliom_extract_resident_batch(liliom_ctx* const* ctxs, int B, const double* q_imu, const double* q_lb,
                                  int* n_surf, int* n_edge, int* n_cut, int* status);
/* liliom_map_update_resident of B independent sessions in one call.  poses7: 7*B doubles.  n_map: B ints (may be NULL).
 * status: B ints.  Session i gets exactly what liliom_map_update_resident(ctxs[i], poses7 + 7*i, &n_map[i]) would give it,
 * bit for bit: status, count, FIFO, filtered cloud (liliom_map_download_cloud), search index (liliom_map_download and every
 * later scan-to-map), incremental entry array, and launch counters.  A session that needs no update this step is simply left
 * out of ctxs.  Horizon (48-byte) and ROT (32-byte) contexts may be mixed.
 * Every kernel of the steady-state update runs once for up to 32 sessions, on ctxs[0]'s stream (other sessions' streams are
 * joined with events), and the call waits four times for all sessions together (the new frames' boxes, their key flags, the
 * voxel counts, the cell grids' escape flags) where B solo calls wait five times each.  It returns, like the solo call,
 * with every session's map complete (one more wait when a session re-built its cell grid or left the steady-state path).  The library sorts and scans stay per
 * session, in order on the same stream.  Sessions off the steady-state path finish on their solo path inside the call: a
 * first update or one after liliom_map_push_frame / liliom_map_clear, voxel keys that do not fit 21 bits, max_map_frames
 * above 64, a cell grid whose box a centroid left.
 * A session's own error (LILIOM_E_ARG: no scan resident; LILIOM_E_GRID: a map extent over 2^29 cells; a CUDA error) is its
 * status; the others run.
 * LILIOM_E_ARG for the whole call, nothing changed: B < 1, a NULL array (ctxs, poses7, status), a NULL or repeated context,
 * contexts on different devices, a context with a communicator.
 * For a single session the solo call is faster (no event joins). */
int liliom_map_update_batch(liliom_ctx* const* ctxs, int B, const double* poses7, int* n_map, int* status);
/* liliom_backend_window_correspond of B independent sessions in one call.  bps: B structs.  kf_ids, poses7_lidar, n_edge_corr,
 * n_surf_corr: B per-session pointers; k, status: B ints.  Session i gets exactly what
 * liliom_backend_window_correspond(ctxs[i], &bps[i], kf_ids[i], poses7_lidar[i], k[i], n_edge_corr[i], n_surf_corr[i]) would give
 * it, bit for bit: status, counts (zeroed up to an unknown id, as the solo call writes them), liliom_last_error, launches, and the
 * window left resident in ctxs[i], so that solo and batched window calls mix freely (liliom_backend_window_blocks,
 * liliom_backend_window_corr, liliom_backend_window_blocks_batch).  A session that has no new keyframe is simply left out of ctxs.
 * Horizon (48-byte, variant 0) and ROT (32-byte, variant 1) sessions may be mixed, with their own k (1..16) and parameters.
 * A session's own error (every error its solo call returns, a NULL per-session pointer included) is its status; the others run.
 * The edge searches of every session run in one launch per 32 sessions (k_backend_edge_batch), the surf searches likewise
 * (k_backend_surf_batch), the counts in one more (k_win_count_batch), all on ctxs[0]'s stream (other sessions' streams are
 * joined with events); a session without edge (surf) queries takes part in no edge (surf) launch, as in its solo call.  The call
 * waits once for all sessions, where B solo calls wait B times.
 * LILIOM_E_ARG for the whole call, nothing changed: B < 1, a NULL array (ctxs, bps, kf_ids, poses7_lidar, k, n_edge_corr,
 * n_surf_corr, status), a NULL or repeated context, contexts on different devices, a context with a communicator. */
int liliom_backend_window_correspond_batch(liliom_ctx* const* ctxs, int B, const liliom_backend_params* bps,
                                           const int* const* kf_ids, const double* const* poses7_lidar, const int* k,
                                           int* const* n_edge_corr, int* const* n_surf_corr, int* status);
/* liliom_backend_window_blocks of B independent sessions in one call.  poses7_body, out29: B per-session pointers (7 k[i] and
 * 2 k[i] 29 doubles); k, status: B ints.  Session i gets exactly what liliom_backend_window_blocks(ctxs[i], poses7_body[i], k[i],
 * out29[i]) would give it, bit for bit (same partition, same fixed-order sums), with status, liliom_last_error and launches as
 * that call's.  A session whose LM has stopped is simply left out of ctxs.  The segments of up to 32 sessions share one
 * k_backend_block_batch launch and one k_backend_block_sum launch on ctxs[0]'s stream, and the call reads the blocks of every
 * session back with one wait.  Per-session errors and whole-call refusals as liliom_backend_window_correspond_batch. */
int liliom_backend_window_blocks_batch(liliom_ctx* const* ctxs, int B, const double* const* poses7_body, const int* k,
                                       double* const* out29, int* status);

/* The settings and the results of one session of liliom_loop_align_batch: liliom_loop_align's arguments and outputs. */
typedef struct { float leaf; double max_corr_dist; int max_iter; double trans_eps, fit_eps; } liliom_loop_params;
typedef struct { double T16[16]; double fitness; int converged, iters, n_src, n_tgt; } liliom_loop_result;
/* liliom_loop_align of B independent sessions in one call.  src_ids, src_poses7, tgt_ids, tgt_poses7: B per-session pointers;
 * k_src, k_tgt, status: B ints; prm, res: B structs.  Session i gets exactly what
 *   liliom_loop_align(ctxs[i], src_ids[i], src_poses7[i], k_src[i], tgt_ids[i], tgt_poses7[i], k_tgt[i], prm[i].leaf,
 *                     prm[i].max_corr_dist, prm[i].max_iter, prm[i].trans_eps, prm[i].fit_eps, res[i].T16, &res[i].fitness,
 *                     &res[i].converged, &res[i].iters, &res[i].n_src, &res[i].n_tgt)
 * would give it, bit for bit: status, results, liliom_last_error, launches and lib_launches, and the state left in ctxs[i] (the
 * loop index and source, no resident scan for liliom_map_update_resident; the odometry map, the local map, the window and the
 * keyframe store untouched), so that solo and batched calls mix freely.  A session without a loop candidate this tick is simply
 * left out of ctxs.  Horizon (48-byte) and ROT (32-byte) sessions may be mixed, each with its own lists and settings.
 * Every kernel of both clouds' composition (gather, VoxelGrid chain, repack) and of the targets' cell grids runs once for up to 32
 * sessions on ctxs[0]'s stream (other sessions' streams are joined with events); the library sorts and scans stay per session, in
 * order on the same stream.  The ICPs share cooperative k_icp_batch launches: each session keeps its solo grid, its own barrier
 * word, partials and pinned results, so its bits do not depend on its neighbours; a session whose solo grid is not co-resident
 * beside nothing else in k_icp_batch runs k_icp_persistent inside the call.  The call waits three times for all sessions together
 * (both clouds' counts, the targets' boxes, the results) where B solo calls wait four times each; a session whose voxel index
 * wraps (wide keys) finishes on its solo path inside the call.  Sessions with an empty source or target get identity,
 * converged = 0 and iters = 0 without an ICP launch, as in the solo call.
 * A session's own error (every error its solo call returns: an unknown id, leaf <= 0, max_corr_dist <= 0, max_iter < 1, a negative
 * k, a NULL list with k > 0; LILIOM_E_GRID) is its status; the others run.
 * LILIOM_E_ARG for the whole call, nothing changed: B < 1, a NULL array (ctxs, src_ids, src_poses7, k_src, tgt_ids, tgt_poses7,
 * k_tgt, prm, res, status), a NULL or repeated context, contexts on different devices, a context with a communicator. */
int liliom_loop_align_batch(liliom_ctx* const* ctxs, int B, const int* const* src_ids, const double* const* src_poses7, const int* k_src,
                            const int* const* tgt_ids, const double* const* tgt_poses7, const int* k_tgt,
                            const liliom_loop_params* prm, liliom_loop_result* res, int* status);
/* liliom_loop_align_multi of B independent sessions in one call (many inter-robot or prior-map loop candidates at once).
 * src_stores, tgt_stores: B per-session arrays (liliom_loop_align_multi's stores); the other arguments as liliom_loop_align_batch.
 * Session i gets exactly what liliom_loop_align_multi(ctxs[i], src_stores[i], src_ids[i], src_poses7[i], k_src[i], tgt_stores[i],
 * tgt_ids[i], tgt_poses7[i], k_tgt[i], prm[i]..., res[i]...) would give it, bit for bit, with everything liliom_loop_align_batch
 * promises (status, results, liliom_last_error, launches and lib_launches, the state left in ctxs[i]); launches and waits as
 * liliom_loop_align_batch.  Stores as liliom_bmap_build_batch_multi: any backend context on the device, only read, every distinct
 * store stream joined into ctxs[0]'s stream before the first read, every read done when the call returns, no other host thread
 * calling into a store meanwhile.  A session's own error (every error its solo call returns, the stores' included) is its status;
 * the others run.  LILIOM_E_ARG for the whole call, nothing changed: as liliom_loop_align_batch, and a NULL src_stores or
 * tgt_stores. */
int liliom_loop_align_batch_multi(liliom_ctx* const* ctxs, int B, liliom_ctx* const* const* src_stores, const int* const* src_ids,
                                  const double* const* src_poses7, const int* k_src, liliom_ctx* const* const* tgt_stores,
                                  const int* const* tgt_ids, const double* const* tgt_poses7, const int* k_tgt,
                                  const liliom_loop_params* prm, liliom_loop_result* res, int* status);

#ifdef __cplusplus
}
#endif
#endif /* LILIOM_H */
