/* ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h header); what is pinned: DESIGN.md §6.
 *
 * C interface of the CPU restatement of LiLi-OM's per-scan hot path.  Loaded through
 * ctypes by tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs — never by
 * the product package (liliom_b200/).  Citations are relative to the reference repository's root.
 */
#ifndef LILIOM_ORACLE_API_H
#define LILIOM_ORACLE_API_H
#ifdef __cplusplus
extern "C" {
#endif

/* PCL point layouts (third-party, from knowledge): 16-byte aligned, float4 #0 = x,y,z,1. */
typedef struct { float x, y, z, w; float nx, ny, nz, nw; float intensity, curvature, p0, p1; } orc_pt48; /* pcl::PointXYZINormal */
typedef struct { float x, y, z, w; float intensity, p0, p1, p2; } orc_pt32;                             /* pcl::PointXYZI */

/* ---- pcl::VoxelGrid (LidarOdometry.cpp:315-323; LiLi-OM-ROT/src/Preprocessing.cpp:502-508) ----
 * stride = 48 or 32.  Returns the output count; when the voxel index would overflow int32
 * PCL warns and returns the input unchanged — the restatement does the same (count = n). */
int orc_voxelgrid(const void* pts, int n, int stride, float leaf, void* out, int cap);

/* ---- exact K=5 nearest neighbours (pcl::KdTreeFLANN, LidarOdometry.cpp:490,360) ----
 * map: float4 {x,y,z,*}.  idx/sqd: nq*5, ascending (squared distance fp32, then index).
 * Entries beyond the cloud size are idx=-1, sqd=+inf. */
void* orc_kdtree_build(const float* map_xyzw, int m);
void  orc_kdtree_free(void* tree);
void  orc_knn5(const void* tree, const float* q_xyzw, int nq, int* idx, float* sqd, int nthreads);
void  orc_knn5_brute(const float* map_xyzw, int m, const float* q_xyzw, int nq, int* idx, float* sqd);

/* ---- LidarOdometry::findCorrespondingSurfFeatures (LidarOdometry.cpp:352-413) ----
 * feats: float4 body-frame points.  Per feature i: corr_valid[i] in {0,1};
 * corr_plane[i] = {w*nx, w*ny, w*nz, w*d} (the `normal` point of :401-405);
 * nn_idx (optional, n*5) = the 5-NN indices; pw (optional, n*4) = transformed point.
 * Returns the number of accepted correspondences (surf_res_cnt). */
int orc_find_surf_corr(const void* tree, const float* map_xyzw, int m, const float* feats_xyzw, int n,
                       const double pose7[7], unsigned char* corr_valid, float* corr_plane,
                       int* nn_idx, float* pw, int nthreads);

/* 27 scalars (upper triangle of J^T J row-major: 21, then J^T r: 6) + cost + count, for the
 * Huber(0.1)-robustified plane residuals of LidarKeyframeFactor.h:111-139 at `pose7`
 * over frozen correspondences.  order of the 6 tangent dims: rot(3) then trans(3). */
void orc_normal_equations(const float* feats_xyzw, int n, const unsigned char* corr_valid,
                          const float* corr_plane, const double pose7[7], double huber_a,
                          double out29[29]);

typedef struct {
    int    n_corr;      /* accepted correspondences at the linearisation pose */
    int    lm_iters;    /* Ceres iterations executed (ceres mode), 1 in GN mode */
    double cost;        /* 1/2 sum rho(r^2) at the linearisation pose */
    double jtj_jtr[27]; /* 21 + 6 at the linearisation pose (unscaled) */
    double pose7[7];    /* pose after this outer iteration */
} orc_iter_stats;

/* GN mode: `iters` iterations of [re-associate, linearise, solve H d = -b, Plus].
 * Returns 0, or -1 when m < 10 (LidarOdometry.cpp:485-488: pose untouched).
 * stats may be NULL, else iters entries. */
int orc_scan_to_map_gn(const void* tree, const float* map_xyzw, int m, const float* feats_xyzw, int n,
                       double pose7[7], int iters, orc_iter_stats* stats, int nthreads);

/* Ceres-faithful mode (LidarOdometry.cpp:483-561): match_cnt outer iterations, each with
 * frozen correspondences and a Ceres-2.0-default trust-region LM of <= max_num_iter
 * iterations, DENSE_QR on [J; D]; the reference's 15 ms wall-clock cap is disabled. */
int orc_scan_to_map_ceres(const void* tree, const float* map_xyzw, int m, const float* feats_xyzw, int n,
                          double pose7[7], int match_cnt, int max_num_iter, orc_iter_stats* stats, int nthreads);

/* Ceres LM on frozen correspondences only (one ceres::Solve). Returns LM iterations run. */
int orc_ceres_solve(const float* feats_xyzw, int n, const unsigned char* corr_valid, const float* corr_plane,
                    double pose7[7], int max_num_iter, double* final_cost);

/* ---- Preprocessing (Horizon), LiLi-OM/src/Preprocessing.cpp:219-383 ----
 * pts: n x 48 B (as published by FormatConvert.cpp:14-22). q_imu: un-normalised (w,x,y,z).
 * Outputs are caller-allocated with capacity >= n (cutted, surf) / n (edge). */
int orc_extract_horizon(const orc_pt48* pts, int n, const double q_imu[4], double surf_thres, double edge_thres,
                        orc_pt48* surf, int* n_surf, orc_pt48* edge, int* n_edge, orc_pt48* cutted, int* n_cut);

/* ---- Preprocessing (ROT), LiLi-OM-ROT/src/Preprocessing.cpp:276-509 ----
 * pts: n x 32 B. label_out (optional, capacity n): cloudLabel per laserCloud point;
 * labels of points not visited by the curvature loop are 0. */
int orc_extract_rot(const orc_pt32* pts, int n, const double q_imu[4], const double q_lb[4], int line_num, int ds_rate,
                    orc_pt32* surf, int* n_surf, orc_pt32* edge, int* n_edge, orc_pt32* cutted, int* n_cut,
                    int* label_out, float* curv_out);

/* ---- BackendFusion correspondences ----
 * edge: LiLi-OM/src/BackendFusion.cpp:1531-1599 (variant 0) /
 *       LiLi-OM-ROT/src/BackendFusion.cpp:1394-1462 (variant 1: extra dist<0.1 gate).
 * valid[i], pa[i*3..], pb[i*3..] (float, as stored in PointType). */
int orc_correspond_edge(const void* tree, const float* map_xyzw, int m, const float* feats_xyzw, int n,
                        const double pose7[7], int variant, unsigned char* valid, float* pa, float* pb);
/* surf (ROT variant, LiLi-OM-ROT/src/BackendFusion.cpp:1464-1520): kd_max_radius, surf_dist_thres,
 * weight gate; plane[i] = {w n, w d}, score[i] = lidar_const*w.
 * Horizon variant (LiLi-OM/src/BackendFusion.cpp:1601-1681) when refl != NULL: map_refl/feat_refl
 * hold the `curvature` (reflectivity) channel; reflect_thres gate; score = lidar_const*(w+exp(-sum)). */
int orc_correspond_surf_backend(const void* tree, const float* map_xyzw, int m, const float* feats_xyzw, int n,
                                const double pose7[7], double kd_max_radius, double surf_dist_thres, double w_gate,
                                double lidar_const, const float* map_refl, const float* feat_refl, double reflect_thres,
                                unsigned char* valid, float* plane, double* score);


/* ---- (f1) backend LiDAR residual blocks of one window keyframe, LiLi-OM/src/BackendFusion.cpp:919-979 ----
 * LidarEdgeFactor / LidarPlaneNormFactor (LidarKeyframeFactor.h:12-108) under CauchyLoss(cauchy_b), reduced to the
 * keyframe's normal-equation block.  Tangent order [t(3), rot(3)] (parameter blocks t, q); out29 = 21 + 6 + cost + count.
 * feats/valid/pa/pb/plane/score are the outputs of the correspondence searches above; pose7_body = [qw..qz, tx..tz] of the
 * keyframe (tmpQuat/tmpTrans), NOT the lidar pose the search ran at. */
void orc_backend_edge_block(const float* feats_xyzw, int n, const unsigned char* valid, const float* pa, const float* pb,
                            double s_weight, const double pose7_body[7], double cauchy_b, double out29[29]);
void orc_backend_surf_block(const float* feats_xyzw, int n, const unsigned char* valid, const float* plane, const double* score,
                            const double pose7_body[7], const double q_lb[4], const double t_lb[3], double cauchy_b,
                            double out29[29]);

/* ---- (f3) FormatConvert, LiLi-OM/src/FormatConvert.cpp:11-24: livox CustomPoint[] -> PointXYZINormal[] ---- */
void orc_convert_livox(const unsigned char* custom_pts, int n, int stride, orc_pt48* out);

/* ---- host glue restated for tests of the node mirror ----
 * math_tools.h:125-138 deltaQ + Preprocessing.cpp:129-133 solveRotation: q <- q * deltaQ(0.5*(g0+g1)*dt) */
void orc_solve_rotation(double q_wxyz[4], const double gyr0[3], const double gyr1[3], double dt);
/* LidarOdometry.cpp:415-442 poseInitialization; :444-480 computeRelative */
void orc_pose_compose(const double abs7[7], const double rel7[7], double out7[7]);
void orc_pose_relative(const double prev7[7], const double cur7[7], double rel7[7]);
/* LidarOdometry.cpp:246-278 transformCloud (48 B: rotates normals; 32 B: xyz+intensity only) */
void orc_transform_cloud(const void* in, int n, int stride, const double pose7[7], void* out);
/* LidarOdometry::undistortion, L/src/LidarOdometry.cpp:178-199 (in place) */
void orc_undistort(void* pts, int n, int stride, const double trans[3], const double quat_wxyz[4]);

/* ---- test hooks for the from-knowledge third-party restatements (oracle_math.h) ---- */
void orc_eigen_sym3(const double a_rowmajor[9], double eval[3], double evec_rowmajor[9]);
void orc_colpiv_qr_solve(int rows, const double* A_rows_x3, const double* b, double x[3]);
void orc_slerp_identity(const double q_wxyz[4], double t, double out_wxyz[4]);

#ifdef __cplusplus
}
#endif
#endif
