// Harness of the reference's LidarOdometry.cpp (LiLi-OM/src, PointXYZINormal; built again as ref_lo_rot.cpp against
// LiLi-OM-ROT/src, PointXYZI), called at member level: undistortion, transformPoint / transformCloud,
// findCorrespondingSurfFeatures, poseInitialization / computeRelative, and buildLocalMap + downSampleCloud over the frame FIFO.
// updateTransformationWithCeres and run() are not driven.  Points cross the API as arrays of the variant's PointType.
#include "harness.h"
#define private public
#include "LidarOdometry.cpp"
#undef private

namespace {
LidarOdometry* g_lo = nullptr;

void set_abs(const double p[7]) { for (int k = 0; k < 7; ++k) g_lo->abs_pose[k] = p[k]; }
}

REF_API int ref_lo_point_size() { return (int)sizeof(PointType); }

REF_API void ref_lo_create() {
    delete g_lo;
    ref::reset_world();
    g_lo = new LidarOdometry();
}

// undistortion(cloud, trans, quat) in place
REF_API void ref_lo_undistort(void* pts, int n, const double trans[3], const double quat[4]) {
    auto c = ref::cloud_of<PointType>(pts, n);
    g_lo->undistortion(c, Eigen::Vector3d(trans[0], trans[1], trans[2]), Eigen::Quaterniond(quat[0], quat[1], quat[2], quat[3]));
    ref::copy_out(c->points, pts, n);
}

// transformCloud(cloud, &PointPoseInfo{pose7})
REF_API void ref_lo_transform_cloud(const void* pts, int n, const double pose7[7], void* out) {
    auto c = ref::cloud_of<PointType>(pts, n);
    PointPoseInfo info;
    info.qw = pose7[0]; info.qx = pose7[1]; info.qy = pose7[2]; info.qz = pose7[3];
    info.x = pose7[4]; info.y = pose7[5]; info.z = pose7[6];
    info.idx = 0; info.time = 0;
    auto o = g_lo->transformCloud(c, &info);
    ref::copy_out(o->points, out, n);
}

// transformPoint at abs_pose = pose7, point by point (po is default-constructed, as findCorrespondingSurfFeatures' point_sel)
REF_API void ref_lo_transform_point(const void* pts, int n, const double pose7[7], void* out) {
    set_abs(pose7);
    const PointType* in = (const PointType*)pts;
    PointType* o = (PointType*)out;
    for (int i = 0; i < n; ++i) { PointType p; g_lo->transformPoint(&in[i], &p); o[i] = p; }
}

// findCorrespondingSurfFeatures with surf_from_map_ds = map (and the kd-tree over it), surf_last_ds = feats, abs_pose = pose7.
// out_pts / out_normal: the accepted points and their `normal` points, in the order the node appends them (capacity n).
REF_API int ref_lo_find_surf_corr(const void* map, int m, const void* feats, int n, const double pose7[7], void* out_pts,
                                  void* out_normal) {
    *g_lo->surf_from_map_ds = *ref::cloud_of<PointType>(map, m);
    g_lo->kd_tree_surf_last->setInputCloud(g_lo->surf_from_map_ds);
    *g_lo->surf_last_ds = *ref::cloud_of<PointType>(feats, n);
    set_abs(pose7);
    g_lo->surf_current_pts->clear();
    g_lo->surf_normal->clear();
    g_lo->findCorrespondingSurfFeatures();
    ref::copy_out(g_lo->surf_current_pts->points, out_pts, n);
    ref::copy_out(g_lo->surf_normal->points, out_normal, n);
    return g_lo->surf_res_cnt;
}

// poseInitialization: abs_pose <- abs_pose (+) rel_pose
REF_API void ref_lo_pose_init(const double abs7[7], const double rel7[7], double out7[7]) {
    set_abs(abs7);
    for (int k = 0; k < 7; ++k) g_lo->rel_pose[k] = rel7[k];
    g_lo->poseInitialization();
    for (int k = 0; k < 7; ++k) out7[k] = g_lo->abs_pose[k];
}

// computeRelative: rel_pose of abs_pose = cur7 against the second-to-last saved pose (prev7), or against the identity when
// no pose has been saved (prev7 == NULL)
REF_API void ref_lo_compute_relative(const double* prev7, const double cur7[7], double rel7[7]) {
    g_lo->pose_info_cloud_frame->clear();
    if (prev7) {
        PointPoseInfo p;
        p.qw = prev7[0]; p.qx = prev7[1]; p.qy = prev7[2]; p.qz = prev7[3]; p.x = prev7[4]; p.y = prev7[5]; p.z = prev7[6];
        p.idx = 0; p.time = 0;
        g_lo->pose_info_cloud_frame->push_back(p);
        g_lo->pose_info_cloud_frame->push_back(p);   // the last entry is the current frame's; computeRelative reads the one before
    }
    set_abs(cur7);
    g_lo->computeRelative();
    for (int k = 0; k < 7; ++k) rel7[k] = g_lo->rel_pose[k];
}

// One scan of run()'s map maintenance with the scan-to-map step replaced by `pose7`: the first call saves the pose and
// initialises (:662-666); every later one runs buildLocalMap and downSampleCloud on surf, takes pose7 as the matched pose,
// saves it and clears (:670-681).  out_map: the down-sampled local map the scan was matched against (capacity cap); out_ds:
// the scan's own down-sampled cloud (capacity n).  Returns the map's size, or -1 on the initialising call.
REF_API int ref_lo_map_step(const void* surf, int n, const double pose7[7], void* out_map, int cap, void* out_ds, int* n_ds) {
    *g_lo->surf_features = *ref::cloud_of<PointType>(surf, n);
    *n_ds = 0;
    if (!g_lo->system_initialized) {
        set_abs(pose7);
        g_lo->savePoses();
        g_lo->checkInitialization();
        return -1;
    }
    g_lo->buildLocalMap();
    g_lo->downSampleCloud();
    const int m = ref::copy_out(g_lo->surf_from_map_ds->points, out_map, cap);
    *n_ds = ref::copy_out(g_lo->surf_last_ds->points, out_ds, n);
    set_abs(pose7);
    g_lo->savePoses();
    g_lo->computeRelative();
    g_lo->clearCloud();
    return m;
}
