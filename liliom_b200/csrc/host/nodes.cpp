// See nodes.h.  Line citations are to the reference tree (L/ = LiLi-OM/, R/ = LiLi-OM-ROT/).
#include "nodes.h"
#include "../pc2_fields.h"
#include <cmath>
#include <cstring>
#include <cstdlib>

namespace liliom {

// ---- the few Eigen operations the node glue uses (fp64, Eigen's formulas)
static inline Quat qmul(const Quat& a, const Quat& b) {
    return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}
static inline Vec3 cross(const Vec3& a, const Vec3& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
static inline Vec3 qrot(const Quat& q, const Vec3& v) {            // Eigen: v + w*uv + qv x uv, uv = 2 qv x v
    Vec3 qv{q.x, q.y, q.z};
    Vec3 uv = cross(qv, v);
    uv = {uv.x + uv.x, uv.y + uv.y, uv.z + uv.z};
    Vec3 c = cross(qv, uv);
    return {v.x + q.w * uv.x + c.x, v.y + q.w * uv.y + c.y, v.z + q.w * uv.z + c.z};
}
static inline Quat qinverse(const Quat& q) {
    double n2 = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
    if (n2 > 0) return {q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
    return {0, 0, 0, 0};
}

// ============================================================ Preprocessing
Preprocessing::Preprocessing(liliom_ctx* g, int var, const double qlb[4]) : gpu(g), variant(var), stride(var == 1 ? 32 : 48) {
    if (qlb) q_lb = Quat{qlb[0], qlb[1], qlb[2], qlb[3]};
}

// L/src/Preprocessing.cpp:173-192
void Preprocessing::imuHandler(double stamp, const double gyro[3]) {
    imu_buf.push_back(ImuMsg{stamp, Vec3{gyro[0], gyro[1], gyro[2]}, true});
    if (imu_buf.size() > 600) imu_buf[imu_buf.size() - 601].valid = false;     // the reference nulls the pointer (:176-177)
    if (current_time_imu < 0) current_time_imu = stamp;
    if (!first_imu) {
        first_imu = true;
        gyr_0 = Vec3{gyro[0], gyro[1], gyro[2]};
    }
}

// :129-133 with math_tools.h:125-138 deltaQ (un-normalised: w = 1, xyz = theta/2)
void Preprocessing::solveRotation(double dt, const Vec3& w) {
    Vec3 un_gyr{0.5 * (gyr_0.x + w.x), 0.5 * (gyr_0.y + w.y), 0.5 * (gyr_0.z + w.z)};
    Vec3 th{un_gyr.x * dt, un_gyr.y * dt, un_gyr.z * dt};
    Quat dq{1.0, th.x / 2.0, th.y / 2.0, th.z / 2.0};
    q_iMU = qmul(q_iMU, dq);
    gyr_0 = w;
}

// :135-171.  The reference dereferences imu_buf[i] even after entry i was released (:176-177, latent UB):
// here a released entry simply stops the integration loop.
void Preprocessing::processIMU(double t_cur) {
    double rx = 0, ry = 0, rz = 0;
    int i = idx_imu;
    if (i >= (int)imu_buf.size()) i--;
    while (i >= 0 && imu_buf[i].valid && imu_buf[i].stamp < t_cur) {
        double t = imu_buf[i].stamp;
        if (current_time_imu < 0) current_time_imu = t;
        double dt = t - current_time_imu;
        current_time_imu = imu_buf[i].stamp;
        rx = imu_buf[i].angular_velocity.x; ry = imu_buf[i].angular_velocity.y; rz = imu_buf[i].angular_velocity.z;
        solveRotation(dt, Vec3{rx, ry, rz});
        i++;
        if (i >= (int)imu_buf.size()) break;
    }
    if (i >= 0 && i < (int)imu_buf.size() && imu_buf[i].valid) {
        double dt1 = t_cur - current_time_imu;
        double dt2 = imu_buf[i].stamp - t_cur;
        double w1 = dt2 / (dt1 + dt2);
        double w2 = dt1 / (dt1 + dt2);
        rx = w1 * rx + w2 * imu_buf[i].angular_velocity.x;
        ry = w1 * ry + w2 * imu_buf[i].angular_velocity.y;
        rz = w1 * rz + w2 * imu_buf[i].angular_velocity.z;
        solveRotation(dt1, Vec3{rx, ry, rz});
    }
    current_time_imu = t_cur;
    idx_imu = i < 0 ? 0 : i;
}

// :194-408 (R: :248-535)
int Preprocessing::cloudHandler(double stamp, const void* pts, int n, void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap,
                                int* n_edge, void* cutted, int cut_cap, int* n_cut, double* stamp_out, double q_imu_out[4]) {
    CloudMsg m;
    m.stamp = stamp; m.n = n;
    m.data.assign((const unsigned char*)pts, (const unsigned char*)pts + (size_t)n * stride);
    return handleCloud(std::move(m), surf, surf_cap, n_surf, edge, edge_cap, n_edge, cutted, cut_cap, n_cut, stamp_out, q_imu_out);
}

// R/src/Preprocessing.cpp:248-535 on the PointCloud2 itself: the queue keeps a copy of the whole message (:251)
int Preprocessing::cloudHandlerPc2(double stamp, const liliom_pc2_msg* msg, void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap,
                                   int* n_edge, void* cutted, int cut_cap, int* n_cut, double* stamp_out, double q_imu_out[4]) {
    lili::Pc2Map map;
    if (variant != 1 || lili::pc2_match(msg, &map) != LILIOM_OK) return LILIOM_E_ARG;
    CloudMsg m;
    m.stamp = stamp; m.n = map.n; m.pc2 = true;
    m.height = msg->height; m.width = msg->width; m.point_step = msg->point_step; m.row_step = msg->row_step;
    if (map.n > 0) m.data.assign((const unsigned char*)msg->data, (const unsigned char*)msg->data + (size_t)msg->height * msg->row_step);
    if (msg->n_fields > 0) m.fields.assign(msg->fields, msg->fields + msg->n_fields);
    return handleCloud(std::move(m), surf, surf_cap, n_surf, edge, edge_cap, n_edge, cutted, cut_cap, n_cut, stamp_out, q_imu_out);
}

int Preprocessing::handleCloud(CloudMsg&& m, void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap, int* n_edge, void* cutted,
                               int cut_cap, int* n_cut, double* stamp_out, double q_imu_out[4]) {
    cloud_queue.push_back(std::move(m));                                   // :196
    if (cloud_queue.size() <= 2) return 0;                                 // :197-198
    CloudMsg cur = std::move(cloud_queue.front());                         // :201-202
    cloud_queue.pop_front();
    time_scan_next = cloud_queue.front().stamp;                            // :206
    int tmp_idx = idx_imu > 0 ? idx_imu - 1 : 0;                           // :209-211
    if (imu_buf.empty() || (tmp_idx < (int)imu_buf.size() && imu_buf[tmp_idx].stamp > time_scan_next)) return 0;   // "Waiting for IMU data ..."
    if ((variant == 0 && !imu_buf.empty()) || (variant == 1 && first_imu)) processIMU(time_scan_next);            // :230-231 / R:297-298
    if (std::isnan(q_iMU.w) || std::isnan(q_iMU.x) || std::isnan(q_iMU.y) || std::isnan(q_iMU.z)) q_iMU = Quat{}; // :232-234
    const double q[4] = {q_iMU.w, q_iMU.x, q_iMU.y, q_iMU.z};
    int rc;
    if (variant == 0)
        rc = liliom_extract_horizon(gpu, (const liliom_pt48*)cur.data.data(), cur.n, q, (liliom_pt48*)surf, surf_cap, n_surf,
                                    (liliom_pt48*)edge, edge_cap, n_edge, (liliom_pt48*)cutted, cut_cap, n_cut);           // :225-383
    else if (cur.pc2) {
        const double ql[4] = {q_lb.w, q_lb.x, q_lb.y, q_lb.z};
        const liliom_pc2_msg msg{cur.data.data(), cur.height, cur.width, cur.point_step, cur.row_step, cur.fields.data(), (int)cur.fields.size(), 0};
        rc = liliom_extract_rot_pc2(gpu, &msg, q, ql, (liliom_pt32*)surf, surf_cap, n_surf, (liliom_pt32*)edge, edge_cap, n_edge,
                                    (liliom_pt32*)cutted, cut_cap, n_cut);                                                   // R:277-509
    } else {
        const double ql[4] = {q_lb.w, q_lb.x, q_lb.y, q_lb.z};
        rc = liliom_extract_rot(gpu, (const liliom_pt32*)cur.data.data(), cur.n, q, ql, (liliom_pt32*)surf, surf_cap, n_surf,
                                (liliom_pt32*)edge, edge_cap, n_edge, (liliom_pt32*)cutted, cut_cap, n_cut);               // R:280-509
    }
    if (stamp_out) *stamp_out = cur.stamp;
    if (q_imu_out) { q_imu_out[0] = q[0]; q_imu_out[1] = q[1]; q_imu_out[2] = q[2]; q_imu_out[3] = q[3]; }
    q_iMU = Quat{};                                                        // :403
    return rc == LILIOM_OK ? 1 : rc;
}

// ============================================================ LidarOdometry
LidarOdometry::LidarOdometry(liliom_ctx* g, int mni, int smc, bool deskew, int md)
    : gpu(g), max_num_iter(mni), scan_match_cnt(smc), mode(md), if_to_deskew(deskew) {
    stride = liliom_point_stride(gpu);
}

static void assign(std::vector<unsigned char>& dst, const void* pts, int n, int stride) {
    dst.assign((const unsigned char*)pts, (const unsigned char*)pts + (size_t)n * stride);
}
// :159-176
void LidarOdometry::laserCloudLessSharpHandler(double stamp, const void* pts, int n) { time_new_edge = stamp; assign(edge_features, pts, n, stride); n_edge_features = n; new_edge = true; }
void LidarOdometry::laserCloudLessFlatHandler(double stamp, const void* pts, int n) { time_new_surf = stamp; assign(surf_features, pts, n, stride); n_surf_features = n; new_surf = true; }
void LidarOdometry::FullPointCloudHandler(double stamp, const void* pts, int n) { time_new_full_points = stamp; cloud_stamp = stamp; assign(full_cloud, pts, n, stride); n_full_cloud = n; new_full_cloud = true; }

// :415-442
void LidarOdometry::poseInitialization() {
    Quat q0{abs_pose[0], abs_pose[1], abs_pose[2], abs_pose[3]};
    Vec3 t0{abs_pose[4], abs_pose[5], abs_pose[6]};
    Quat dq{rel_pose[0], rel_pose[1], rel_pose[2], rel_pose[3]};
    Vec3 dt{rel_pose[4], rel_pose[5], rel_pose[6]};
    Vec3 r = qrot(q0, dt);
    t0 = Vec3{r.x + t0.x, r.y + t0.y, r.z + t0.z};
    q0 = qmul(q0, dq);
    abs_pose[0] = q0.w; abs_pose[1] = q0.x; abs_pose[2] = q0.y; abs_pose[3] = q0.z;
    abs_pose[4] = t0.x; abs_pose[5] = t0.y; abs_pose[6] = t0.z;
}

// :280-303 + :316-317 + :490 : the library owns recent_surf_frames (FIFO of 20), the VoxelGrid and the search grid
int LidarOdometry::buildLocalMap() {
    const int nposes = (int)pose_info_cloud_frame.size();
    int rc;
    if (nposes <= 1) {                                                     // :283-287 map = the current (raw) surf features
        liliom_map_clear(gpu);
        const double I[7] = {1, 0, 0, 0, 0, 0, 0};
        temp_map = true;
        return liliom_map_update(gpu, surf_features.data(), n_surf_features, I, &n_map);
    }
    if (temp_map) { liliom_map_clear(gpu); temp_map = false; map_current = false; }
    if (recent_frames < 20 || latest_frame_idx != nposes - 1) {            // :290-299
        const int i = nposes - 1;
        const PoseInfo& P = pose_info_cloud_frame[i];
        const double pose[7] = {P.qw, P.qx, P.qy, P.qz, P.x, P.y, P.z};
        if (recent_frames < 20) recent_frames++;
        else latest_frame_idx = nposes - 1;
        // transformCloud :246-278 + FIFO :290-299 + concatenation :301-302 + VoxelGrid(0.4) :316-317 + search structure :490, as ONE
        // incremental call: the filtered map lives on the device across scans (SURVEY §8 f2, liliom_map_update)
        rc = liliom_map_update(gpu, surf_frames[i].data(), surf_frames_n[i], pose, &n_map);
        map_current = rc == LILIOM_OK;
        return rc;
    }
    // No frame entered the FIFO: the reference re-concatenates and re-filters the same 20 clouds (:301-302, :316-317) and gets
    // the cloud it already had; the resident map is that cloud.
    if (map_current) return LILIOM_OK;
    rc = liliom_map_rebuild(gpu, &n_map);
    map_current = rc == LILIOM_OK;
    return rc;
}

// :319-322 + :483-561 + keyframe decision :565-585
int LidarOdometry::updateTransformation() {
    const int match_cnt = pose_info_cloud_frame.size() < 2 ? 8 : scan_match_cnt;   // :500-504
    surf_last_ds.resize((size_t)(n_surf_features > 0 ? n_surf_features : 1) * stride);
    n_surf_last_ds = 0;
    int rc = liliom_odometry(gpu, surf_features.data(), n_surf_features, abs_pose, match_cnt, max_num_iter, mode, nullptr,
                             surf_last_ds.data(), n_surf_features, &n_surf_last_ds);
    last_status = rc;
    if (rc == LILIOM_E_FEWMAP || rc == LILIOM_E_NOMAP) return LILIOM_OK;   // :485-488 "Not enough feature points from the map": return, kf unchanged
    if (rc != LILIOM_OK) return rc;
    Vec3 transCur{abs_pose[4], abs_pose[5], abs_pose[6]};
    Quat quatCur{abs_pose[0], abs_pose[1], abs_pose[2], abs_pose[3]};
    const double dx = transCur.x - trans_last_kf.x, dy = transCur.y - trans_last_kf.y, dz = transCur.z - trans_last_kf.z;
    const double dis = std::sqrt(dx * dx + dy * dy + dz * dz);
    const double ang = 2 * std::acos(qmul(qinverse(quat_last_kF), quatCur).w);
    const size_t sz = pose_info_cloud_frame.size();
    if ((((dis > 0.2 || ang > 0.1) && (sz - kf_num > 1)) || (sz - kf_num > 2)) || sz <= 1) {   // :575 (size_t arithmetic as in the reference)
        kf = true;
        trans_last_kf = transCur;
        quat_last_kF = quatCur;
    } else
        kf = false;
    return LILIOM_OK;
}

// :325-350
void LidarOdometry::savePoses() {
    PoseInfo p;
    p.x = abs_pose[4]; p.y = abs_pose[5]; p.z = abs_pose[6];
    p.qw = abs_pose[0]; p.qx = abs_pose[1]; p.qy = abs_pose[2]; p.qz = abs_pose[3];
    p.idx = (int)pose_info_cloud_frame.size();
    p.time = time_new_surf;
    pose_info_cloud_frame.push_back(p);
    surf_frames.emplace_back(surf_last_ds.begin(), surf_last_ds.begin() + (size_t)n_surf_last_ds * stride);
    surf_frames_n.push_back(n_surf_last_ds);
}

// :444-480
void LidarOdometry::computeRelative() {
    Quat q1; Vec3 t1;
    const int max_idx = (int)pose_info_cloud_frame.size();
    if (max_idx >= 2) {      // the reference indexes [max_idx-2] unconditionally (UB when size is 1, SURVEY App. C.12)
        const PoseInfo& P = pose_info_cloud_frame[max_idx - 2];
        q1 = Quat{P.qw, P.qx, P.qy, P.qz};
        t1 = Vec3{P.x, P.y, P.z};
    }
    Quat q2{abs_pose[0], abs_pose[1], abs_pose[2], abs_pose[3]};
    Vec3 t2{abs_pose[4], abs_pose[5], abs_pose[6]};
    Quat qi = qinverse(q1);
    Quat qr = qmul(qi, q2);
    Vec3 tr = qrot(qi, Vec3{t2.x - t1.x, t2.y - t1.y, t2.z - t1.z});
    rel_pose[0] = qr.w; rel_pose[1] = qr.x; rel_pose[2] = qr.y; rel_pose[3] = qr.z;
    rel_pose[4] = tr.x; rel_pose[5] = tr.y; rel_pose[6] = tr.z;
}

// :178-199, called with quat = identity (:626); the per-point loop runs on the device (liliom_undistort)
int LidarOdometry::undistortion(std::vector<unsigned char>& cloud, int n, const Vec3& trans) {
    const double t[3] = {trans.x, trans.y, trans.z}, ident[4] = {1.0, 0.0, 0.0, 0.0};
    return liliom_undistort(gpu, cloud.data(), n, t, ident);
}

int LidarOdometry::publishClouds(void* kf_edge, int edge_cap, int* n_edge, void* kf_surf, int surf_cap, int* n_surf, void* kf_full,
                                 int full_cap, int* n_full) {
    if ((kf_edge && n_edge_features > edge_cap) || (kf_surf && n_surf_features > surf_cap) || (kf_full && n_full_cloud > full_cap)) return LILIOM_E_CAPACITY;
    if (kf_edge) std::memcpy(kf_edge, edge_features.data(), (size_t)n_edge_features * stride);
    if (kf_surf) std::memcpy(kf_surf, surf_features.data(), (size_t)n_surf_features * stride);
    if (kf_full) std::memcpy(kf_full, full_cloud.data(), (size_t)n_full_cloud * stride);
    if (n_edge) *n_edge = n_edge_features;
    if (n_surf) *n_surf = n_surf_features;
    if (n_full) *n_full = n_full_cloud;
    return LILIOM_OK;
}

// :652-686
int LidarOdometry::run(liliom_lo_output* out, void* kf_edge, int edge_cap, int* n_edge, void* kf_surf, int surf_cap, int* n_surf,
                       void* kf_full, int full_cap, int* n_full) {
    std::memset(out, 0, sizeof(*out));
    if (n_edge) *n_edge = 0;
    if (n_surf) *n_surf = 0;
    if (n_full) *n_full = 0;
    if (new_surf && new_full_cloud && new_edge && std::fabs(time_new_full_points - time_new_surf) < 0.1 &&
        std::fabs(time_new_full_points - time_new_edge) < 0.1) {                       // :653-660
        new_surf = false; new_edge = false; new_full_cloud = false;
    } else
        return LILIOM_OK;
    out->ran = 1;
    out->stamp = cloud_stamp;
    if (!system_initialized) {                                                          // :662-666
        savePoses();
        int rc = publishClouds(kf_edge, edge_cap, n_edge, kf_surf, surf_cap, n_surf, kf_full, full_cap, n_full);   // checkInitialization :201-219
        system_initialized = true;
        out->initialized = 0; out->kf = 0;
        std::memcpy(out->abs_pose, abs_pose, sizeof(abs_pose));
        std::memcpy(out->rel_pose, rel_pose, sizeof(rel_pose));
        return rc;
    }
    out->initialized = 1;
    poseInitialization();                                                               // :668
    int rc = buildLocalMap();                                                           // :670
    if (rc != LILIOM_OK) return rc;
    rc = updateTransformation();                                                        // :671-672
    if (rc != LILIOM_OK) return rc;
    savePoses();                                                                        // :673
    computeRelative();                                                                  // :674
    if (kf) {                                                                           // :675-679
        kf_num = (int)pose_info_cloud_frame.size();
        if (if_to_deskew) {                                                             // publishCloudLast :624-632
            Vec3 trans{rel_pose[4], rel_pose[5], rel_pose[6]};
            if ((rc = undistortion(surf_features, n_surf_features, trans)) != LILIOM_OK) return rc;
            if ((rc = undistortion(edge_features, n_edge_features, trans)) != LILIOM_OK) return rc;
            if ((rc = undistortion(full_cloud, n_full_cloud, trans)) != LILIOM_OK) return rc;
        }
        rc = publishClouds(kf_edge, edge_cap, n_edge, kf_surf, surf_cap, n_surf, kf_full, full_cap, n_full);
    }
    out->kf = kf ? 1 : 0;
    out->n_map = n_map; out->n_surf_ds = n_surf_last_ds; out->status = last_status;
    std::memcpy(out->abs_pose, abs_pose, sizeof(abs_pose));
    std::memcpy(out->rel_pose, rel_pose, sizeof(rel_pose));
    // clearCloud :305-313 — host copies of frames older than 8 are released
    if (surf_frames.size() > 7) { std::vector<unsigned char>().swap(surf_frames[surf_frames.size() - 8]); }
    return rc;
}

}  // namespace liliom

// ============================================================ C interface
struct liliom_pre_node { liliom::Preprocessing impl; liliom_pre_node(liliom_ctx* g, int v, const double* q) : impl(g, v, q) {} };
struct liliom_lo_node { liliom::LidarOdometry impl; liliom_lo_node(liliom_ctx* g, int a, int b, bool c, int d) : impl(g, a, b, c, d) {} };

extern "C" {
liliom_pre_node* liliom_pre_create(liliom_ctx* gpu, int variant, const double q_lb[4]) { return gpu ? new liliom_pre_node(gpu, variant, q_lb) : nullptr; }
void liliom_pre_destroy(liliom_pre_node* n) { delete n; }
void liliom_pre_imu(liliom_pre_node* n, double stamp, const double gyro[3]) { if (n) n->impl.imuHandler(stamp, gyro); }
int liliom_pre_cloud(liliom_pre_node* n, double stamp, const void* pts, int np, void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap,
                     int* n_edge, void* cutted, int cut_cap, int* n_cut, double* stamp_out, double q_imu_out[4]) {
    if (!n || np < 0 || (np > 0 && !pts)) return LILIOM_E_ARG;
    return n->impl.cloudHandler(stamp, pts, np, surf, surf_cap, n_surf, edge, edge_cap, n_edge, cutted, cut_cap, n_cut, stamp_out, q_imu_out);
}
int liliom_pre_cloud_pc2(liliom_pre_node* n, double stamp, const liliom_pc2_msg* msg, void* surf, int surf_cap, int* n_surf, void* edge,
                         int edge_cap, int* n_edge, void* cutted, int cut_cap, int* n_cut, double* stamp_out, double q_imu_out[4]) {
    if (!n) return LILIOM_E_ARG;
    return n->impl.cloudHandlerPc2(stamp, msg, surf, surf_cap, n_surf, edge, edge_cap, n_edge, cutted, cut_cap, n_cut, stamp_out, q_imu_out);
}
liliom_lo_node* liliom_lo_create(liliom_ctx* gpu, int max_num_iter, int scan_match_cnt, int if_to_deskew, int mode) {
    return gpu ? new liliom_lo_node(gpu, max_num_iter, scan_match_cnt, if_to_deskew != 0, mode) : nullptr;
}
void liliom_lo_destroy(liliom_lo_node* n) { delete n; }
void liliom_lo_edge(liliom_lo_node* n, double stamp, const void* pts, int np) { if (n) n->impl.laserCloudLessSharpHandler(stamp, pts, np); }
void liliom_lo_surf(liliom_lo_node* n, double stamp, const void* pts, int np) { if (n) n->impl.laserCloudLessFlatHandler(stamp, pts, np); }
void liliom_lo_full(liliom_lo_node* n, double stamp, const void* pts, int np) { if (n) n->impl.FullPointCloudHandler(stamp, pts, np); }
int liliom_lo_run(liliom_lo_node* n, liliom_lo_output* out, void* kf_edge, int edge_cap, int* n_edge, void* kf_surf, int surf_cap, int* n_surf,
                  void* kf_full, int full_cap, int* n_full) {
    if (!n || !out) return LILIOM_E_ARG;
    return n->impl.run(out, kf_edge, edge_cap, n_edge, kf_surf, surf_cap, n_surf, kf_full, full_cap, n_full);
}
}
