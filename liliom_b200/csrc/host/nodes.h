// Host-side C++ mirror of the two hot-path ROS nodes of the reference (no ROS / PCL / Eigen / Ceres
// dependency: plain buffers in, plain buffers out; all heavy work goes through the liliom.h C ABI).
// Method and member names follow the reference so that the classes read like the originals:
//   class Preprocessing  — L/src/Preprocessing.cpp:5-409, R/src/Preprocessing.cpp:7-536
//   class LidarOdometry  — L/src/LidarOdometry.cpp:6-687 (R/src/LidarOdometry.cpp identical but for normals)
#pragma once
#include <deque>
#include <vector>
#include <cstdint>
#include "../../../include/liliom_nodes.h"

namespace liliom {

struct Quat { double w = 1, x = 0, y = 0, z = 0; };
struct Vec3 { double x = 0, y = 0, z = 0; };

struct ImuMsg { double stamp; Vec3 angular_velocity; bool valid; };
struct CloudMsg {
    double stamp; std::vector<unsigned char> data; int n;
    // a PointCloud2 as received (liliom_pre_cloud_pc2): data is its payload, these are the rest of the message it needs
    bool pc2 = false;
    unsigned int height = 0, width = 0, point_step = 0, row_step = 0;
    std::vector<liliom_pc2_field> fields;
};

class Preprocessing {
public:
    Preprocessing(liliom_ctx* gpu, int variant, const double q_lb[4]);
    void imuHandler(double stamp, const double gyro[3]);
    int cloudHandler(double stamp, const void* pts, int n, void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap, int* n_edge,
                     void* cutted, int cut_cap, int* n_cut, double* stamp_out, double q_imu_out[4]);
    int cloudHandlerPc2(double stamp, const liliom_pc2_msg* msg, void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap, int* n_edge,
                        void* cutted, int cut_cap, int* n_cut, double* stamp_out, double q_imu_out[4]);

private:
    int handleCloud(CloudMsg&& msg, void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap, int* n_edge,
                    void* cutted, int cut_cap, int* n_cut, double* stamp_out, double q_imu_out[4]);
    void solveRotation(double dt, const Vec3& angular_velocity);
    void processIMU(double t_cur);

    liliom_ctx* gpu;
    int variant, stride;
    std::vector<ImuMsg> imu_buf;
    int idx_imu = 0;
    double current_time_imu = -1;
    Vec3 gyr_0;
    Quat q_iMU;
    bool first_imu = false;
    std::deque<CloudMsg> cloud_queue;
    double time_scan_next = 0;
    Quat q_lb;
};

class LidarOdometry {
public:
    LidarOdometry(liliom_ctx* gpu, int max_num_iter, int scan_match_cnt, bool if_to_deskew, int mode);
    void laserCloudLessSharpHandler(double stamp, const void* pts, int n);
    void laserCloudLessFlatHandler(double stamp, const void* pts, int n);
    void FullPointCloudHandler(double stamp, const void* pts, int n);
    int run(liliom_lo_output* out, void* kf_edge, int edge_cap, int* n_edge, void* kf_surf, int surf_cap, int* n_surf,
            void* kf_full, int full_cap, int* n_full);

private:
    void poseInitialization();
    int buildLocalMap();
    int updateTransformation();          // downSampleCloud(scan) + updateTransformationWithCeres
    void savePoses();
    void computeRelative();
    int undistortion(std::vector<unsigned char>& cloud, int n, const Vec3& trans);
    int publishClouds(void* kf_edge, int edge_cap, int* n_edge, void* kf_surf, int surf_cap, int* n_surf, void* kf_full, int full_cap, int* n_full);

    liliom_ctx* gpu;
    int stride;
    int max_num_iter, scan_match_cnt, mode;
    bool if_to_deskew;

    std::vector<unsigned char> edge_features, surf_features, full_cloud, surf_last_ds;
    int n_edge_features = 0, n_surf_features = 0, n_full_cloud = 0, n_surf_last_ds = 0;
    bool new_edge = false, new_surf = false, new_full_cloud = false;
    double time_new_surf = 0, time_new_full_points = 0, time_new_edge = 0;
    double cloud_stamp = 0;

    double abs_pose[7] = {1, 0, 0, 0, 0, 0, 0};
    double rel_pose[7] = {1, 0, 0, 0, 0, 0, 0};
    bool system_initialized = false;

    struct PoseInfo { double x, y, z, qw, qx, qy, qz; int idx; double time; };
    std::vector<PoseInfo> pose_info_cloud_frame;           // pose of each frame (== pose_cloud_frame in size)
    std::vector<std::vector<unsigned char>> surf_frames;   // surf_last_ds of each frame
    std::vector<int> surf_frames_n;
    int recent_frames = 0;                                  // recent_surf_frames.size()
    int latest_frame_idx = 0;
    bool temp_map = false;                                  // the initialization map (:283-287) is in the library FIFO
    bool map_current = false;                               // the resident filtered map describes the present FIFO
    int n_map = 0;

    bool kf = true;
    int kf_num = 0;
    Vec3 trans_last_kf;
    Quat quat_last_kF;
    int last_status = LILIOM_OK;
};

}  // namespace liliom
