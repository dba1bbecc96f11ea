/* liliom_nodes.h — C interface of the host-side C++ mirror of the reference's two hot-path ROS nodes
 * (liliom_b200/csrc/host/nodes.{h,cpp}).  ROS is not available in this image, so the node classes take
 * plain buffers where the reference takes sensor_msgs; their control flow, state and method names
 * follow L/src/Preprocessing.cpp:5-409 (R/src/Preprocessing.cpp:7-536) and L/src/LidarOdometry.cpp:6-687.
 * A ROS adapter is ~30 lines per node: fromROSMsg -> *_cloud() (the ROT node: the PointCloud2 itself ->
 * liliom_pre_cloud_pc2()), publish the returned buffers.
 * Every compute step goes through the C ABI of liliom.h on the context passed at creation. */
#ifndef LILIOM_NODES_H
#define LILIOM_NODES_H
#include "liliom.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct liliom_pre_node liliom_pre_node;   /* class Preprocessing */
typedef struct liliom_lo_node  liliom_lo_node;    /* class LidarOdometry  */

/* variant 0 = Horizon (48-byte points), 1 = ROT (32-byte points, q_lb = /backend_fusion/ql2b_*). */
liliom_pre_node* liliom_pre_create(liliom_ctx* gpu, int variant, const double q_lb_wxyz[4]);
void liliom_pre_destroy(liliom_pre_node*);
/* imuHandler (L/src/Preprocessing.cpp:173-192) */
void liliom_pre_imu(liliom_pre_node*, double stamp, const double gyro_xyz[3]);
/* cloudHandler (:194-408).  Returns 1 when a scan was processed and published (the reference processes
 * the scan that is two messages behind, :196-207), 0 when it only queued the message or is waiting for
 * IMU data (:212-216), <0 = LILIOM_E_*.  Output buffers (capacity in points) receive the three clouds of
 * the processed scan; *stamp_out = its header stamp; q_imu_out (optional) = the q_iMU that was used. */
int liliom_pre_cloud(liliom_pre_node*, double stamp, const void* pts, int n,
                     void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap, int* n_edge,
                     void* cutted, int cut_cap, int* n_cut, double* stamp_out, double q_imu_out[4]);
/* cloudHandler of the ROT package (R/src/Preprocessing.cpp:248-535) on the driver's PointCloud2 as received: the queued message
 * keeps its payload and field list (the reference copies the whole message, :251), and the processed one goes through
 * liliom_extract_rot_pc2 (fromROSMsg on the device, :277).  Same outputs and return values as liliom_pre_cloud; ROT nodes
 * only.  A message liliom_convert_pc2 would reject: LILIOM_E_ARG, nothing queued. */
int liliom_pre_cloud_pc2(liliom_pre_node*, double stamp, const liliom_pc2_msg* msg,
                         void* surf, int surf_cap, int* n_surf, void* edge, int edge_cap, int* n_edge,
                         void* cutted, int cut_cap, int* n_cut, double* stamp_out, double q_imu_out[4]);

/* mode = LILIOM_MODE_CERES (reference semantics) or LILIOM_MODE_GN. */
liliom_lo_node* liliom_lo_create(liliom_ctx* gpu, int max_num_iter, int scan_match_cnt, int if_to_deskew, int mode);
void liliom_lo_destroy(liliom_lo_node*);
/* laserCloudLessSharpHandler / laserCloudLessFlatHandler / FullPointCloudHandler (:159-176) */
void liliom_lo_edge(liliom_lo_node*, double stamp, const void* pts, int n);
void liliom_lo_surf(liliom_lo_node*, double stamp, const void* pts, int n);
void liliom_lo_full(liliom_lo_node*, double stamp, const void* pts, int n);

typedef struct {
    int    ran;            /* 1 when run() passed the synchronisation gate (:653-660) */
    int    initialized;    /* 0 on the call that only performed checkInitialization (:662-666) */
    int    kf;             /* keyframe decision (:573-585): /odom, /path and the three clouds are published iff 1 */
    int    n_map;          /* surf_from_map_ds size */
    int    n_surf_ds;      /* surf_last_ds size */
    int    status;         /* LILIOM_OK or the error of the scan-to-map call (LILIOM_E_FEWMAP leaves the pose) */
    double abs_pose[7];    /* /odom         (:588-597) */
    double rel_pose[7];    /* /each_odom    (:609-622) */
    double stamp;
} liliom_lo_output;
/* run() (:652-686).  kf clouds (what publishCloudLast sends, incl. the optional translation de-skew :178-199,
 * :624-650) are written to the optional buffers when out->kf == 1 (or on the initialization call). */
int liliom_lo_run(liliom_lo_node*, liliom_lo_output* out,
                  void* kf_edge, int edge_cap, int* n_edge, void* kf_surf, int surf_cap, int* n_surf,
                  void* kf_full, int full_cap, int* n_full);

#ifdef __cplusplus
}
#endif
#endif
