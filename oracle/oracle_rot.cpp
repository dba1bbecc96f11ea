// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h).  Pinned to the reference's own code: DESIGN.md §6.
// Spinning-LiDAR (LOAM-style) feature extractor restated: the body of
// Preprocessing::cloudHandler in LiLi-OM-ROT/src/Preprocessing.cpp:276-509, with
// undistortion (:153-177) and removeClosedPointCloud (:120-145).  qIMU is an input (the
// gyro integration :179-223 stays host-side).  The class arrays cloudCurvature / SortInd /
// NeighborPicked / Label (:9-12) persist across scans in the reference; every entry that is
// read is first re-initialised at :390-393, so per-call arrays are equivalent.
// std::sort at :410 is unstable; the order of equal curvatures is DEFINED as ascending index.  Its comparator `curv[a] < curv[b]`
// is no strict weak ordering once a curvature is NaN (returns of magnitude ~1e38 inside one 11-point window give inf - inf), and
// the order is then undefined; DEFINED here: a NaN sorts after +inf (NaNs among themselves by index) and is never a candidate,
// since both `> 2.0` and `< 0.1` are false for it.  rot_curv_less is that total order.
#include "oracle_api.h"
#include "oracle_math.h"
#include <vector>
#include <cstring>

using namespace orc;

extern "C" int orc_extract_rot(const orc_pt32* pts, int n, const double q_imu_in[4], const double q_lb_in[4], int N_SCANS, int ds_rate,
                               orc_pt32* surf, int* n_surf, orc_pt32* edge, int* n_edge, orc_pt32* cutted, int* n_cut,
                               int* label_out, float* curv_out) {
    *n_surf = *n_edge = *n_cut = 0;
    if (N_SCANS != 16 && N_SCANS != 32 && N_SCANS != 64) return -2;   // :344-347 ROS_BREAK
    Quat qIMU{q_imu_in[0], q_imu_in[1], q_imu_in[2], q_imu_in[3]};
    if (std::isnan(qIMU.w) || std::isnan(qIMU.x) || std::isnan(qIMU.y) || std::isnan(qIMU.z)) qIMU = Quat{1, 0, 0, 0};  // :299-301
    Quat q_lb{q_lb_in[0], q_lb_in[1], q_lb_in[2], q_lb_in[3]};
    Quat q_lb_inv = qinv(q_lb);

    // :280-281 removeNaN + removeClosedPointCloud(3.0)
    std::vector<orc_pt32> in;
    in.reserve(n);
    const float thres = 3.0f;
    for (int i = 0; i < n; ++i) {
        const orc_pt32& p = pts[i];
        if (!std::isfinite(p.x) || !std::isfinite(p.y) || !std::isfinite(p.z)) continue;
        if (p.x * p.x + p.y * p.y + p.z * p.z < thres * thres) continue;
        in.push_back(p);
    }
    int cloudSize = (int)in.size();
    if (cloudSize == 0) return 0;   // reference dereferences points[0] (UB); guarded

    float startOri = -std::atan2(in[0].y, in[0].x);                                   // :285
    float endOri = -std::atan2(in[cloudSize - 1].y, in[cloudSize - 1].x) + 2 * M_PI;  // :286-288
    if (endOri - startOri > 3 * M_PI) endOri -= 2 * M_PI;                             // :290-294
    else if (endOri - startOri < M_PI) endOri += 2 * M_PI;

    bool halfPassed = false;
    int count = cloudSize;
    std::vector<std::vector<orc_pt32>> rings(N_SCANS);
    for (int i = 0; i < cloudSize; i++) {                                             // :308
        float px = in[i].x, py = in[i].y, pz = in[i].z;
        float angle = std::atan(pz / std::sqrt(px * px + py * py)) * 180 / M_PI;      // :315
        int scanID = 0;
        if (N_SCANS == 16) {
            scanID = int((angle + 15) / 2 + 0.5);
            if (scanID > (N_SCANS - 1) || scanID < 0) { count--; continue; }
        } else if (N_SCANS == 32) {
            scanID = int((angle + 92.0 / 3.0) * 3.0 / 4.0);
            if (scanID > (N_SCANS - 1) || scanID < 0) { count--; continue; }
        } else {
            if (angle >= -8.83) scanID = int((2 - angle) * 3.0 + 0.5);
            else scanID = N_SCANS / 2 + int((-8.83 - angle) * 2.0 + 0.5);
            if (angle > 2 || angle < -24.33 || scanID > 50 || scanID < 0) { count--; continue; }
        }
        float ori = -std::atan2(py, px);                                              // :349
        if (!halfPassed) {
            if (ori < startOri - M_PI / 2) ori += 2 * M_PI;
            else if (ori > startOri + M_PI * 3 / 2) ori -= 2 * M_PI;
            if (ori - startOri > M_PI) halfPassed = true;
        } else {
            ori += 2 * M_PI;
            if (ori < endOri - M_PI * 3 / 2) ori += 2 * M_PI;
            else if (ori > endOri + M_PI / 2) ori -= 2 * M_PI;
        }
        float relTime = (ori - startOri) / (endOri - startOri);                       // :367
        float intensity = scanID + 0.1 * relTime;                                     // :368
        // undistortion, :153-177
        int line = int(intensity);
        double dt_i = intensity - line;
        double ratio_i = dt_i / 0.1;
        if (ratio_i >= 1.0) ratio_i = 1.0;
        Quat q_si = qslerp(Quat{1, 0, 0, 0}, ratio_i, qIMU);
        q_si = qmul(qmul(q_lb, q_si), q_lb_inv);                                      // :168
        V3 ps = qrot(q_si, V3{px, py, pz});
        orc_pt32 o;
        std::memset(&o, 0, sizeof(o));
        o.x = (float)ps.x; o.y = (float)ps.y; o.z = (float)ps.z; o.w = 1.0f;
        o.intensity = intensity;
        rings[scanID].push_back(o);                                                   // :371
    }
    cloudSize = count;

    std::vector<orc_pt32> cloud;
    cloud.reserve(cloudSize);
    std::vector<int> scanStartInd(N_SCANS, 0), scanEndInd(N_SCANS, 0);
    for (int i = 0; i < N_SCANS; i++) {                                               // :378-382
        scanStartInd[i] = (int)cloud.size() + 5;
        cloud.insert(cloud.end(), rings[i].begin(), rings[i].end());
        scanEndInd[i] = (int)cloud.size() - 6;
    }
    for (int i = 0; i < cloudSize; ++i) cutted[i] = cloud[i];
    *n_cut = cloudSize;

    std::vector<float> curv(cloudSize, 0.f);
    std::vector<int> sortInd(cloudSize, 0), picked(cloudSize, 0), label(cloudSize, 0);
    const orc_pt32* P = cloud.data();
    for (int i = 5; i < cloudSize - 5; i++) {                                         // :385-394
        float diffX = P[i - 5].x + P[i - 4].x + P[i - 3].x + P[i - 2].x + P[i - 1].x - 10 * P[i].x + P[i + 1].x + P[i + 2].x + P[i + 3].x + P[i + 4].x + P[i + 5].x;
        float diffY = P[i - 5].y + P[i - 4].y + P[i - 3].y + P[i - 2].y + P[i - 1].y - 10 * P[i].y + P[i + 1].y + P[i + 2].y + P[i + 3].y + P[i + 4].y + P[i + 5].y;
        float diffZ = P[i - 5].z + P[i - 4].z + P[i - 3].z + P[i - 2].z + P[i - 1].z - 10 * P[i].z + P[i + 1].z + P[i + 2].z + P[i + 3].z + P[i + 4].z + P[i + 5].z;
        curv[i] = diffX * diffX + diffY * diffY + diffZ * diffZ;
        sortInd[i] = i;
    }

    auto gap2 = [&](int a, int b) {   // :435-438 squared gap between consecutive points, fp32
        float dX = P[a].x - P[b].x, dY = P[a].y - P[b].y, dZ = P[a].z - P[b].z;
        return dX * dX + dY * dY + dZ * dZ;
    };
    auto range2 = [&](int k) { return P[k].x * P[k].x + P[k].y * P[k].y + P[k].z * P[k].z; };
    auto suppress = [&](int ind) {    // :434-451 / :473-490
        for (int l = 1; l <= 5; l++) {
            if (gap2(ind + l, ind + l - 1) > 0.05) break;
            picked[ind + l] = 1;
        }
        for (int l = -1; l >= -5; l--) {
            if (gap2(ind + l, ind + l + 1) > 0.05) break;
            picked[ind + l] = 1;
        }
    };

    int ns = 0, ne = 0;
    for (int i = 0; i < N_SCANS; i++) {                                               // :401
        if (scanEndInd[i] - scanStartInd[i] < 6 || i % ds_rate != 0) continue;
        std::vector<orc_pt32> lessFlatScan;
        for (int j = 0; j < 6; j++) {
            const int span = scanEndInd[i] - scanStartInd[i];
            int sp = scanStartInd[i] + span * j / 6;
            int ep = scanStartInd[i] + span * (j + 1) / 6 - 1;
            std::stable_sort(sortInd.begin() + sp, sortInd.begin() + ep + 1, [&](int a, int b) { return rot_curv_less(curv[a], curv[b]); });  // :410

            int largestPickedNum = 0;
            for (int k = ep; k >= sp; k--) {                                          // :413-453
                int ind = sortInd[k];
                if (picked[ind] == 0 && curv[ind] > 2.0) {
                    largestPickedNum++;
                    if (largestPickedNum <= 2) { label[ind] = 2; edge[ne++] = P[ind]; }
                    else if (largestPickedNum <= 10) { label[ind] = 1; edge[ne++] = P[ind]; }
                    else break;
                    picked[ind] = 1;
                    suppress(ind);
                }
            }
            int smallestPickedNum = 0;
            for (int k = sp; k <= ep; k++) {                                          // :456-492
                int ind = sortInd[k];
                if (range2(ind) < 0.25) continue;
                if (picked[ind] == 0 && curv[ind] < 0.1) {
                    label[ind] = -1;
                    smallestPickedNum++;
                    if (smallestPickedNum >= 4) break;
                    picked[ind] = 1;
                    suppress(ind);
                }
            }
            for (int k = sp; k <= ep; k++) {                                          // :494-499
                if (range2(k) < 0.25) continue;
                if (label[k] <= 0) lessFlatScan.push_back(P[k]);
            }
        }
        if (!lessFlatScan.empty()) {                                                  // :502-508
            std::vector<orc_pt32> ds(lessFlatScan.size());
            int m = orc_voxelgrid(lessFlatScan.data(), (int)lessFlatScan.size(), 32, 0.6f, ds.data(), (int)ds.size());
            for (int k = 0; k < m; ++k) surf[ns++] = ds[k];
        }
    }
    *n_surf = ns; *n_edge = ne;
    if (label_out) for (int i = 0; i < cloudSize; ++i) label_out[i] = label[i];
    if (curv_out) for (int i = 0; i < cloudSize; ++i) curv_out[i] = curv[i];
    return 0;
}
