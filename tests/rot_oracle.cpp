// TEST INFRASTRUCTURE: the CPU oracle of the ROT extractor's side channels, the ring taken from the driver's `ring` field
// (LILIOM_RING_FIELD) and relTime from its per-point time field (LILIOM_TIME_FIELD).  The body of Preprocessing::cloudHandler
// (R/src/Preprocessing.cpp:276-509) as oracle/oracle_rot.cpp restates it, behind one function that takes an optional per-point
// ring array and an optional per-point time array:
//   rings == nullptr   scanID from the elevation tables (:315-347, N_SCANS 16 / 32 / 64); else scanID = rings[i], kept iff
//                      0 <= ring < N_SCANS (LILIOM_RING_FIELD, N_SCANS 1..128)
//   times == nullptr   relTime from the azimuth rule (:285-294, 349-367); else a point with a non-finite time is removed with
//                      the NaN points, and relTime = (t_i - t_min) / (t_max - t_min) in double over the surviving points (0 for
//                      a span of 0) — the only substitution.
// It lives beside the tests so that the oracle library stays as it is; tests/test_rot_rings_cpu.py and tests/test_rot_time_cpu.py
// pin its untimed modes to orc_extract_rot byte for byte.
//   orc_extract_rot_timed   the extractor with optional rings and optional times
//   orc_rot_scan_ids        the tables' per-point verdict: scanID, or -1 for a dropped point (removed or a table miss)
#include "oracle_api.h"
#include "oracle_math.h"
#include <vector>
#include <cstring>

using namespace orc;

namespace {

bool rot_removed(const orc_pt32& p) {   // :280-281 removeNaN + removeClosedPointCloud(3.0)
    const float thres = 3.0f;
    if (!std::isfinite(p.x) || !std::isfinite(p.y) || !std::isfinite(p.z)) return true;
    return p.x * p.x + p.y * p.y + p.z * p.z < thres * thres;
}

int table_scan_id(const orc_pt32& p, int N_SCANS) {   // :315-347, -1 for `count--; continue`
    float px = p.x, py = p.y, pz = p.z;
    float angle = std::atan(pz / std::sqrt(px * px + py * py)) * 180 / M_PI;
    int scanID = 0;
    if (N_SCANS == 16) {
        scanID = int((angle + 15) / 2 + 0.5);
        if (scanID > (N_SCANS - 1) || scanID < 0) return -1;
    } else if (N_SCANS == 32) {
        scanID = int((angle + 92.0 / 3.0) * 3.0 / 4.0);
        if (scanID > (N_SCANS - 1) || scanID < 0) return -1;
    } else {
        if (angle >= -8.83) scanID = int((2 - angle) * 3.0 + 0.5);
        else scanID = N_SCANS / 2 + int((-8.83 - angle) * 2.0 + 0.5);
        if (angle > 2 || angle < -24.33 || scanID > 50 || scanID < 0) return -1;
    }
    return scanID;
}

int extract_rot(const orc_pt32* pts, const int* rings, const double* times, int n, const double q_imu_in[4], const double q_lb_in[4],
                int N_SCANS, int ds_rate, orc_pt32* surf, int* n_surf, orc_pt32* edge, int* n_edge, orc_pt32* cutted, int* n_cut,
                int* label_out, float* curv_out) {
    *n_surf = *n_edge = *n_cut = 0;
    Quat qIMU{q_imu_in[0], q_imu_in[1], q_imu_in[2], q_imu_in[3]};
    if (std::isnan(qIMU.w) || std::isnan(qIMU.x) || std::isnan(qIMU.y) || std::isnan(qIMU.z)) qIMU = Quat{1, 0, 0, 0};  // :299-301
    Quat q_lb{q_lb_in[0], q_lb_in[1], q_lb_in[2], q_lb_in[3]};
    Quat q_lb_inv = qinv(q_lb);

    std::vector<orc_pt32> in;
    std::vector<int> in_ring;
    std::vector<double> in_time;
    in.reserve(n);
    for (int i = 0; i < n; ++i) {
        if (rot_removed(pts[i])) continue;
        if (times && !std::isfinite(times[i])) continue;                              // LILIOM_TIME_FIELD: with the NaN points
        in.push_back(pts[i]);
        in_ring.push_back(rings ? rings[i] : 0);
        in_time.push_back(times ? times[i] : 0.0);
    }
    int cloudSize = (int)in.size();
    if (cloudSize == 0) return 0;
    double t_min = 0.0, t_max = 0.0;                                                  // LILIOM_TIME_FIELD: the span
    if (times) {
        t_min = t_max = in_time[0];
        for (double t : in_time) { if (t < t_min) t_min = t; if (t > t_max) t_max = t; }
    }

    float startOri = -std::atan2(in[0].y, in[0].x);                                   // :285
    float endOri = -std::atan2(in[cloudSize - 1].y, in[cloudSize - 1].x) + 2 * M_PI;  // :286-288
    if (endOri - startOri > 3 * M_PI) endOri -= 2 * M_PI;                             // :290-294
    else if (endOri - startOri < M_PI) endOri += 2 * M_PI;

    bool halfPassed = false;
    int count = cloudSize;
    std::vector<std::vector<orc_pt32>> ringv(N_SCANS);
    for (int i = 0; i < cloudSize; i++) {                                             // :308
        float px = in[i].x, py = in[i].y, pz = in[i].z;
        int scanID;
        if (rings) {                                                                  // LILIOM_RING_FIELD: the substitution
            scanID = in_ring[i];
            if (scanID > (N_SCANS - 1) || scanID < 0) { count--; continue; }
        } else {
            scanID = table_scan_id(in[i], N_SCANS);
            if (scanID < 0) { count--; continue; }
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
        if (times) relTime = t_max == t_min ? 0.0f : (float)((in_time[i] - t_min) / (t_max - t_min));   // the substitution
        float intensity = scanID + 0.1 * relTime;                                     // :368
        int line = int(intensity);                                                    // undistortion, :153-177
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
        ringv[scanID].push_back(o);                                                   // :371
    }
    cloudSize = count;

    std::vector<orc_pt32> cloud;
    cloud.reserve(cloudSize);
    std::vector<int> scanStartInd(N_SCANS, 0), scanEndInd(N_SCANS, 0);
    for (int i = 0; i < N_SCANS; i++) {                                               // :378-382
        scanStartInd[i] = (int)cloud.size() + 5;
        cloud.insert(cloud.end(), ringv[i].begin(), ringv[i].end());
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

    auto gap2 = [&](int a, int b) {   // :435-438
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

}  // namespace

// rings == nullptr: the elevation tables (line_num 16 / 32 / 64), else scanID = rings[i] (1..128); times == nullptr: the azimuth
// rule, else relTime from the times
extern "C" int orc_extract_rot_timed(const orc_pt32* pts, const int* rings, const double* times, int n, const double q_imu[4],
                                     const double q_lb[4], int line_num, int ds_rate, orc_pt32* surf, int* n_surf, orc_pt32* edge,
                                     int* n_edge, orc_pt32* cutted, int* n_cut, int* label_out, float* curv_out) {
    *n_surf = *n_edge = *n_cut = 0;
    if (rings ? (line_num < 1 || line_num > 128) : (line_num != 16 && line_num != 32 && line_num != 64)) return -2;
    return extract_rot(pts, rings, times, n, q_imu, q_lb, line_num, ds_rate, surf, n_surf, edge, n_edge, cutted, n_cut, label_out, curv_out);
}

extern "C" int orc_rot_scan_ids(const orc_pt32* pts, int n, int line_num, int* ids) {
    if (line_num != 16 && line_num != 32 && line_num != 64) return -2;
    for (int i = 0; i < n; ++i) ids[i] = rot_removed(pts[i]) ? -1 : table_scan_id(pts[i], line_num);
    return 0;
}
