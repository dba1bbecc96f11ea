// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.h).  Pinned to the reference's own code: DESIGN.md §6.
// Livox-Horizon feature extractor restated: the body of Preprocessing::cloudHandler between
// fromROSMsg and toROSMsg, LiLi-OM/src/Preprocessing.cpp:219-383, plus getDepth (:99-102),
// undistortion (:104-127) and removeClosedPointCloud (:72-97).  The gyro integration that
// produces q_iMU (:129-171) stays on the host side of the boundary and is an input here.
// Expression widths (fp32 vs fp64) are kept exactly as the reference's C++ resolves them
// (`using namespace std` => float overloads of sqrt/fabs, LiLi-OM/include/utils/common.h:48).
#include "oracle_api.h"
#include "oracle_math.h"
#include <vector>
#include <cstring>

using namespace orc;

namespace {
constexpr int N_SCANS = 6;      // Preprocessing.cpp:34
constexpr int H_SCANS = 4000;   // Preprocessing.cpp:35

struct Cell { float x, y, z, intensity, curvature, nx, ny, nz; };  // PointXYZINormal payload, zero = empty

static inline double get_depth(const Cell& c) {                 // :99-102 (fp32 inside, widened on return)
    return std::sqrt(c.x * c.x + c.y * c.y + c.z * c.z);
}

static inline orc_pt48 to_pt(const Cell& c) {
    orc_pt48 p;
    std::memset(&p, 0, sizeof(p));
    p.x = c.x; p.y = c.y; p.z = c.z; p.w = 1.0f;
    p.nx = c.nx; p.ny = c.ny; p.nz = c.nz;
    p.intensity = c.intensity; p.curvature = c.curvature;
    return p;
}
}  // namespace

extern "C" int orc_extract_horizon(const orc_pt48* pts, int n, const double q_imu_in[4], double surf_thres, double edge_thres,
                                   orc_pt48* surf, int* n_surf, orc_pt48* edge, int* n_edge, orc_pt48* cutted, int* n_cut) {
    Quat q_imu{q_imu_in[0], q_imu_in[1], q_imu_in[2], q_imu_in[3]};
    if (std::isnan(q_imu.w) || std::isnan(q_imu.x) || std::isnan(q_imu.y) || std::isnan(q_imu.z)) q_imu = Quat{1, 0, 0, 0};  // :232-234
    std::vector<Cell> mat((size_t)N_SCANS * H_SCANS);
    std::memset(mat.data(), 0, mat.size() * sizeof(Cell));
    auto M = [&](int k, int c) -> Cell& { return mat[(size_t)k * H_SCANS + c]; };
    const double t_interval = 0.1 / (H_SCANS - 1);                 // :239
    const float thres = 0.1f;                                      // :226
    int ncut = 0, ns = 0, ne = 0;

    for (int i = 0; i < n; ++i) {
        const orc_pt48& in = pts[i];
        if (!std::isfinite(in.x) || !std::isfinite(in.y) || !std::isfinite(in.z)) continue;     // :225 removeNaN
        if (in.x * in.x + in.y * in.y + in.z * in.z < thres * thres) continue;                  // :83-86
        Cell point;
        std::memset(&point, 0, sizeof(point));
        point.x = in.x; point.y = in.y; point.z = in.z;
        point.intensity = in.intensity; point.curvature = in.curvature;
        int scan_id = scan_id_of(point.intensity);                   // :250-252
        if (scan_id < 0) continue;                                   // :253
        // undistortion, :104-127
        int line = scan_id_of(point.intensity);
        double dt_i = point.intensity - line;
        double ratio_i = dt_i / 0.1;
        if (ratio_i >= 1.0) ratio_i = 1.0;
        Quat q_si = qslerp(Quat{1, 0, 0, 0}, ratio_i, q_imu);
        V3 ps = qrot(q_si, V3{point.x, point.y, point.z});
        Cell u;
        std::memset(&u, 0, sizeof(u));
        u.x = (float)ps.x; u.y = (float)ps.y; u.z = (float)ps.z;
        u.intensity = point.intensity; u.curvature = point.curvature;
        cutted[ncut++] = to_pt(u);                                   // :257

        double dep = u.x * u.x + u.y * u.y + u.z * u.z;              // :259 (fp32 sum, widened)
        if (dep > 40000.0 || dep < 4.0 || u.curvature < 0.05 || u.curvature > 25.45) continue;   // :260
        int col = int(std::round((u.intensity - scan_id) / t_interval));                         // :262
        if (col >= H_SCANS || col < 0) continue;                     // :263
        if (scan_id >= N_SCANS) continue;   // reference indexes mat[scan_id] out of bounds here (UB); guarded
        if (M(scan_id, col).curvature != 0) continue;                // :265 first writer wins
        M(scan_id, col) = u;                                         // :267
    }

    for (int i = 5; i < H_SCANS - 12; i = i + 6) {                   // :270
        double cx = 0, cy = 0, cz = 0;
        double npx[36], npy[36], npz[36];
        int cntp = 0;
        int num = 36;
        for (int j = 0; j < 6; j++) {
            for (int k = 0; k < N_SCANS; k++) {
                const Cell& c = M(k, i + j);
                if (c.curvature <= 0) { num--; continue; }           // :276-279
                cx += c.x; cy += c.y; cz += c.z;
                npx[cntp] = c.x; npy[cntp] = c.y; npz[cntp] = c.z; ++cntp;
            }
        }
        if (num < 25) continue;                                       // :287
        cx /= num; cy /= num; cz /= num;                              // :289
        double A[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
        for (int j = 0; j < cntp; ++j) {                              // :292-296
            double z0 = npx[j] - cx, z1 = npy[j] - cy, z2 = npz[j] - cz;
            const double zm[3] = {z0, z1, z2};
            for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) A[a][b] += zm[a] * zm[b];
        }
        double ev[3], evec[3][3];
        eigen_sym3(A, ev, evec);                                      // :298

        int idsx[N_SCANS], idsy[N_SCANS], nedge = 0;
        for (int k = 0; k < N_SCANS; k++) {                           // :302-331
            double max_s = 0;
            int idx = i;
            for (int j = 0; j < 6; j++) {
                if (M(k, i + j).curvature <= 0) continue;
                double g1 = get_depth(M(k, i + j - 4)) + get_depth(M(k, i + j - 3)) +
                            get_depth(M(k, i + j - 2)) + get_depth(M(k, i + j - 1)) - 8 * get_depth(M(k, i + j)) +
                            get_depth(M(k, i + j + 1)) + get_depth(M(k, i + j + 2)) + get_depth(M(k, i + j + 3)) +
                            get_depth(M(k, i + j + 4));
                g1 = g1 / (8 * get_depth(M(k, i + j)) + 1e-3);
                if (g1 > 0.06) {
                    if (g1 > max_s) { max_s = g1; idx = i + j; }
                }
            }
            if (max_s != 0) { idsx[nedge] = k; idsy[nedge] = idx; ++nedge; }
        }

        if (nedge > 0) {                                              // :333-365 (size 0: NaN centre, no edge)
            double ex = 0, ey = 0, ez = 0;
            for (int j = 0; j < nedge; ++j) { const Cell& c = M(idsx[j], idsy[j]); ex += c.x; ey += c.y; ez += c.z; }
            ex /= nedge; ey /= nedge; ez /= nedge;
            double E[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
            for (int j = 0; j < nedge; ++j) {
                const Cell& c = M(idsx[j], idsy[j]);
                const double zm[3] = {c.x - ex, c.y - ey, c.z - ez};
                for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) E[a][b] += zm[a] * zm[b];
            }
            double eev[3], eevec[3][3];
            eigen_sym3(E, eev, eevec);                                // :351
            if (eev[2] > edge_thres * eev[1] && nedge > 3) {          // :353
                for (int j = 0; j < nedge; ++j) {
                    Cell& c = M(idsx[j], idsy[j]);
                    if (c.curvature <= 0 && c.intensity <= 0) continue;   // :356
                    c.nx = (float)eevec[0][2]; c.ny = (float)eevec[1][2]; c.nz = (float)eevec[2][2];
                    edge[ne++] = to_pt(c);                            // :362
                    c.curvature *= -1;                                // :363
                }
            }
        }

        if (ev[0] < surf_thres * ev[1]) {                             // :367
            for (int j = 0; j < 6; j++) {
                for (int k = 0; k < N_SCANS; k++) {
                    Cell& c = M(k, i + j);
                    if (c.curvature <= 0) continue;                   // :371
                    c.nx = (float)evec[0][0]; c.ny = (float)evec[1][0]; c.nz = (float)evec[2][0];
                    surf[ns++] = to_pt(c);                            // :378
                    c.curvature *= -1;                                // :379
                }
            }
        }
    }
    *n_surf = ns; *n_edge = ne; *n_cut = ncut;
    return 0;
}
