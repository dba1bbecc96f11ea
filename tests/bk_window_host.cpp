// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/bk_window.h (the window's query -> keyframe lookup and the variant
// weights), so that the CPU test tier checks the SAME SOURCE the backend kernels use.
#include "../liliom_b200/csrc/bk_window.h"

extern "C" int bw_find(const long long* start, int k, long long qi) { return lili::bkw_find(start, k, qi); }
extern "C" double bw_edge_weight(int variant, double lidar_const, int n) { return lili::bkw_edge_weight(variant, lidar_const, n); }
extern "C" double bw_surf_score(int variant, double score, int n) { return lili::bkw_surf_score(variant, score, n); }
