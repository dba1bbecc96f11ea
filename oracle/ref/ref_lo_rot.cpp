// Harness of the reference's LiLi-OM-ROT/src/LidarOdometry.cpp (PointXYZI): the same API as ref_lo.cpp, built against the
// ROT tree's sources and headers.
#include "ref_lo.cpp"
