// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/pc2_fields.h, the PointCloud2 field matching and validation of
// liliom_convert_pc2 / liliom_extract_rot_pc2 / liliom_pre_cloud_pc2, so that the CPU test tier checks the SAME SOURCE they use.
#include "../liliom_b200/csrc/pc2_fields.h"

// out = {src x, src y, src z, src intensity, n}; untouched unless the message is accepted
extern "C" int ph_match(const liliom_pc2_msg* msg, int out[5]) {
    lili::Pc2Map m;
    const int rc = lili::pc2_match(msg, &m);
    if (rc == LILIOM_OK) {
        for (int k = 0; k < 4; ++k) out[k] = m.src[k];
        out[4] = m.n;
    }
    return rc;
}
