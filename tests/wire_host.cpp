// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/wire_decode.h, the per-point decode of the Livox CustomPoint records and
// of PointCloud2 messages that the decode stages of the convert calls (WireStLivox, WireStPc2 in api.cu) run, so that the
// CPU test tier checks the SAME SOURCE they run.
#include "../liliom_b200/csrc/wire_decode.h"

// n records of `stride` bytes -> n PointXYZINormal (48 bytes each) at out
extern "C" void wh_livox(const unsigned char* in, int n, int stride, unsigned char* out) {
    for (int i = 0; i < n; ++i) lili::livox_point_at(in, n, stride, out, i);
}

// msg matched as liliom_convert_pc2 matches it under the sources want_ring / time_name (nullptr: no time field), then every
// point decoded into out (32 bytes each) and, when the source is asked for, rings (u16) and times (double).  Returns the point
// count, or -1 when the message is refused.
extern "C" int wh_pc2(const liliom_pc2_msg* msg, int want_ring, const char* time_name, unsigned char* out, uint16_t* rings,
                      double* times) {
    lili::Pc2Map m;
    if (lili::pc2_match(msg, &m, want_ring != 0, time_name) != LILIOM_OK) return -1;
    const lili::Pc2Wire w = lili::pc2_wire(msg, m);
    const unsigned char* data = static_cast<const unsigned char*>(msg->data);
    for (int i = 0; i < m.n; ++i)
        lili::pc2_point_at(data, m.n, w, out, m.ring_src >= 0 ? rings : nullptr, m.time_src >= 0 ? times : nullptr, i);
    return m.n;
}
