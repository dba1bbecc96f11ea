// TEST INFRASTRUCTURE: host build of the `ring` field rules of liliom_b200/csrc/pc2_fields.h (LILIOM_RING_FIELD): the match
// liliom_convert_pc2 / liliom_extract_rot_pc2 run, and the per-point read k_pc2_to_pt32 shares with the host (pc2_ring_value).
#include "../liliom_b200/csrc/pc2_fields.h"

// out = {src x, src y, src z, src intensity, n, ring_src, ring_bytes}; untouched unless the message is accepted
extern "C" int prh_match(const liliom_pc2_msg* msg, int want_ring, int out[7]) {
    lili::Pc2Map m;
    const int rc = lili::pc2_match(msg, &m, want_ring != 0);
    if (rc == LILIOM_OK) {
        for (int k = 0; k < 4; ++k) out[k] = m.src[k];
        out[4] = m.n;
        out[5] = m.ring_src;
        out[6] = m.ring_bytes;
    }
    return rc;
}

// the ring id of every point, row-major over (row, column) as the device decode writes it; -1: message refused
extern "C" int prh_decode_rings(const liliom_pc2_msg* msg, unsigned short* out) {
    lili::Pc2Map m;
    if (lili::pc2_match(msg, &m, true) != LILIOM_OK) return -1;
    const unsigned char* data = static_cast<const unsigned char*>(msg->data);
    for (unsigned r = 0; r < msg->height; ++r)
        for (unsigned c = 0; c < msg->width; ++c)
            out[(size_t)r * msg->width + c] =
                (unsigned short)lili::pc2_ring_value(data + (size_t)r * msg->row_step + (size_t)c * msg->point_step, m.ring_src, m.ring_bytes);
    return m.n;
}
