// TEST INFRASTRUCTURE: host build of the time field rules of liliom_b200/csrc/pc2_fields.h (LILIOM_TIME_FIELD): the match
// liliom_convert_pc2 / liliom_extract_rot_pc2 run, the per-point read k_pc2_to_pt32 shares with the host (pc2_time_value) and the
// relTime expression k_rot_build uses (pc2_rel_time).
#include "../liliom_b200/csrc/pc2_fields.h"

// out = {src x, src y, src z, src intensity, n, ring_src, ring_bytes, time_src, time_type}; untouched unless the message is
// accepted.  time_name == nullptr: no time field is asked for.
extern "C" int pth_match(const liliom_pc2_msg* msg, int want_ring, const char* time_name, int out[9]) {
    lili::Pc2Map m;
    const int rc = lili::pc2_match(msg, &m, want_ring != 0, time_name);
    if (rc == LILIOM_OK) {
        for (int k = 0; k < 4; ++k) out[k] = m.src[k];
        out[4] = m.n;
        out[5] = m.ring_src;
        out[6] = m.ring_bytes;
        out[7] = m.time_src;
        out[8] = m.time_type;
    }
    return rc;
}

// the time of every point, row-major over (row, column) as the device decode writes it; -1: message refused
extern "C" int pth_decode_times(const liliom_pc2_msg* msg, const char* time_name, double* out) {
    lili::Pc2Map m;
    if (lili::pc2_match(msg, &m, false, time_name) != LILIOM_OK || m.time_src < 0) return -1;
    const unsigned char* data = static_cast<const unsigned char*>(msg->data);
    for (unsigned r = 0; r < msg->height; ++r)
        for (unsigned c = 0; c < msg->width; ++c)
            out[(size_t)r * msg->width + c] =
                lili::pc2_time_value(data + (size_t)r * msg->row_step + (size_t)c * msg->point_step, m.time_src, m.time_type);
    return m.n;
}

extern "C" void pth_rel_times(const double* t, int n, double t_min, double t_max, float* out) {
    for (int i = 0; i < n; ++i) out[i] = lili::pc2_rel_time(t[i], t_min, t_max);
}
