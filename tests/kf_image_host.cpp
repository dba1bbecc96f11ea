// TEST INFRASTRUCTURE: host build of liliom_b200/csrc/kf_image.h (the keyframe image's header, checksums and checks), so that the
// CPU test tier checks the SAME SOURCE liliom_kf_export and liliom_kf_import use.  The points checksum, which the library checks
// on the device, is summed here with the header's kfi_sum.
#include "../liliom_b200/csrc/kf_image.h"
#include <vector>

using namespace lili;

extern "C" unsigned long long kih_term(unsigned long long w, unsigned long long j) { return kfi_term(w, j); }
extern "C" unsigned long long kih_sum(const unsigned char* p, long long words, unsigned long long j0) { return kfi_sum(p, words, j0); }
extern "C" const char* kih_check_name(int e) { return kfi_check_name(e); }
extern "C" long long kih_size(int stride, long long k, long long n_scan, long long n_full) { return kfi_size(stride, k, n_scan, n_full); }

// Every host check of the library (kfi_check); *k_out = the header's k when it passes
extern "C" int kih_check(const unsigned char* img, long long bytes, int stride, int* k_out) {
    KfiHeader h;
    const int e = kfi_check(img, bytes, stride, &h);
    if (e == kKfiOk && k_out) *k_out = h.k;
    return e;
}

// ... and then the points checksum, as the device sums it (the words of A and F, j from the start of A)
extern "C" int kih_check_all(const unsigned char* img, long long bytes, int stride) {
    KfiHeader h;
    const int e = kfi_check(img, bytes, stride, &h);
    if (e != kKfiOk) return e;
    const long long a0 = kKfiHeader + kKfiRecord * (long long)h.k;
    return kfi_sum(img + a0, (bytes - a0) / 8, 0) == h.points_sum ? kKfiOk : kKfiBadPointsSum;
}

// The image liliom_kf_export writes for k keyframes of counts[3i..3i+2] (n_edge, n_surf, n_full) whose section A and F bytes are
// a and f: the header (kfi_header), the table, the points, both checksums.  out: kfi_size bytes.
extern "C" void kih_encode(int stride, int k, unsigned flags, const int* counts, const unsigned char* a, long long a_bytes,
                           const unsigned char* f, long long f_bytes, unsigned char* out) {
    std::vector<KfiRecord> tab(k);
    long long ns = 0, nf = 0;
    for (int i = 0; i < k; ++i) {
        tab[i] = KfiRecord{counts[3 * i], counts[3 * i + 1], counts[3 * i + 2], 0};
        ns += (long long)counts[3 * i] + counts[3 * i + 1];
        nf += counts[3 * i + 2] > 0 ? counts[3 * i + 2] : 0;
    }
    KfiHeader h = kfi_header(stride, k, flags, ns, nf);
    unsigned char* pts = out + kKfiHeader + kKfiRecord * (long long)k;
    memcpy(pts, a, (size_t)a_bytes);
    memcpy(pts + a_bytes, f, (size_t)f_bytes);
    h.points_sum = kfi_sum(pts, (a_bytes + f_bytes) / 8, 0);
    kfi_write_head(out, h, tab.data(), k);
}
