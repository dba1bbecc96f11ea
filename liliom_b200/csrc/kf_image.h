// The keyframe image (liliom_kf_export / liliom_kf_import): a keyframe store's clouds as one checked byte image, shared by host
// and device (keyframes.cu; tests/kf_image_host.cpp compiles this same file for the CPU test tier).
//
// Layout, little-endian, byte offsets 64-bit:
//   header   64 bytes: magic "LILIKF01", u32 version (1), u32 point_stride, i32 k, u32 flags, u64 edge+surf points, u64 full
//            points, u64 table checksum, u64 points checksum, u64 reserved (0)
//   table    k records of 16 bytes: i32 n_edge, i32 n_surf, i32 n_full (-1: no full cloud), i32 reserved (0)
//   A        every keyframe's edge points, then its surf points, in table order, point_stride bytes each
//   F        the full clouds, in table order
//   size  =  64 + 16 k + point_stride * (sum E + sum S + sum F)
// Checksum: h = sum_j mix(w_j ^ j * 0x9E3779B97F4A7C15) mod 2^64 over little-endian u64 words w_j, mix = splitmix64's
// finaliser.  The sum is order-independent and keyed by position, so a parallel reduction gives the same bits as a serial loop,
// and truncation, flipped bits and swapped words all change it.  Points checksum: the words of A then F, j from the start of A.
// Table checksum: the words of the header (both checksum fields zero) then the table, j from the start of the header.
// The point strides (48, 32) are multiples of 16 bytes, so A and F are whole 16-byte vectors.
#pragma once
#include "vg_box.h"          // VGB_HD
#include <cstdint>
#include <cstring>

namespace lili {

constexpr uint64_t kKfiMagic = 0x3130464B494C494CULL;   // "LILIKF01" as a little-endian u64
constexpr uint32_t kKfiVersion = 1;
constexpr uint32_t kKfiFlagFull = 1;                     // LILIOM_KF_IMAGE_FULL
constexpr long long kKfiHeader = 64, kKfiRecord = 16;
constexpr uint64_t kKfiGolden = 0x9E3779B97F4A7C15ULL;

struct KfiHeader {
    uint64_t magic;
    uint32_t version, point_stride;
    int32_t k;
    uint32_t flags;
    uint64_t n_scan, n_full;             // edge + surf points (section A), full points (section F)
    uint64_t table_sum, points_sum;
    uint64_t reserved;
};
struct KfiRecord { int32_t n_edge, n_surf, n_full, reserved; };
static_assert(sizeof(KfiHeader) == kKfiHeader && sizeof(KfiRecord) == kKfiRecord, "the image's header and record sizes");

// one word's term of the checksum: splitmix64's finaliser of w ^ j * golden
VGB_HD uint64_t kfi_term(uint64_t w, uint64_t j) {
    uint64_t z = w ^ (j * kKfiGolden);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}

// the checksum terms of n words at p, the first one at position j0
inline uint64_t kfi_sum(const unsigned char* p, long long n, uint64_t j0) {
    uint64_t h = 0;
    for (long long i = 0; i < n; ++i) {
        uint64_t w;
        memcpy(&w, p + 8 * i, 8);
        h += kfi_term(w, j0 + (uint64_t)i);
    }
    return h;
}

// The image's size from its counts
inline long long kfi_size(int stride, long long k, long long n_scan, long long n_full) {
    return kKfiHeader + kKfiRecord * k + (long long)stride * (n_scan + n_full);
}

// The table checksum of a header and its k records (the header's checksum fields taken as zero)
inline uint64_t kfi_table_sum(const KfiHeader& h, const unsigned char* tab, long long k) {
    KfiHeader z = h;
    z.table_sum = 0; z.points_sum = 0;
    return kfi_sum((const unsigned char*)&z, kKfiHeader / 8, 0) + kfi_sum(tab, k * kKfiRecord / 8, kKfiHeader / 8);
}

// The header of an image of k keyframes holding n_scan edge + surf and n_full full points, its checksums still zero
inline KfiHeader kfi_header(int stride, int k, uint32_t flags, long long n_scan, long long n_full) {
    KfiHeader h{};
    h.magic = kKfiMagic; h.version = kKfiVersion; h.point_stride = (uint32_t)stride; h.k = k; h.flags = flags;
    h.n_scan = (uint64_t)n_scan; h.n_full = (uint64_t)n_full;
    return h;
}

// Writes the table and then the header, with its table checksum, at the front of an image (h.points_sum already set)
inline void kfi_write_head(unsigned char* out, KfiHeader h, const KfiRecord* tab, int k) {
    memcpy(out + kKfiHeader, tab, (size_t)k * kKfiRecord);
    h.table_sum = kfi_table_sum(h, out + kKfiHeader, k);
    memcpy(out, &h, sizeof(h));
}

// The checks of an image, in the order they are made; the points checksum needs the points (the library checks it on the device)
enum KfiCheck { kKfiOk = 0, kKfiBadMagic, kKfiBadVersion, kKfiBadStride, kKfiBadFlags, kKfiBadCounts, kKfiBadTotals, kKfiBadLength,
                kKfiBadTableSum, kKfiBadPointsSum };

inline const char* kfi_check_name(int e) {
    switch (e) {
        case kKfiOk: return "ok";
        case kKfiBadMagic: return "bad magic: not a keyframe image";
        case kKfiBadVersion: return "unknown version";
        case kKfiBadStride: return "point_stride differs from the context's";
        case kKfiBadFlags: return "unknown flags";
        case kKfiBadCounts: return "bad counts: a count below its minimum or a reserved word not zero in the table";
        case kKfiBadTotals: return "totals disagree with the table";
        case kKfiBadLength: return "length differs from the header";
        case kKfiBadTableSum: return "table checksum mismatch";
        case kKfiBadPointsSum: return "points checksum mismatch";
    }
    return "?";
}

// Every check but the points checksum, in order, on an image of `bytes` bytes for a context of point_stride `stride`.  An image
// too short to hold its header, or its table, fails the length check at the first check that would read past its end.  On
// success *h is the header and the table starts at img + kKfiHeader.
inline int kfi_check(const unsigned char* img, long long bytes, int stride, KfiHeader* h) {
    if (bytes < kKfiHeader) return kKfiBadLength;
    memcpy(h, img, sizeof(KfiHeader));
    if (h->magic != kKfiMagic) return kKfiBadMagic;
    if (h->version != kKfiVersion || h->reserved != 0) return kKfiBadVersion;
    if (h->point_stride != (uint32_t)stride) return kKfiBadStride;
    if (h->flags & ~kKfiFlagFull) return kKfiBadFlags;
    if (h->k < 0) return kKfiBadCounts;
    if (bytes - kKfiHeader < kKfiRecord * (long long)h->k) return kKfiBadLength;
    const bool full = h->flags & kKfiFlagFull;
    long long ns = 0, nf = 0;
    for (int i = 0; i < h->k; ++i) {
        KfiRecord r;
        memcpy(&r, img + kKfiHeader + kKfiRecord * i, sizeof(r));
        // without the full flag every keyframe has no full cloud (-1); with it, -1 or a count
        if (r.n_edge < 0 || r.n_surf < 0 || r.n_full < -1 || (!full && r.n_full != -1) || r.reserved != 0) return kKfiBadCounts;
        ns += (long long)r.n_edge + r.n_surf;
        nf += r.n_full > 0 ? r.n_full : 0;
    }
    if ((uint64_t)ns != h->n_scan || (uint64_t)nf != h->n_full) return kKfiBadTotals;
    const long long rest = bytes - kKfiHeader - kKfiRecord * (long long)h->k;   // >= 0 (the table fits)
    if (rest % stride != 0 || rest / stride != ns + nf) return kKfiBadLength;
    if (kfi_table_sum(*h, img + kKfiHeader, h->k) != h->table_sum) return kKfiBadTableSum;
    return kKfiOk;
}

}  // namespace lili
