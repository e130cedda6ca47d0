// xxhash64_device.cuh — the hashes and bit positions of Paimon's bloom-filter file index, for the device kernel
// (file_index.cu) and a host build of the same source (tests/native/file_index_host_check.cc):
//   FastHash (paimon-common/.../fileindex/bloomfilter/FastHash.java): Thomas Wang's 64-bit integer hash of integers,
//     DATE / TIME / TIMESTAMP and of the IEEE bits of FLOAT / DOUBLE (NaN folded to the canonical NaN), XXH64 with seed
//     0 of the bytes of CHAR / VARCHAR / BINARY / VARBINARY;
//   BloomFilter64 (paimon-common/.../utils/BloomFilter64.java): the sizing from items / fpp and the k bit positions of
//     one hash.
// XXH64 follows the published specification (https://github.com/Cyan4973/xxHash/blob/dev/doc/xxhash_spec.md); its
// input is read one byte at a time, so any alignment is fine.
#pragma once

#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define FI_HD __host__ __device__ __forceinline__
#else
#define FI_HD inline
#endif

namespace fi {

constexpr uint64_t kP1 = 0x9E3779B185EBCA87ull, kP2 = 0xC2B2AE3D27D4EB4Full, kP3 = 0x165667B19E3779F9ull,
                   kP4 = 0x85EBCA77C2B2AE63ull, kP5 = 0x27D4EB2F165667C5ull;

FI_HD uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

FI_HD uint64_t load_le(const uint8_t *p, int n) {         // n little-endian bytes
    uint64_t v = 0;
    for (int i = n - 1; i >= 0; i--) v = (v << 8) | p[i];
    return v;
}

FI_HD uint64_t xxh_round(uint64_t acc, uint64_t lane) { return rotl64(acc + lane * kP2, 31) * kP1; }
FI_HD uint64_t xxh_merge(uint64_t acc, uint64_t v) { return (acc ^ xxh_round(0, v)) * kP1 + kP4; }

// XXH64(p[0..n), seed 0): LongHashFunction.xx().hashBytes
FI_HD uint64_t xxh64(const uint8_t *p, int64_t n) {
    const uint8_t *const end = p + n;
    uint64_t h;
    if (n >= 32) {
        uint64_t v1 = kP1 + kP2, v2 = kP2, v3 = 0, v4 = 0ull - kP1;
        for (; end - p >= 32; p += 32) {
            v1 = xxh_round(v1, load_le(p, 8));
            v2 = xxh_round(v2, load_le(p + 8, 8));
            v3 = xxh_round(v3, load_le(p + 16, 8));
            v4 = xxh_round(v4, load_le(p + 24, 8));
        }
        h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = xxh_merge(h, v1);
        h = xxh_merge(h, v2);
        h = xxh_merge(h, v3);
        h = xxh_merge(h, v4);
    } else {
        h = kP5;
    }
    h += (uint64_t)n;
    for (; end - p >= 8; p += 8) h = rotl64(h ^ xxh_round(0, load_le(p, 8)), 27) * kP1 + kP4;
    if (end - p >= 4) {
        h = rotl64(h ^ (load_le(p, 4) * kP1), 23) * kP2 + kP3;
        p += 4;
    }
    for (; p < end; p++) h = rotl64(h ^ (*p * kP5), 11) * kP1;
    h ^= h >> 33;
    h *= kP2;
    h ^= h >> 29;
    h *= kP3;
    h ^= h >> 32;
    return h;
}

// Thomas Wang's 64-bit integer hash with Java's arithmetic >> (FastHash.getLongHash)
FI_HD int64_t wang64(int64_t key) {
    uint64_t k = (uint64_t)key;
    k = ~k + (k << 21);
    k ^= (uint64_t)((int64_t)k >> 24);
    k = k + (k << 3) + (k << 8);
    k ^= (uint64_t)((int64_t)k >> 14);
    k = k + (k << 2) + (k << 4);
    k ^= (uint64_t)((int64_t)k >> 28);
    k = k + (k << 31);
    return (int64_t)k;
}

// Float.floatToIntBits / Double.doubleToLongBits: every NaN is the canonical one
FI_HD int64_t float_key(uint32_t bits) {
    if ((bits & 0x7f800000u) == 0x7f800000u && (bits & 0x007fffffu)) bits = 0x7fc00000u;
    return (int64_t)(int32_t)bits;
}
FI_HD int64_t double_key(uint64_t bits) {
    if ((bits & 0x7ff0000000000000ull) == 0x7ff0000000000000ull && (bits & 0x000fffffffffffffull))
        bits = 0x7ff8000000000000ull;
    return (int64_t)bits;
}

// bit position i (1..k) of a hash in a filter of num_bits bits (BloomFilter64.addHash): h1 + i * h2 in wrapping 32-bit
// arithmetic, its bits flipped when negative, modulo num_bits
FI_HD uint32_t bloom_bit(int64_t hash, int i, uint32_t num_bits) {
    const uint32_t h1 = (uint32_t)(uint64_t)hash, h2 = (uint32_t)((uint64_t)hash >> 32);
    uint32_t c = h1 + (uint32_t)i * h2;
    if (c & 0x80000000u) c = ~c;
    return c % num_bits;
}

// BloomFilter64(items, fpp): nb = (int)(-items * ln fpp / (ln 2)^2), num_bits = nb + 8 - nb % 8 (8 more even when nb
// is a multiple of 8), k = max(1, Math.round(num_bits / items * ln 2)).  items > 0 and 0 < fpp < 1; false when
// num_bits would not fit a Java int (the reference then fails to allocate the bit set).
FI_HD bool bloom_sizing(int32_t items, double fpp, int32_t *num_bits, int32_t *k) {
    const double x = -(double)items * log(fpp) / (log(2.0) * log(2.0));
    const int64_t nb = x >= 2147483647.0 ? 2147483647 : (int64_t)x;       // Java's saturating (int) cast
    const int64_t bits = nb + (8 - nb % 8);
    if (bits > 2147483647) return false;
    const double r = (double)bits / (double)items * log(2.0);
    double f = floor(r);
    if (r - f >= 0.5) f += 1;                                            // Math.round: half up
    *num_bits = (int32_t)bits;
    *k = f < 1 ? 1 : (int32_t)f;
    return true;
}

}  // namespace fi
