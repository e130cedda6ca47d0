// murmur3_device.cuh — the hash and sizing of ORC's bloom filters (BLOOM_FILTER_UTF8 streams of a row index), for the
// device kernel (orc_encode.cu, k_oe_bloom) and host builds of the same source:
//   Murmur3.hash64 with seed 104729 of the bytes of STRING / VARCHAR / BINARY values, restated from the public
//     MurmurHash3 algorithm as ORC's writers use it: one 64-bit state over little-endian 8-byte blocks, the tail bytes
//     mixed in the same way, then the length and the 64-bit finalizer;
//   the bit set's size and hash count from the expected entries (the row index stride) and the fpp, as orc-core's
//     BloomFilter sizes them.
// Integers, DATE, FLOAT and DOUBLE go through Thomas Wang's hash (fi::wang64) and the bit positions are fi::bloom_bit,
// both in xxhash64_device.cuh.
#pragma once

#include "xxhash64_device.cuh"

namespace fi {

constexpr uint64_t kMurmurC1 = 0x87c37b91114253d5ull, kMurmurC2 = 0x4cf5ad432745937full;
constexpr uint64_t kOrcBloomSeed = 104729;

FI_HD uint64_t murmur_fmix64(uint64_t h) {
    h ^= h >> 33;
    h *= 0xff51afd7ed558ccdull;
    h ^= h >> 33;
    h *= 0xc4ceb9fe1a85ec53ull;
    h ^= h >> 33;
    return h;
}

FI_HD uint64_t murmur_mix(uint64_t k) { return rotl64(k * kMurmurC1, 31) * kMurmurC2; }

// Murmur3.hash64(p[0..n), seed): any alignment, bytes read one at a time
FI_HD int64_t murmur3_hash64(const uint8_t *p, int64_t n, uint64_t seed = kOrcBloomSeed) {
    uint64_t h = seed;
    const int64_t blocks = n >> 3;
    for (int64_t b = 0; b < blocks; b++) {
        h ^= murmur_mix(load_le(p + 8 * b, 8));
        h = rotl64(h, 27) * 5 + 0x52dce729;
    }
    const int tail = (int)(n & 7);
    if (tail) h ^= murmur_mix(load_le(p + 8 * blocks, tail));
    h ^= (uint64_t)n;
    return (int64_t)murmur_fmix64(h);
}

// orc-core's BloomFilter(expectedEntries, fpp): nb = (int)(-n ln fpp / (ln 2)^2), num_bits = nb + 64 - nb % 64 (64
// more even when nb is a multiple of 64), k = max(1, Math.round(num_bits / n * ln 2)).  n > 0 and 0 < fpp < 1; false
// when num_bits would not fit a Java int.
FI_HD bool orc_bloom_sizing(int64_t entries, double fpp, int32_t *num_bits, int32_t *k) {
    const double x = -(double)entries * log(fpp) / (log(2.0) * log(2.0));
    const int64_t nb = x >= 2147483647.0 ? 2147483647 : (int64_t)x;
    const int64_t bits = nb + (64 - nb % 64);
    if (bits > 2147483647) return false;
    const double r = (double)bits / (double)entries * log(2.0);
    double f = floor(r);
    if (r - f >= 0.5) f += 1;
    *num_bits = (int32_t)bits;
    *k = f < 1 ? 1 : (int32_t)f;
    return true;
}

}  // namespace fi
