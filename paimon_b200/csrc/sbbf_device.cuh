// sbbf_device.cuh — the Parquet split-block bloom filter (SBBF) of a column chunk, for the device kernel k_pw_sbbf
// (parquet_encode.cu) and a host build of the same source (tests/native/parquet_bloom_host_check.cc).  Restated from
// the Parquet format specification (BloomFilter.md):
//   hash   XXH64 (seed 0, fi::xxh64) of the value's PLAIN bytes: INT8 / INT16 / INT32 / DATE as 4 little-endian bytes
//          (sign-extended), INT64 as 8, FLOAT / DOUBLE as their raw IEEE bits (no NaN folding), STRING / BINARY as
//          the value bytes without the length word;
//   block  ((h >> 32) * num_blocks) >> 32, of 32 bytes: eight little-endian 32-bit words;
//   mask   key = (uint32_t)h, word i of the block gets bit (key * SALT[i]) >> 27.
// The sizing restates parquet-mr 1.16's BlockSplitBloomFilter.optimalNumOfBits and its constructor, as
// ColumnValueCollector calls them: parquet-mr's sources are not vendored, so this is written from its documented
// behaviour and pinned against pyarrow's writer where the two agree (tests/test_parquet_bloom_cpu.py).  A reader
// accepts any power-of-two size within the specification's bounds, so a slip here costs space or false-positive rate,
// never an answer.
#pragma once

#include <math.h>
#include <stdint.h>

#include "xxhash64_device.cuh"

namespace sbbf {

constexpr int64_t kMinBytes = 32;                 // one block
constexpr int64_t kMaxBytes = 1 << 20;            // parquet.bloom.filter.max.bytes default; Paimon does not set it
constexpr int64_t kUpperBoundBytes = 128 << 20;   // the specification's largest filter

// XXH64 (seed 0) of 4 and of 8 little-endian bytes: fi::xxh64 with the length known
FI_HD uint64_t avalanche(uint64_t h) {
    h ^= h >> 33;
    h *= fi::kP2;
    h ^= h >> 29;
    h *= fi::kP3;
    h ^= h >> 32;
    return h;
}
FI_HD uint64_t hash4(uint32_t v) {
    return avalanche(fi::rotl64((fi::kP5 + 4) ^ ((uint64_t)v * fi::kP1), 23) * fi::kP2 + fi::kP3);
}
FI_HD uint64_t hash8(uint64_t v) {
    return avalanche(fi::rotl64((fi::kP5 + 8) ^ fi::xxh_round(0, v), 27) * fi::kP1 + fi::kP4);
}

FI_HD uint32_t block_of(uint64_t h, uint32_t n_blocks) { return (uint32_t)(((h >> 32) * n_blocks) >> 32); }

// the bit that hash h sets in word i (0..7) of its block
FI_HD uint32_t mask_word(uint64_t h, int i) {
    const uint32_t salt[8] = {0x47b6137bu, 0x44974d91u, 0x8824ad5bu, 0xa2b7289du,
                              0x705495c7u, 0x2df1424bu, 0x9efc4947u, 0x5c6bfb31u};
    return 1u << (((uint32_t)h * salt[i]) >> 27);
}

// The bitset bytes of a filter for `ndv` distinct values at `fpp` (0 < fpp < 1); ndv 0 = unset: kMaxBytes.
// optimalNumOfBits: bits = (int)(-8 ndv / ln(1 - fpp^(1/8))), kUpperBoundBytes * 8 when larger, then
// (bits + 255) & ~256 and at least kMinBytes * 8; the constructor takes bits / 8 bytes, at least kMinBytes, rounded up
// to a power of two, at most kMaxBytes.
FI_HD int64_t num_bytes(int64_t ndv, double fpp) {
    if (ndv <= 0) return kMaxBytes;
    const double m = -8.0 * (double)ndv / log(1.0 - pow(fpp, 1.0 / 8));
    int64_t bits = m >= 2147483647.0 ? 2147483647 : (int64_t)m;          // Java's saturating (int) cast
    if (bits > (kUpperBoundBytes << 3) || m < 0) bits = kUpperBoundBytes << 3;
    bits = (bits + 255) & ~(int64_t)256;
    if (bits < (kMinBytes << 3)) bits = kMinBytes << 3;
    int64_t bytes = bits / 8;
    if (bytes < kMinBytes) bytes = kMinBytes;
    int64_t p = kMinBytes;
    while (p < bytes) p <<= 1;
    return p > kMaxBytes ? kMaxBytes : p;
}

}  // namespace sbbf
