// lz4_device.cuh — LZ4 block decoder for Parquet LZ4 pages (Hadoop block framing) and ORC LZ4 compression chunks,
// written once for host and device.
//
// Paimon's per-level compression example is '0:lz4,1:zstd' (paimon-api/.../CoreOptions.java:299-305), so every
// level-0 file of such a table is LZ4.  Parquet codec 5 (LZ4) goes through Hadoop's Lz4Codec: the page body is a
// sequence of blocks, each a big-endian u32 uncompressed length followed by chunks, each a big-endian u32 compressed
// length and one raw LZ4 block.  ORC CompressionKind 4 stores one raw LZ4 block per compression chunk.  The format
// restated here is the public LZ4 block format description: a token (literal length high nibble, match length - 4 low
// nibble, 15 = more length bytes follow, each added, until one is not 255), the literals, a little-endian u16 offset.
// The last sequence holds literals only and ends the block.
//
// End-of-block rules, as liblz4's safe decoder enforces them when a sequence is decoded on its checked path: a match
// must start at least 12 bytes before the end of the output buffer and end at least 5 bytes before it, and a
// sequence that is followed by a match must leave at least 8 input bytes behind its literals.  liblz4 skips these
// checks on its unchecked fast paths and also takes offset 0; this decoder refuses both, so every block it accepts
// liblz4 accepts with the same bytes.  tests/test_lz4_cpu.py pins the host build against pyarrow's lz4_raw codec.
//
// One decoder = one warp on the device: every lane parses the same token stream, literal and match bytes move
// lane-parallel, byte i of an overlapping match (offset < length) comes from out - offset + (i mod offset).
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define LZ4_HD __host__ __device__
#else
#define LZ4_HD
#endif

namespace lz4 {

constexpr int64_t kMatchStartMargin = 12;   // a match starts at least this many bytes before the end of the output
constexpr int64_t kLastLiterals = 5;        // ... and ends at least this many bytes before it
constexpr int64_t kTailAfterLiterals = 8;   // offset (2) + final token (1) + last literals (5)

// dst[0, len) = from[0, len), byte i of an overlapping copy from from[i mod dist]
LZ4_HD inline void copy(uint8_t *dst, const uint8_t *from, int64_t len, int64_t dist) {
#if defined(__CUDA_ARCH__)
    __syncwarp();                                   // bytes other lanes wrote are visible
    const int lane = threadIdx.x & 31;
    if (dist >= len) { for (int64_t i = lane; i < len; i += 32) dst[i] = from[i]; }
    else { for (int64_t i = lane; i < len; i += 32) dst[i] = from[i % dist]; }
    __syncwarp();
#else
    for (int64_t i = 0; i < len; i++) dst[i] = from[i];   // serial: a forward copy repeats the overlap by itself
    (void)dist;
#endif
}

// one raw LZ4 block src[0, n) -> dst[0, cap).  Returns the bytes produced, or -1 (malformed / does not fit `cap`).
LZ4_HD inline int64_t decode_block(const uint8_t *src, int64_t n, uint8_t *dst, int64_t cap) {
    if (n <= 0) return -1;
    if (cap == 0) return (n == 1 && src[0] == 0) ? 0 : -1;
    int64_t ip = 0, op = 0;
    while (ip < n) {
        const uint32_t token = src[ip++];
        int64_t len = token >> 4;
        if (len == 15) {
            uint32_t s;
            do {
                if (ip >= n) return -1;
                s = src[ip++];
                len += s;
            } while (s == 255);
        }
        if (len > n - ip || len > cap - op) return -1;
        copy(dst + op, src + ip, len, len);
        ip += len;
        op += len;
        if (ip == n) return op;                     // the last sequence: literals only
        if (op > cap - kMatchStartMargin || n - ip < kTailAfterLiterals) return -1;
        const int64_t offset = src[ip] | (src[ip + 1] << 8);
        ip += 2;
        if (offset == 0 || offset > op) return -1;
        int64_t mlen = (token & 15) + 4;
        if ((token & 15) == 15) {
            uint32_t s;
            do {
                s = src[ip++];                      // in bounds: ip <= n - 4 before every read
                if (ip > n - 4) return -1;
                mlen += s;
            } while (s == 255);
        }
        if (mlen > cap - kLastLiterals - op) return -1;
        copy(dst + op, dst + op - offset, mlen, offset);
        op += mlen;
    }
    return -1;                                      // (not reached: a match leaves at least 4 input bytes)
}

LZ4_HD inline int64_t be32(const uint8_t *p) {
    return ((int64_t)p[0] << 24) | ((int64_t)p[1] << 16) | ((int64_t)p[2] << 8) | (int64_t)p[3];
}

// Hadoop Lz4Codec framing (Parquet codec 5) src[0, n) -> dst: blocks of [u32 BE uncompressed length] then chunks of
// [u32 BE compressed length][raw LZ4 block] until the block's length is produced.  Returns `want`, or -1 unless the
// blocks use every input byte and add up to exactly `want` bytes.
LZ4_HD inline int64_t decode_hadoop(const uint8_t *src, int64_t n, uint8_t *dst, int64_t want) {
    int64_t pos = 0, out = 0;
    while (pos < n) {
        if (n - pos < 4) return -1;
        const int64_t block = be32(src + pos);
        pos += 4;
        if (block > want - out) return -1;
        const int64_t end = out + block;
        while (out < end) {
            if (n - pos < 4) return -1;
            const int64_t clen = be32(src + pos);
            pos += 4;
            if (clen > n - pos) return -1;
            const int64_t got = decode_block(src + pos, clen, dst + out, end - out);
            if (got < 0) return -1;
            out += got;
            pos += clen;
        }
    }
    return out == want ? out : -1;
}

}  // namespace lz4
