// snappy_device.cuh — Snappy decoder for Parquet SNAPPY pages, written once for host and device.
//
// parquet-mr hands compressed pages to snappy-java 1.1.10.8; the format restated here is the public Snappy format
// description: a varint preamble holding the uncompressed length (at most 32 bits, so at most 5 bytes, the fifth
// below 16), then elements until the input ends.  The low 2 bits of a tag pick the element:
//   00 literal: length - 1 in the upper 6 bits when below 60; 60..63 = 1..4 little-endian length bytes follow
//   01 copy-1:  length 4..11 in bits 2..4, offset bits 8..10 in bits 5..7, one more offset byte
//   10 copy-2:  length 1..64 in the upper 6 bits, a little-endian u16 offset
//   11 copy-4:  length 1..64 in the upper 6 bits, a little-endian u32 offset
// A copy reads from `offset` bytes behind the output position and may overlap its own output (offset < length).
//
// Lengths and positions are 64-bit and every bound compares against what remains, so no length byte pattern can
// wrap a check.  Refused: an empty stream, a preamble over 32 bits, a preamble other than the page size, offset 0, an
// offset past the bytes produced, a literal or copy past the end of the input or the output, a truncated tag, length
// bytes or copy operand, and an output short of the preamble.  These are libsnappy's checks, so every stream this
// decoder accepts libsnappy accepts with the same bytes; tests/test_codecs_cpu.py pins the host build against it.
//
// One decoder = one warp on the device, the shape of lz4_device.cuh: every lane parses the same element stream, the
// bytes of a literal or copy move lane-parallel, byte i of an overlapping copy comes from out - offset + (i mod offset).
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define SN_HD __host__ __device__
#else
#define SN_HD
#endif

namespace snappy {

// dst[0, len) = from[0, len), byte i of an overlapping copy (dist < len, so len <= 64) from from[i mod dist]
SN_HD inline void copy(uint8_t *dst, const uint8_t *from, int64_t len, int64_t dist) {
#if defined(__CUDA_ARCH__)
    const int lane = threadIdx.x & 31;
    if (dist >= len) { for (int64_t i = lane; i < len; i += 32) dst[i] = from[i]; }
    else { for (int i = lane; i < (int)len; i += 32) dst[i] = from[(uint32_t)i % (uint32_t)dist]; }
    __syncwarp();                                   // later copies may read what other lanes just wrote
#else
    for (int64_t i = 0; i < len; i++) dst[i] = from[i];   // serial: a forward copy repeats the overlap by itself
    (void)dist;
#endif
}

// one Snappy stream src[0, n_src) -> dst[0, n_dst).  Returns n_dst, or -1 unless the stream is well-formed and its
// preamble and elements produce exactly n_dst bytes.
SN_HD inline int64_t decode(const uint8_t *src, int64_t n_src, uint8_t *dst, int64_t n_dst) {
    int64_t pos = 0;
    uint32_t ulen = 0;
    for (int sh = 0;; sh += 7) {                    // preamble
        if (pos >= n_src) return -1;
        const uint32_t b = src[pos++];
        if (sh == 28 && b > 15) return -1;          // above 32 bits, or a sixth byte
        ulen |= (b & 0x7f) << sh;
        if (!(b & 0x80)) break;
    }
    if ((int64_t)ulen != n_dst) return -1;
    int64_t out = 0;
    while (pos < n_src) {
        const uint32_t tag = src[pos++];
        int64_t len;
        if ((tag & 3) == 0) {
            len = (tag >> 2) + 1;
            if (len > 60) {
                const int extra = (int)len - 60;
                if (extra > n_src - pos) return -1;
                len = 0;
                for (int b = 0; b < extra; b++) len |= (int64_t)src[pos + b] << (8 * b);
                len += 1;                           // up to 2^32: never wraps to a short literal
                pos += extra;
            }
            if (len > n_src - pos || len > n_dst - out) return -1;
            copy(dst + out, src + pos, len, len);
            pos += len;
        } else {
            int64_t offset;
            if ((tag & 3) == 1) {
                if (n_src - pos < 1) return -1;
                len = 4 + ((tag >> 2) & 7);
                offset = ((tag >> 5) << 8) | src[pos];
                pos += 1;
            } else if ((tag & 3) == 2) {
                if (n_src - pos < 2) return -1;
                len = 1 + (tag >> 2);
                offset = src[pos] | (src[pos + 1] << 8);
                pos += 2;
            } else {
                if (n_src - pos < 4) return -1;
                len = 1 + (tag >> 2);
                offset = (int64_t)(src[pos] | (src[pos + 1] << 8) | (src[pos + 2] << 16) | ((uint32_t)src[pos + 3] << 24));
                pos += 4;
            }
            if (offset == 0 || offset > out || len > n_dst - out) return -1;
            copy(dst + out, dst + out - offset, len, offset);
        }
        out += len;
    }
    return out == n_dst ? out : -1;
}

}  // namespace snappy
