// inflate_device.cuh — DEFLATE (RFC 1951) decoder for ORC ZLIB compression chunks and Parquet GZIP pages, written
// once for host and device.
//
// ORC's default 'compress' is ZLIB: every stream is a sequence of compression chunks, each a raw DEFLATE stream
// (orc-core 1.9.2 behind paimon-format/.../orc/OrcReaderFactory.java:107-118; not under /root/reference).  Parquet
// GZIP pages are gzip members (RFC 1952: 10-byte header, DEFLATE, CRC32 + ISIZE) produced by parquet-mr's codec
// factory.  The algorithm restated here is the public DEFLATE specification: stored / fixed-Huffman /
// dynamic-Huffman blocks, canonical Huffman codes (LSB-first bit stream, codes packed MSB-first), LZ77 copies over a
// 32 KiB window.
//
// One decoder = one warp on the device, like zstd_device.cuh: every lane runs the same control flow, lane 0 builds
// the code tables and writes literals, match copies are lane-parallel (byte i of an overlapping copy comes from
// out - dist + (i mod dist)).  tests/test_inflate_cpu.py pins the host build against zlib, and tests/test_codecs_cpu.py
// fuzzes it under sanitizers: every stream it accepts, zlib accepts with the same bytes once the CRCs it skips are right.
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define IF_HD __host__ __device__
#else
#define IF_HD
#endif

namespace inflate {

constexpr int kFastBits = 9;

struct Huff {
    uint16_t fast[1 << kFastBits];     // (symbol << 4) | length for codes of <= kFastBits bits, 0 = take the slow path
    uint16_t count[16];                // codes per length
    uint16_t first[16];                // first canonical code of each length
    uint16_t index[16];                // index into sym[] of the first symbol of each length
    uint16_t sym[288];                 // symbols ordered by (length, symbol)
};
struct Tables {
    Huff lit, dist;
    uint8_t lens[320];
};

IF_HD inline int lane_id() {
#if defined(__CUDA_ARCH__)
    return threadIdx.x & 31;
#else
    return 0;
#endif
}
IF_HD inline void warp_sync() {
#if defined(__CUDA_ARCH__)
    __syncwarp();
#endif
}
IF_HD inline int bcast0(int v) {
#if defined(__CUDA_ARCH__)
    __syncwarp();
    return __shfl_sync(0xffffffffu, v, 0);
#else
    return v;
#endif
}

struct Bits {
    const uint8_t *p;
    int64_t n, pos;       // bytes, next byte to load
    uint64_t buf;
    int cnt;              // valid bits in buf (bytes past the end of the input are loaded as zeros)
};
// true when more bits have been CONSUMED than the input holds
IF_HD inline bool overrun(const Bits &b) { return b.pos * 8 - b.cnt > b.n * 8; }
IF_HD inline void refill(Bits &b) {
    while (b.cnt <= 56) {
        uint64_t byte = 0;
        if (b.pos < b.n) byte = b.p[b.pos];
        b.pos++;
        b.buf |= byte << b.cnt;
        b.cnt += 8;
    }
}
IF_HD inline uint32_t getbits(Bits &b, int n) {           // n <= 32
    if (b.cnt < n) refill(b);
    const uint32_t v = (uint32_t)(b.buf & ((n >= 32) ? 0xffffffffull : ((1ull << n) - 1)));
    b.buf >>= n;
    b.cnt -= n;
    return v;
}

// canonical Huffman code from code lengths (RFC 1951 §3.2.2).  Returns 0, or -1 for an over-subscribed code and for
// an incomplete code of a dynamic block.  zlib's rule: a code with no symbols is allowed (using it is an error), and a
// literal/length or distance code may be a single code of 1 bit; the fixed distance code is incomplete by design.
enum CodeKind { kFixed, kCodeLengths, kLitDist };
IF_HD inline int build(Huff &h, const uint8_t *lens, int n, CodeKind kind) {
    for (int i = 0; i < 16; i++) h.count[i] = 0;
    for (int i = 0; i < n; i++) h.count[lens[i]]++;
    h.count[0] = 0;
    int code = 0, idx = 0, left = 1;
    for (int l = 1; l < 16; l++) {
        left <<= 1;
        left -= h.count[l];
        if (left < 0) return -1;
        code = (code + h.count[l - 1]) << 1;
        h.first[l] = (uint16_t)code;
        h.index[l] = (uint16_t)idx;
        idx += h.count[l];
    }
    if (left > 0 && kind != kFixed) {
        int max = 15;
        while (max > 0 && !h.count[max]) max--;
        if (max > 0 && (kind == kCodeLengths || max != 1)) return -1;
    }
    // symbols in (length, symbol) order
    uint16_t next[16];
    for (int l = 0; l < 16; l++) next[l] = h.index[l];
    for (int s = 0; s < n; s++) if (lens[s]) h.sym[next[lens[s]]++] = (uint16_t)s;
    // fast table: index = the next kFastBits stream bits (LSB first) = the code bit-reversed
    for (int i = 0; i < (1 << kFastBits); i++) h.fast[i] = 0;
    for (int l = 1; l <= kFastBits; l++) {
        for (int k = 0; k < h.count[l]; k++) {
            const int c = h.first[l] + k;
            int rev = 0;
            for (int b = 0; b < l; b++) rev |= ((c >> b) & 1) << (l - 1 - b);
            const uint16_t e = (uint16_t)((h.sym[h.index[l] + k] << 4) | l);
            for (int i = rev; i < (1 << kFastBits); i += 1 << l) h.fast[i] = e;
        }
    }
    return 0;
}

IF_HD inline int decode_sym(Bits &b, const Huff &h) {
    if (b.cnt < 16) refill(b);
    const uint16_t e = h.fast[b.buf & ((1u << kFastBits) - 1)];
    if (e) {
        const int l = e & 15;
        b.buf >>= l;
        b.cnt -= l;
        return e >> 4;
    }
    int code = 0;
    for (int l = 1; l < 16; l++) {
        code = (code << 1) | (int)(b.buf & 1);
        b.buf >>= 1;
        b.cnt -= 1;
        const int d = code - h.first[l];
        if (d >= 0 && d < h.count[l]) return h.sym[h.index[l] + d];
    }
    return -1;
}

// A raw DEFLATE stream -> dst.  Returns the bytes produced, or -1 (malformed / does not fit `cap`).
// *consumed (optional) receives the input bytes used.
IF_HD inline int64_t inflate_raw(const uint8_t *src, int64_t n, uint8_t *dst, int64_t cap, Tables &T, int64_t *consumed) {
    Bits b;
    b.p = src; b.n = n; b.pos = 0; b.buf = 0; b.cnt = 0;
    int64_t out = 0;
    const uint16_t len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
    const uint8_t len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
    const uint16_t dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
                                    4097, 6145, 8193, 12289, 16385, 24577};
    const uint8_t dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
    const uint8_t clc_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    while (true) {
        const int final = (int)getbits(b, 1);
        const int type = (int)getbits(b, 2);
        if (type == 0) {
            // stored: skip to the byte boundary, LEN / NLEN, bytes
            const int drop = b.cnt & 7;
            b.buf >>= drop; b.cnt -= drop;
            const uint32_t len = getbits(b, 16), nlen = getbits(b, 16);
            if ((len ^ 0xffff) != nlen) return -1;
            // the bit buffer holds whole bytes now: hand them back
            int64_t bytepos = b.pos - b.cnt / 8;
            if (overrun(b) || bytepos + len > n || out + len > cap) return -1;
#if defined(__CUDA_ARCH__)
            __syncwarp();
            for (int64_t i = lane_id(); i < (int64_t)len; i += 32) dst[out + i] = src[bytepos + i];
            __syncwarp();
#else
            for (int64_t i = 0; i < (int64_t)len; i++) dst[out + i] = src[bytepos + i];
#endif
            out += len;
            b.pos = bytepos + len; b.buf = 0; b.cnt = 0;
        } else if (type == 1 || type == 2) {
            int rc = 0;
            if (type == 1) {
                if (lane_id() == 0) {
                    for (int i = 0; i < 144; i++) T.lens[i] = 8;
                    for (int i = 144; i < 256; i++) T.lens[i] = 9;
                    for (int i = 256; i < 280; i++) T.lens[i] = 7;
                    for (int i = 280; i < 288; i++) T.lens[i] = 8;
                    rc = build(T.lit, T.lens, 288, kFixed);
                    for (int i = 0; i < 30; i++) T.lens[i] = 5;
                    rc |= build(T.dist, T.lens, 30, kFixed);
                }
                rc = bcast0(rc);
            } else {
                const int hlit = (int)getbits(b, 5) + 257, hdist = (int)getbits(b, 5) + 1, hclen = (int)getbits(b, 4) + 4;
                if (hlit > 286 || hdist > 30) return -1;
                // the code-length code is read by every lane (it moves the bit position); lane 0 builds the tables
                uint8_t cl[19];
                for (int i = 0; i < 19; i++) cl[i] = 0;
                for (int i = 0; i < hclen; i++) cl[clc_order[i]] = (uint8_t)getbits(b, 3);
                warp_sync();                              // (nobody still decodes with the previous block's tables)
                if (lane_id() == 0) rc = build(T.lit, cl, 19, kCodeLengths);          // borrowed: T.lit is rebuilt below
                rc = bcast0(rc);
                if (rc) return -1;
                // code lengths of the literal/length and distance alphabets, run-length coded
                int i = 0, prev = 0;
                const bool w = lane_id() == 0;
                while (i < hlit + hdist) {
                    const int s = decode_sym(b, T.lit);
                    if (s < 0) return -1;
                    if (s < 16) { if (w) T.lens[i] = (uint8_t)s; i++; prev = s; }
                    else {
                        int rep, val = 0;
                        if (s == 16) { if (i == 0) return -1; rep = 3 + (int)getbits(b, 2); val = prev; }
                        else if (s == 17) { rep = 3 + (int)getbits(b, 3); prev = 0; }
                        else { rep = 11 + (int)getbits(b, 7); prev = 0; }
                        if (i + rep > hlit + hdist) return -1;
                        for (int r = 0; r < rep; r++) { if (w) T.lens[i] = (uint8_t)val; i++; }
                    }
                }
                warp_sync();                              // every lane is done decoding with the code-length code
                if (lane_id() == 0) {
                    if (T.lens[256] == 0) rc = -1;         // no end-of-block code
                    else {
                        uint8_t tmp[32];
                        for (int k = 0; k < hdist; k++) tmp[k] = T.lens[hlit + k];
                        rc = build(T.lit, T.lens, hlit, kLitDist);
                        rc |= build(T.dist, tmp, hdist, kLitDist);
                    }
                }
                rc = bcast0(rc);
            }
            if (rc) return -1;
            while (true) {
                const int s = decode_sym(b, T.lit);
                if (s < 0 || overrun(b)) return -1;
                if (s < 256) {
                    if (out >= cap) return -1;
                    if (lane_id() == 0) dst[out] = (uint8_t)s;
                    out++;
                } else if (s == 256) break;
                else {
                    if (s > 285) return -1;
                    const int len = len_base[s - 257] + (int)getbits(b, len_extra[s - 257]);
                    const int ds = decode_sym(b, T.dist);
                    if (ds < 0 || ds > 29) return -1;
                    const int64_t dist = dist_base[ds] + (int64_t)getbits(b, dist_extra[ds]);
                    if (dist > out || out + len > cap) return -1;
                    const uint8_t *from = dst + out - dist;
#if defined(__CUDA_ARCH__)
                    __syncwarp();                          // literals written by lane 0 are visible to every lane
                    if (dist >= len) { for (int i = lane_id(); i < len; i += 32) dst[out + i] = from[i]; }
                    else { for (int i = lane_id(); i < len; i += 32) dst[out + i] = from[i % dist]; }
                    __syncwarp();
#else
                    for (int i = 0; i < len; i++) dst[out + i] = from[i];
#endif
                    out += len;
                }
            }
        } else return -1;
        if (final) break;
    }
    if (overrun(b)) return -1;
    if (consumed) *consumed = b.pos - b.cnt / 8;
    warp_sync();
    return out;
}

// a gzip member (RFC 1952) -> dst; Parquet GZIP pages.  Returns bytes produced or -1.
IF_HD inline int64_t inflate_gzip(const uint8_t *src, int64_t n, uint8_t *dst, int64_t cap, Tables &T) {
    int64_t pos = 0, out = 0;
    while (pos < n) {                                     // concatenated members are legal
        if (n - pos < 18 || src[pos] != 0x1f || src[pos + 1] != 0x8b || src[pos + 2] != 8) return -1;
        const int flg = src[pos + 3];
        if (flg & 0xE0) return -1;                        // reserved flags
        int64_t p = pos + 10;
        if (flg & 4) { if (p + 2 > n) return -1; p += 2 + (src[p] | (src[p + 1] << 8)); }
        if (flg & 8) { while (p < n && src[p]) p++; p++; }
        if (flg & 16) { while (p < n && src[p]) p++; p++; }
        if (flg & 2) p += 2;
        if (p >= n) return -1;
        int64_t used = 0;
        const int64_t got = inflate_raw(src + p, n - p, dst + out, cap - out, T, &used);
        if (got < 0) return -1;
        out += got;
        pos = p + used + 8;                               // the header CRC16 and CRC32 are not verified; ISIZE is
        if (pos > n) return -1;
        const uint32_t isize = src[pos - 4] | (src[pos - 3] << 8) | (src[pos - 2] << 16) | ((uint32_t)src[pos - 1] << 24);
        if (isize != (uint32_t)got) return -1;
    }
    return out;
}

// a zlib stream (RFC 1950: 2-byte header, DEFLATE, Adler-32) -> dst.  The Adler-32 must be there; it is not verified.
IF_HD inline int64_t inflate_zlib(const uint8_t *src, int64_t n, uint8_t *dst, int64_t cap, Tables &T) {
    if (n < 6 || (src[0] & 15) != 8 || (src[0] >> 4) > 7 || ((src[0] << 8) | src[1]) % 31 != 0 || (src[1] & 32)) return -1;
    int64_t used = 0;
    const int64_t got = inflate_raw(src + 2, n - 2, dst, cap, T, &used);
    return got >= 0 && n - 2 - used >= 4 ? got : -1;
}

}  // namespace inflate
