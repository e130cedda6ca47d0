// orc_encode_device.cuh — ORC stream encoders, written once for host and device, beside the decoders of
// orc_device.cuh (whose width tables they share).
//
// The encodings are those of the public ORC specification v1 that orc_device.cuh reads.  Run boundaries are fixed in
// advance so that every run is encoded on its own and its size is known before any byte is written:
//   * integer RLE v2: runs of at most kRunValues values; each run takes the smallest of SHORT_REPEAT (3 to 10 equal
//     values), DELTA (deltas of one sign, none overflowing int64) and DIRECT.  PATCHED_BASE is not written.
//   * byte RLE: groups of at most kByteGroup bytes; a group of 3 or more equal bytes is one run, any other a literal.
// A run is sized by rle2_plan / brle_size and written by rle2_write / brle_write, by one thread on the device or by the
// host harness (tests/native/orc_encode_host_check.cc).
#pragma once

#include "orc_device.cuh"

namespace orcdev {

constexpr int kRunValues = 512;   // the longest run integer RLE v2 can express
constexpr int kByteGroup = 128;   // the longest literal byte RLE can express

ORC_HD inline uint64_t zigzag(int64_t v) { return ((uint64_t)v << 1) ^ (uint64_t)(v >> 63); }

ORC_HD inline int bits_of(uint64_t v) {
    int n = 0;
    while (v) { n++; v >>= 1; }
    return n;
}
ORC_HD inline int varint_size(uint64_t v) {
    int n = 1;
    while (v >= 0x80) { n++; v >>= 7; }
    return n;
}
// the 5-bit code of a width closest_fixed_bits returns (the inverse of decode_width)
ORC_HD inline int encode_width(int w) {
    if (w <= 24) return w - 1;
    switch (w) {
        case 26: return 24;
        case 28: return 25;
        case 30: return 26;
        case 32: return 27;
        case 40: return 28;
        case 48: return 29;
        case 56: return 30;
        default: return 31;
    }
}

struct Out {
    uint8_t *p;   // NULL = count only
    int64_t n;
};
ORC_HD inline void put(Out &o, uint32_t b) {
    if (o.p) o.p[o.n] = (uint8_t)b;
    o.n++;
}
ORC_HD inline void put_varint(Out &o, uint64_t v) {
    while (v >= 0x80) { put(o, (uint32_t)(v & 0x7f) | 0x80); v >>= 7; }
    put(o, (uint32_t)v);
}
// big-endian bit packing of `count` values of `width` bits, from a byte boundary, the last byte zero-padded
struct BitPack {
    uint32_t cur;
    int used;
};
ORC_HD inline void pack(Out &o, BitPack &b, uint64_t v, int width) {
    for (int left = width; left > 0;) {
        const int take = left < 8 - b.used ? left : 8 - b.used;
        const uint32_t bits = (uint32_t)(v >> (left - take)) & ((1u << take) - 1);
        b.cur |= bits << (8 - b.used - take);
        b.used += take;
        left -= take;
        if (b.used == 8) { put(o, b.cur); b.cur = 0; b.used = 0; }
    }
}
ORC_HD inline void pack_flush(Out &o, BitPack &b) {
    if (b.used) put(o, b.cur);
    b.cur = 0;
    b.used = 0;
}

// ---- integer RLE v2
enum : int { R2_SHORT_REPEAT = 0, R2_DIRECT = 1, R2_DELTA = 3 };

struct Rle2Plan {
    int form;
    int width;    // SHORT_REPEAT: bytes of the value; DIRECT / DELTA: bit width (DELTA 0 = fixed delta)
    int size;     // bytes of the run
};

// the stored (zigzagged when signed) form of a value
ORC_HD inline uint64_t stored(int64_t v, int is_signed) { return is_signed ? zigzag(v) : (uint64_t)v; }

// b - a, or false when it leaves int64 (INT64_MIN is refused too: its magnitude does not fit a signed delta)
ORC_HD inline bool delta_of(int64_t a, int64_t b, int64_t &d) {
    d = (int64_t)((uint64_t)b - (uint64_t)a);
    if (((a ^ b) & (b ^ d)) < 0) return false;           // signs of a and b differ and d took a's sign
    return d != INT64_MIN;
}

ORC_HD inline Rle2Plan rle2_plan(const int64_t *v, int n, int is_signed) {
    // DIRECT is always valid
    uint64_t mx = 0;
    bool equal = true;
    for (int i = 0; i < n; i++) {
        const uint64_t s = stored(v[i], is_signed);
        mx = s > mx ? s : mx;
        equal = equal && v[i] == v[0];
    }
    const int dw = closest_fixed_bits(bits_of(mx));
    Rle2Plan best{R2_DIRECT, dw, 2 + (int)(((int64_t)n * dw + 7) / 8)};
    if (equal && n >= 3 && n <= 10) {
        const int bytes = (bits_of(stored(v[0], is_signed)) + 7) / 8;
        const int size = 1 + (bytes ? bytes : 1);
        if (size < best.size) best = Rle2Plan{R2_SHORT_REPEAT, bytes ? bytes : 1, size};
    }
    if (n >= 3) {
        // DELTA: the first delta gives the direction; every later delta has its sign (a zero first delta: upwards)
        int64_t d0;
        bool ok = delta_of(v[0], v[1], d0), fixed = true;
        uint64_t dmax = 0;
        for (int i = 2; i < n && ok; i++) {
            int64_t d;
            ok = delta_of(v[i - 1], v[i], d) && (d0 < 0 ? d <= 0 : d >= 0);
            fixed = fixed && d == d0;
            const uint64_t m = d < 0 ? (uint64_t)(-d) : (uint64_t)d;
            dmax = m > dmax ? m : dmax;
        }
        if (ok) {
            // width code 0 means a fixed delta, so a 1-bit width is written as 2 bits
            int w = fixed ? 0 : closest_fixed_bits(bits_of(dmax));
            if (w == 1) w = 2;
            const int size = 2 + varint_size(stored(v[0], is_signed)) + varint_size(zigzag(d0)) +
                             (int)(((int64_t)(n - 2) * w + 7) / 8);
            if (size < best.size || (size == best.size && best.form == R2_DIRECT)) best = Rle2Plan{R2_DELTA, w, size};
        }
    }
    return best;
}

// writes the run as planned: exactly p.size bytes
ORC_HD inline void rle2_write(const int64_t *v, int n, int is_signed, const Rle2Plan &p, uint8_t *dst) {
    Out o{dst, 0};
    if (p.form == R2_SHORT_REPEAT) {
        put(o, (uint32_t)((p.width - 1) << 3) | (uint32_t)(n - 3));
        const uint64_t s = stored(v[0], is_signed);
        for (int b = p.width - 1; b >= 0; b--) put(o, (uint32_t)(s >> (8 * b)) & 0xff);
        return;
    }
    const int wcode = p.form == R2_DELTA && p.width == 0 ? 0 : encode_width(p.width);
    put(o, ((uint32_t)p.form << 6) | ((uint32_t)wcode << 1) | ((uint32_t)(n - 1) >> 8));
    put(o, (uint32_t)(n - 1) & 0xff);
    BitPack b{0, 0};
    if (p.form == R2_DIRECT) {
        for (int i = 0; i < n; i++) pack(o, b, stored(v[i], is_signed), p.width);
    } else {
        put_varint(o, stored(v[0], is_signed));
        const int64_t d0 = (int64_t)((uint64_t)v[1] - (uint64_t)v[0]);
        put_varint(o, zigzag(d0));
        if (p.width)
            for (int i = 2; i < n; i++) {
                const int64_t d = (int64_t)((uint64_t)v[i] - (uint64_t)v[i - 1]);
                pack(o, b, d < 0 ? (uint64_t)(-d) : (uint64_t)d, p.width);
            }
    }
    pack_flush(o, b);
}

// ---- byte RLE over a group of 1 to kByteGroup bytes
ORC_HD inline bool brle_is_run(const uint8_t *v, int n) {
    if (n < 3) return false;
    for (int i = 1; i < n; i++)
        if (v[i] != v[0]) return false;
    return true;
}
ORC_HD inline int brle_size(const uint8_t *v, int n) { return brle_is_run(v, n) ? 2 : 1 + n; }
ORC_HD inline void brle_write(const uint8_t *v, int n, uint8_t *dst) {
    if (brle_is_run(v, n)) {
        dst[0] = (uint8_t)(n - 3);
        dst[1] = v[0];
        return;
    }
    dst[0] = (uint8_t)(256 - n);
    for (int i = 0; i < n; i++) dst[1 + i] = v[i];
}

// a PRESENT or BOOLEAN stream byte from 8 validity bits (LSB first, as in an Arrow bitmap): MSB first
ORC_HD inline uint8_t bit_reverse8(uint32_t b) {
    b = ((b & 0xF0u) >> 4) | ((b & 0x0Fu) << 4);
    b = ((b & 0xCCu) >> 2) | ((b & 0x33u) << 2);
    b = ((b & 0xAAu) >> 1) | ((b & 0x55u) << 1);
    return (uint8_t)b;
}

}  // namespace orcdev
