// orc_device.cuh — ORC stream decoders and the per-(stripe, column) decode task, written once for host and device.
//
// The reference reads ORC through orc-core 1.9.2 (paimon-format/.../orc/OrcReaderFactory.java:98-163 createReader /
// :280-330 createRecordReader; the vector adapters in orc/reader/*): all decode arithmetic lives in that dependency,
// which is not under /root/reference.  The encodings restated here are the public ORC specification v1: byte RLE,
// boolean (bit) streams, integer RLE v1 and v2 (SHORT_REPEAT / DIRECT / PATCHED_BASE / DELTA), base-128 varints with
// zigzag, string DIRECT / DICTIONARY encodings, decimals (varint + scale), PRESENT streams.
//
// A task = one column of one stripe.  It is decoded serially (the streams are run-length coded without random
// access inside a stripe; the parallelism is stripes x columns: a 128 MiB-stripe file of 50 columns per run and 16
// runs gives thousands of tasks), by one thread on the device or by the host harness that pins this code against
// pyarrow.orc and the reference's golden files (tests/test_orc_cpu.py).
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define ORC_HD __host__ __device__
#else
#define ORC_HD
#endif

namespace orcdev {

enum : int { T_BOOLEAN = 0, T_BYTE = 1, T_SHORT = 2, T_INT = 3, T_LONG = 4, T_FLOAT = 5, T_DOUBLE = 6, T_STRING = 7, T_BINARY = 8,
             T_TIMESTAMP = 9, T_DECIMAL = 14, T_DATE = 15, T_VARCHAR = 16, T_CHAR = 17 };
enum : int { ENC_DIRECT = 0, ENC_DICTIONARY = 1, ENC_DIRECT_V2 = 2, ENC_DICTIONARY_V2 = 3 };

struct Src {
    const uint8_t *p;
    int64_t n, pos;
    int bad;
};
ORC_HD inline void src_init(Src &s, const uint8_t *p, int64_t n) { s.p = p; s.n = n; s.pos = 0; s.bad = 0; }
ORC_HD inline uint32_t src_byte(Src &s) {
    if (s.pos >= s.n) { s.bad = 1; return 0; }
    return s.p[s.pos++];
}
ORC_HD inline uint64_t read_vulong(Src &s) {
    uint64_t v = 0;
    for (int sh = 0; sh < 70; sh += 7) {
        const uint32_t b = src_byte(s);
        if (sh < 64) v |= (uint64_t)(b & 0x7f) << sh;
        if (!(b & 0x80)) return v;
    }
    s.bad = 1;
    return v;
}
ORC_HD inline int64_t unzigzag(uint64_t v) { return (int64_t)(v >> 1) ^ -(int64_t)(v & 1); }
ORC_HD inline int64_t read_vslong(Src &s) { return unzigzag(read_vulong(s)); }

// ---- byte RLE: header 0..127 = run of header + 3 copies of the next byte, 128..255 = 256 - header literal bytes
struct ByteRle {
    Src s;
    int run, lit;
    uint8_t val;
};
ORC_HD inline void brle_init(ByteRle &r, const uint8_t *p, int64_t n) { src_init(r.s, p, n); r.run = r.lit = 0; r.val = 0; }
ORC_HD inline uint8_t brle_next(ByteRle &r) {
    if (r.run == 0 && r.lit == 0) {
        const uint32_t h = src_byte(r.s);
        if (h < 128) { r.run = (int)h + 3; r.val = (uint8_t)src_byte(r.s); }
        else r.lit = 256 - (int)h;
    }
    if (r.run) { r.run--; return r.val; }
    r.lit--;
    return (uint8_t)src_byte(r.s);
}

// ---- boolean stream (PRESENT, BOOLEAN data): byte RLE, bits most significant first
struct BoolRle {
    ByteRle b;
    int left;
    uint8_t cur;
    int all;             // no stream: every bit is 1
};
ORC_HD inline void bool_init(BoolRle &r, const uint8_t *p, int64_t n) { brle_init(r.b, p, n); r.left = 0; r.cur = 0; r.all = p == nullptr; }
ORC_HD inline int bool_next(BoolRle &r) {
    if (r.all) return 1;
    if (!r.left) { r.cur = brle_next(r.b); r.left = 8; }
    r.left--;
    return (r.cur >> r.left) & 1;
}

ORC_HD inline int decode_width(int enc) {
    if (enc <= 23) return enc + 1;
    const int t[8] = {26, 28, 30, 32, 40, 48, 56, 64};
    return t[enc - 24];
}
ORC_HD inline int closest_fixed_bits(int n) {
    if (n == 0) return 1;
    if (n <= 24) return n;
    if (n <= 26) return 26;
    if (n <= 28) return 28;
    if (n <= 30) return 30;
    if (n <= 32) return 32;
    if (n <= 40) return 40;
    if (n <= 48) return 48;
    if (n <= 56) return 56;
    return 64;
}

// big-endian bit-packed values of `width` bits, starting at a byte boundary
ORC_HD inline void read_packed(Src &s, int width, int count, int64_t *out) {
    uint32_t cur = 0;
    int left = 0;
    for (int i = 0; i < count; i++) {
        uint64_t v = 0;
        int need = width;
        while (need > 0) {
            if (left == 0) { cur = src_byte(s); left = 8; }
            const int take = need < left ? need : left;
            v = (v << take) | ((cur >> (left - take)) & ((1u << take) - 1));
            left -= take;
            need -= take;
        }
        out[i] = (int64_t)v;
    }
}

// ---- integer RLE v1 / v2: a run at a time into buf
struct IntRle {
    Src s;
    int v2, is_signed;
    int n, i;
    int64_t buf[512];
};
ORC_HD inline void irle_init(IntRle &r, const uint8_t *p, int64_t len, int v2, int is_signed) {
    src_init(r.s, p, len);
    r.v2 = v2; r.is_signed = is_signed; r.n = r.i = 0;
}
ORC_HD inline void irle_fill(IntRle &r) {
    Src &s = r.s;
    r.i = 0;
    r.n = 0;
    if (!r.v2) {
        const uint32_t h = src_byte(s);
        if (h < 128) {
            const int run = (int)h + 3;
            const int64_t delta = (int8_t)src_byte(s);
            const int64_t base = r.is_signed ? read_vslong(s) : (int64_t)read_vulong(s);
            for (int j = 0; j < run; j++) r.buf[j] = base + j * delta;
            r.n = run;
        } else {
            const int lit = 256 - (int)h;
            for (int j = 0; j < lit; j++) r.buf[j] = r.is_signed ? read_vslong(s) : (int64_t)read_vulong(s);
            r.n = lit;
        }
        return;
    }
    const uint32_t fb = src_byte(s);
    const int enc = (int)(fb >> 6);
    if (enc == 0) {                                       // SHORT_REPEAT
        const int w = (int)((fb >> 3) & 7) + 1, count = (int)(fb & 7) + 3;
        uint64_t v = 0;
        for (int b = 0; b < w; b++) v = (v << 8) | src_byte(s);
        const int64_t val = r.is_signed ? unzigzag(v) : (int64_t)v;
        for (int j = 0; j < count; j++) r.buf[j] = val;
        r.n = count;
    } else if (enc == 1) {                                // DIRECT
        const int w = decode_width((int)((fb >> 1) & 31));
        const int len = (int)(((fb & 1) << 8) | src_byte(s)) + 1;
        read_packed(s, w, len, r.buf);
        if (r.is_signed) for (int j = 0; j < len; j++) r.buf[j] = unzigzag((uint64_t)r.buf[j]);
        r.n = len;
    } else if (enc == 2) {                                // PATCHED_BASE
        const int w = decode_width((int)((fb >> 1) & 31));
        const int len = (int)(((fb & 1) << 8) | src_byte(s)) + 1;
        const uint32_t b3 = src_byte(s), b4 = src_byte(s);
        const int bw = (int)(b3 >> 5) + 1, pw = decode_width((int)(b3 & 31));
        const int pgw = (int)(b4 >> 5) + 1, pll = (int)(b4 & 31);
        uint64_t ub = 0;
        for (int b = 0; b < bw; b++) ub = (ub << 8) | src_byte(s);
        const uint64_t sign = 1ull << (bw * 8 - 1);
        int64_t base = (int64_t)(ub & (sign - 1));
        if (ub & sign) base = -base;
        read_packed(s, w, len, r.buf);
        if (pll > 0) {
            if (pw + pgw > 64) { s.bad = 1; return; }
            const int cfb = closest_fixed_bits(pw + pgw);
            int64_t patches[32];
            read_packed(s, cfb, pll, patches);
            int idx = 0;
            const uint64_t pmask = pw >= 64 ? ~0ull : ((1ull << pw) - 1);
            for (int q = 0; q < pll; q++) {
                const uint64_t e = (uint64_t)patches[q];
                idx += (int)(e >> pw);
                const uint64_t patch = e & pmask;
                if (idx >= len) { s.bad = 1; return; }
                r.buf[idx] = (int64_t)((uint64_t)r.buf[idx] | (patch << w));
            }
        }
        for (int j = 0; j < len; j++) r.buf[j] += base;
        r.n = len;
    } else {                                              // DELTA
        const int we = (int)((fb >> 1) & 31);
        const int w = we == 0 ? 0 : decode_width(we);
        const int len = (int)(((fb & 1) << 8) | src_byte(s)) + 1;
        const int64_t base = r.is_signed ? read_vslong(s) : (int64_t)read_vulong(s);
        const int64_t db = read_vslong(s);
        r.buf[0] = base;
        if (len > 1) r.buf[1] = base + db;
        if (w == 0) {
            for (int j = 2; j < len; j++) r.buf[j] = r.buf[j - 1] + db;
        } else if (len > 2) {
            read_packed(s, w, len - 2, r.buf + 2);
            for (int j = 2; j < len; j++) r.buf[j] = db < 0 ? r.buf[j - 1] - r.buf[j] : r.buf[j - 1] + r.buf[j];
        }
        r.n = len;
    }
}
ORC_HD inline int64_t irle_next(IntRle &r) {
    if (r.i >= r.n) {
        irle_fill(r);
        if (r.n == 0) { r.s.bad = 1; return 0; }
    }
    return r.buf[r.i++];
}

// ---- one (stripe, column)
struct Task {
    const uint8_t *present, *data, *length, *dict_data, *secondary;    // decompressed streams (NULL = absent)
    int64_t present_n, data_n, length_n, dict_data_n, secondary_n;
    int64_t row0;              // first row of the stripe inside the output run
    int64_t rows;
    int32_t kind;              // ORC type kind
    int32_t enc;               // column encoding
    int32_t dict_size;
    int32_t scale;             // DECIMAL: the type's scale
    int32_t out_width;         // bytes of the output type, 0 = var-len
    int32_t cast;              // 1: the read type is BIGINT over a narrower integer (sign extension happens anyway)
    void *out_data;            // fixed width values
    int32_t *out_offsets;      // var-len: lengths are written to out_offsets[row + 1] in phase A, scanned, then phase B
    uint32_t *out_validity;    // NULL = the run's column has no bitmap
    uint8_t *out_payload;      // phase B
    int32_t *dict_off;         // scratch [dict_size + 1]
    int64_t payload_bytes;     // phase A result
    int32_t bad;
};

ORC_HD inline void or_word(uint32_t *p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    if (v) atomicOr(p, v);
#else
    *p |= v;
#endif
}

// the validity bits of the task's rows: accumulated 32 at a time; words shared with neighbouring stripes are OR-ed
struct BitSink {
    uint32_t *bm;
    int64_t row;               // next row
    uint32_t cur;
};
ORC_HD inline void sink_init(BitSink &k, uint32_t *bm, int64_t row0) { k.bm = bm; k.row = row0; k.cur = 0; }
ORC_HD inline void sink_put(BitSink &k, int bit) {
    if (bit) k.cur |= 1u << (k.row & 31);
    k.row++;
    if ((k.row & 31) == 0) { if (k.bm) or_word(&k.bm[(k.row - 1) >> 5], k.cur); k.cur = 0; }
}
ORC_HD inline void sink_flush(BitSink &k) {
    if ((k.row & 31) != 0 && k.bm) or_word(&k.bm[k.row >> 5], k.cur);
}

ORC_HD inline void store_val(void *out, int width, int64_t row, uint64_t v) {
    switch (width) {
        case 1: ((uint8_t *)out)[row] = (uint8_t)v; break;
        case 2: ((uint16_t *)out)[row] = (uint16_t)v; break;
        case 4: ((uint32_t *)out)[row] = (uint32_t)v; break;
        default: ((uint64_t *)out)[row] = v; break;
    }
}

// phase A: validity, fixed-width values, var-len lengths (+ the task's payload bytes)
ORC_HD inline void decode_task_a(Task &t) {
    BoolRle pres;
    bool_init(pres, t.present, t.present_n);
    BitSink sink;
    sink_init(sink, t.out_validity, t.row0);
    const bool v2 = t.enc == ENC_DIRECT_V2 || t.enc == ENC_DICTIONARY_V2;
    const bool dict = t.enc == ENC_DICTIONARY || t.enc == ENC_DICTIONARY_V2;
    int bad = 0;
    int64_t payload = 0;
    const int k = t.kind;
    IntRle r, len;                                        // (declared once: their run buffers are 4 KiB of stack each)
    if (k == T_SHORT || k == T_INT || k == T_LONG || k == T_DATE) {
        irle_init(r, t.data, t.data_n, v2, 1);
        for (int64_t i = 0; i < t.rows; i++) {
            const int ok = bool_next(pres);
            sink_put(sink, ok);
            store_val(t.out_data, t.out_width, t.row0 + i, ok ? (uint64_t)irle_next(r) : 0);
        }
        bad |= r.s.bad;
    } else if (k == T_BYTE) {
        ByteRle br;
        brle_init(br, t.data, t.data_n);
        for (int64_t i = 0; i < t.rows; i++) {
            const int ok = bool_next(pres);
            sink_put(sink, ok);
            store_val(t.out_data, t.out_width, t.row0 + i, ok ? (uint64_t)(int64_t)(int8_t)brle_next(br) : 0);
        }
        bad |= br.s.bad;
    } else if (k == T_BOOLEAN) {
        BoolRle bo;
        bool_init(bo, t.data, t.data_n);
        bo.all = 0;
        for (int64_t i = 0; i < t.rows; i++) {
            const int ok = bool_next(pres);
            sink_put(sink, ok);
            store_val(t.out_data, t.out_width, t.row0 + i, ok ? (uint64_t)bool_next(bo) : 0);
        }
        bad |= bo.b.s.bad;
    } else if (k == T_FLOAT || k == T_DOUBLE) {
        const int w = k == T_FLOAT ? 4 : 8;
        int64_t pos = 0;
        for (int64_t i = 0; i < t.rows; i++) {
            const int ok = bool_next(pres);
            sink_put(sink, ok);
            uint64_t v = 0;
            if (ok) {
                if (pos + w > t.data_n) { bad = 1; break; }
                for (int b = 0; b < w; b++) v |= (uint64_t)t.data[pos + b] << (8 * b);
                pos += w;
                if (w == 4 && t.out_width == 8) {          // FLOAT file column read as DOUBLE
                    union { uint32_t u; float f; } a;
                    union { uint64_t u; double d; } c;
                    a.u = (uint32_t)v; c.d = (double)a.f; v = c.u;
                }
            }
            store_val(t.out_data, t.out_width, t.row0 + i, v);
        }
    } else if (k == T_DECIMAL) {
        Src d;
        src_init(d, t.data, t.data_n);
        IntRle &sc = r;
        irle_init(sc, t.secondary, t.secondary_n, v2, 1);
        for (int64_t i = 0; i < t.rows; i++) {
            const int ok = bool_next(pres);
            sink_put(sink, ok);
            int64_t v = 0;
            if (ok) {
                v = read_vslong(d);
                int64_t s = irle_next(sc);
                // a value's own scale is 0..38 and at most 18 away from the type's (any other is a corrupt stream):
                // the rescale to the type's scale (DecimalColumnVector semantics) then takes at most 18 steps
                if (s < 0 || s > 38 || s - t.scale > 18 || t.scale - s > 18) { bad = 1; break; }
                for (; s < t.scale; s++) {
                    if (v > INT64_MAX / 10 || v < INT64_MIN / 10) { bad = 1; break; }
                    v *= 10;
                }
                if (bad) break;
                for (; s > t.scale; s--) v /= 10;
            }
            store_val(t.out_data, t.out_width, t.row0 + i, (uint64_t)v);
        }
        bad |= d.bad | sc.s.bad;
    } else if (k == T_STRING || k == T_VARCHAR || k == T_CHAR || k == T_BINARY) {
        if (dict) {
            irle_init(len, t.length, t.length_n, v2, 0);
            int64_t acc = 0;
            for (int j = 0; j < t.dict_size && !bad; j++) {    // (stops where the LENGTH stream runs dry)
                t.dict_off[j] = (int32_t)acc;
                const int64_t l = irle_next(len);
                acc += l;
                if (len.s.bad || l < 0 || acc > t.dict_data_n || acc > 0x7fffffffLL) bad = 1;
            }
            if (t.dict_size < 0) bad = 1;
            if (!bad) t.dict_off[t.dict_size] = (int32_t)acc;
            IntRle &ids = r;
            irle_init(ids, t.data, t.data_n, v2, 0);
            for (int64_t i = 0; i < t.rows && !bad; i++) {
                const int ok = bool_next(pres);
                sink_put(sink, ok);
                int32_t l = 0;
                if (ok) {
                    const int64_t id = irle_next(ids);
                    if (id < 0 || id >= t.dict_size) { bad = 1; break; }
                    l = t.dict_off[id + 1] - t.dict_off[id];
                }
                t.out_offsets[t.row0 + i + 1] = l;
                payload += l;
            }
            bad |= ids.s.bad;
        } else {
            irle_init(len, t.length, t.length_n, v2, 0);
            for (int64_t i = 0; i < t.rows; i++) {
                const int ok = bool_next(pres);
                sink_put(sink, ok);
                int64_t l = ok ? irle_next(len) : 0;
                if (l < 0 || l > 0x7fffffffLL) { bad = 1; break; }
                t.out_offsets[t.row0 + i + 1] = (int32_t)l;
                payload += l;
            }
            bad |= len.s.bad;
            if (payload > t.data_n) bad = 1;
        }
    } else bad = 1;
    sink_flush(sink);
    bad |= pres.b.s.bad && !pres.all;
    t.payload_bytes = bad ? 0 : payload;
    t.bad = bad;
}

// phase B (var-len columns): the payload bytes at their final offsets (out_offsets is scanned by now)
ORC_HD inline void decode_task_b(Task &t) {
    const int k = t.kind;
    if (!(k == T_STRING || k == T_VARCHAR || k == T_CHAR || k == T_BINARY) || t.bad) return;
    BoolRle pres;
    bool_init(pres, t.present, t.present_n);
    const bool v2 = t.enc == ENC_DIRECT_V2 || t.enc == ENC_DICTIONARY_V2;
    const bool dict = t.enc == ENC_DICTIONARY || t.enc == ENC_DICTIONARY_V2;
    if (dict) {
        IntRle ids;
        irle_init(ids, t.data, t.data_n, v2, 0);
        for (int64_t i = 0; i < t.rows; i++) {
            if (!bool_next(pres)) continue;
            const int64_t id = irle_next(ids);
            if (id < 0 || id >= t.dict_size) { t.bad = 1; return; }
            const uint8_t *src = t.dict_data + t.dict_off[id];
            const int32_t l = t.dict_off[id + 1] - t.dict_off[id];
            uint8_t *dst = t.out_payload + t.out_offsets[t.row0 + i];
            for (int32_t b = 0; b < l; b++) dst[b] = src[b];
        }
    } else {
        // the DATA stream is the concatenation of the non-null values: one contiguous copy
        const int64_t o0 = t.out_offsets[t.row0], o1 = t.out_offsets[t.row0 + t.rows];
        uint8_t *dst = t.out_payload + o0;
        for (int64_t b = 0; b < o1 - o0; b++) dst[b] = t.data[b];
    }
}

}  // namespace orcdev
