// zstd_device.cuh — Zstandard frame decoder for Parquet pages, written once for host and device.
//
// Paimon's default 'file.compression' is zstd (paimon-api/.../CoreOptions.java:318-321; the Parquet writer takes it
// in ParquetFileFormat.java:98-101).  The reference hands compressed pages to zstd-jni 1.5.5-11 through parquet-mr's
// codec factory; that dependency is not under /root/reference.  The algorithm restated here is the public
// Zstandard format specification (RFC 8878): frame header, raw / RLE / compressed blocks, literals section (raw, RLE,
// Huffman with 1 or 4 streams, treeless), Huffman tree descriptions (direct or FSE-compressed weights), sequences
// section (predefined / RLE / FSE-compressed / repeat tables, three interleaved FSE states read from a backward
// bit stream, repeat offsets) and sequence execution.  No dictionaries (Parquet pages never use them), content
// checksums are skipped, skippable frames are skipped; a frame that declares its content size must produce exactly it.
//
// One decoder instance = one page = one warp on the device: every lane runs the same control flow over the same
// bytes (the stream is inherently sequential), byte moves are lane-parallel (literal copies, match copies — a match
// may overlap its own output: byte i comes from out - offset + (i mod offset)) and the four Huffman literal streams
// are decoded by four lanes.  The same source compiles for the host (tests/native/codec_host_check.cc runs it under
// sanitizers: tests/test_zstd_cpu.py pins it against pyarrow-compressed buffers, tests/test_codecs_cpu.py fuzzes it
// against libzstd).
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define ZS_HD __host__ __device__
#else
#define ZS_HD
#endif

namespace zs {

constexpr int kMaxBlock = 128 * 1024;
constexpr int kLLLog = 9, kOFLog = 8, kMLLog = 9, kHufLog = 11;
constexpr int kLLDefLog = 6, kOFDefLog = 5, kMLDefLog = 6;

// predefined distributions of the sequence codes (RFC 8878 §3.1.1.3.2.2), as initialisers of local arrays so that the
// decoder and the encoder (zstd_encode_device.cuh) read the same numbers on the host and on the device
#define ZS_LL_DEFAULT_NORM {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, \
                            -1, -1, -1, -1}
#define ZS_ML_DEFAULT_NORM {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, \
                            1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1}
#define ZS_OF_DEFAULT_NORM {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1}

struct FseEntry { uint16_t base; uint8_t sym; uint8_t nbits; };
struct HufEntry { uint8_t sym; uint8_t nbits; };

// the tables of one decoder: shared memory on the device (one set per warp), ordinary memory on the host
struct Tables {
    FseEntry ll[1 << kLLLog];
    FseEntry of[1 << kOFLog];
    FseEntry ml[1 << kMLLog];
    HufEntry huf[1 << kHufLog];
    FseEntry wtab[64];           // FSE table of a Huffman tree description (accuracy log <= 6)
    int ll_log, of_log, ml_log, huf_log;
    int have_huf, have_ll, have_of, have_ml;
    uint8_t weights[256];
    int16_t norm[64];
    uint16_t next[64];
};

ZS_HD inline int lane_id() {
#if defined(__CUDA_ARCH__)
    return threadIdx.x & 31;
#else
    return 0;
#endif
}
ZS_HD inline void warp_sync() {
#if defined(__CUDA_ARCH__)
    __syncwarp();
#endif
}
// lane 0's value for every lane (tables are built by lane 0 only: the builders update shared state in place, which
// 32 lanes running ahead of each other would corrupt)
ZS_HD inline int bcast0(int v) {
#if defined(__CUDA_ARCH__)
    __syncwarp();
    return __shfl_sync(0xffffffffu, v, 0);
#else
    return v;
#endif
}
ZS_HD inline int highbit(uint32_t v) {                 // position of the highest set bit, v != 0
#if defined(__CUDA_ARCH__)
    return 31 - __clz((int)v);
#else
    return 31 - __builtin_clz(v);
#endif
}

// forward copy dst[i] = src[i], the regions do not overlap (or src is behind dst by at least n).
// (sequences of columnar data are short — a few literal bytes, a match of the previous value's high bytes — so the
// <= 32-byte case is one predicated byte move, no loop)
ZS_HD inline void copy_bytes(uint8_t *dst, const uint8_t *src, int64_t n) {
#if defined(__CUDA_ARCH__)
    const int l = lane_id(), m = (int)n;
    if (m <= 32) { if (l < m) dst[l] = src[l]; }
    else for (int i = l; i < m; i += 32) dst[i] = src[i];
    __syncwarp();
#else
    for (int64_t i = 0; i < n; i++) dst[i] = src[i];
#endif
}
ZS_HD inline void fill_bytes(uint8_t *dst, uint8_t v, int64_t n) {
#if defined(__CUDA_ARCH__)
    for (int i = lane_id(); i < (int)n; i += 32) dst[i] = v;
    __syncwarp();
#else
    for (int64_t i = 0; i < n; i++) dst[i] = v;
#endif
}
// match copy: dst[i] = dst[i - offset]; overlapping when offset < n (then dst[i] = from[i mod offset])
ZS_HD inline void copy_match(uint8_t *dst, int64_t offset, int64_t n) {
    const uint8_t *from = dst - offset;
#if defined(__CUDA_ARCH__)
    const int l = lane_id(), m = (int)n;
    if (offset >= n) {
        if (m <= 32) { if (l < m) dst[l] = from[l]; }
        else for (int i = l; i < m; i += 32) dst[i] = from[i];
    } else if (offset == 1) {
        const uint8_t v = from[0];
        for (int i = l; i < m; i += 32) dst[i] = v;
    } else {
        const uint32_t o = (uint32_t)offset;
        for (int i = l; i < m; i += 32) dst[i] = from[(uint32_t)i % o];
    }
    __syncwarp();
#else
    for (int64_t i = 0; i < n; i++) dst[i] = from[i];
#endif
}

// ---- backward bit stream (RFC 8878 §4.1): bits are read from the end of the buffer towards its start; the last
// byte carries a 1-bit end mark above the last data bit
struct BitsR {
    const uint8_t *p;
    int len;              // bytes in the stream (a block is <= 128 KiB: bit positions fit an int)
    int nbits;            // bits not read yet
    int bad;
    uint64_t w;           // cached window: stream bits [base, base + 64), refilled as the read position moves down
    int base;             // (a read costs a shift and a mask instead of up to 8 byte loads)
};
ZS_HD inline void bits_init(BitsR &b, const uint8_t *p, int64_t len) {
    b.p = p;
    b.len = (int)len;
    b.bad = 0;
    b.w = 0;
    b.base = 1 << 30;                                   // no window yet: every position is below it
    if (len <= 0 || len > (1 << 27) || p[len - 1] == 0) { b.nbits = 0; b.bad = 1; return; }
    b.nbits = 8 * ((int)len - 1) + highbit(p[len - 1]);
}
// the n bits below the read position (n <= 32); positions before the start of the stream read as zero
ZS_HD inline uint32_t bits_peek_at(BitsR &b, int pos, int n) {
    if (n == 0) return 0;
    const uint32_t mask = n >= 32 ? 0xffffffffu : ((1u << n) - 1);
    if (pos >= 0) {
        // (unsigned compare: pos below the window wraps to a huge value)
        if ((unsigned)(pos - b.base) > (unsigned)(64 - n)) {
            // window whose top byte holds bit pos + n - 1: it reaches 57+ bits below the read position
            int nb = ((pos + n + 7) & ~7) - 64;
            if (nb < 0) nb = 0;
            const int byte0 = nb >> 3;
            const uint8_t *q = b.p + byte0;
            uint64_t v = 0;
            if (byte0 + 8 <= b.len) {
#pragma unroll
                for (int i = 0; i < 8; i++) v |= (uint64_t)q[i] << (8 * i);
            } else {
                for (int i = 0; i < 8; i++)
                    if (byte0 + i < b.len) v |= (uint64_t)q[i] << (8 * i);
            }
            b.w = v;
            b.base = nb;
        }
        return (uint32_t)(b.w >> (pos - b.base)) & mask;
    }
    // (rare: the read reaches below the first bit)
    const int shift = -pos;
    if (shift >= n) return 0;
    uint64_t v = 0;
    const int need = (pos + n + 7) >> 3;                   // bytes that hold the bits
    for (int i = 0; i < need && i < 8; i++) v |= (uint64_t)b.p[i] << (8 * i);
    v <<= shift;
    return (uint32_t)v & mask;
}
ZS_HD inline uint32_t bits_read(BitsR &b, int n) {
    b.nbits -= n;
    return bits_peek_at(b, b.nbits, n);
}

// ---- FSE table description (RFC 8878 §4.1.1): normalised counts -> decoding table
// Returns the number of bytes consumed, or -1.
ZS_HD inline int fse_read_table(const uint8_t *p, int len, int max_log, int max_sym, FseEntry *table, int *out_log, Tables &T) {
    if (len < 1) return -1;
    // forward bit reader, little endian
    int64_t bitpos = 0;
    const int64_t total_bits = (int64_t)len * 8;
    auto rd = [&](int n) -> uint32_t {
        uint64_t v = 0;
        const int64_t b0 = bitpos >> 3;
        for (int i = 0; i < 5 && b0 + i < len; i++) v |= (uint64_t)p[b0 + i] << (8 * i);
        v >>= (bitpos & 7);
        bitpos += n;
        return (uint32_t)(v & ((1ull << n) - 1));
    };
    const int log = (int)rd(4) + 5;
    if (log > max_log) return -1;
    int remaining = (1 << log) + 1;
    int sym = 0;
    for (int i = 0; i < 64; i++) T.norm[i] = 0;
    while (remaining > 1 && sym <= max_sym) {
        if (bitpos > total_bits) return -1;
        const int nb = highbit((uint32_t)remaining) + 1;            // bits of values up to `remaining`
        const int lower_mask = (1 << (nb - 1)) - 1;
        const int threshold = (1 << nb) - 1 - remaining;
        // a value takes nb - 1 bits when its low bits are below `threshold`, else nb bits
        const uint32_t full = rd(nb);
        int val;
        if ((int)(full & lower_mask) < threshold) { val = (int)(full & lower_mask); bitpos -= 1; }
        else { val = (int)full; if (val >= (1 << (nb - 1))) val -= threshold; }
        const int prob = val - 1;                                  // -1 = "less than 1"
        remaining -= prob < 0 ? 1 : prob;
        T.norm[sym++] = (int16_t)prob;
        if (prob == 0) {
            // zero run: 2-bit repeat counts, 3 = more follow
            while (true) {
                const int rep = (int)rd(2);
                for (int r = 0; r < rep && sym <= max_sym; r++) T.norm[sym++] = 0;
                if (rep != 3) break;
                if (bitpos > total_bits) return -1;
            }
        }
    }
    if (remaining != 1 || sym > max_sym + 1) return -1;
    const int n_sym = sym;
    // build (RFC 8878 §4.1.1 "from normalized distribution to decoding tables")
    const int size = 1 << log;
    int high = size - 1;
    for (int s = 0; s < n_sym; s++) {
        if (T.norm[s] == -1) { table[high].sym = (uint8_t)s; high--; T.next[s] = 1; }
        else T.next[s] = (uint16_t)T.norm[s];
    }
    const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
    int pos = 0;
    for (int s = 0; s < n_sym; s++) {
        for (int i = 0; i < T.norm[s]; i++) {
            table[pos].sym = (uint8_t)s;
            do { pos = (pos + step) & mask; } while (pos > high);
        }
    }
    if (pos != 0) return -1;
    for (int i = 0; i < size; i++) {
        const int s = table[i].sym;
        const int x = T.next[s]++;
        const int nb = log - highbit((uint32_t)x);
        table[i].nbits = (uint8_t)nb;
        table[i].base = (uint16_t)((x << nb) - size);
    }
    *out_log = log;
    return (int)((bitpos + 7) >> 3);
}

ZS_HD inline void fse_build_predefined(const int8_t *dist, int n_sym, int log, FseEntry *table, Tables &T) {
    const int size = 1 << log;
    int high = size - 1;
    for (int s = 0; s < n_sym; s++) {
        T.norm[s] = dist[s];
        if (dist[s] == -1) { table[high].sym = (uint8_t)s; high--; T.next[s] = 1; }
        else T.next[s] = (uint16_t)dist[s];
    }
    const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
    int pos = 0;
    for (int s = 0; s < n_sym; s++)
        for (int i = 0; i < T.norm[s]; i++) {
            table[pos].sym = (uint8_t)s;
            do { pos = (pos + step) & mask; } while (pos > high);
        }
    for (int i = 0; i < size; i++) {
        const int s = table[i].sym;
        const int x = T.next[s]++;
        const int nb = log - highbit((uint32_t)x);
        table[i].nbits = (uint8_t)nb;
        table[i].base = (uint16_t)((x << nb) - size);
    }
}

// ---- Huffman tree description (RFC 8878 §4.2.1) -> single-symbol decoding table.  Returns bytes consumed or -1.
ZS_HD inline int huf_read_table(const uint8_t *p, int len, Tables &T) {
    if (len < 1) return -1;
    const int hb = p[0];
    int n_w = 0, used = 1;
    if (hb >= 128) {
        n_w = hb - 127;
        const int nbytes = (n_w + 1) / 2;
        if (1 + nbytes > len) return -1;
        for (int i = 0; i < n_w; i++) {
            const uint8_t b = p[1 + i / 2];
            T.weights[i] = (i & 1) ? (b & 15) : (b >> 4);
        }
        used = 1 + nbytes;
    } else {
        // FSE-compressed weights: table (accuracy log <= 6), then two interleaved states over a backward stream
        if (1 + hb > len || hb < 1) return -1;
        FseEntry *tab = T.wtab;
        int log = 0;
        const int hdr = fse_read_table(p + 1, hb, 6, 12, tab, &log, T);         // weights 0..11 (12 bounds the alphabet)
        if (hdr < 0 || hdr >= hb) return -1;
        BitsR br;
        bits_init(br, p + 1 + hdr, hb - hdr);
        if (br.bad) return -1;
        uint32_t s1 = bits_read(br, log), s2 = bits_read(br, log);
        while (true) {
            if (n_w >= 255) return -1;
            T.weights[n_w++] = tab[s1].sym;
            if (br.nbits < (int64_t)tab[s1].nbits) { if (n_w >= 255) return -1; T.weights[n_w++] = tab[s2].sym; break; }
            s1 = tab[s1].base + bits_read(br, tab[s1].nbits);
            if (n_w >= 255) return -1;
            T.weights[n_w++] = tab[s2].sym;
            if (br.nbits < (int64_t)tab[s2].nbits) { if (n_w >= 255) return -1; T.weights[n_w++] = tab[s1].sym; break; }
            s2 = tab[s2].base + bits_read(br, tab[s2].nbits);
        }
        used = 1 + hb;
    }
    // last weight is implied: the weights must sum (as 2^(w-1)) to a power of two
    uint32_t sum = 0;
    for (int i = 0; i < n_w; i++) {
        if (T.weights[i] > kHufLog) return -1;
        if (T.weights[i]) sum += 1u << (T.weights[i] - 1);
    }
    if (sum == 0) return -1;
    const int max_bits = highbit(sum) + 1;
    if (max_bits > kHufLog) return -1;
    const uint32_t rest = (1u << max_bits) - sum;
    if (rest == 0 || (rest & (rest - 1))) return -1;
    T.weights[n_w++] = (uint8_t)(highbit(rest) + 1);
    // table: for weight w ascending, symbols in natural order, each takes 2^(w-1) consecutive entries
    uint32_t rank_start[kHufLog + 2];
    uint32_t cnt[kHufLog + 2];
    for (int w = 0; w <= kHufLog + 1; w++) cnt[w] = 0;
    for (int i = 0; i < n_w; i++) cnt[T.weights[i]]++;
    uint32_t nxt = 0;
    for (int w = 1; w <= max_bits; w++) { rank_start[w] = nxt; nxt += cnt[w] << (w - 1); }
    if (nxt != (1u << max_bits)) return -1;
    for (int s = 0; s < n_w; s++) {
        const int w = T.weights[s];
        if (!w) continue;
        const uint32_t n = 1u << (w - 1);
        const uint8_t nb = (uint8_t)(max_bits + 1 - w);
        for (uint32_t i = 0; i < n; i++) { T.huf[rank_start[w] + i].sym = (uint8_t)s; T.huf[rank_start[w] + i].nbits = nb; }
        rank_start[w] += n;
    }
    T.huf_log = max_bits;
    T.have_huf = 1;
    return used;
}

// one Huffman stream: `count` symbols into dst.  Returns 0 / -1.
ZS_HD inline int huf_decode_stream(const uint8_t *p, int len, uint8_t *dst, int count, const Tables &T) {
    BitsR br;
    bits_init(br, p, len);
    if (br.bad) return -1;
    const int log = T.huf_log;
    for (int i = 0; i < count; i++) {
        const uint32_t idx = bits_peek_at(br, br.nbits - log, log);
        const HufEntry e = T.huf[idx];
        br.nbits -= e.nbits;
        dst[i] = e.sym;
    }
    return br.nbits == 0 ? 0 : -1;
}

struct Literals {
    const uint8_t *ptr;      // raw / decoded literals (NULL for RLE)
    int size;
    int rle;                 // 1: `size` copies of `value`
    uint8_t value;
};

// literals section (RFC 8878 §3.1.1.3.1).  `lit_buf` (kMaxBlock bytes, private to this decoder) receives Huffman
// output.  Returns bytes consumed or -1.
ZS_HD inline int read_literals(const uint8_t *p, int len, uint8_t *lit_buf, Tables &T, Literals &L) {
    if (len < 1) return -1;
    const int type = p[0] & 3, fmt = (p[0] >> 2) & 3;
    if (type < 2) {
        int hdr, size;
        if (fmt == 0 || fmt == 2) { hdr = 1; size = p[0] >> 3; }
        else if (fmt == 1) { if (len < 2) return -1; hdr = 2; size = (p[0] >> 4) | (p[1] << 4); }
        else { if (len < 3) return -1; hdr = 3; size = (p[0] >> 4) | (p[1] << 4) | (p[2] << 12); }
        if (size > kMaxBlock) return -1;
        if (type == 0) {
            if (hdr + size > len) return -1;
            L.ptr = p + hdr; L.size = size; L.rle = 0; L.value = 0;
            return hdr + size;
        }
        if (hdr + 1 > len) return -1;
        L.ptr = nullptr; L.size = size; L.rle = 1; L.value = p[hdr];
        return hdr + 1;
    }
    int hdr, regen, comp, streams;
    if (fmt == 0 || fmt == 1) {
        if (len < 3) return -1;
        const uint32_t h = p[0] | (p[1] << 8) | (p[2] << 16);
        hdr = 3; regen = (h >> 4) & 0x3ff; comp = (h >> 14) & 0x3ff; streams = fmt == 0 ? 1 : 4;
    } else if (fmt == 2) {
        if (len < 4) return -1;
        const uint32_t h = p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24);
        hdr = 4; regen = (h >> 4) & 0x3fff; comp = (h >> 18) & 0x3fff; streams = 4;
    } else {
        if (len < 5) return -1;
        const uint64_t h = (uint64_t)p[0] | ((uint64_t)p[1] << 8) | ((uint64_t)p[2] << 16) | ((uint64_t)p[3] << 24) | ((uint64_t)p[4] << 32);
        hdr = 5; regen = (int)((h >> 4) & 0x3ffff); comp = (int)((h >> 22) & 0x3ffff); streams = 4;
    }
    if (regen > kMaxBlock || hdr + comp > len) return -1;
    const uint8_t *q = p + hdr;
    int left = comp;
    if (type == 2) {
        int used = 0;
        if (lane_id() == 0) used = huf_read_table(q, left, T);
        used = bcast0(used);                               // (the table is in place for every lane)
        if (used < 0) return -1;
        q += used; left -= used;
    } else {
        warp_sync();
        if (!T.have_huf) return -1;
    }
    int rc = 0;
    if (streams == 1) {
        if (lane_id() == 0) rc = huf_decode_stream(q, left, lit_buf, regen, T);
    } else {
        if (left < 6) return -1;
        const int s1 = q[0] | (q[1] << 8), s2 = q[2] | (q[3] << 8), s3 = q[4] | (q[5] << 8);
        const int s4 = left - 6 - s1 - s2 - s3;
        if (s4 < 1 || s1 < 1 || s2 < 1 || s3 < 1) return -1;
        const int per = (regen + 3) / 4;
        const int last = regen - 3 * per;
        if (last < 0) return -1;
        const uint8_t *b = q + 6;
#if defined(__CUDA_ARCH__)
        const int l = lane_id();
        if (l == 0) rc = huf_decode_stream(b, s1, lit_buf, per, T);
        else if (l == 1) rc = huf_decode_stream(b + s1, s2, lit_buf + per, per, T);
        else if (l == 2) rc = huf_decode_stream(b + s1 + s2, s3, lit_buf + 2 * per, per, T);
        else if (l == 3) rc = huf_decode_stream(b + s1 + s2 + s3, s4, lit_buf + 3 * per, last, T);
#else
        rc |= huf_decode_stream(b, s1, lit_buf, per, T);
        rc |= huf_decode_stream(b + s1, s2, lit_buf + per, per, T);
        rc |= huf_decode_stream(b + s1 + s2, s3, lit_buf + 2 * per, per, T);
        rc |= huf_decode_stream(b + s1 + s2 + s3, s4, lit_buf + 3 * per, last, T);
#endif
    }
#if defined(__CUDA_ARCH__)
    __syncwarp();                                           // lanes 0..3 wrote lit_buf: order it before every lane reads
    rc = __any_sync(0xffffffffu, rc != 0) ? -1 : 0;        // (a vote alone implies no memory ordering)
#endif
    if (rc) return -1;
    L.ptr = lit_buf; L.size = regen; L.rle = 0; L.value = 0;
    return hdr + comp;
}

ZS_HD inline void ll_code_info(int code, uint32_t &base, int &bits) {
    if (code < 16) { base = (uint32_t)code; bits = 0; return; }
    const uint32_t b[20] = {16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
    const int n[20] = {1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
    base = b[code - 16]; bits = n[code - 16];
}
ZS_HD inline void ml_code_info(int code, uint32_t &base, int &bits) {
    if (code < 32) { base = (uint32_t)code + 3; bits = 0; return; }
    const uint32_t b[21] = {35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539};
    const int n[21] = {1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
    base = b[code - 32]; bits = n[code - 32];
}

// one symbol-compression mode of the sequences section -> table.  Returns bytes consumed or -1.
ZS_HD inline int read_seq_table(int mode, const uint8_t *p, int len, int max_log, int max_sym, const int8_t *predef, int predef_n,
                                int predef_log, FseEntry *table, int *log, int *have, Tables &T) {
    if (mode == 0) { fse_build_predefined(predef, predef_n, predef_log, table, T); *log = predef_log; *have = 1; return 0; }
    if (mode == 1) {
        if (len < 1 || p[0] > max_sym) return -1;
        table[0].sym = p[0]; table[0].nbits = 0; table[0].base = 0;
        *log = 0; *have = 1;
        return 1;
    }
    if (mode == 2) {
        const int used = fse_read_table(p, len, max_log, max_sym, table, log, T);
        if (used < 0) return -1;
        *have = 1;
        return used;
    }
    return *have ? 0 : -1;                                  // repeat: the previous block's table
}

struct FrameState {
    uint32_t rep[3];
};

// one compressed block.  `out` = where the block's bytes go, `out_start` = first byte of the frame's output (matches
// may reach back into earlier blocks), `cap` = room left.  Returns bytes produced or -1.
ZS_HD inline int64_t decode_block(const uint8_t *p, int len, uint8_t *out, const uint8_t *out_start, int64_t cap,
                                  uint8_t *lit_buf, Tables &T, FrameState &F) {
    Literals L;
    const int lit_used = read_literals(p, len, lit_buf, T, L);
    if (lit_used < 0) return -1;
    const uint8_t *q = p + lit_used;
    int left = len - lit_used;
    if (left < 1) return -1;
    int n_seq = q[0], used = 1;
    if (n_seq >= 128) {
        if (n_seq < 255) { if (left < 2) return -1; n_seq = ((n_seq - 128) << 8) + q[1]; used = 2; }
        else { if (left < 3) return -1; n_seq = q[1] + (q[2] << 8) + 0x7F00; used = 3; }
    }
    int64_t produced = 0;
    int lit_pos = 0;
    auto put_literals = [&](int n) -> bool {
        if (n > L.size - lit_pos || produced + n > cap) return false;
        if (L.rle) fill_bytes(out + produced, L.value, n);
        else copy_bytes(out + produced, L.ptr + lit_pos, n);
        lit_pos += n;
        produced += n;
        return true;
    };
    if (n_seq > 0) {
        q += used; left -= used;
        if (left < 1) return -1;
        const int modes = q[0];
        if (modes & 3) return -1;
        q++; left--;
        const int8_t ll_def[36] = ZS_LL_DEFAULT_NORM;
        const int8_t ml_def[53] = ZS_ML_DEFAULT_NORM;
        const int8_t of_def[29] = ZS_OF_DEFAULT_NORM;
        int u = 0;
        if (lane_id() == 0) u = read_seq_table((modes >> 6) & 3, q, left, kLLLog, 35, ll_def, 36, 6, T.ll, &T.ll_log, &T.have_ll, T);
        u = bcast0(u);
        if (u < 0) return -1;
        q += u; left -= u;
        if (lane_id() == 0) u = read_seq_table((modes >> 4) & 3, q, left, kOFLog, 31, of_def, 29, 5, T.of, &T.of_log, &T.have_of, T);
        u = bcast0(u);
        if (u < 0) return -1;
        q += u; left -= u;
        if (lane_id() == 0) u = read_seq_table((modes >> 2) & 3, q, left, kMLLog, 52, ml_def, 53, 6, T.ml, &T.ml_log, &T.have_ml, T);
        u = bcast0(u);
        if (u < 0) return -1;
        q += u; left -= u;
        BitsR br;
        bits_init(br, q, left);
        if (br.bad) return -1;
        uint32_t sl = bits_read(br, T.ll_log), so = bits_read(br, T.of_log), sm = bits_read(br, T.ml_log);
        for (int i = 0; i < n_seq; i++) {
            const FseEntry el = T.ll[sl], eo = T.of[so], em = T.ml[sm];
            const int of_code = eo.sym;
            if (of_code > 31) return -1;
            uint32_t ofv = (1u << of_code) + bits_read(br, of_code);
            uint32_t mb, lb;
            int mbits, lbits;
            ml_code_info(em.sym, mb, mbits);
            ll_code_info(el.sym, lb, lbits);
            const uint32_t mlen = mb + bits_read(br, mbits);
            const uint32_t llen = lb + bits_read(br, lbits);
            if (i + 1 < n_seq) {
                sl = el.base + bits_read(br, el.nbits);
                sm = em.base + bits_read(br, em.nbits);
                so = eo.base + bits_read(br, eo.nbits);
            }
            if (br.nbits < 0) return -1;
            // repeat offsets (RFC 8878 §3.1.1.5)
            uint32_t offset;
            if (ofv > 3) {
                offset = ofv - 3;
                F.rep[2] = F.rep[1]; F.rep[1] = F.rep[0]; F.rep[0] = offset;
            } else {
                uint32_t idx = ofv - 1;                      // 0..2
                if (llen == 0) idx++;                        // 1..3
                if (idx == 0) offset = F.rep[0];
                else {
                    offset = idx < 3 ? F.rep[idx] : F.rep[0] - 1;
                    if (idx > 1) F.rep[2] = F.rep[1];
                    F.rep[1] = F.rep[0];
                    F.rep[0] = offset;
                }
            }
            if (!put_literals((int)llen)) return -1;
            if (offset == 0 || (int64_t)offset > (out + produced) - out_start || produced + mlen > cap) return -1;
            copy_match(out + produced, offset, mlen);
            produced += mlen;
        }
        if (br.nbits != 0) return -1;
    }
    if (!put_literals(L.size - lit_pos)) return -1;
    return produced;
}

// A whole zstd stream (one or more frames) -> dst.  Returns the number of bytes produced, or -1 when the stream is
// malformed / does not fit `cap`.  `lit_buf`: kMaxBlock bytes private to this decoder; `T`: its tables.
ZS_HD inline int64_t decode(const uint8_t *src, int64_t n, uint8_t *dst, int64_t cap, uint8_t *lit_buf, Tables &T) {
    int64_t pos = 0, out = 0;
    while (pos < n) {
        if (n - pos < 4) return -1;
        const uint32_t magic = src[pos] | (src[pos + 1] << 8) | (src[pos + 2] << 16) | ((uint32_t)src[pos + 3] << 24);
        if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {         // skippable frame
            if (n - pos < 8) return -1;
            const uint32_t sz = src[pos + 4] | (src[pos + 5] << 8) | (src[pos + 6] << 16) | ((uint32_t)src[pos + 7] << 24);
            if ((int64_t)sz > n - pos - 8) return -1;
            pos += 8 + (int64_t)sz;
            continue;
        }
        if (magic != 0xFD2FB528u) return -1;
        pos += 4;
        if (pos >= n) return -1;
        const int fhd = src[pos++];
        const int fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, checksum = (fhd >> 2) & 1, did_flag = fhd & 3;
        if (fhd & 8) return -1;                             // reserved bit
        if (!single) pos += 1;                              // window descriptor
        const int did_bytes = did_flag == 0 ? 0 : (did_flag == 1 ? 1 : (did_flag == 2 ? 2 : 4));
        for (int i = 0; i < did_bytes; i++) if (pos + i < n && src[pos + i]) return -1;   // dictionaries: not in Parquet pages
        pos += did_bytes;
        const int fcs_bytes = fcs_flag == 0 ? (single ? 1 : 0) : (fcs_flag == 1 ? 2 : (fcs_flag == 2 ? 4 : 8));
        if (fcs_bytes > n - pos) return -1;
        uint64_t fcs = 0;                                   // frame content size: the frame must produce exactly it
        for (int i = 0; i < fcs_bytes; i++) fcs |= (uint64_t)src[pos + i] << (8 * i);
        if (fcs_bytes == 2) fcs += 256;
        pos += fcs_bytes;
        FrameState F;
        F.rep[0] = 1; F.rep[1] = 4; F.rep[2] = 8;
        warp_sync();
        if (lane_id() == 0) T.have_huf = T.have_ll = T.have_of = T.have_ml = 0;
        warp_sync();
        const int64_t frame_out = out;
        while (true) {
            if (n - pos < 3) return -1;
            const uint32_t bh = src[pos] | (src[pos + 1] << 8) | (src[pos + 2] << 16);
            pos += 3;
            const int last = bh & 1, type = (bh >> 1) & 3;
            const int64_t bsize = bh >> 3;
            if (type == 0) {
                if (bsize > n - pos || bsize > cap - out) return -1;
                copy_bytes(dst + out, src + pos, bsize);
                pos += bsize; out += bsize;
            } else if (type == 1) {
                if (n - pos < 1 || bsize > cap - out) return -1;
                fill_bytes(dst + out, src[pos], bsize);
                pos += 1; out += bsize;
            } else if (type == 2) {
                if (bsize > n - pos || bsize > kMaxBlock) return -1;
                const int64_t got = decode_block(src + pos, (int)bsize, dst + out, dst + frame_out, cap - out, lit_buf, T, F);
                if (got < 0) return -1;
                pos += bsize; out += got;
            } else return -1;
            if (last) break;
        }
        if (fcs_bytes && (uint64_t)(out - frame_out) != fcs) return -1;
        if (checksum) pos += 4;
        if (pos > n) return -1;
    }
    return out;
}

}  // namespace zs
