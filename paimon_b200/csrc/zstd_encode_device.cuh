// zstd_encode_device.cuh — Zstandard frame encoder for Parquet page bodies, written once for host and device.
//
// Paimon compresses every data file it writes with zstd level 1 unless told otherwise (CoreOptions.java:318-330,
// 'file.compression' / 'file.compression.zstd-level'), so the compaction output encoders write one zstd frame per
// Parquet page body or ORC compression chunk (ZstdFrames, encoded_file.cu).  The format is the public Zstandard specification (RFC 8878), the same one the decoder in
// zstd_device.cuh restates; the code tables (ll_code_info / ml_code_info) and the predefined distributions are that
// header's.
//
// What is written:
//   frame    single segment, Frame_Content_Size, no checksum, no dictionary; blocks of at most 128 KiB
//   block    Raw, RLE or Compressed, whichever is smallest
//   parse    greedy LZ77 inside the block, minimum match 4, candidates from a hash table of every position
//            (the most recent earlier position with the same 4-byte hash), positions taken in rounds of 32
//   literals raw, RLE, or Huffman (code lengths <= 11, 1 stream below 256 literals, else 4) with the weights written
//            direct or FSE-compressed, whichever is shorter
//   sequences LL / OF / ML each Predefined, RLE or FSE_Compressed, chosen per block by estimated bit cost; an offset
//            equal to a repeat offset is written as the repeat code once this block has set that repeat offset (the
//            blocks of a frame are compressed independently, so the history entering a block is not known)
//
// Unit of work = one block.  On the device a block is one warp: the 32 positions of a round look up the hash table
// together (__match_any_sync gives each position its most recent same-hash predecessor inside the round), a ballot
// finds the next position where a match starts, a match is extended 32 bytes per step, literal copies are
// lane-parallel; the entropy stage (histograms, Huffman / FSE tables, the bit streams) runs on lane 0.  The host build
// runs the same rounds serially and produces the same bytes, which is what tests/native/zstd_encode_host_check.cc
// checks against libzstd.
#pragma once

#include "zstd_device.cuh"

namespace zs {

constexpr int kMinMatch = 4;
constexpr int kHashLog = 13;                             // 32 KiB of shared memory per block encoder
constexpr int kRound = 32;                               // positions per parse round (one per lane)

struct Seq { uint32_t ll, ml, off; };                    // literal length, match length, offset (then offset value)

// scratch of one block encoder: shared memory on the device, ordinary memory on the host
struct FseCT {
    uint16_t state[1 << kLLLog];
    uint32_t dnb[64];                                    // deltaNbBits
    int32_t dfs[64];                                     // deltaFindState
    int log;
};
struct EncWork {
    uint32_t hist[256];
    uint32_t hcnt[256];
    uint16_t hcode[256];
    uint8_t hlen[256];
    uint8_t hweight[256];
    uint16_t hsym[256];
    uint32_t hw[512];
    uint16_t hparent[512];
    uint8_t hdepth[512];
    uint8_t spread[1 << kLLLog];
    uint32_t cnt[3][64];                                 // LL, OF, ML code histograms
    int16_t norm[3][64];
    FseCT ct[3];
};

struct BlockOut { int type, size; };                     // type: 0 raw, 1 RLE, 2 compressed; size: payload bytes

ZS_HD inline uint32_t rd32(const uint8_t *p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
ZS_HD inline uint32_t hash4(const uint8_t *p) { return (rd32(p) * 2654435761u) >> (32 - kHashLog); }

// ---- forward bit writer (LSB first); a write past `cap` marks the stream as overflowed instead of storing
struct BitW {
    uint8_t *p;
    int cap, pos, cnt, over;
    uint64_t acc;
};
ZS_HD inline void bw_init(BitW &b, uint8_t *p, int cap) { b.p = p; b.cap = cap; b.pos = 0; b.cnt = 0; b.over = 0; b.acc = 0; }
ZS_HD inline void bw_add(BitW &b, uint32_t v, int n) {  // v < 2^n, n <= 32
    b.acc |= (uint64_t)v << b.cnt;
    b.cnt += n;
    while (b.cnt >= 8) {
        if (b.pos < b.cap) b.p[b.pos] = (uint8_t)b.acc;
        else b.over = 1;
        b.pos++;
        b.acc >>= 8;
        b.cnt -= 8;
    }
}
ZS_HD inline int bw_flush_bytes(BitW &b) {               // pad the last byte with zeros; bytes written or -1
    if (b.cnt > 0) bw_add(b, 0, 8 - b.cnt);
    return b.over ? -1 : b.pos;
}
ZS_HD inline int bw_close(BitW &b) {                     // backward stream: end mark above the last bit
    bw_add(b, 1, 1);
    return bw_flush_bytes(b);
}

// ---- value -> code (the inverse of ll_code_info / ml_code_info)
ZS_HD inline int ll_code(uint32_t v) {
    if (v < 16) return (int)v;
    if (v < 24) return 16 + (int)(v - 16) / 2;
    if (v < 32) return 20 + (int)(v - 24) / 4;
    if (v < 48) return 22 + (int)(v - 32) / 8;
    if (v < 64) return 24;
    return highbit(v) + 19;
}
ZS_HD inline int ml_code(uint32_t ml) {                  // ml >= 3
    const uint32_t v = ml - 3;
    if (v < 32) return (int)v;
    if (v < 40) return 32 + (int)(v - 32) / 2;
    if (v < 48) return 36 + (int)(v - 40) / 4;
    if (v < 64) return 38 + (int)(v - 48) / 8;
    if (v < 96) return 40 + (int)(v - 64) / 16;
    if (v < 128) return 42;
    return highbit(v) + 36;
}

// 256 * log2(x), x >= 1 (linear between powers of two: integer, so host and device agree on every choice it drives)
ZS_HD inline uint32_t lg256(uint32_t x) {
    const int hb = highbit(x);
    const uint32_t f = hb >= 8 ? (x >> (hb - 8)) & 255u : (x << (8 - hb)) & 255u;
    return (uint32_t)hb * 256u + f;
}

// ---- FSE: normalised counts, table description, encoding table
// counts -> normalised counts summing to 2^log, every present symbol >= 1; `cap_half`: no symbol above 2^(log-1)
// (then every state of the table reads at least one bit, which the Huffman weight stream needs to end unambiguously)
ZS_HD inline void fse_normalize(const uint32_t *cnt, int n_sym, uint32_t total, int log, int16_t *norm, int cap_half) {
    const int size = 1 << log;
    int sum = 0, big = -1;
    for (int s = 0; s < n_sym; s++) {
        if (!cnt[s]) { norm[s] = 0; continue; }
        int v = (int)((((uint64_t)cnt[s] << log) + total / 2) / total);
        if (v < 1) v = 1;
        norm[s] = (int16_t)v;
        sum += v;
        if (big < 0 || cnt[s] > cnt[big]) big = s;
    }
    while (sum > size) {                                  // rounding and the minimum of 1 overshot: the largest give
        int m = -1;
        for (int s = 0; s < n_sym; s++) if (norm[s] > 1 && (m < 0 || norm[s] > norm[m])) m = s;
        norm[m]--;
        sum--;
    }
    if (sum < size) norm[big] = (int16_t)(norm[big] + size - sum);
    if (cap_half && norm[big] > size / 2) {
        int excess = norm[big] - size / 2;
        norm[big] = (int16_t)(size / 2);
        while (excess > 0)
            for (int s = 0; s < n_sym && excess > 0; s++)
                if (s != big && norm[s] > 0 && norm[s] < size / 2) { norm[s]++; excess--; }
    }
}

// estimated cost in 1/256 bits of coding the counts with a table; ~0 when a used symbol has no probability
ZS_HD inline uint64_t fse_cost(const uint32_t *cnt, int n_cnt, const int16_t *norm, int n_norm, int log) {
    uint64_t c = 0;
    for (int s = 0; s < n_cnt; s++) {
        if (!cnt[s]) continue;
        const int n = s < n_norm ? (norm[s] == -1 ? 1 : norm[s]) : 0;
        if (n <= 0) return ~0ull;
        c += (uint64_t)cnt[s] * ((uint32_t)log * 256u - lg256((uint32_t)n));
    }
    return c;
}

// the table description (RFC 8878 §4.1.1), the inverse of fse_read_table.  Returns bytes written or -1.
ZS_HD inline int fse_write_ncount(uint8_t *dst, int cap, const int16_t *norm, int n_sym, int log) {
    BitW b;
    bw_init(b, dst, cap);
    bw_add(b, (uint32_t)(log - 5), 4);
    int remaining = (1 << log) + 1, s = 0;
    while (remaining > 1 && s < n_sym) {
        const int prob = norm[s++];
        const int value = prob + 1;
        const int nb = highbit((uint32_t)remaining) + 1;
        const int threshold = (1 << nb) - 1 - remaining;
        if (value < threshold) bw_add(b, (uint32_t)value, nb - 1);
        else if (value < (1 << (nb - 1))) bw_add(b, (uint32_t)value, nb);
        else bw_add(b, (uint32_t)(value + threshold), nb);
        remaining -= prob < 0 ? 1 : prob;
        if (prob == 0) {
            int run = 0;
            while (s < n_sym && norm[s] == 0) { run++; s++; }
            while (run >= 3) { bw_add(b, 3, 2); run -= 3; }
            bw_add(b, (uint32_t)run, 2);
        }
    }
    if (remaining != 1) return -1;
    return bw_flush_bytes(b);
}

// symbol spread of the decoding table, as fse_read_table / fse_build_predefined lay it out
ZS_HD inline void fse_spread(const int16_t *norm, int n_sym, int log, uint8_t *spread) {
    const int size = 1 << log;
    int high = size - 1;
    for (int s = 0; s < n_sym; s++) if (norm[s] == -1) spread[high--] = (uint8_t)s;
    const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
    int pos = 0;
    for (int s = 0; s < n_sym; s++)
        for (int i = 0; i < norm[s]; i++) {
            spread[pos] = (uint8_t)s;
            do { pos = (pos + step) & mask; } while (pos > high);
        }
}

ZS_HD inline void fse_build_ct(const int16_t *norm, int n_sym, int log, FseCT &ct, uint8_t *spread) {
    fse_spread(norm, n_sym, log, spread);
    const int size = 1 << log;
    uint16_t cumul[64];
    int acc = 0;
    for (int s = 0; s < n_sym; s++) { cumul[s] = (uint16_t)acc; acc += norm[s] == -1 ? 1 : norm[s]; }
    for (int u = 0; u < size; u++) ct.state[cumul[spread[u]]++] = (uint16_t)(size + u);
    int total = 0;
    for (int s = 0; s < n_sym; s++) {
        const int n = norm[s];
        if (n == 0) { ct.dnb[s] = ((uint32_t)(log + 1) << 16) - (uint32_t)size; ct.dfs[s] = 0; }
        else if (n == -1 || n == 1) { ct.dnb[s] = ((uint32_t)log << 16) - (uint32_t)size; ct.dfs[s] = total - 1; total++; }
        else {
            const uint32_t mbo = (uint32_t)(log - highbit((uint32_t)(n - 1)));
            ct.dnb[s] = (mbo << 16) - ((uint32_t)n << mbo);
            ct.dfs[s] = total - n;
            total += n;
        }
    }
    ct.log = log;
}
ZS_HD inline uint32_t fse_init_state(const FseCT &ct, int s) {
    const uint32_t nb = (ct.dnb[s] + (1u << 15)) >> 16;
    const uint32_t v = (nb << 16) - ct.dnb[s];
    return ct.state[(int)(v >> nb) + ct.dfs[s]];
}
ZS_HD inline void fse_encode(BitW &b, const FseCT &ct, uint32_t &st, int s) {
    const uint32_t nb = (st + ct.dnb[s]) >> 16;
    bw_add(b, st & ((1u << nb) - 1), (int)nb);
    st = ct.state[(int)(st >> nb) + ct.dfs[s]];
}
ZS_HD inline void fse_flush(BitW &b, const FseCT &ct, uint32_t st) { bw_add(b, st & ((1u << ct.log) - 1), ct.log); }

// table log for n samples of an alphabet of n_sym symbols (RFC 8878 leaves it to the encoder; this is libzstd's rule)
ZS_HD inline int fse_table_log(int n, int n_sym, int max_log) {
    const int src_bits = highbit((uint32_t)(n > 1 ? n - 1 : 1));
    int log = src_bits - 2 < max_log ? src_bits - 2 : max_log;
    const int min_bits = (src_bits + 1) < (highbit((uint32_t)(n_sym > 1 ? n_sym - 1 : 1)) + 2)
                             ? src_bits + 1 : highbit((uint32_t)(n_sym > 1 ? n_sym - 1 : 1)) + 2;
    if (log < min_bits) log = min_bits;
    if (log < 5) log = 5;
    if (log > max_log) log = max_log;
    return log;
}

// ---- Huffman
// code lengths of the present symbols of W.hcnt (two-queue Huffman); returns the largest
ZS_HD inline int huf_depths(EncWork &W) {
    int n = 0;
    for (int s = 0; s < 256; s++) { W.hlen[s] = 0; if (W.hcnt[s]) W.hsym[n++] = (uint16_t)s; }
    for (int i = 1; i < n; i++) {                         // by (count, symbol)
        const uint16_t x = W.hsym[i];
        int k = i - 1;
        while (k >= 0 && W.hcnt[W.hsym[k]] > W.hcnt[x]) { W.hsym[k + 1] = W.hsym[k]; k--; }
        W.hsym[k + 1] = x;
    }
    if (n < 2) return 0;                                  // (callers have two symbols at least)
    for (int i = 0; i < n; i++) W.hw[i] = W.hcnt[W.hsym[i]];
    int leaf = 0, node = n, next = n;
    for (int k = 0; k < n - 1; k++) {
        int ab[2];
        for (int t = 0; t < 2; t++)
            ab[t] = (leaf < n && (node >= next || W.hw[leaf] <= W.hw[node])) ? leaf++ : node++;
        W.hw[next] = W.hw[ab[0]] + W.hw[ab[1]];
        W.hparent[ab[0]] = W.hparent[ab[1]] = (uint16_t)next;
        next++;
    }
    W.hdepth[2 * n - 2] = 0;
    for (int i = 2 * n - 3; i >= 0; i--) W.hdepth[i] = (uint8_t)(W.hdepth[W.hparent[i]] + 1);
    int maxd = 0;
    for (int i = 0; i < n; i++) {
        W.hlen[W.hsym[i]] = W.hdepth[i];
        if (W.hdepth[i] > maxd) maxd = W.hdepth[i];
    }
    return maxd;
}

// Huffman code of the histogram W.hist (>= 2 symbols): lengths <= kHufLog, weights and canonical codes laid out the way
// huf_read_table builds its decoding table.  Returns the largest code length.
ZS_HD inline int huf_build(EncWork &W) {
    for (int s = 0; s < 256; s++) W.hcnt[s] = W.hist[s];
    int max_bits;
    while ((max_bits = huf_depths(W)) > kHufLog)          // flatten until the limit holds
        for (int s = 0; s < 256; s++) if (W.hcnt[s]) W.hcnt[s] = (W.hcnt[s] + 1) >> 1;
    uint32_t start[kHufLog + 2], cw[kHufLog + 2];
    for (int w = 0; w <= kHufLog + 1; w++) cw[w] = 0;
    for (int s = 0; s < 256; s++) {
        W.hweight[s] = W.hlen[s] ? (uint8_t)(max_bits + 1 - W.hlen[s]) : 0;
        cw[W.hweight[s]]++;
    }
    uint32_t nxt = 0;
    for (int w = 1; w <= max_bits; w++) { start[w] = nxt; nxt += cw[w] << (w - 1); }
    for (int s = 0; s < 256; s++) {
        const int w = W.hweight[s];
        if (!w) continue;
        W.hcode[s] = (uint16_t)(start[w] >> (w - 1));
        start[w] += 1u << (w - 1);
    }
    return max_bits;
}

// Huffman tree description: the weights of symbols [0, last_sym) (the last one is implied), FSE-compressed or direct,
// whichever is shorter.  Returns bytes written or -1.
ZS_HD inline int huf_write_tree(uint8_t *dst, int cap, int last_sym, EncWork &W) {
    const int n_w = last_sym;
    int best = -1;
    if (n_w >= 2 && cap >= 2) {
        uint32_t wc[16];
        int max_w = 0, distinct = 0;
        for (int w = 0; w < 16; w++) wc[w] = 0;
        for (int i = 0; i < n_w; i++) { wc[W.hweight[i]]++; if (W.hweight[i] > max_w) max_w = W.hweight[i]; }
        for (int w = 0; w <= max_w; w++) distinct += wc[w] != 0;
        if (distinct >= 2) {
            const int log = 6;
            int16_t *norm = W.norm[0];
            fse_normalize(wc, max_w + 1, (uint32_t)n_w, log, norm, 1);
            const int lim = cap - 1 < 127 ? cap - 1 : 127;
            const int hdr = fse_write_ncount(dst + 1, lim, norm, max_w + 1, log);
            if (hdr > 0 && hdr < lim) {
                FseCT &ct = W.ct[0];
                fse_build_ct(norm, max_w + 1, log, ct, W.spread);
                BitW b;
                bw_init(b, dst + 1 + hdr, lim - hdr);
                const uint8_t *w = W.hweight;
                int ip = n_w;
                uint32_t s1, s2;
                if (n_w & 1) {
                    s1 = fse_init_state(ct, w[--ip]);
                    s2 = fse_init_state(ct, w[--ip]);
                    fse_encode(b, ct, s1, w[--ip]);
                } else {
                    s2 = fse_init_state(ct, w[--ip]);
                    s1 = fse_init_state(ct, w[--ip]);
                }
                while (ip > 0) {
                    fse_encode(b, ct, s2, w[--ip]);
                    fse_encode(b, ct, s1, w[--ip]);
                }
                fse_flush(b, ct, s2);
                fse_flush(b, ct, s1);
                const int sb = bw_close(b);
                if (sb > 0 && hdr + sb <= 127) { dst[0] = (uint8_t)(hdr + sb); best = 1 + hdr + sb; }
            }
        }
    }
    if (n_w <= 128) {
        const int size = 1 + (n_w + 1) / 2;
        if ((best < 0 || size < best) && size <= cap) {
            dst[0] = (uint8_t)(127 + n_w);
            for (int i = 0; i < n_w; i += 2)
                dst[1 + i / 2] = (uint8_t)((W.hweight[i] << 4) | (i + 1 < n_w ? W.hweight[i + 1] : 0));
            best = size;
        }
    }
    return best;
}

ZS_HD inline int huf_stream(const uint8_t *lit, int n, uint8_t *dst, int cap, const EncWork &W) {
    BitW b;
    bw_init(b, dst, cap);
    for (int i = n - 1; i >= 0; i--) bw_add(b, W.hcode[lit[i]], W.hlen[lit[i]]);
    return bw_close(b);
}

// ---- literals section (RFC 8878 §3.1.1.3.1).  Returns bytes written or -1 when it does not fit `cap`.
ZS_HD inline int lit_header_raw(uint8_t *d, int type, int n) {
    if (n < 32) { d[0] = (uint8_t)(type | (n << 3)); return 1; }
    if (n < 4096) { d[0] = (uint8_t)(type | (1 << 2) | ((n & 15) << 4)); d[1] = (uint8_t)(n >> 4); return 2; }
    d[0] = (uint8_t)(type | (3 << 2) | ((n & 15) << 4)); d[1] = (uint8_t)(n >> 4); d[2] = (uint8_t)(n >> 12); return 3;
}
ZS_HD inline int write_literals(const uint8_t *lit, int n, uint8_t *dst, int cap, EncWork &W) {
    const int raw_hdr = n < 32 ? 1 : (n < 4096 ? 2 : 3);
    for (int s = 0; s < 256; s++) W.hist[s] = 0;
    for (int i = 0; i < n; i++) W.hist[lit[i]]++;
    int distinct = 0, last_sym = 0;
    for (int s = 0; s < 256; s++) if (W.hist[s]) { distinct++; last_sym = s; }
    if (n > 0 && distinct == 1) {                         // RLE
        if (raw_hdr + 1 > cap) return -1;
        const int h = lit_header_raw(dst, 1, n);
        dst[h] = lit[0];
        return h + 1;
    }
    const int raw_size = raw_hdr + n;
    if (n >= 64) {
        const int hdr = n <= 1023 ? 3 : (n <= 16383 ? 4 : 5);
        const int streams = n < 256 ? 1 : 4;
        const int lim = (raw_size < cap ? raw_size : cap) - hdr;       // worth it only below the raw size
        if (lim > 8) {
            huf_build(W);
            uint8_t *q = dst + hdr;
            int comp = huf_write_tree(q, lim, last_sym, W);
            if (comp > 0) {
                if (streams == 1) {
                    const int s = huf_stream(lit, n, q + comp, lim - comp, W);
                    comp = s < 0 ? -1 : comp + s;
                } else if (comp + 6 < lim) {
                    const int per = (n + 3) / 4;
                    int at = comp + 6;
                    uint8_t *jump = q + comp;
                    for (int k = 0; k < 4 && at > 0; k++) {
                        const int cnt = k < 3 ? per : n - 3 * per;
                        const int s = huf_stream(lit + k * per, cnt, q + at, lim - at, W);
                        if (s < 0 || s > 65535) { at = -1; break; }
                        if (k < 3) { jump[2 * k] = (uint8_t)s; jump[2 * k + 1] = (uint8_t)(s >> 8); }
                        at += s;
                    }
                    comp = at;
                } else comp = -1;
            }
            if (comp > 0 && hdr + comp < raw_size) {
                const int fmt = streams == 1 ? 0 : (hdr == 3 ? 1 : (hdr == 4 ? 2 : 3));
                const int sb = hdr == 3 ? 10 : (hdr == 4 ? 14 : 18);
                const uint64_t h = 2u | ((uint64_t)fmt << 2) | ((uint64_t)n << 4) | ((uint64_t)comp << (4 + sb));
                for (int i = 0; i < hdr; i++) dst[i] = (uint8_t)(h >> (8 * i));
                return hdr + comp;
            }
        }
    }
    if (raw_size > cap) return -1;
    const int h = lit_header_raw(dst, 0, n);
    for (int i = 0; i < n; i++) dst[h + i] = lit[i];
    return raw_size;
}

// ---- sequences section (RFC 8878 §3.1.1.3.2).  seqs[i].off is rewritten to the offset value.  Returns bytes or -1.
ZS_HD inline int write_sequences(Seq *seqs, int ns, uint8_t *dst, int cap, EncWork &W) {
    if (cap < 3) return -1;
    int at;
    if (ns < 128) { dst[0] = (uint8_t)ns; at = 1; }
    else if (ns < 0x7F00) { dst[0] = (uint8_t)((ns >> 8) + 128); dst[1] = (uint8_t)ns; at = 2; }
    else { dst[0] = 255; dst[1] = (uint8_t)(ns - 0x7F00); dst[2] = (uint8_t)((ns - 0x7F00) >> 8); at = 3; }
    if (ns == 0) return at;
    // offsets -> offset values (repeat codes where the repeat offset is known), code histograms
    for (int t = 0; t < 3; t++) for (int s = 0; s < 64; s++) W.cnt[t][s] = 0;
    uint32_t rep[3] = {0, 0, 0};                           // 0 = not known inside this block
    for (int i = 0; i < ns; i++) {
        Seq &q = seqs[i];
        const uint32_t off = q.off;
        uint32_t ob;
        if (q.ll > 0) ob = off == rep[0] ? 1 : (off == rep[1] ? 2 : (off == rep[2] ? 3 : off + 3));
        else ob = off == rep[1] ? 1 : (off == rep[2] ? 2 : (rep[0] > 1 && off == rep[0] - 1 ? 3 : off + 3));
        if (ob > 3) { rep[2] = rep[1]; rep[1] = rep[0]; rep[0] = off; }
        else {
            const uint32_t idx = ob - 1 + (q.ll == 0 ? 1 : 0);
            if (idx > 0) { if (idx > 1) rep[2] = rep[1]; rep[1] = rep[0]; rep[0] = off; }
        }
        q.off = ob;
        W.cnt[0][ll_code(q.ll)]++;
        W.cnt[1][highbit(ob)]++;
        W.cnt[2][ml_code(q.ml)]++;
    }
    // per table: RLE, Predefined or FSE_Compressed by estimated bits
    const int8_t ll_def[36] = ZS_LL_DEFAULT_NORM;
    const int8_t ml_def[53] = ZS_ML_DEFAULT_NORM;
    const int8_t of_def[29] = ZS_OF_DEFAULT_NORM;
    const int8_t *defs[3] = {ll_def, of_def, ml_def};
    const int def_n[3] = {36, 29, 53}, def_log[3] = {kLLDefLog, kOFDefLog, kMLDefLog};
    const int max_log[3] = {kLLLog, kOFLog, kMLLog}, n_codes[3] = {36, 32, 53};
    int mode[3], rle_sym[3];
    const int modes_at = at++;
    for (int t = 0; t < 3; t++) {
        int distinct = 0, top = 0;
        for (int s = 0; s < n_codes[t]; s++) if (W.cnt[t][s]) { distinct++; top = s; }
        int16_t pre[64];
        for (int s = 0; s < def_n[t]; s++) pre[s] = defs[t][s];
        uint64_t best = fse_cost(W.cnt[t], top + 1, pre, def_n[t], def_log[t]);
        mode[t] = 0;
        if (distinct == 1 && 8 * 256 < best) { mode[t] = 1; best = 8 * 256; rle_sym[t] = top; }
        if (ns >= 4 && distinct > 1) {
            const int log = fse_table_log(ns, top + 1, max_log[t]);
            fse_normalize(W.cnt[t], top + 1, (uint32_t)ns, log, W.norm[t], 0);
            uint8_t hdr[96];
            const int hb = fse_write_ncount(hdr, 96, W.norm[t], top + 1, log);
            const uint64_t c = fse_cost(W.cnt[t], top + 1, W.norm[t], top + 1, log);
            if (hb > 0 && c != ~0ull && c + (uint64_t)hb * 8 * 256 < best) {
                if (at + hb > cap) return -1;
                for (int i = 0; i < hb; i++) dst[at + i] = hdr[i];
                mode[t] = 2;
                fse_build_ct(W.norm[t], top + 1, log, W.ct[t], W.spread);
                at += hb;
                continue;
            }
        }
        if (mode[t] == 1) {
            if (at + 1 > cap) return -1;
            dst[at++] = (uint8_t)rle_sym[t];
        } else fse_build_ct(pre, def_n[t], def_log[t], W.ct[t], W.spread);
    }
    dst[modes_at] = (uint8_t)((mode[0] << 6) | (mode[1] << 4) | (mode[2] << 2));
    // the bit stream, last sequence first; per sequence the decoder reads OF, ML, LL extra bits, then LL, ML, OF states
    BitW b;
    bw_init(b, dst + at, cap - at);
    uint32_t st[3] = {0, 0, 0};
    for (int i = ns - 1; i >= 0; i--) {
        const Seq q = seqs[i];
        const int c[3] = {ll_code(q.ll), highbit(q.off), ml_code(q.ml)};
        if (i == ns - 1) {
            for (int t = 2; t >= 0; t--) if (mode[t] != 1) st[t] = fse_init_state(W.ct[t], c[t]);   // ML, OF, LL
        } else {
            if (mode[1] != 1) fse_encode(b, W.ct[1], st[1], c[1]);
            if (mode[2] != 1) fse_encode(b, W.ct[2], st[2], c[2]);
            if (mode[0] != 1) fse_encode(b, W.ct[0], st[0], c[0]);
        }
        uint32_t lb, mb;
        int lbits, mbits;
        ll_code_info(c[0], lb, lbits);
        ml_code_info(c[2], mb, mbits);
        bw_add(b, q.ll - lb, lbits);
        bw_add(b, q.ml - mb, mbits);
        bw_add(b, q.off - (1u << c[1]), c[1]);
        if (b.over) return -1;
    }
    if (mode[2] != 1) fse_flush(b, W.ct[2], st[2]);
    if (mode[1] != 1) fse_flush(b, W.ct[1], st[1]);
    if (mode[0] != 1) fse_flush(b, W.ct[0], st[0]);
    const int sb = bw_close(b);
    return sb < 0 ? -1 : at + sb;
}

// ---- LZ parse of one block: sequences and literals.  On the device every lane of the warp calls it.
struct ParseOut { int n_seq, n_lit; };

ZS_HD inline ParseOut parse_block(const uint8_t *src, int n, int32_t *htab, Seq *seqs, uint8_t *lits) {
    const int n_hash = n >= kMinMatch ? n - kMinMatch + 1 : 0;   // positions with 4 bytes to hash
    int cur = 0, anchor = 0, ns = 0, nl = 0;
#if defined(__CUDA_ARCH__)
    const int lane = lane_id();
    for (int i = lane; i < (1 << kHashLog); i += 32) htab[i] = -1;
    __syncwarp();
    for (int c0 = 0; c0 < n_hash; c0 += kRound) {
        if (c0 + kRound <= cur) continue;                  // the round lies inside the current match
        const int p = c0 + lane;
        const bool valid = p < n_hash;
        const uint32_t h = valid ? hash4(src + p) : (1u << kHashLog) + lane;
        const unsigned peers = __match_any_sync(0xffffffffu, h);
        const unsigned below = peers & ((1u << lane) - 1);
        const int cand = below ? c0 + 31 - __clz((int)below) : (valid ? htab[h] : -1);
        __syncwarp();
        if (valid && (peers >> lane) == 1u) htab[h] = p;   // the last position of its hash in this round
        __syncwarp();
        const bool ok = valid && cand >= 0 && rd32(src + cand) == rd32(src + p);
        const unsigned m = __ballot_sync(0xffffffffu, ok);
        while (true) {
            const int from = cur - c0;
            if (from >= kRound) break;
            const unsigned sel = from <= 0 ? m : (m & (0xffffffffu << from));
            if (!sel) break;
            const int l = __ffs((int)sel) - 1;
            const int pp = c0 + l, cc = __shfl_sync(0xffffffffu, cand, l);
            int len = kMinMatch;
            while (true) {
                const int i = pp + len + lane;
                const bool eq = i < n && src[i] == src[cc + len + lane];
                const unsigned ne = __ballot_sync(0xffffffffu, !eq);
                if (ne) { len += __ffs((int)ne) - 1; break; }
                len += 32;
            }
            for (int i = lane; i < pp - anchor; i += 32) lits[nl + i] = src[anchor + i];
            if (lane == 0) seqs[ns] = Seq{(uint32_t)(pp - anchor), (uint32_t)len, (uint32_t)(pp - cc)};
            ns++;
            nl += pp - anchor;
            cur = anchor = pp + len;
        }
    }
    for (int i = lane; i < n - anchor; i += 32) lits[nl + i] = src[anchor + i];
    nl += n - anchor;
    __syncwarp();
#else
    for (int i = 0; i < (1 << kHashLog); i++) htab[i] = -1;
    int cand[kRound];
    for (int c0 = 0; c0 < n_hash; c0 += kRound) {
        if (c0 + kRound <= cur) continue;
        for (int l = 0; l < kRound && c0 + l < n_hash; l++) {
            const uint32_t h = hash4(src + c0 + l);
            cand[l] = htab[h];
            htab[h] = c0 + l;
        }
        for (int l = 0; l < kRound && c0 + l < n_hash; l++) {
            const int p = c0 + l, c = cand[l];
            if (p < cur || c < 0 || rd32(src + c) != rd32(src + p)) continue;
            int len = kMinMatch;
            while (p + len < n && src[p + len] == src[c + len]) len++;
            for (int i = 0; i < p - anchor; i++) lits[nl + i] = src[anchor + i];
            seqs[ns++] = Seq{(uint32_t)(p - anchor), (uint32_t)len, (uint32_t)(p - c)};
            nl += p - anchor;
            cur = anchor = p + len;
        }
    }
    for (int i = 0; i < n - anchor; i++) lits[nl + i] = src[anchor + i];
    nl += n - anchor;
#endif
    return ParseOut{ns, nl};
}

// ---- one block: RLE when every byte is the same, else the compressed form when it is smaller than the input, else
// raw.  The payload (RLE byte or compressed block) goes to `out` (room for n bytes); a raw block's payload is the input.
ZS_HD inline BlockOut compress_block(const uint8_t *src, int n, uint8_t *out, int32_t *htab, Seq *seqs, uint8_t *lits,
                                     EncWork &W) {
    if (n == 0) return BlockOut{0, 0};
    int same = 1;
#if defined(__CUDA_ARCH__)
    for (int i0 = 0; i0 < n && same; i0 += 32) {
        const int i = i0 + lane_id();
        same = __all_sync(0xffffffffu, i >= n || src[i] == src[0]);
    }
#else
    for (int i = 1; i < n && same; i++) same = src[i] == src[0];
#endif
    if (same) {
        if (lane_id() == 0) out[0] = src[0];
        return BlockOut{1, 1};
    }
    const ParseOut P = parse_block(src, n, htab, seqs, lits);
    int size = -1;
    if (lane_id() == 0) {
        const int a = write_literals(lits, P.n_lit, out, n - 1, W);
        if (a >= 0) {
            const int b = write_sequences(seqs, P.n_seq, out + a, n - 1 - a, W);
            if (b >= 0) size = a + b;
        }
    }
    size = bcast0(size);
    return size > 0 ? BlockOut{2, size} : BlockOut{0, n};
}

// ---- frame and block headers
ZS_HD inline int frame_header_size(uint64_t n) { return 5 + (n <= 255 ? 1 : (n <= 65791 ? 2 : (n <= 0xFFFFFFFFull ? 4 : 8))); }
ZS_HD inline int write_frame_header(uint8_t *d, uint64_t n) {
    d[0] = 0x28; d[1] = 0xB5; d[2] = 0x2F; d[3] = 0xFD;
    const int f = n <= 255 ? 0 : (n <= 65791 ? 1 : (n <= 0xFFFFFFFFull ? 2 : 3));
    d[4] = (uint8_t)((f << 6) | (1 << 5));                    // single segment
    const uint64_t v = f == 1 ? n - 256 : n;
    const int bytes = f == 0 ? 1 : (f == 1 ? 2 : (f == 2 ? 4 : 8));
    for (int i = 0; i < bytes; i++) d[5 + i] = (uint8_t)(v >> (8 * i));
    return 5 + bytes;
}
ZS_HD inline void write_block_header(uint8_t *d, int last, int type, uint32_t size) {
    const uint32_t h = (uint32_t)last | ((uint32_t)type << 1) | (size << 3);
    d[0] = (uint8_t)h; d[1] = (uint8_t)(h >> 8); d[2] = (uint8_t)(h >> 16);
}
ZS_HD inline int64_t frame_bound(int64_t n) { return frame_header_size((uint64_t)n) + n + 3 * (n / kMaxBlock + 1); }

// A whole frame, block after block (the host build; the device runs the blocks as separate warps and places them with
// a gather, encoded_file.cu).  `htab` 2^kHashLog entries, `seqs` kMaxBlock / 4 + 1, `lits` and `out_blk` kMaxBlock
// bytes.  Returns the frame size, or -1 when it does not fit `cap`.
ZS_HD inline int64_t compress_frame(const uint8_t *src, int64_t n, uint8_t *dst, int64_t cap, int32_t *htab, Seq *seqs,
                                    uint8_t *lits, uint8_t *out_blk, EncWork &W) {
    if (cap < frame_bound(n)) return -1;
    int64_t at = write_frame_header(dst, (uint64_t)n);
    int64_t pos = 0;
    do {
        const int bn = (int)(n - pos < kMaxBlock ? n - pos : kMaxBlock);
        const BlockOut r = compress_block(src + pos, bn, out_blk, htab, seqs, lits, W);
        write_block_header(dst + at, pos + bn >= n, r.type, r.type == 2 ? (uint32_t)r.size : (uint32_t)bn);
        at += 3;
        const uint8_t *pay = r.type == 0 ? src + pos : out_blk;
        for (int i = 0; i < r.size; i++) dst[at + i] = pay[i];
        at += r.size;
        pos += bn;
    } while (pos < n);
    return at;
}

}  // namespace zs
