// orc_encode.cu — compaction output encode: a device-resident columnar batch -> one ORC data file.
//
// The rewrite step of parquet_encode.cu for tables whose file format at the output level is orc
// (KeyValueFileWriterFactory.java:301-310 picks the writer per level; OrcWriterFactory drives orc-core's writer, types
// by OrcTypeUtil.convertToOrcType).  The byte layout is the public ORC v1 specification that orc_meta.h restates:
//   "ORC" | stripes: [index: per column ROW_INDEX, BLOOM_FILTER_UTF8?] per column PRESENT? DATA LENGTH|SECONDARY?,
//   stripe footer | Metadata | Footer | PostScript | len
// No dictionaries.  Stripes start at multiples of 8 rows, so a PRESENT stream's bytes are the bit-reversed bytes of the
// validity bitmap.  The row index (pg_orc_encode_indexed) cuts each stripe into row groups of `stride` rows, also a
// multiple of 8; without it a stripe is one row group, and the code below is the same.
//
// Pipeline (the launch count does not depend on the number of columns; a task = one column of one stripe, a span =
// one column of one row group):
//   1. k_oe_count + k_pw_stats per span: non-null values, payload bytes, exact sums, true count, VARCHAR lengths; min /
//      max / NaN / retracts.  k_oe_bloom per row group of a bloom column: its filter.  One read-back.  The ORC
//      statistics come from both (task_stats, merge_stats over a stripe's row groups); the file statistics of
//      pg_parquet_file_column_stats and pg_file_meta from the k_pw_stats words (FileStats).
//   2. k_oe_values (phase 0): the non-null values that are run-length coded are compacted into scratch (int64 values,
//      string lengths, decimal scales; BYTE values, BOOLEAN bits; PRESENT bytes).
//   3. k_oe_rle_size: one thread per integer RLE v2 run (kRunValues values) or byte-RLE group (kByteGroup bytes), the
//      runs cut where a row group starts, so every row index position starts a run.  One read-back; the host lays out
//      the streams and computes the positions.
//   4. k_oe_rle_write and k_oe_values (phase 1): the runs, and the streams that are the values themselves (FLOAT /
//      DOUBLE, string bytes, DECIMAL varints) straight from the batch, at their positions in the image.
//   5. ZSTD: every stream cut into chunks of at most the block size, every chunk one zstd frame (ZstdFrames); one
//      read-back of the frame sizes; the host keeps the original bytes of a chunk whose frame is not smaller, lays
//      out the stripes, and the gather places each chunk, compressed or original, behind its 3-byte header.
// The chunk headers, the row index sections, the stripe footers and the file tail are written on the host
// (orc_meta.cc) as host parts, like Parquet's page headers and footer.
#include <math.h>

#include <algorithm>
#include <memory>
#include <string>

#include "device_utils.cuh"
#include "encoded_file.h"
#include "murmur3_device.cuh"
#include "orc_encode_device.cuh"
#include "orc_meta.h"

namespace pg {

namespace {

using orc::OutType;

struct OeTask {                   // one column of one stripe (k_oe_count: of one row group)
    int32_t col, kind;            // batch column, ORC kind
    int32_t max_len, scale;       // VARCHAR(n): n, else 0; DECIMAL: the scale
    int64_t row0, rows;           // batch rows of the stripe (row0 a multiple of 8)
    int64_t present;              // byte scratch: the PRESENT bytes, -1 = no PRESENT stream
    int64_t bytes;                // byte scratch: BYTE values / BOOLEAN bits, -1 = none
    int64_t ints;                 // int64 scratch: SHORT / INT / LONG / DATE values, string lengths, decimal scales; -1
    int64_t direct;               // image offset of a DATA stream written from the values themselves, -1 = none
};
constexpr int kCountWords = 6;    // per task: non-null values, payload bytes, trues, sum (lo, hi), a VARCHAR too long

struct RleJob {                   // one integer RLE v2 run or one byte-RLE group
    int64_t src;                  // first value in the int64 / byte scratch
    int64_t dst;                  // image offset
    int32_t n;
    int32_t mode;                 // 0 unsigned RLE v2, 1 signed RLE v2, 2 byte RLE
};

struct BloomTask {                // the filter of one bloom column over one row group
    int32_t col, kind;
    int64_t row0, rows;
    int64_t out;                  // first word of the filter in the filter buffer
};
// the largest filter k_oe_bloom holds: the shared memory one CTA can take on sm_90
constexpr int64_t kBloomMaxBytes = 227 << 10;

__device__ __forceinline__ bool is_int_rle(int k) {
    return k == orc::K_SHORT || k == orc::K_INT || k == orc::K_LONG || k == orc::K_DATE;
}
__device__ __forceinline__ bool is_bytes(int k) { return k == orc::K_STRING || k == orc::K_VARCHAR || k == orc::K_BINARY; }

__device__ __forceinline__ __int128 shfl_xor128(__int128 v, int d) {
    const unsigned long long lo = __shfl_xor_sync(0xffffffffu, (unsigned long long)v, d);
    const unsigned long long hi = __shfl_xor_sync(0xffffffffu, (unsigned long long)((unsigned __int128)v >> 64), d);
    return (__int128)(((unsigned __int128)hi << 64) | lo);
}

__global__ void __launch_bounds__(256)
k_oe_count(const EncColumn *cols, const OeTask *tasks, int64_t *out) {
    const OeTask t = tasks[blockIdx.x];
    const EncColumn c = cols[t.col];
    long long nn = 0, payload = 0, trues = 0, too_long = 0;
    __int128 sum = 0;
    for (int64_t i = threadIdx.x; i < t.rows; i += blockDim.x) {
        const int64_t row = t.row0 + i;
        if (!valid_bit(c.validity, row)) continue;
        nn++;
        if (c.width == 0) {
            const int32_t s = c.offsets[row], len = c.offsets[row + 1] - s;
            payload += len;
            if (t.max_len) {                               // characters = UTF-8 bytes that are not continuation bytes
                const uint8_t *p = (const uint8_t *)c.data + s;
                int chars = 0;
                for (int b = 0; b < len; b++) chars += (p[b] & 0xC0) != 0x80;
                too_long |= chars > t.max_len;
            }
            continue;
        }
        const int64_t x = sext(load_fixed(c.data, c.width, row), c.width);
        if (t.kind == orc::K_BOOLEAN) trues += x != 0;
        else if (t.kind != orc::K_FLOAT && t.kind != orc::K_DOUBLE && t.kind != orc::K_DATE) sum += x;
        if (t.kind == orc::K_DECIMAL) payload += orcdev::varint_size(orcdev::zigzag(x));
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        nn += __shfl_xor_sync(0xffffffffu, nn, d);
        payload += __shfl_xor_sync(0xffffffffu, payload, d);
        trues += __shfl_xor_sync(0xffffffffu, trues, d);
        too_long |= __shfl_xor_sync(0xffffffffu, too_long, d);
        sum += shfl_xor128(sum, d);
    }
    __shared__ long long s_w[8][4];
    __shared__ __int128 s_sum[8];
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        s_w[warp][0] = nn; s_w[warp][1] = payload; s_w[warp][2] = trues; s_w[warp][3] = too_long;
        s_sum[warp] = sum;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long a = 0, b = 0, e = 0, f = 0;
        __int128 s = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) {
            a += s_w[w][0]; b += s_w[w][1]; e += s_w[w][2]; f |= s_w[w][3];
            s += s_sum[w];
        }
        int64_t *o = out + kCountWords * (int64_t)blockIdx.x;
        o[0] = a; o[1] = b; o[2] = e;
        o[3] = (int64_t)(uint64_t)s;
        o[4] = (int64_t)(s >> 64);
        o[5] = f;
    }
}

// phase 0: PRESENT bytes and the compacted values the run-length coders read; phase 1: the DATA streams that are the
// values themselves, at t.direct in the image.  One CTA per task; ranks and byte offsets by block-wide scans.
__global__ void __launch_bounds__(256)
k_oe_values(const EncColumn *cols, const OeTask *tasks, int phase, int64_t *ints, uint8_t *bytes, uint8_t *image) {
    const OeTask t = tasks[blockIdx.x];
    const EncColumn c = cols[t.col];
    const int k = t.kind;
    if (phase == 0 && t.present >= 0) {
        const int64_t nb = (t.rows + 7) >> 3;
        for (int64_t b = threadIdx.x; b < nb; b += blockDim.x) {
            uint32_t v = c.validity ? c.validity[(t.row0 >> 3) + b] : 0xFFu;
            const int64_t rem = t.rows - b * 8;
            if (rem < 8) v &= (1u << rem) - 1;
            bytes[t.present + b] = orcdev::bit_reverse8(v);
        }
    }
    const bool work = phase == 0 ? (t.bytes >= 0 || t.ints >= 0) : t.direct >= 0;
    if (!work) return;
    __shared__ int ws[33];
    int64_t base_rank = 0, base_bytes = 0;
    for (int64_t i0 = 0; i0 < t.rows; i0 += blockDim.x) {
        const int64_t i = i0 + threadIdx.x;
        const int64_t row = t.row0 + i;
        const bool v = i < t.rows && valid_bit(c.validity, row);
        int len = 0;
        int32_t st = 0;
        int64_t x = 0;
        if (v && c.width == 0) { st = c.offsets[row]; len = c.offsets[row + 1] - st; }
        else if (v) x = sext(load_fixed(c.data, c.width, row), c.width);
        if (phase == 1 && v && k == orc::K_DECIMAL) len = orcdev::varint_size(orcdev::zigzag(x));
        int n_valid, n_bytes;
        const int64_t rank = base_rank + block_scan_excl(v ? 1 : 0, ws, &n_valid);
        const int64_t boff = base_bytes + block_scan_excl(phase == 1 ? len : 0, ws, &n_bytes);
        if (v) {
            if (phase == 0) {
                if (k == orc::K_BYTE) bytes[t.bytes + rank] = (uint8_t)x;
                else if (k == orc::K_BOOLEAN) {
                    // bits most significant first; the scratch is zeroed, the aligned word may hold neighbouring bytes
                    if (x) {
                        uint8_t *byte = bytes + t.bytes + (rank >> 3);
                        unsigned int *word = (unsigned int *)((uintptr_t)byte & ~(uintptr_t)3);
                        atomicOr(word, 1u << ((((uintptr_t)byte & 3) << 3) + (7 - (rank & 7))));
                    }
                } else if (is_int_rle(k)) ints[t.ints + rank] = x;
                else if (is_bytes(k)) ints[t.ints + rank] = len;
                else if (k == orc::K_DECIMAL) ints[t.ints + rank] = t.scale;
            } else {
                uint8_t *d = image + t.direct;
                if (k == orc::K_FLOAT) { const uint32_t u = (uint32_t)x; memcpy(d + 4 * rank, &u, 4); }
                else if (k == orc::K_DOUBLE) { const uint64_t u = (uint64_t)x; memcpy(d + 8 * rank, &u, 8); }
                else if (k == orc::K_DECIMAL) {
                    orcdev::Out o{d + boff, 0};
                    orcdev::put_varint(o, orcdev::zigzag(x));
                } else {
                    const uint8_t *s = (const uint8_t *)c.data + st;
                    for (int b = 0; b < len; b++) d[boff + b] = s[b];
                }
            }
        }
        base_rank += n_valid;
        base_bytes += n_bytes;
    }
}

// One CTA per row group of a bloom column: the filter is zeroed in shared memory, every non-null value's k bits are set
// there (ORC's BloomFilter.addLong / addDouble / addBytes: integers and DATE sign-extended through Thomas Wang's hash,
// FLOAT widened to double and DOUBLE by their bits with NaN canonical, strings and BINARY through Murmur3 hash64), and
// the words are stored at t.out.  num_bits is a multiple of 64.
__global__ void __launch_bounds__(256)
k_oe_bloom(const EncColumn *cols, const BloomTask *tasks, uint32_t num_bits, int k, uint32_t *out) {
    extern __shared__ uint32_t s_bits[];
    const BloomTask t = tasks[blockIdx.x];
    const EncColumn c = cols[t.col];
    const int n_words = (int)(num_bits >> 5);
    for (int i = threadIdx.x; i < n_words; i += blockDim.x) s_bits[i] = 0;
    __syncthreads();
    for (int64_t i = threadIdx.x; i < t.rows; i += blockDim.x) {
        const int64_t row = t.row0 + i;
        if (!valid_bit(c.validity, row)) continue;
        int64_t h;
        if (c.width == 0) {
            const int32_t s = c.offsets[row];
            h = fi::murmur3_hash64((const uint8_t *)c.data + s, c.offsets[row + 1] - s);
        } else {
            const uint64_t v = load_fixed(c.data, c.width, row);
            int64_t key;
            if (t.kind == orc::K_FLOAT) key = fi::double_key((uint64_t)__double_as_longlong((double)__uint_as_float((uint32_t)v)));
            else if (t.kind == orc::K_DOUBLE) key = fi::double_key(v);
            else key = sext(v, c.width);
            h = fi::wang64(key);
        }
        for (int j = 1; j <= k; j++) {
            const uint32_t p = fi::bloom_bit(h, j, num_bits);
            atomicOr(s_bits + (p >> 5), 1u << (p & 31));
        }
    }
    __syncthreads();
    uint32_t *o = out + t.out;
    for (int i = threadIdx.x; i < n_words; i += blockDim.x) o[i] = s_bits[i];
}

__global__ void k_oe_rle_size(const RleJob *jobs, int n, const int64_t *ints, const uint8_t *bytes, int32_t *sizes) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const RleJob r = jobs[j];
    sizes[j] = r.mode == 2 ? orcdev::brle_size(bytes + r.src, r.n) : orcdev::rle2_plan(ints + r.src, r.n, r.mode).size;
}

__global__ void k_oe_rle_write(const RleJob *jobs, int n, const int64_t *ints, const uint8_t *bytes, uint8_t *image) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const RleJob r = jobs[j];
    if (r.mode == 2) orcdev::brle_write(bytes + r.src, r.n, image + r.dst);
    else {
        const orcdev::Rle2Plan p = orcdev::rle2_plan(ints + r.src, r.n, r.mode);
        orcdev::rle2_write(ints + r.src, r.n, r.mode, p, image + r.dst);
    }
}

// ------------------------------------------------------------------ host side

int default_kind(int t) {
    switch (t) {
        case PG_INT8: return orc::K_BYTE;
        case PG_INT16: return orc::K_SHORT;
        case PG_INT32: return orc::K_INT;
        case PG_INT64: return orc::K_LONG;
        case PG_FLOAT: return orc::K_FLOAT;
        case PG_DOUBLE: return orc::K_DOUBLE;
        case PG_BOOL: return orc::K_BOOLEAN;
        case PG_STRING: return orc::K_STRING;
        default: return orc::K_BINARY;
    }
}

// the ORC type of every column: the caller's, checked against the physical types, or the default for each
pg_status resolve_types(const Schema &s, const pg_orc_column_type *in, std::vector<OutType> &out) {
    const int nc = s.n_cols();
    out.assign(nc, OutType{});
    for (int c = 0; c < nc; c++) {
        const int t = s.field(c).type;
        OutType &o = out[c];
        if (!in) { o.kind = default_kind(t); continue; }
        const pg_orc_column_type &x = in[c];
        const std::string who = "orc encode: column " + std::to_string(c) + ": ";
        if (x.kind < 0 || x.kind > orc::K_TIMESTAMP_INSTANT)
            return fail(PG_ERR_INVALID, who + "kind " + std::to_string(x.kind) + " is not an ORC TypeKind");
        if (x.kind == orc::K_TIMESTAMP || x.kind == orc::K_TIMESTAMP_INSTANT || x.kind == orc::K_CHAR ||
            (x.kind >= orc::K_LIST && x.kind <= orc::K_UNION))
            return fail(PG_ERR_UNSUPPORTED, who + "kind " + std::to_string(x.kind) +
                                                " is not written on the device (TIMESTAMP, CHAR and nested kinds are not)");
        bool fits;
        switch (x.kind) {
            case orc::K_BYTE: fits = t == PG_INT8; break;
            case orc::K_SHORT: fits = t == PG_INT16; break;
            case orc::K_INT: case orc::K_DATE: fits = t == PG_INT32; break;
            case orc::K_LONG: fits = t == PG_INT64; break;
            case orc::K_DECIMAL: fits = t == PG_INT64 && x.precision >= 1 && x.precision <= 18 && x.scale >= 0 &&
                                        x.scale <= x.precision; break;
            case orc::K_FLOAT: fits = t == PG_FLOAT; break;
            case orc::K_DOUBLE: fits = t == PG_DOUBLE; break;
            case orc::K_BOOLEAN: fits = t == PG_BOOL; break;
            case orc::K_STRING: fits = t == PG_STRING; break;
            case orc::K_VARCHAR: fits = t == PG_STRING && x.max_length >= 1; break;
            default: fits = t == PG_BINARY; break;       // K_BINARY
        }
        if (!fits)
            return fail(PG_ERR_INVALID, who + "kind " + std::to_string(x.kind) + " (precision " + std::to_string(x.precision) +
                                            ", scale " + std::to_string(x.scale) + ", max_length " + std::to_string(x.max_length) +
                                            ") does not fit physical type " + std::to_string(t));
        o.kind = x.kind;
        if (x.kind == orc::K_DECIMAL) { o.precision = (uint32_t)x.precision; o.scale = (uint32_t)x.scale; }
        if (x.kind == orc::K_VARCHAR) o.max_length = (uint32_t)x.max_length;
    }
    return PG_OK;
}

bool is_int_kind(int k) { return k == orc::K_BYTE || k == orc::K_SHORT || k == orc::K_INT || k == orc::K_LONG; }
bool is_bytes_kind(int k) { return k == orc::K_STRING || k == orc::K_VARCHAR || k == orc::K_BINARY; }
bool fits_int64(__int128 v) { return v >= (__int128)INT64_MIN && v <= (__int128)INT64_MAX; }

double as_double(int64_t bits) {
    double x;
    memcpy(&x, &bits, 8);
    return x;
}

// the ORC statistics of a task from its counts and k_pw_stats words
orc::ColumnStats task_stats(const OeTask &t, const int64_t *cnt, const int64_t *st) {
    orc::ColumnStats s;
    s.values = (uint64_t)cnt[0];
    s.has_null = cnt[0] < t.rows;
    if (!s.values) return s;
    const int k = t.kind;
    s.sum = (__int128)(((unsigned __int128)(uint64_t)cnt[4] << 64) | (uint64_t)cnt[3]);
    if (is_int_kind(k) || k == orc::K_DATE || k == orc::K_DECIMAL) {
        s.has_minmax = true;
        s.imin = st[0];
        s.imax = st[1];
        s.has_sum = k == orc::K_DECIMAL || (is_int_kind(k) && fits_int64(s.sum));
    } else if (k == orc::K_FLOAT || k == orc::K_DOUBLE) {
        s.has_minmax = true;
        if (st[4]) { s.dmin = -INFINITY; s.dmax = NAN; }
        else { s.dmin = as_double(zero_as(st[0], -0.0)); s.dmax = as_double(zero_as(st[1], 0.0)); }
    } else if (k == orc::K_BOOLEAN) s.trues = (uint64_t)cnt[2];
    else s.bytes = cnt[1];
    return s;
}

// a column's stripe statistics: the merge of its row groups', its file statistics: of its stripes' (a NaN anywhere
// gives [-Infinity, NaN])
void merge_stats(int kind, orc::ColumnStats &f, const orc::ColumnStats &s, bool first) {
    if (first) { f = s; return; }
    f.values += s.values;
    f.has_null |= s.has_null;
    f.trues += s.trues;
    f.bytes += s.bytes;
    f.sum += s.sum;
    f.has_sum = kind == orc::K_DECIMAL || (is_int_kind(kind) && fits_int64(f.sum));
    if (!s.has_minmax) return;
    if (!f.has_minmax) { f.has_minmax = true; f.imin = s.imin; f.imax = s.imax; f.dmin = s.dmin; f.dmax = s.dmax; return; }
    f.imin = std::min(f.imin, s.imin);
    f.imax = std::max(f.imax, s.imax);
    if (isnan(f.dmax) || isnan(s.dmax)) { f.dmin = -INFINITY; f.dmax = NAN; }
    else { f.dmin = std::min(f.dmin, s.dmin); f.dmax = std::max(f.dmax, s.dmax); }
}

struct Stream {
    int task, kind;
    int64_t length = 0;           // raw bytes
    size_t job0 = 0, job1 = 0;    // its run-length jobs
    bool runs = false;            // run-length coded (else the values themselves)
    std::vector<int64_t> at;      // per row group of the stripe, where it starts: a job index while the run sizes are
                                  // not back (runs), then the offset in the raw stream
    std::vector<uint8_t> bit;     // BOOLEAN DATA: per row group, the bit of its first value in the byte at `at`
    int64_t raw_off = 0;          // offset in the raw image
    size_t chunk0 = 0, chunk1 = 0;
    int64_t stored = 0;           // bytes in the file
};

pg_status encode_orc(uint64_t source, const char *const *names, int64_t row0, int64_t n_rows,
                     const pg_orc_write_options *opt, const pg_orc_index_options *ix, uint64_t *out_file) {
    const int codec = opt ? opt->compression : orc::C_NONE;
    const int level = opt ? opt->zstd_level : 1;
    const int64_t block = opt && opt->compression_block_size > 0 ? opt->compression_block_size : 256 << 10;
    if (codec < 0 || codec > 6)
        return fail(PG_ERR_INVALID, "orc encode: compression " + std::to_string(codec) + " is not an ORC CompressionKind");
    if (codec != orc::C_NONE && codec != orc::C_ZSTD)
        return fail(PG_ERR_UNSUPPORTED, "orc encode: compression " + std::to_string(codec) +
                                            " is not written on the device (NONE and ZSTD are)");
    if (codec == orc::C_ZSTD && (level == 0 || level > 1))
        return fail(PG_ERR_UNSUPPORTED, "orc encode: zstd level " + std::to_string(level) +
                                            " is not written on the device (level 1 and the negative fast levels are)");
    if (opt && (opt->compression_block_size < 0 || opt->compression_block_size >= ((int64_t)1 << 23)))
        return fail(PG_ERR_INVALID, "orc encode: compression block size " + std::to_string(opt->compression_block_size) +
                                        " outside [0, 2^23) (a chunk header holds 23 bits of length)");
    const int64_t stride = ix ? ix->row_index_stride : 0;
    const int n_bloom = ix ? ix->n_bloom_columns : 0;
    if (stride < 0 || (stride > 0 && stride < 1000))
        return fail(PG_ERR_INVALID, "orc encode: row index stride " + std::to_string(stride) +
                                        " is negative or below 1000 (orc-core's minimum)");
    if (n_bloom < 0 || (n_bloom > 0 && !ix->bloom_columns))
        return fail(PG_ERR_INVALID, "orc encode: " + std::to_string(n_bloom) + " bloom filter columns");
    if (n_bloom > 0 && stride == 0)
        return fail(PG_ERR_INVALID, "orc encode: bloom filters are written per row group and need a row index stride");
    if (n_bloom > 0 && !(ix->bloom_fpp > 0 && ix->bloom_fpp < 1))
        return fail(PG_ERR_INVALID, "orc encode: bloom filter fpp " + std::to_string(ix->bloom_fpp) + " outside (0, 1)");
    if (stride % 8)
        return fail(PG_ERR_UNSUPPORTED, "orc encode: row index stride " + std::to_string(stride) +
                                            " is not a multiple of 8 (row groups start on whole PRESENT bytes)");
    int32_t bloom_bits = 0, bloom_k = 0;
    if (n_bloom > 0 && (!fi::orc_bloom_sizing(stride, ix->bloom_fpp, &bloom_bits, &bloom_k) || bloom_bits / 8 > kBloomMaxBytes))
        return fail(PG_ERR_UNSUPPORTED, "orc encode: a bloom filter for " + std::to_string(stride) + " rows at fpp " +
                                            std::to_string(ix->bloom_fpp) + " is larger than the " +
                                            std::to_string(kBloomMaxBytes) + " bytes one CTA holds in shared memory");
    BatchColumns batch;                                      // held until the encode below is done
    pg_status st = encode_source(source, "orc encode", row0, &n_rows, &batch);
    if (st) return st;
    const Schema *s = batch.schema.get();
    const std::vector<DevColumn> &dcols = batch.cols;
    const int nc = s->n_cols();
    std::vector<OutType> types;
    if ((st = resolve_types(*s, opt ? opt->types : nullptr, types))) return st;
    std::vector<int> bloom_cols;                             // file columns
    for (int b = 0; b < n_bloom; b++) {
        const int c = ix->bloom_columns[b];
        const std::string who = "orc encode: bloom filter column " + std::to_string(c);
        if (c < 0 || c >= nc) return fail(PG_ERR_INVALID, who + " outside the " + std::to_string(nc) + " columns");
        if (std::find(bloom_cols.begin(), bloom_cols.end(), c) != bloom_cols.end())
            return fail(PG_ERR_INVALID, who + " is listed twice");
        if (types[c].kind == orc::K_BOOLEAN || types[c].kind == orc::K_DECIMAL)
            return fail(PG_ERR_UNSUPPORTED, who + " is BOOLEAN or DECIMAL (their filters are not written on the device)");
        bloom_cols.push_back(c);
    }

    SectionTimer tm;
    if ((st = start_encode(tm))) return st;

    // ---- tasks: stripe major, then column; spans: stripe, row group, column; bloom tasks: stripe, bloom column, row
    // group.  Without a row index a stripe is one row group.
    int64_t stripe_rows = opt && opt->stripe_rows > 0 ? opt->stripe_rows : (int64_t)1 << 20;
    stripe_rows = (stripe_rows + 7) & ~(int64_t)7;
    const int64_t n_stripes = n_rows == 0 ? 0 : (n_rows + stripe_rows - 1) / stripe_rows;
    const int64_t group_rows = stride > 0 ? stride : stripe_rows;
    std::vector<EncColumn> cols;
    for (int c = 0; c < nc; c++) {
        const pg_field f = s->field(c);
        cols.push_back(EncColumn{dcols[c].data, dcols[c].offsets, dcols[c].validity, f.type, type_width(f.type), 1, 0});
    }
    std::vector<OeTask> tasks, spans;
    std::vector<StatJob> sjobs;
    std::vector<BloomTask> btasks;
    std::vector<int64_t> group0(n_stripes + 1, 0);           // the stripe's first row group in the file
    const int64_t bloom_words = bloom_bits / 32;
    for (int64_t g = 0; g < n_stripes; g++) {
        const int64_t g0 = row0 + g * stripe_rows, g1 = std::min(row0 + n_rows, g0 + stripe_rows);
        for (int c = 0; c < nc; c++)
            tasks.push_back(OeTask{c, types[c].kind, (int32_t)types[c].max_length, (int32_t)types[c].scale, g0, g1 - g0,
                                   -1, -1, -1, -1});
        for (int64_t r0 = g0; r0 < g1; r0 += group_rows) {
            const int64_t r1 = std::min(g1, r0 + group_rows);
            for (int c = 0; c < nc; c++) {
                spans.push_back(OeTask{c, types[c].kind, (int32_t)types[c].max_length, (int32_t)types[c].scale, r0,
                                       r1 - r0, -1, -1, -1, -1});
                sjobs.push_back(StatJob{c, 0, r0, r1 - r0});
            }
        }
        group0[g + 1] = (int64_t)spans.size() / nc;
        for (int c : bloom_cols)
            for (int64_t r0 = g0; r0 < g1; r0 += group_rows)
                btasks.push_back(BloomTask{c, types[c].kind, r0, std::min(g1, r0 + group_rows) - r0,
                                           (int64_t)btasks.size() * bloom_words});
    }
    const size_t nt = tasks.size(), ns = spans.size(), nbt = btasks.size();
    Scratch scratch(0);                                      // temporaries, released on every path out of this function
    EncColumn *d_cols = (EncColumn *)scratch.take(sizeof(EncColumn) * nc);
    OeTask *d_tasks = (OeTask *)scratch.take(sizeof(OeTask) * std::max<size_t>(nt, 1));
    OeTask *d_spans = (OeTask *)scratch.take(sizeof(OeTask) * std::max<size_t>(ns, 1));
    StatJob *d_sjobs = (StatJob *)scratch.take(sizeof(StatJob) * std::max<size_t>(ns, 1));
    int64_t *d_counts = (int64_t *)scratch.take(sizeof(int64_t) * kCountWords * (ns + 1));
    int64_t *d_stats = (int64_t *)scratch.take(sizeof(int64_t) * kStatWords * (ns + 1));
    BloomTask *d_btasks = (BloomTask *)scratch.take(sizeof(BloomTask) * std::max<size_t>(nbt, 1));
    uint32_t *d_filters = (uint32_t *)scratch.take(sizeof(uint32_t) * (nbt * bloom_words + 1));
    if (!d_cols || !d_tasks || !d_spans || !d_sjobs || !d_counts || !d_stats || !d_btasks || !d_filters)
        return fail(PG_ERR_CUDA, "orc encode: out of device memory for the task tables");
    PG_CUDA(cudaMemcpy(d_cols, cols.data(), sizeof(EncColumn) * nc, cudaMemcpyHostToDevice));
    int launches = 0;
    std::vector<int64_t> counts(kCountWords * (ns + 1)), stats(kStatWords * (ns + 1));
    std::vector<uint64_t> filters(nbt * bloom_words / 2);
    if (ns) {
        PG_CUDA(cudaMemcpy(d_spans, spans.data(), sizeof(OeTask) * ns, cudaMemcpyHostToDevice));
        PG_CUDA(cudaMemcpy(d_sjobs, sjobs.data(), sizeof(StatJob) * ns, cudaMemcpyHostToDevice));
        k_oe_count<<<(unsigned)ns, 256>>>(d_cols, d_spans, d_counts);
        launch_pw_stats(d_cols, d_sjobs, (int)ns, d_stats);
        launches += 2;
        if (nbt) {
            const int smem = bloom_bits / 8;
            if (smem > (48 << 10))
                PG_CUDA(cudaFuncSetAttribute(k_oe_bloom, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            PG_CUDA(cudaMemcpy(d_btasks, btasks.data(), sizeof(BloomTask) * nbt, cudaMemcpyHostToDevice));
            k_oe_bloom<<<(unsigned)nbt, 256, smem>>>(d_cols, d_btasks, (uint32_t)bloom_bits, bloom_k, d_filters);
            PG_CUDA(cudaGetLastError());
            launches++;
        }
        SmallReads rd(0);
        if ((st = rd.add(counts.data(), d_counts, sizeof(int64_t) * kCountWords * ns))) return st;
        if ((st = rd.add(stats.data(), d_stats, sizeof(int64_t) * kStatWords * ns))) return st;
        if ((st = rd.add(filters.data(), d_filters, sizeof(uint64_t) * filters.size()))) return st;
        launches++;
        if ((st = rd.finish())) return st;
    }

    // ---- statistics (per row group, folded per stripe and file), scratch slots, streams and their run-length jobs
    auto ef = std::make_unique<EncodedFile>();
    std::vector<orc::ColumnStats> file_stats(nc + 1), span_stats(ns);
    file_stats[0].values = (uint64_t)n_rows;
    std::vector<orc::OutStripe> stripes(n_stripes);
    FileStats fs(*s);                                         // the accessor's statistics: those of the Parquet output
    std::vector<Stream> streams;
    std::vector<RleJob> jobs;
    int64_t n_ints = 0, n_bytes = 0;
    // the jobs of n values (bytes) from scratch `src`, cut where each row group starts (starts[r], from 0)
    auto add_runs = [&](Stream &sm, int64_t src, int64_t n, int mode, const std::vector<int64_t> &starts) {
        const int per = mode == 2 ? orcdev::kByteGroup : orcdev::kRunValues;
        sm.runs = true;
        sm.job0 = jobs.size();
        sm.at.resize(starts.size());
        for (size_t r = 0; r < starts.size(); r++) {
            const int64_t end = r + 1 < starts.size() ? starts[r + 1] : n;
            sm.at[r] = (int64_t)jobs.size();
            for (int64_t i = starts[r]; i < end; i += per)
                jobs.push_back(RleJob{src + i, 0, (int32_t)std::min<int64_t>(per, end - i), mode});
        }
        sm.job1 = jobs.size();
    };
    auto scaled = [](const std::vector<int64_t> &v, int64_t mul, int shift) {
        std::vector<int64_t> o(v.size());
        for (size_t r = 0; r < v.size(); r++) o[r] = (v[r] * mul) >> shift;
        return o;
    };
    for (size_t i = 0; i < nt; i++) {
        OeTask &t = tasks[i];
        const int64_t g = (int64_t)(i / nc), ng = group0[g + 1] - group0[g];
        orc::OutStripe &sp = stripes[g];
        if (sp.stats.empty()) {
            sp.stats.resize(nc + 1);
            sp.stats[0].values = (uint64_t)t.rows;
            sp.rows = (uint64_t)t.rows;
        }
        int64_t nn = 0, payload = 0;
        std::vector<int64_t> rank(ng), bytes_at(ng), row_at(ng);   // where each row group starts in the stripe's column
        for (int64_t r = 0; r < ng; r++) {
            const size_t j = (size_t)((group0[g] + r) * nc + t.col);
            const int64_t *cnt = &counts[kCountWords * j], *sw = &stats[kStatWords * j];
            if (cnt[5])
                return fail(PG_ERR_UNSUPPORTED, "orc encode: column " + std::to_string(t.col) + " holds a value longer than "
                                                "its VARCHAR(" + std::to_string(t.max_len) + ") (orc-core would truncate it)");
            rank[r] = nn;
            bytes_at[r] = payload;
            row_at[r] = spans[j].row0 - t.row0;
            nn += cnt[0];
            payload += cnt[1];
            span_stats[j] = task_stats(spans[j], cnt, sw);
            merge_stats(t.kind, sp.stats[t.col + 1], span_stats[j], r == 0);
            fs.add(t.col, cols[t.col], sw, spans[j].rows);
        }
        merge_stats(t.kind, file_stats[t.col + 1], sp.stats[t.col + 1], g == 0);

        if (nn < t.rows) {
            Stream sm{(int)i, orc::S_PRESENT};
            t.present = n_bytes;
            add_runs(sm, n_bytes, (t.rows + 7) / 8, 2, scaled(row_at, 1, 3));
            n_bytes += (t.rows + 7) / 8;
            streams.push_back(sm);
        }
        Stream data{(int)i, orc::S_DATA};
        const int k = t.kind;
        if (k == orc::K_BYTE) { t.bytes = n_bytes; add_runs(data, n_bytes, nn, 2, rank); n_bytes += nn; }
        else if (k == orc::K_BOOLEAN) {
            t.bytes = n_bytes;
            add_runs(data, n_bytes, (nn + 7) / 8, 2, scaled(rank, 1, 3));
            for (int64_t r : rank) data.bit.push_back((uint8_t)(r & 7));
            n_bytes += (nn + 7) / 8;
        } else if (k == orc::K_SHORT || k == orc::K_INT || k == orc::K_LONG || k == orc::K_DATE) {
            t.ints = n_ints;
            add_runs(data, n_ints, nn, 1, rank);
            n_ints += nn;
        } else if (k == orc::K_FLOAT) { data.length = 4 * nn; data.at = scaled(rank, 4, 0); }
        else if (k == orc::K_DOUBLE) { data.length = 8 * nn; data.at = scaled(rank, 8, 0); }
        else { data.length = payload; data.at = bytes_at; }  // string bytes, decimal varints
        streams.push_back(data);
        if (is_bytes_kind(k) || k == orc::K_DECIMAL) {
            Stream second{(int)i, is_bytes_kind(k) ? orc::S_LENGTH : orc::S_SECONDARY};
            t.ints = n_ints;
            add_runs(second, n_ints, nn, is_bytes_kind(k) ? 0 : 1, rank);
            n_ints += nn;
            streams.push_back(second);
        }
    }
    fs.finish(*ef);

    // ---- compaction and run sizes
    const size_t nj = jobs.size();
    int64_t *d_ints = (int64_t *)scratch.take(sizeof(int64_t) * (size_t)n_ints + 64);
    uint8_t *d_bytes = (uint8_t *)scratch.take((size_t)n_bytes + 64);
    RleJob *d_jobs = (RleJob *)scratch.take(sizeof(RleJob) * std::max<size_t>(nj, 1));
    int32_t *d_sizes = (int32_t *)scratch.take(sizeof(int32_t) * std::max<size_t>(nj, 1));
    if (!d_ints || !d_bytes || !d_jobs || !d_sizes) return fail(PG_ERR_CUDA, "orc encode: out of device memory for the run scratch");
    std::vector<int32_t> sizes(nj);
    if (nt) {
        PG_CUDA(cudaMemsetAsync(d_bytes, 0, (size_t)n_bytes + 64, 0));
        PG_CUDA(cudaMemcpy(d_tasks, tasks.data(), sizeof(OeTask) * nt, cudaMemcpyHostToDevice));
        k_oe_values<<<(unsigned)nt, 256>>>(d_cols, d_tasks, 0, d_ints, d_bytes, nullptr);
        launches++;
    }
    if (nj) {
        PG_CUDA(cudaMemcpy(d_jobs, jobs.data(), sizeof(RleJob) * nj, cudaMemcpyHostToDevice));
        k_oe_rle_size<<<(unsigned)((nj + 127) / 128), 128>>>(d_jobs, (int)nj, d_ints, d_bytes, d_sizes);
        launches++;
        SmallReads rd(0);
        if ((st = rd.add(sizes.data(), d_sizes, sizeof(int32_t) * nj))) return st;
        launches++;
        if ((st = rd.finish())) return st;
    }
    for (Stream &sm : streams) {                             // lengths; a row group's job index -> its raw offset
        size_t r = 0;
        for (size_t j = sm.job0; j < sm.job1; j++) {
            for (; r < sm.at.size() && sm.at[r] == (int64_t)j; r++) sm.at[r] = sm.length;
            sm.length += sizes[j];
        }
        for (; sm.runs && r < sm.at.size(); r++) sm.at[r] = sm.length;
    }

    // ---- the raw streams: contiguous for ZSTD (a scratch image), at their file offsets for NONE (the file image)
    const bool zstd = codec == orc::C_ZSTD;
    std::vector<uint8_t> magic = {'O', 'R', 'C'};
    ef->host_parts.push_back({0, magic});
    std::vector<int> encodings(nc + 1, orc::E_DIRECT);
    for (int c = 0; c < nc; c++) {
        const int k = types[c].kind;
        if (k != orc::K_BYTE && k != orc::K_BOOLEAN && k != orc::K_FLOAT && k != orc::K_DOUBLE) encodings[c + 1] = orc::E_DIRECT_V2;
    }
    // the index streams of every stripe, stored, from the streams' positions (ZSTD: from the chunks' stored sizes):
    // per column, root first, its ROW_INDEX and for a bloom column its BLOOM_FILTER_UTF8
    std::vector<std::vector<std::pair<orc::OutStream, std::vector<uint8_t>>>> index(n_stripes);
    auto build_index = [&](const std::vector<int64_t> &chunk_stored) -> pg_status {
        if (!stride) return PG_OK;
        OutType root;
        root.kind = orc::K_STRUCT;
        const int64_t w64 = bloom_words / 2;
        size_t si = 0;
        for (int64_t g = 0; g < n_stripes; g++) {
            const int64_t ng = group0[g + 1] - group0[g];
            std::vector<std::vector<uint64_t>> pos(ng);
            std::vector<orc::ColumnStats> gs(ng);
            auto add = [&](int kind, int column, const std::vector<uint8_t> &raw) {
                std::vector<uint8_t> b = orc::compress_section(raw, codec, (uint64_t)block);
                index[g].push_back({orc::OutStream{kind, (uint32_t)column, (uint64_t)b.size()}, std::move(b)});
            };
            try {
                for (int64_t r = 0; r < ng; r++) gs[r].values = (uint64_t)spans[(size_t)((group0[g] + r) * nc)].rows;
                add(orc::S_ROW_INDEX, 0, orc::row_index(root, pos, gs));
                for (int c = 0; c < nc; c++) {
                    for (std::vector<uint64_t> &p : pos) p.clear();
                    for (; si < streams.size() && streams[si].task == (int)(g * nc + c); si++) {
                        const Stream &sm = streams[si];
                        size_t ch = 0;                           // ZSTD: the chunk holding the position, its offset
                        int64_t ch_off = 0;
                        for (int64_t r = 0; r < ng; r++) {
                            const int64_t raw = sm.at[r];
                            if (zstd) {
                                for (; ch < sm.chunk1 - sm.chunk0 && (int64_t)(ch + 1) * block <= raw; ch++)
                                    ch_off += 3 + chunk_stored[sm.chunk0 + ch];
                                pos[r].push_back((uint64_t)ch_off);
                                pos[r].push_back((uint64_t)(raw - (int64_t)ch * block));
                            } else pos[r].push_back((uint64_t)raw);
                            if (sm.runs) pos[r].push_back(0);    // every position starts a run
                            if (sm.kind == orc::S_PRESENT) pos[r].push_back(0);
                            else if (!sm.bit.empty()) pos[r].push_back(sm.bit[r]);
                        }
                    }
                    for (int64_t r = 0; r < ng; r++) gs[r] = span_stats[(size_t)((group0[g] + r) * nc + c)];
                    add(orc::S_ROW_INDEX, c + 1, orc::row_index(types[c], pos, gs));
                    const size_t b = std::find(bloom_cols.begin(), bloom_cols.end(), c) - bloom_cols.begin();
                    if (b < bloom_cols.size())
                        add(orc::S_BLOOM_FILTER_UTF8, c + 1,
                            orc::bloom_filter_index(bloom_k, filters.data() + (group0[g] * n_bloom + (int64_t)b * ng) * w64,
                                                    (size_t)w64, (size_t)ng));
                }
            } catch (const std::exception &e) { return fail(PG_ERR_INVALID, std::string("orc encode: ") + e.what()); }
        }
        return PG_OK;
    };
    // lays out the stripes from the streams' stored sizes: offsets, index streams, stripe footers, the tail
    auto layout = [&](std::vector<int64_t> &stream_off) -> pg_status {
        int64_t pos = 3;
        size_t si = 0;
        stream_off.assign(streams.size(), 0);
        for (int64_t g = 0; g < n_stripes; g++) {
            orc::OutStripe &sp = stripes[g];
            sp.offset = (uint64_t)pos;
            std::vector<orc::OutStream> list;
            for (const auto &x : index[g]) {
                list.push_back(x.first);
                ef->host_parts.push_back({pos, x.second});
                pos += (int64_t)x.second.size();
            }
            sp.index_length = (uint64_t)pos - sp.offset;
            for (; si < streams.size() && streams[si].task / nc == g; si++) {
                stream_off[si] = pos;
                pos += streams[si].stored;
                list.push_back(orc::OutStream{streams[si].kind, (uint32_t)(tasks[streams[si].task].col + 1),
                                              (uint64_t)streams[si].stored});
            }
            sp.data_length = (uint64_t)pos - sp.offset - sp.index_length;
            std::vector<uint8_t> foot;
            try {
                foot = orc::compress_section(orc::stripe_footer(list, encodings), codec, (uint64_t)block);
            } catch (const std::exception &e) { return fail(PG_ERR_INVALID, std::string("orc encode: ") + e.what()); }
            sp.footer_length = foot.size();
            ef->host_parts.push_back({pos, std::move(foot)});
            pos += (int64_t)sp.footer_length;
        }
        ef->data_end = pos;
        std::vector<std::string> col_names(nc);
        for (int c = 0; c < nc; c++) col_names[c] = names && names[c] ? names[c] : "c" + std::to_string(c);
        try {
            ef->host_parts.push_back({pos, orc::file_tail(types, col_names, stripes, file_stats, (uint64_t)n_rows,
                                                          (uint64_t)pos, codec, (uint64_t)block, (uint64_t)stride)});
        } catch (const std::exception &e) { return fail(PG_ERR_INVALID, std::string("orc encode: ") + e.what()); }
        ef->file_bytes = pos + (int64_t)ef->host_parts.back().second.size();
        return PG_OK;
    };
    std::vector<int64_t> stream_off;
    int64_t raw_bytes = 0;
    if (zstd) {
        for (Stream &sm : streams) { sm.raw_off = raw_bytes; raw_bytes += sm.length; }
    } else {
        for (Stream &sm : streams) sm.stored = sm.length;
        if ((st = build_index({}))) return st;
        if ((st = layout(stream_off))) return st;
        for (size_t i = 0; i < streams.size(); i++) streams[i].raw_off = stream_off[i];
    }
    for (Stream &sm : streams) {
        int64_t at = sm.raw_off;
        for (size_t j = sm.job0; j < sm.job1; j++) { jobs[j].dst = at; at += sizes[j]; }
        const int k = tasks[sm.task].kind;
        if (sm.kind == orc::S_DATA && (k == orc::K_FLOAT || k == orc::K_DOUBLE || k == orc::K_DECIMAL || is_bytes_kind(k)))
            tasks[sm.task].direct = sm.raw_off;
    }
    uint8_t *d_raw = nullptr;
    if (zstd) d_raw = (uint8_t *)scratch.take((size_t)raw_bytes + 64);
    else {
        if ((st = ef->alloc_image())) return st;
        d_raw = ef->d_file;
    }
    if (!d_raw) return fail(PG_ERR_CUDA, "orc encode: out of device memory for the stream image");
    if (nj) {
        PG_CUDA(cudaMemcpy(d_jobs, jobs.data(), sizeof(RleJob) * nj, cudaMemcpyHostToDevice));
        k_oe_rle_write<<<(unsigned)((nj + 127) / 128), 128>>>(d_jobs, (int)nj, d_ints, d_bytes, d_raw);
        launches++;
    }
    if (nt) {
        PG_CUDA(cudaMemcpy(d_tasks, tasks.data(), sizeof(OeTask) * nt, cudaMemcpyHostToDevice));
        k_oe_values<<<(unsigned)nt, 256>>>(d_cols, d_tasks, 1, d_ints, d_bytes, d_raw);
        launches++;
    }

    // ---- ZSTD: chunks of at most `block` bytes, one frame each; sizes back; layout; the chunk headers among the host
    // parts, each chunk behind its header, compressed or original
    if (zstd) {
        std::vector<ZstdFrames::Body> chunks;
        for (Stream &sm : streams) {
            sm.chunk0 = chunks.size();
            for (int64_t c0 = 0; c0 < sm.length; c0 += block)
                chunks.push_back({sm.raw_off + c0, std::min<int64_t>(block, sm.length - c0)});
            sm.chunk1 = chunks.size();
        }
        ZstdFrames frames("orc encode");
        std::vector<int64_t> stored, chunk_off(chunks.size());  // the frame sizes, then the bytes of each chunk's body
        if ((st = frames.compress(scratch, d_raw, chunks, &stored, &launches))) return st;
        std::vector<uint8_t> original(chunks.size());           // the frame is not smaller: the bytes as they are
        for (Stream &sm : streams) {
            sm.stored = 0;
            for (size_t c = sm.chunk0; c < sm.chunk1; c++) {
                original[c] = stored[c] >= chunks[c].bytes;
                if (original[c]) stored[c] = chunks[c].bytes;
                sm.stored += 3 + stored[c];
            }
        }
        if ((st = build_index(stored))) return st;
        if ((st = layout(stream_off))) return st;
        for (size_t i = 0; i < streams.size(); i++) {
            int64_t at = stream_off[i];
            for (size_t c = streams[i].chunk0; c < streams[i].chunk1; c++) {
                const uint32_t h = (uint32_t)stored[c] << 1 | original[c];
                ef->host_parts.push_back({at, {(uint8_t)h, (uint8_t)(h >> 8), (uint8_t)(h >> 16)}});
                chunk_off[c] = at + 3;
                at += 3 + stored[c];
            }
        }
        if ((st = ef->alloc_image())) return st;
        if ((st = frames.gather(chunk_off, original, ef->d_file, &launches))) return st;
    }
    ef->meta.n_rows = n_rows;
    ef->meta.n_row_groups = (int32_t)n_stripes;
    ef->meta.n_pages = (int32_t)streams.size();
    return finish_encode(tm, std::move(ef), launches, "orc encode", out_file);
}

}  // namespace

}  // namespace pg

extern "C" pg_status pg_orc_encode_indexed(uint64_t source, const char *const *column_names, int64_t row0,
                                           int64_t n_rows, const pg_orc_write_options *options,
                                           const pg_orc_index_options *index, uint64_t *out_file) {
    if (!out_file) return pg::fail(PG_ERR_INVALID, "null argument");
    return pg::encode_orc(source, column_names, row0, n_rows, options, index, out_file);
}

extern "C" pg_status pg_orc_encode(uint64_t source, const char *const *column_names, int64_t row0, int64_t n_rows,
                                   const pg_orc_write_options *options, uint64_t *out_file) {
    return pg_orc_encode_indexed(source, column_names, row0, n_rows, options, nullptr, out_file);
}
