// parquet_encode.cu — compaction output encode: a device-resident columnar batch -> one Parquet data file.
//
// Replaces, for the rewrite side of MergeTreeCompactRewriter.rewriteCompaction
// (paimon-core/.../mergetree/compact/MergeTreeCompactRewriter.java:78-116):
//   KeyValueDataFileWriter.write / result()  paimon-core/.../io/KeyValueDataFileWriter.java:108-184
//       (row count, min / max key, min / max sequence number, delete row count, per-column stats -> DataFileMeta)
//   ParquetRowDataWriter + RowDataParquetBuilder   paimon-format/.../parquet/writer/ParquetRowDataWriter.java,
//       RowDataParquetBuilder.java:58-119 (which drive parquet-mr 1.16.0's ParquetWriter; the byte layout restated
//       here is the public Parquet format specification, conformance is pinned by reading the files back with
//       pyarrow and with this library's own decoder)
//   Paimon -> Parquet type mapping   paimon-format/.../parquet/ParquetSchemaConverter.java:76-160
//       (TINYINT / SMALLINT / INT -> INT32 with INT_8 / INT_16 annotations, BIGINT -> INT64, STRING -> BYTE_ARRAY UTF8,
//        nullable -> OPTIONAL (max definition level 1), NOT NULL -> REQUIRED)
//
// Layout written: PAR1 | per row group, per column: data pages V1, PLAIN, uncompressed or one zstd frame per page
// body (pg_parquet_encode_compressed) | with page_index: every ColumnIndex, then every OffsetIndex (parquet-mr's
// order) | with bloom columns (pg_parquet_encode_bloom): every bloom filter, row group major, each a BloomFilterHeader
// and its bitset (32-byte aligned) | FileMetaData | len | PAR1.  Page bounds come from k_pw_stats, run per page (the
// chunk statistics are folded from the page words on the host), and for STRING / BINARY from k_pw_minmax_bytes.  The
// bloom filters' bits (sbbf_device.cuh) are set by k_pw_sbbf straight into the file image.
// Pages start at multiples of 8 rows, so a nullable column's definition levels (bit width 1, bit-packed LSB first)
// ARE the bytes of the Arrow validity bitmap: they are copied, not re-encoded.  Values of non-null rows are
// compacted by a block-wide scan; BYTE_ARRAY values are written as [len:int32][bytes].
#include <memory>
#include <string>

#include "device_utils.cuh"
#include "encoded_file.h"
#include "parquet_meta.h"
#include "sbbf_device.cuh"

namespace pg {

// ------------------------------------------------------------------ page jobs

struct EncJob {                   // one data page of one column
    int32_t col;
    int32_t n_rows;
    int64_t row0;                 // first row (multiple of 8 relative to the batch slice start, see row_shift)
    int64_t def_off;              // file offset of the definition-level bytes (the copied bitmap bytes), -1 = none
    int64_t val_off;              // file offset of the PLAIN values
};

// per job: non-null rows and (var-len) payload bytes of the non-null rows
__global__ void k_pw_count(const EncColumn *cols, const EncJob *jobs, int64_t *counts) {
    const EncJob j = jobs[blockIdx.x];
    const EncColumn c = cols[j.col];
    long long nn = 0, vb = 0;
    for (int i = threadIdx.x; i < j.n_rows; i += blockDim.x) {
        const int64_t row = j.row0 + i;
        const bool v = c.validity == nullptr || valid_bit(c.validity, row);
        if (v) {
            nn++;
            if (c.width == 0) vb += c.offsets[row + 1] - c.offsets[row];
        }
    }
    __shared__ long long s_nn, s_vb;
    if (threadIdx.x == 0) { s_nn = 0; s_vb = 0; }
    __syncthreads();
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        nn += __shfl_xor_sync(0xffffffffu, nn, d);
        vb += __shfl_xor_sync(0xffffffffu, vb, d);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd((unsigned long long *)&s_nn, (unsigned long long)nn);
        atomicAdd((unsigned long long *)&s_vb, (unsigned long long)vb);
    }
    __syncthreads();
    if (threadIdx.x == 0) { counts[2 * blockIdx.x] = s_nn; counts[2 * blockIdx.x + 1] = s_vb; }
}

// the page bodies: definition-level bytes (= bitmap bytes) and compacted PLAIN values
__global__ void __launch_bounds__(256)
k_pw_encode(const EncColumn *cols, const EncJob *jobs, uint8_t *file) {
    const EncJob j = jobs[blockIdx.x];
    const EncColumn c = cols[j.col];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ int ws[2][9];
    // definition levels: bit width 1, LSB first == the validity bitmap; an OPTIONAL column without a bitmap has
    // no nulls
    if (j.def_off >= 0) {
        const int nb = (j.n_rows + 7) >> 3;
        for (int b = tid; b < nb; b += blockDim.x) {
            uint8_t byte = c.validity ? c.validity[(j.row0 >> 3) + b] : 0xFF;
            const int rem = j.n_rows - b * 8;
            if (rem < 8) byte &= (uint8_t)((1u << rem) - 1);
            file[j.def_off + b] = byte;
        }
    }
    uint8_t *vals = file + j.val_off;
    int base_rank = 0, base_bytes = 0;
    for (int i0 = 0; i0 < j.n_rows; i0 += blockDim.x) {
        const int i = i0 + tid;
        const int64_t row = j.row0 + i;
        const bool v = i < j.n_rows && (c.validity == nullptr || valid_bit(c.validity, row));
        int len = 0, st = 0;
        if (v && c.width == 0) { st = c.offsets[row]; len = c.offsets[row + 1] - st; }
        // block-wide exclusive scans of (valid, len)
        const unsigned bal = __ballot_sync(0xffffffffu, v);
        const int wrank = __popc(bal & ((1u << lane) - 1));
        const int wincl = warp_scan_incl(len);
        if (lane == 31) { ws[0][warp] = __popc(bal); ws[1][warp] = wincl; }
        __syncthreads();
        if (warp == 0) {
            int a = lane < 8 ? ws[0][lane] : 0, b = lane < 8 ? ws[1][lane] : 0;
            const int ai = warp_scan_incl(a), bi = warp_scan_incl(b);
            if (lane < 8) { ws[0][lane] = ai - a; ws[1][lane] = bi - b; }
            if (lane == 7) { ws[0][8] = ai; ws[1][8] = bi; }
        }
        __syncthreads();
        const int rank = base_rank + ws[0][warp] + wrank;
        const int boff = base_bytes + ws[1][warp] + wincl - len;
        if (v) {
            if (c.width == 0) {
                uint8_t *d = vals + 4 * (int64_t)rank + boff;
                d[0] = (uint8_t)len; d[1] = (uint8_t)(len >> 8); d[2] = (uint8_t)(len >> 16); d[3] = (uint8_t)(len >> 24);
                const uint8_t *s = (const uint8_t *)c.data + st;
                for (int b = 0; b < len; b++) d[4 + b] = s[b];
            } else if (c.type == PG_BOOL) {
                // bit-packed, LSB first; the page region is zeroed, the containing aligned word may reach into
                // neighbouring bytes, which an OR of zero bits leaves alone
                if (((const uint8_t *)c.data)[row]) {
                    uint8_t *byte = vals + (rank >> 3);
                    unsigned int *word = (unsigned int *)((uintptr_t)byte & ~(uintptr_t)3);
                    atomicOr(word, 1u << ((((uintptr_t)byte & 3) << 3) + (rank & 7)));
                }
            } else if (c.width == 8) {
                uint64_t x = ((const uint64_t *)c.data)[row];
                memcpy(vals + 8 * (int64_t)rank, &x, 8);
            } else {
                // TINYINT / SMALLINT / INT -> INT32 (sign extended), FLOAT stays 4 bytes
                int32_t x;
                if (c.width == 4) x = ((const int32_t *)c.data)[row];
                else if (c.width == 2) x = ((const int16_t *)c.data)[row];
                else x = ((const int8_t *)c.data)[row];
                memcpy(vals + 4 * (int64_t)rank, &x, 4);
            }
        }
        base_rank += ws[0][8];
        base_bytes += ws[1][8];
        __syncthreads();
    }
}

// ------------------------------------------------------------------ bloom filters (SBBF)

struct SbbfJob {                  // the filter of one column chunk
    int32_t col;
    uint32_t n_blocks;            // bitset bytes / 32
    int64_t row0, n_rows;         // the chunk's rows
    int64_t bits_off;             // file offset of the bitset, a multiple of 32
};

// One thread per row of a chunk, blockIdx.y (strided) = the job: skip NULLs, hash the value's PLAIN bytes, set its
// eight bits in the bitset inside the file image (zeroed at allocation) with word atomics.
__global__ void __launch_bounds__(256) k_pw_sbbf(const EncColumn *cols, const SbbfJob *jobs, int n_jobs, uint8_t *file) {
    for (int jb = blockIdx.y; jb < n_jobs; jb += gridDim.y) {
        const SbbfJob j = jobs[jb];
        const EncColumn c = cols[j.col];
        uint32_t *bits = (uint32_t *)(file + j.bits_off);
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < j.n_rows;
             i += (int64_t)gridDim.x * blockDim.x) {
            const int64_t row = j.row0 + i;
            if (!valid_bit(c.validity, row)) continue;
            uint64_t h;
            if (c.width == 0) {
                const int32_t a = c.offsets[row], b = c.offsets[row + 1];
                h = fi::xxh64((const uint8_t *)c.data + a, b - a);
            } else if (c.width == 8) {
                h = sbbf::hash8(((const uint64_t *)c.data)[row]);
            } else {                                           // INT8 / INT16 sign-extended to INT32, FLOAT's bits
                const uint64_t v = load_fixed(c.data, c.width, row);
                h = sbbf::hash4(c.type == PG_FLOAT ? (uint32_t)v : (uint32_t)(int32_t)sext(v, c.width));
            }
            // the block as four 64-bit words (little-endian word pairs); an atomic only where a bit is still clear,
            // so that the rows of a low-cardinality column do not all queue on the same few addresses (a bit once
            // set stays set, so a stale read costs an atomic, never a bit)
            unsigned long long *blk = (unsigned long long *)(bits + 8 * (size_t)sbbf::block_of(h, j.n_blocks));
#pragma unroll
            for (int w = 0; w < 4; w++) {
                const unsigned long long m =
                    sbbf::mask_word(h, 2 * w) | (unsigned long long)sbbf::mask_word(h, 2 * w + 1) << 32;
                if ((__ldcg(blk + w) & m) != m) atomicOr(blk + w, m);
            }
        }
    }
}

// The bitset bytes of each file column's filter (0 = none) from `bloom`, or the refusal of a bad list
static pg_status bloom_sizes(const Schema &s, const pg_parquet_bloom_options *bloom, std::vector<int64_t> *bytes) {
    const int nc = s.n_cols();
    bytes->assign(nc, 0);
    if (!bloom || bloom->n_columns == 0) return PG_OK;
    if (bloom->n_columns < 0 || !bloom->columns)
        return fail(PG_ERR_INVALID, "parquet encode: bloom n_columns " + std::to_string(bloom->n_columns) +
                                        " is negative or its columns are NULL");
    for (int i = 0; i < bloom->n_columns; i++) {
        const pg_parquet_bloom_column &b = bloom->columns[i];
        const std::string col = "parquet encode: bloom column " + std::to_string(b.column);
        if (b.column < 0 || b.column >= nc) return fail(PG_ERR_INVALID, col + " is outside the schema");
        if ((*bytes)[b.column]) return fail(PG_ERR_INVALID, col + " is listed twice");
        if (b.ndv < 0) return fail(PG_ERR_INVALID, col + ": ndv " + std::to_string(b.ndv) + " is negative");
        if (!(b.fpp > 0 && b.fpp < 1))
            return fail(PG_ERR_INVALID, col + ": fpp " + std::to_string(b.fpp) + " is outside (0, 1)");
        if (s.field(b.column).type == PG_BOOL)
            return fail(PG_ERR_UNSUPPORTED, col + " is BOOLEAN, which Parquet bloom filters do not cover");
        (*bytes)[b.column] = sbbf::num_bytes(b.ndv, b.fpp);
    }
    return PG_OK;
}

// BloomFilterHeader: numBytes, algorithm BLOCK, hash XXHASH, compression UNCOMPRESSED (each union's first member, an
// empty struct)
static std::vector<uint8_t> bloom_header(int64_t bytes) {
    pq::ThriftWriter w;
    w.i32(1, (int32_t)bytes);
    for (int f = 2; f <= 4; f++) {
        w.struct_field(f);
        w.struct_field(1);
        w.end();
        w.end();
    }
    w.end();
    return std::move(w.b);
}

// ------------------------------------------------------------------ page index: bounds of var-len pages

constexpr int kTruncate = 64;     // parquet-mr's default column-index truncation length
constexpr int kHeadBytes = kTruncate + 1;

struct BytesBound {               // per page of a var-len column: its least [0] and its greatest [1] non-null value
    int64_t row[2];               // -1: the page has no non-null value
    int32_t start[2], len[2];     // where the value's bytes lie in the column's payload, and how many
    uint8_t head[2][kHeadBytes];  // its first min(len, kHeadBytes) bytes
};

// a candidate bound of a var-len page: its row (-1 = none) and where its bytes lie in the column's payload, kept in
// registers so that a comparison reads the payload of the row it is offered only
struct Cand { int64_t row; int32_t start, len; };

// unsigned-byte lexicographic order, a proper prefix first: < 0, 0 or > 0
__device__ __forceinline__ int cmp_values(const uint8_t *data, const Cand &a, const Cand &b) {
    const uint8_t *pa = data + a.start, *pb = data + b.start;
    const int n = min(a.len, b.len);
    for (int i = 0; i < n; i++)
        if (pa[i] != pb[i]) return (int)pa[i] - (int)pb[i];
    return a.len - b.len;
}

// x replaces lo when it is smaller, hi when it is greater
__device__ __forceinline__ void take_bounds(const uint8_t *data, Cand &lo, Cand &hi, const Cand &xlo, const Cand &xhi) {
    if (xlo.row >= 0 && (lo.row < 0 || cmp_values(data, xlo, lo) < 0)) lo = xlo;
    if (xhi.row >= 0 && (hi.row < 0 || cmp_values(data, xhi, hi) > 0)) hi = xhi;
}

__device__ __forceinline__ Cand shfl_xor(const Cand &c, int d) {
    return Cand{__shfl_xor_sync(0xffffffffu, c.row, d), __shfl_xor_sync(0xffffffffu, c.start, d),
                __shfl_xor_sync(0xffffffffu, c.len, d)};
}

// One CTA per var-len page (jobs[which[blockIdx.x]]): the rows of its least and greatest non-null value, found by a
// strided scan per thread, a shuffle reduction per warp and one across the warps, and the first kHeadBytes bytes of
// each, so that the host reads the bounds back in one small read.
__global__ void __launch_bounds__(256)
k_pw_minmax_bytes(const EncColumn *cols, const EncJob *jobs, const int32_t *which, BytesBound *out) {
    const EncJob j = jobs[which[blockIdx.x]];
    const EncColumn c = cols[j.col];
    const uint8_t *data = (const uint8_t *)c.data;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    Cand lo{-1, 0, 0}, hi{-1, 0, 0};
    for (int i = threadIdx.x; i < j.n_rows; i += blockDim.x) {
        const int64_t row = j.row0 + i;
        if (!valid_bit(c.validity, row)) continue;
        const int32_t st = c.offsets[row];
        const Cand x{row, st, c.offsets[row + 1] - st};
        take_bounds(data, lo, hi, x, x);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const Cand xlo = shfl_xor(lo, d), xhi = shfl_xor(hi, d);
        take_bounds(data, lo, hi, xlo, xhi);
    }
    __shared__ Cand s_lo[8], s_hi[8];
    if (lane == 0) { s_lo[warp] = lo; s_hi[warp] = hi; }
    __syncthreads();
    if (warp) return;
    const int nw = blockDim.x >> 5;
    if (lane < nw) { lo = s_lo[lane]; hi = s_hi[lane]; }
    else lo.row = hi.row = -1;
#pragma unroll
    for (int d = 4; d > 0; d >>= 1) {
        const Cand xlo = shfl_xor(lo, d), xhi = shfl_xor(hi, d);
        take_bounds(data, lo, hi, xlo, xhi);
    }
    BytesBound &o = out[blockIdx.x];
    for (int k = 0; k < 2; k++) {
        Cand b = k ? hi : lo;
        b = Cand{__shfl_sync(0xffffffffu, b.row, 0), __shfl_sync(0xffffffffu, b.start, 0),
                 __shfl_sync(0xffffffffu, b.len, 0)};
        if (lane == 0) { o.row[k] = b.row; o.start[k] = b.start; o.len[k] = b.len; }
        for (int i = lane; i < min(b.len, kHeadBytes); i += 32) o.head[k][i] = data[b.start + i];
    }
}

static int parquet_type_of(int t) {
    switch (t) {
        case PG_BOOL: return pq::T_BOOLEAN;
        case PG_INT8: case PG_INT16: case PG_INT32: return pq::T_INT32;
        case PG_INT64: return pq::T_INT64;
        case PG_FLOAT: return pq::T_FLOAT;
        case PG_DOUBLE: return pq::T_DOUBLE;
        default: return pq::T_BYTE_ARRAY;
    }
}

// The column chunks and data pages of a file, built in one pass over (row group, column, page).  jobs[p] and
// sjobs[p] are what the kernels read for pages[p], in arrays that go to the device as they are.
struct Page {
    std::vector<uint8_t> prefix;  // RLE-hybrid definition levels: [length:int32][run header varint]; empty = REQUIRED
    int64_t def_bytes = 0;        // prefix and level bytes
    int64_t body = 0;             // page body bytes
    int64_t stored = 0;           // bytes in the file: the body, or its zstd frame
    int64_t null_count = 0;
    bool nan = false;             // a non-null value is NaN
    std::vector<uint8_t> min, max;  // ColumnIndex bounds, PLAIN-encoded; empty for a page of NULLs only
    int64_t header_off = 0, header_bytes = 0;  // PageLocation: offset, and with `stored`, compressed_page_size
};
struct Chunk {
    int col;
    int64_t row0, n_rows;         // its rows (row0: the batch row its row group starts at)
    size_t page0, page1;          // its pages
    ColStats st;                  // the footer's Statistics
    int64_t first_page = 0, total_uncompressed = 0, total_compressed = 0;
    int64_t column_index_off = -1, offset_index_off = -1;   // -1: not written
    int32_t column_index_len = 0, offset_index_len = 0;
    int64_t bloom_off = -1;       // its BloomFilterHeader, -1: no filter
    int32_t bloom_len = 0;        // header and bitset
};
struct Plan {
    int64_t n_groups = 0;
    std::vector<EncColumn> cols;
    std::vector<EncJob> jobs;
    std::vector<Page> pages;
    std::vector<StatJob> sjobs;
    std::vector<Chunk> chunks;    // row group major, then column
};

static Plan make_plan(const Schema &s, const std::vector<DevColumn> &dcols, int64_t row0, int64_t n_rows,
                      const pg_parquet_write_options *opt) {
    Plan pl;
    int64_t page_rows = opt && opt->page_rows > 0 ? opt->page_rows : 32768;
    page_rows = (page_rows + 7) & ~(int64_t)7;
    int64_t group_rows = opt && opt->row_group_rows > 0 ? opt->row_group_rows : (int64_t)1 << 20;
    group_rows = ((group_rows + page_rows - 1) / page_rows) * page_rows;
    pl.n_groups = n_rows == 0 ? 0 : (n_rows + group_rows - 1) / group_rows;
    const int nc = s.n_cols();
    for (int c = 0; c < nc; c++) {
        pg_field f = s.field(c);
        pl.cols.push_back(EncColumn{dcols[c].data, dcols[c].offsets, dcols[c].validity, f.type, type_width(f.type),
                                    (f.nullable || dcols[c].validity) ? 1 : 0, 0});
    }
    for (int64_t g = 0; g < pl.n_groups; g++) {
        const int64_t g0 = row0 + g * group_rows, g1 = std::min(row0 + n_rows, g0 + group_rows);
        for (int c = 0; c < nc; c++) {
            const size_t page0 = pl.jobs.size();
            for (int64_t p0 = g0; p0 < g1; p0 += page_rows) {
                const int64_t n = std::min(g1, p0 + page_rows) - p0;
                pl.jobs.push_back(EncJob{c, (int32_t)n, p0, -1, 0});
                pl.sjobs.push_back(StatJob{c, 0, p0, n});
            }
            pl.chunks.push_back(Chunk{c, g0, g1 - g0, page0, pl.jobs.size(), ColStats{}});
        }
    }
    pl.pages.resize(pl.jobs.size());
    return pl;
}

// The k_pw_stats words of a chunk from those of its pages: min of the mins, max of the maxes (as doubles for FLOAT /
// DOUBLE: the words of a page without a non-NaN value are +inf / -inf), summed counts, NaN OR-ed.
static void fold_page_words(const EncColumn &ec, const int64_t *sw, size_t n_pages, int64_t *out) {
    const bool fp = ec.type == PG_FLOAT || ec.type == PG_DOUBLE;
    for (int w = 0; w < kStatWords; w++) out[w] = sw[w];
    for (size_t p = 1; p < n_pages; p++) {
        const int64_t *x = sw + kStatWords * p;
        if (fp) {
            double a, b, lo, hi;
            memcpy(&a, &out[0], 8); memcpy(&b, &out[1], 8); memcpy(&lo, &x[0], 8); memcpy(&hi, &x[1], 8);
            a = std::min(a, lo); b = std::max(b, hi);
            memcpy(&out[0], &a, 8); memcpy(&out[1], &b, 8);
        } else {
            out[0] = std::min(out[0], x[0]);
            out[1] = std::max(out[1], x[1]);
        }
        out[2] += x[2];
        out[3] += x[3];
        out[4] |= x[4];
    }
}

// a fixed-width bound PLAIN-encoded in the column's physical type: INT8 / INT16 / INT32 as 4 bytes, BOOLEAN as 1,
// FLOAT as 4 (`v` holds the double)
static std::vector<uint8_t> plain_bound(const EncColumn &ec, int64_t v) {
    uint8_t b[8];
    size_t n = ec.width == 8 ? 8 : 4;
    if (ec.type == PG_FLOAT) {
        double d; memcpy(&d, &v, 8);
        const float f = (float)d; memcpy(b, &f, 4);
    } else if (ec.type == PG_BOOL) {
        n = 1; b[0] = (uint8_t)v;
    } else if (n == 4) {
        const int32_t x = (int32_t)v; memcpy(b, &x, 4);
    } else memcpy(b, &v, 8);
    return std::vector<uint8_t>(b, b + n);
}

// The device's counts -> each page's level prefix and body size, each chunk's statistics (folded into the file's by
// `fs`) and, for a fixed-width column, each page's ColumnIndex entry.  counts: per page, non-null rows and payload
// bytes (k_pw_count); stats: per page, kStatWords (k_pw_stats).
static pg_status fold_counts(Plan &pl, const int64_t *counts, const int64_t *stats, FileStats &fs) {
    for (Chunk &ch : pl.chunks) {
        const EncColumn &ec = pl.cols[ch.col];
        int64_t words[kStatWords];
        fold_page_words(ec, &stats[kStatWords * ch.page0], ch.page1 - ch.page0, words);
        ch.st = fs.add(ch.col, ec, words, ch.n_rows);
        for (size_t p = ch.page0; p < ch.page1; p++) {
            Page &pg = pl.pages[p];
            const int64_t nn = counts[2 * p], vb = counts[2 * p + 1];
            const ColStats ps = piece_stats(ec, &stats[kStatWords * p], pl.jobs[p].n_rows);
            pg.null_count = ps.null_count;
            pg.nan = stats[kStatWords * p + 4] != 0;
            if (ps.has_minmax) { pg.min = plain_bound(ec, ps.min); pg.max = plain_bound(ec, ps.max); }
            if (ec.optional) {                                 // one bit-packed run of bit width 1
                const int64_t groups = (pl.jobs[p].n_rows + 7) / 8;
                std::vector<uint8_t> run;
                pq::put_varint(run, (uint64_t)(groups << 1) | 1);
                const uint32_t len = (uint32_t)(run.size() + groups);
                pg.prefix = {(uint8_t)len, (uint8_t)(len >> 8), (uint8_t)(len >> 16), (uint8_t)(len >> 24)};
                pg.prefix.insert(pg.prefix.end(), run.begin(), run.end());
                pg.def_bytes = (int64_t)pg.prefix.size() + groups;
            }
            int64_t val_bytes;
            if (ec.width == 0) val_bytes = 4 * nn + vb;
            else if (ec.type == PG_BOOL) val_bytes = (nn + 7) / 8;
            else val_bytes = nn * (ec.width == 8 ? 8 : 4);
            pg.body = pg.stored = pg.def_bytes + val_bytes;
            if (pg.body > 0x7fffffffLL) return fail(PG_ERR_UNSUPPORTED, "parquet encode: page larger than 2 GiB");
        }
    }
    return PG_OK;
}

// Places the body of page p at base[p]: its level prefix, the definition-level bytes behind it, the values behind
// those.  Sets the jobs' def_off / val_off and returns the prefixes, which the caller puts in place.
static std::vector<Part> place_bodies(Plan &pl, const std::vector<int64_t> &base) {
    std::vector<Part> prefixes;
    for (size_t p = 0; p < pl.pages.size(); p++) {
        const Page &pg = pl.pages[p];
        if (!pg.prefix.empty()) {
            prefixes.push_back({base[p], pg.prefix});
            pl.jobs[p].def_off = base[p] + (int64_t)pg.prefix.size();
        }
        pl.jobs[p].val_off = base[p] + pg.def_bytes;
    }
    return prefixes;
}

// PageHeader of a data page V1: PLAIN values, RLE levels
static std::vector<uint8_t> page_header(const Page &pg, int32_t n_rows) {
    pq::ThriftWriter w;
    w.i32(1, pq::P_DATA);
    w.i32(2, (int32_t)pg.body);
    w.i32(3, (int32_t)pg.stored);
    w.struct_field(5);                                         // DataPageHeader
    w.i32(1, n_rows);
    w.i32(2, pq::E_PLAIN);
    w.i32(3, pq::E_RLE);
    w.i32(4, pq::E_RLE);
    w.end();
    w.end();
    return std::move(w.b);
}

// Statistics max_value / min_value: a chunk's bounds, PLAIN-encoded in the column's physical type
static void write_min_max(pq::ThriftWriter &w, const EncColumn &ec, const ColStats &st) {
    const std::vector<uint8_t> mn = plain_bound(ec, st.min), mx = plain_bound(ec, st.max);
    w.bin(5, mx.data(), mx.size());
    w.bin(6, mn.data(), mn.size());
}

// ------------------------------------------------------------------ page index (ColumnIndex, OffsetIndex)

// The var-len bounds of the ColumnIndex, truncated to kTruncate bytes as parquet-mr truncates them.  `v` holds the
// first min(len, kHeadBytes) bytes of a value of `len` bytes.  A longer min becomes its prefix (STRING: cut back to a
// code-point boundary); a longer max becomes that prefix up to its last position that can be incremented, incremented
// (BINARY: a byte below 0xFF; STRING: a code point below U+10FFFF, the surrogates skipped), so min <= value <= max
// holds.  When no position can be incremented the max is the whole value, and *whole is set.
static int utf8_cut(const uint8_t *v, bool utf8) {
    int n = kTruncate;
    if (utf8)
        while (n > 0 && (v[n] & 0xC0) == 0x80) n--;
    return n;
}

static std::vector<uint8_t> truncate_min(const uint8_t *v, int len, bool utf8) {
    return std::vector<uint8_t>(v, v + (len <= kTruncate ? len : utf8_cut(v, utf8)));
}

// the code point of the UTF-8 sequence v[s, e), -1 if it is not one well-formed sequence
static int32_t utf8_decode(const uint8_t *v, int s, int e) {
    const int n = e - s;
    const uint8_t b0 = v[s];
    int want;
    int32_t cp;
    if (b0 < 0x80) { want = 1; cp = b0; }
    else if ((b0 & 0xE0) == 0xC0) { want = 2; cp = b0 & 0x1F; }
    else if ((b0 & 0xF0) == 0xE0) { want = 3; cp = b0 & 0x0F; }
    else if ((b0 & 0xF8) == 0xF0) { want = 4; cp = b0 & 0x07; }
    else return -1;
    if (n != want) return -1;
    for (int i = 1; i < n; i++) {
        if ((v[s + i] & 0xC0) != 0x80) return -1;
        cp = (cp << 6) | (v[s + i] & 0x3F);
    }
    static const int32_t least[5] = {0, 0, 0x80, 0x800, 0x10000};
    if (cp < least[n] || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return -1;
    return cp;
}

static void utf8_encode(std::vector<uint8_t> &b, int32_t cp) {
    if (cp < 0x80) b.push_back((uint8_t)cp);
    else if (cp < 0x800) { b.push_back((uint8_t)(0xC0 | (cp >> 6))); b.push_back((uint8_t)(0x80 | (cp & 0x3F))); }
    else if (cp < 0x10000) {
        b.push_back((uint8_t)(0xE0 | (cp >> 12)));
        b.push_back((uint8_t)(0x80 | ((cp >> 6) & 0x3F)));
        b.push_back((uint8_t)(0x80 | (cp & 0x3F)));
    } else {
        b.push_back((uint8_t)(0xF0 | (cp >> 18)));
        b.push_back((uint8_t)(0x80 | ((cp >> 12) & 0x3F)));
        b.push_back((uint8_t)(0x80 | ((cp >> 6) & 0x3F)));
        b.push_back((uint8_t)(0x80 | (cp & 0x3F)));
    }
}

static std::vector<uint8_t> truncate_max(const uint8_t *v, int len, bool utf8, bool *whole) {
    *whole = false;
    if (len <= kTruncate) return std::vector<uint8_t>(v, v + len);
    int end = utf8_cut(v, utf8);
    while (end > 0) {
        if (!utf8) {
            if (v[end - 1] != 0xFF) {
                std::vector<uint8_t> out(v, v + end);
                out.back()++;
                return out;
            }
            end--;
            continue;
        }
        int s = end - 1;
        while (s > 0 && end - s < 4 && (v[s] & 0xC0) == 0x80) s--;
        int32_t cp = utf8_decode(v, s, end);
        if (cp < 0) { end--; continue; }                        // not a code point: that byte is skipped
        if (cp < 0x10FFFF) {
            std::vector<uint8_t> out(v, v + s);
            utf8_encode(out, cp + 1 == 0xD800 ? 0xE000 : cp + 1);
            return out;
        }
        end = s;
    }
    *whole = true;
    return {};
}

// two PLAIN-encoded bounds in the column's order: signed integers, numeric FLOAT / DOUBLE, unsigned bytes
template <typename T> static int cmp_as(const std::vector<uint8_t> &a, const std::vector<uint8_t> &b) {
    T x, y;
    memcpy(&x, a.data(), sizeof(T)); memcpy(&y, b.data(), sizeof(T));
    return (x > y) - (x < y);
}
static int cmp_bound(const EncColumn &ec, const std::vector<uint8_t> &a, const std::vector<uint8_t> &b) {
    switch (ec.type) {
        case PG_FLOAT: return cmp_as<float>(a, b);
        case PG_DOUBLE: return cmp_as<double>(a, b);
        case PG_BOOL: return cmp_as<uint8_t>(a, b);
        default:
            if (ec.width == 0) return a < b ? -1 : (b < a ? 1 : 0);
            return ec.width == 8 ? cmp_as<int64_t>(a, b) : cmp_as<int32_t>(a, b);
    }
}

enum BoundaryOrder { B_UNORDERED = 0, B_ASCENDING = 1, B_DESCENDING = 2 };

// ColumnIndex of a chunk: null_pages, min_values, max_values, boundary_order (over the non-null pages), null_counts
static std::vector<uint8_t> column_index(const Plan &pl, const Chunk &ch) {
    const EncColumn &ec = pl.cols[ch.col];
    bool asc = true, desc = true;
    const Page *prev = nullptr;
    for (size_t p = ch.page0; p < ch.page1; p++) {
        const Page &pg = pl.pages[p];
        if (pg.null_count == pl.jobs[p].n_rows) continue;
        if (prev) {
            const int lo = cmp_bound(ec, prev->min, pg.min), hi = cmp_bound(ec, prev->max, pg.max);
            asc = asc && lo <= 0 && hi <= 0;
            desc = desc && lo >= 0 && hi >= 0;
        }
        prev = &pg;
    }
    const size_t n = ch.page1 - ch.page0;
    pq::ThriftWriter w;
    w.list(1, pq::CT_TRUE, n);                                 // (bool elements: 1 true, 2 false)
    for (size_t p = ch.page0; p < ch.page1; p++)
        w.b.push_back(pl.pages[p].null_count == pl.jobs[p].n_rows ? pq::CT_TRUE : pq::CT_FALSE);
    w.list(2, pq::CT_BINARY, n);
    for (size_t p = ch.page0; p < ch.page1; p++) w.binary(pl.pages[p].min.data(), pl.pages[p].min.size());
    w.list(3, pq::CT_BINARY, n);
    for (size_t p = ch.page0; p < ch.page1; p++) w.binary(pl.pages[p].max.data(), pl.pages[p].max.size());
    w.i32(4, asc ? B_ASCENDING : desc ? B_DESCENDING : B_UNORDERED);
    w.list(5, pq::CT_I64, n);
    for (size_t p = ch.page0; p < ch.page1; p++) w.zigzag(pl.pages[p].null_count);
    w.end();
    return std::move(w.b);
}

// OffsetIndex of a chunk: per page {offset, compressed_page_size, first_row_index (in the row group)}
static std::vector<uint8_t> offset_index(const Plan &pl, const Chunk &ch) {
    pq::ThriftWriter w;
    w.list(1, pq::CT_STRUCT, ch.page1 - ch.page0);
    for (size_t p = ch.page0; p < ch.page1; p++) {
        const Page &pg = pl.pages[p];
        w.struct_elem();
        w.i64(1, pg.header_off);
        w.i32(2, (int32_t)(pg.header_bytes + pg.stored));
        w.i64(3, pl.jobs[p].row0 - ch.row0);
        w.end();
    }
    w.end();
    return std::move(w.b);
}

// The ColumnIndex bounds of the var-len pages pl.jobs[which[i]] from their k_pw_minmax_bytes records bb[i].  A max
// that has to be written whole is read in one more round of small reads.
static pg_status varlen_bounds(Plan &pl, const std::vector<int32_t> &which, const std::vector<BytesBound> &bb) {
    struct Whole { int32_t page; std::vector<uint8_t> bytes; const uint8_t *src; };
    std::vector<Whole> whole;
    for (size_t i = 0; i < which.size(); i++) {
        const BytesBound &b = bb[i];
        if (b.row[0] < 0) continue;                            // NULLs only
        const EncColumn &ec = pl.cols[pl.jobs[which[i]].col];
        const bool utf8 = ec.type == PG_STRING;
        Page &pg = pl.pages[which[i]];
        bool need_whole;
        pg.min = truncate_min(b.head[0], b.len[0], utf8);
        pg.max = truncate_max(b.head[1], b.len[1], utf8, &need_whole);
        if (need_whole)
            whole.push_back({which[i], std::vector<uint8_t>((size_t)b.len[1]), (const uint8_t *)ec.data + b.start[1]});
    }
    if (whole.empty()) return PG_OK;
    SmallReads rd(0);
    for (Whole &x : whole)
        if (pg_status st = rd.add(x.bytes.data(), x.src, x.bytes.size())) return st;
    if (pg_status st = rd.finish()) return st;
    for (Whole &x : whole) pl.pages[x.page].max = std::move(x.bytes);
    return PG_OK;
}

// A chunk gets a ColumnIndex unless a page holds a NaN (parquet-mr drops the column index of such a chunk)
static bool has_column_index(const Plan &pl, const Chunk &ch) {
    for (size_t p = ch.page0; p < ch.page1; p++)
        if (pl.pages[p].nan) return false;
    return true;
}

// FileMetaData, its length and "PAR1": the end of the file
static std::vector<uint8_t> footer(const Plan &pl, const char *const *names, int64_t n_rows, bool zstd) {
    const int nc = (int)pl.cols.size();
    std::vector<std::string> col_names(nc);
    for (int c = 0; c < nc; c++) col_names[c] = names && names[c] ? names[c] : "c" + std::to_string(c);
    pq::ThriftWriter w;
    w.i32(1, 1);                                               // version
    w.list(2, pq::CT_STRUCT, (size_t)nc + 1);                  // schema
    w.struct_elem();
    w.str(4, "paimon_schema");
    w.i32(5, nc);
    w.end();
    for (int c = 0; c < nc; c++) {
        const EncColumn &ec = pl.cols[c];
        w.struct_elem();
        w.i32(1, parquet_type_of(ec.type));
        w.i32(3, ec.optional ? pq::R_OPTIONAL : pq::R_REQUIRED);
        w.str(4, col_names[c]);
        if (ec.type == PG_STRING) w.i32(6, 0);                 // UTF8
        else if (ec.type == PG_INT8) w.i32(6, 15);             // INT_8
        else if (ec.type == PG_INT16) w.i32(6, 16);            // INT_16
        w.end();
    }
    w.i64(3, n_rows);
    w.list(4, pq::CT_STRUCT, (size_t)pl.n_groups);
    for (int64_t g = 0; g < pl.n_groups; g++) {
        w.struct_elem();                                       // RowGroup
        w.list(1, pq::CT_STRUCT, (size_t)nc);
        int64_t group_bytes = 0;
        for (int c = 0; c < nc; c++) {
            const size_t k = (size_t)g * nc + c;
            const Chunk &ch = pl.chunks[k];
            group_bytes += ch.total_uncompressed;
            w.struct_elem();                                   // ColumnChunk
            w.i64(2, ch.first_page);
            w.struct_field(3);                                 // ColumnMetaData
            w.i32(1, parquet_type_of(pl.cols[c].type));
            w.list(2, pq::CT_I32, 2); w.zigzag(pq::E_PLAIN); w.zigzag(pq::E_RLE);
            w.list(3, pq::CT_BINARY, 1); w.binary(col_names[c].data(), col_names[c].size());
            w.i32(4, zstd ? pq::C_ZSTD : pq::C_UNCOMPRESSED);
            w.i64(5, ch.n_rows);
            w.i64(6, ch.total_uncompressed);
            w.i64(7, ch.total_compressed);
            w.i64(9, ch.first_page);
            w.struct_field(12);                                // Statistics
            w.i64(3, ch.st.null_count);
            if (ch.st.has_minmax) write_min_max(w, pl.cols[c], ch.st);
            w.end();
            if (ch.bloom_off >= 0) {
                w.i64(14, ch.bloom_off);
                w.i32(15, ch.bloom_len);
            }
            w.end();                                           // ColumnMetaData
            if (ch.offset_index_off >= 0) {
                w.i64(4, ch.offset_index_off);
                w.i32(5, ch.offset_index_len);
            }
            if (ch.column_index_off >= 0) {
                w.i64(6, ch.column_index_off);
                w.i32(7, ch.column_index_len);
            }
            w.end();                                           // ColumnChunk
        }
        w.i64(2, group_bytes);
        w.i64(3, pl.chunks[(size_t)g * nc].n_rows);            // the rows of the group: those of any of its chunks
        w.end();
    }
    w.str(6, "paimon-b200 (libpaimon_gpu)");
    // column_orders: TYPE_ORDER (TypeDefinedOrder) for every column.  Readers take min_value / max_value only from a
    // file that declares the order they were computed in; without it parquet-cpp (pyarrow) ignores them.
    w.list(7, pq::CT_STRUCT, (size_t)nc);
    for (int c = 0; c < nc; c++) {
        w.struct_elem();                                       // ColumnOrder (union)
        w.struct_field(1);                                     // TYPE_ORDER: TypeDefinedOrder, no fields
        w.end();
        w.end();
    }
    w.end();
    const uint32_t flen = (uint32_t)w.b.size();
    w.b.insert(w.b.end(), {(uint8_t)flen, (uint8_t)(flen >> 8), (uint8_t)(flen >> 16), (uint8_t)(flen >> 24), 'P', 'A', 'R', '1'});
    return std::move(w.b);
}

static pg_status encode(uint64_t source, const char *const *names, int64_t row0, int64_t n_rows,
                        const pg_parquet_write_options *opt, int codec, const pg_parquet_bloom_options *bloom,
                        uint64_t *out_file) {
    if (opt && opt->page_index != 0 && opt->page_index != 1)
        return fail(PG_ERR_INVALID, "parquet encode: page_index " + std::to_string(opt->page_index) + " is not 0 or 1");
    const bool page_index = opt && opt->page_index == 1;
    BatchColumns batch;                                      // held until the encode below is done
    pg_status st = encode_source(source, "parquet encode", row0, &n_rows, &batch);
    if (st) return st;
    const Schema *s = batch.schema.get();
    const int nc = s->n_cols();
    std::vector<int64_t> bloom_bytes;                        // per column: its filters' bitset bytes, 0 = none
    if ((st = bloom_sizes(*s, bloom, &bloom_bytes))) return st;

    SectionTimer tm;
    if ((st = start_encode(tm))) return st;

    Plan pl = make_plan(*s, batch.cols, row0, n_rows, opt);
    const size_t nj = pl.jobs.size();
    std::vector<int32_t> vpages;                             // the var-len pages, whose bounds k_pw_minmax_bytes finds
    for (size_t p = 0; page_index && p < nj; p++)
        if (pl.cols[pl.jobs[p].col].width == 0) vpages.push_back((int32_t)p);
    const size_t nv = vpages.size();
    std::vector<int64_t> counts(2 * nj + 2), stats(kStatWords * (nj + 1));
    std::vector<BytesBound> bounds(nv);
    Scratch scratch(0);                                      // temporaries, released on every path out of this function
    EncColumn *d_cols = (EncColumn *)scratch.take(sizeof(EncColumn) * nc);
    EncJob *d_jobs = (EncJob *)scratch.take(sizeof(EncJob) * std::max<size_t>(nj, 1));
    StatJob *d_sjobs = (StatJob *)scratch.take(sizeof(StatJob) * std::max<size_t>(nj, 1));
    int64_t *d_counts = (int64_t *)scratch.take(sizeof(int64_t) * (2 * nj + 2));
    int64_t *d_stats = (int64_t *)scratch.take(sizeof(int64_t) * kStatWords * (nj + 1));
    int32_t *d_vpages = (int32_t *)scratch.take(sizeof(int32_t) * std::max<size_t>(nv, 1));
    BytesBound *d_bounds = (BytesBound *)scratch.take(sizeof(BytesBound) * std::max<size_t>(nv, 1));
    if (!d_cols || !d_jobs || !d_sjobs || !d_counts || !d_stats || !d_vpages || !d_bounds)
        return fail(PG_ERR_CUDA, "parquet encode: out of device memory for the page tables");
    PG_CUDA(cudaMemcpy(d_cols, pl.cols.data(), sizeof(EncColumn) * nc, cudaMemcpyHostToDevice));
    int launches = 0;
    if (nj) {
        PG_CUDA(cudaMemcpy(d_jobs, pl.jobs.data(), sizeof(EncJob) * nj, cudaMemcpyHostToDevice));
        PG_CUDA(cudaMemcpy(d_sjobs, pl.sjobs.data(), sizeof(StatJob) * nj, cudaMemcpyHostToDevice));
        k_pw_count<<<(unsigned)nj, 256>>>(d_cols, d_jobs, d_counts);
        launch_pw_stats(d_cols, d_sjobs, (int)nj, d_stats);
        launches += 2;
        if (nv) {
            PG_CUDA(cudaMemcpy(d_vpages, vpages.data(), sizeof(int32_t) * nv, cudaMemcpyHostToDevice));
            k_pw_minmax_bytes<<<(unsigned)nv, 256>>>(d_cols, d_jobs, d_vpages, d_bounds);
            launches++;
        }
        PG_CUDA(cudaMemcpy(counts.data(), d_counts, sizeof(int64_t) * 2 * nj, cudaMemcpyDeviceToHost));
        PG_CUDA(cudaMemcpy(stats.data(), d_stats, sizeof(int64_t) * kStatWords * nj, cudaMemcpyDeviceToHost));
        if (nv) {
            SmallReads rd(0);
            if ((st = rd.add(bounds.data(), d_bounds, sizeof(BytesBound) * nv)) || (st = rd.finish())) return st;
            launches++;
        }
    }
    auto ef = std::make_unique<EncodedFile>();
    FileStats fs(*s);
    if ((st = fold_counts(pl, counts.data(), stats.data(), fs))) return st;
    fs.finish(*ef);
    if ((st = varlen_bounds(pl, vpages, bounds))) return st;

    // ---- zstd: bodies into a scratch image, one frame per body; the frame sizes come back before the layout
    const bool zstd = codec == pq::C_ZSTD;
    ZstdFrames frames("parquet encode");
    if (zstd && nj) {
        std::vector<ZstdFrames::Body> bodies;
        std::vector<int64_t> img_off(nj), frame_bytes;
        int64_t img = 0;
        for (size_t p = 0; p < nj; p++) {
            img_off[p] = img;
            bodies.push_back({img, pl.pages[p].body});
            img += pl.pages[p].body;
        }
        const std::vector<Part> prefixes = place_bodies(pl, img_off);
        uint8_t *d_img = (uint8_t *)scratch.take((size_t)img + 64);
        if (!d_img) return fail(PG_ERR_CUDA, "parquet encode: out of device memory for the zstd page images");
        PG_CUDA(cudaMemsetAsync(d_img, 0, (size_t)img + 64, 0));
        PG_CUDA(cudaMemcpy(d_jobs, pl.jobs.data(), sizeof(EncJob) * nj, cudaMemcpyHostToDevice));
        k_pw_encode<<<(unsigned)nj, 256>>>(d_cols, d_jobs, d_img);
        launches++;
        if ((st = patch(scratch, prefixes, d_img, "the zstd page images"))) return st;
        if (!prefixes.empty()) launches++;
        if ((st = frames.compress(scratch, d_img, bodies, &frame_bytes, &launches))) return st;
        for (size_t p = 0; p < nj; p++) pl.pages[p].stored = frame_bytes[p];
    }

    // ---- layout: "PAR1", per page its header and its stored body, with the page index every ColumnIndex and then
    // every OffsetIndex (row group major, then column), the footer
    int64_t pos = 4;
    ef->host_parts.push_back({0, {'P', 'A', 'R', '1'}});
    std::vector<int64_t> body_off(nj);
    for (Chunk &ch : pl.chunks) {
        ch.first_page = pos;
        for (size_t p = ch.page0; p < ch.page1; p++) {
            Page &pg = pl.pages[p];
            std::vector<uint8_t> header = page_header(pg, pl.jobs[p].n_rows);
            const int64_t hb = (int64_t)header.size();
            ef->host_parts.push_back({pos, std::move(header)});
            pg.header_off = pos;
            pg.header_bytes = hb;
            body_off[p] = pos + hb;
            pos += hb + pg.stored;
            ch.total_uncompressed += hb + pg.body;
            ch.total_compressed += hb + pg.stored;
        }
    }
    ef->data_end = pos;
    if (page_index) {
        for (Chunk &ch : pl.chunks) {
            if (!has_column_index(pl, ch)) continue;
            std::vector<uint8_t> ci = column_index(pl, ch);
            ch.column_index_off = pos;
            ch.column_index_len = (int32_t)ci.size();
            pos += (int64_t)ci.size();
            ef->host_parts.push_back({ch.column_index_off, std::move(ci)});
        }
        for (Chunk &ch : pl.chunks) {
            std::vector<uint8_t> oi = offset_index(pl, ch);
            ch.offset_index_off = pos;
            ch.offset_index_len = (int32_t)oi.size();
            pos += (int64_t)oi.size();
            ef->host_parts.push_back({ch.offset_index_off, std::move(oi)});
        }
    }
    // every bloom filter (row group major, then column), each header placed so that its bitset starts on a 32-byte
    // boundary; the bitsets are written on the device, so the device's part of the image reaches to the last one
    std::vector<SbbfJob> bjobs;
    int64_t bloom_rows = 0;
    for (Chunk &ch : pl.chunks) {
        const int64_t nb = bloom_bytes[ch.col];
        if (!nb) continue;
        std::vector<uint8_t> hdr = bloom_header(nb);
        const int64_t hb = (int64_t)hdr.size(), bits_off = (pos + hb + 31) & ~(int64_t)31;
        ch.bloom_off = bits_off - hb;
        ch.bloom_len = (int32_t)(hb + nb);
        ef->host_parts.push_back({ch.bloom_off, std::move(hdr)});
        bjobs.push_back(SbbfJob{ch.col, (uint32_t)(nb / 32), ch.row0, ch.n_rows, bits_off});
        bloom_rows = std::max(bloom_rows, ch.n_rows);
        pos = bits_off + nb;
        ef->data_end = pos;
    }
    ef->host_parts.push_back({pos, footer(pl, names, n_rows, zstd)});
    ef->file_bytes = pos + (int64_t)ef->host_parts.back().second.size();

    // ---- page bodies on the device: the zstd frames gathered, or the bodies written in place behind their prefixes
    if ((st = ef->alloc_image())) return st;
    if (nj && zstd) {
        if ((st = frames.gather(body_off, {}, ef->d_file, &launches))) return st;
    } else if (nj) {
        for (Part &prefix : place_bodies(pl, body_off)) ef->host_parts.push_back(std::move(prefix));
        PG_CUDA(cudaMemcpy(d_jobs, pl.jobs.data(), sizeof(EncJob) * nj, cudaMemcpyHostToDevice));
        k_pw_encode<<<(unsigned)nj, 256>>>(d_cols, d_jobs, ef->d_file);
        launches++;
    }
    if (!bjobs.empty()) {
        SbbfJob *d_bjobs = (SbbfJob *)scratch.take(sizeof(SbbfJob) * bjobs.size());
        if (!d_bjobs) return fail(PG_ERR_CUDA, "parquet encode: out of device memory for the bloom filter jobs");
        PG_CUDA(cudaMemcpy(d_bjobs, bjobs.data(), sizeof(SbbfJob) * bjobs.size(), cudaMemcpyHostToDevice));
        const int64_t bx = std::min<int64_t>(std::max<int64_t>((bloom_rows + 255) / 256, 1), 4096);
        const unsigned by = (unsigned)std::min<size_t>(bjobs.size(), 65535);
        k_pw_sbbf<<<dim3((unsigned)bx, by), 256>>>(d_cols, d_bjobs, (int)bjobs.size(), ef->d_file);
        launches++;
    }
    ef->meta.n_rows = n_rows;
    ef->meta.n_row_groups = (int32_t)pl.n_groups;
    ef->meta.n_pages = (int)nj;
    return finish_encode(tm, std::move(ef), launches, "parquet encode", out_file);
}

}  // namespace pg

using namespace pg;

extern "C" {

pg_status pg_parquet_encode(uint64_t source, const char *const *column_names, int64_t row0, int64_t n_rows,
                            const pg_parquet_write_options *options, uint64_t *out_file) {
    if (!out_file) return fail(PG_ERR_INVALID, "null argument");
    return encode(source, column_names, row0, n_rows, options, pq::C_UNCOMPRESSED, nullptr, out_file);
}

pg_status pg_parquet_encode_compressed(uint64_t source, const char *const *column_names, int64_t row0, int64_t n_rows,
                                       const pg_parquet_write_options *options, int32_t codec, int32_t level,
                                       uint64_t *out_file) {
    return pg_parquet_encode_bloom(source, column_names, row0, n_rows, options, codec, level, nullptr, out_file);
}

pg_status pg_parquet_encode_bloom(uint64_t source, const char *const *column_names, int64_t row0, int64_t n_rows,
                                  const pg_parquet_write_options *options, int32_t codec, int32_t level,
                                  const pg_parquet_bloom_options *bloom, uint64_t *out_file) {
    if (!out_file) return fail(PG_ERR_INVALID, "null argument");
    if (codec < pq::C_UNCOMPRESSED || codec > pq::C_LZ4_RAW)
        return fail(PG_ERR_INVALID, "parquet encode: codec " + std::to_string(codec) + " is not a Parquet CompressionCodec");
    if (codec != pq::C_UNCOMPRESSED && codec != pq::C_ZSTD)
        return fail(PG_ERR_UNSUPPORTED, "parquet encode: codec " + std::to_string(codec) +
                                            " is not written on the device (UNCOMPRESSED and ZSTD are)");
    if (codec == pq::C_ZSTD && (level == 0 || level > 1))
        return fail(PG_ERR_UNSUPPORTED, "parquet encode: file.compression.zstd-level " + std::to_string(level) +
                                            " is not written on the device (level 1 and the negative fast levels are)");
    return encode(source, column_names, row0, n_rows, options, codec, bloom, out_file);
}

}  // extern "C"
