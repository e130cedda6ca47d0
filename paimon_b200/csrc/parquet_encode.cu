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
// body (pg_parquet_encode_compressed) | FileMetaData | len | PAR1.
// Pages start at multiples of 8 rows, so a nullable column's definition levels (bit width 1, bit-packed LSB first)
// ARE the bytes of the Arrow validity bitmap: they are copied, not re-encoded.  Values of non-null rows are
// compacted by a block-wide scan; BYTE_ARRAY values are written as [len:int32][bytes].
#include <memory>
#include <string>

#include "device_utils.cuh"
#include "parquet_meta.h"
#include "zstd_encode_device.cuh"

namespace pg {

// ------------------------------------------------------------------ page jobs

struct EncColumn {
    const void *data;
    const int32_t *offsets;
    const uint8_t *validity;     // NULL = no nulls
    int32_t type;                // pg_type
    int32_t width;               // bytes in memory, 0 = var-len
    int32_t optional;            // OPTIONAL in the file (definition levels are written)
    int32_t pad;
};

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

// per column chunk (one CTA): min / max of the non-null values of a fixed-width numeric column, as int64 / double
// bit patterns (FLOAT / DOUBLE: of the non-NaN values, whichever zero comes first; the host applies the zero rule),
// whether a non-null value is NaN; also used for the sequence number range and the delete count (kind column)
struct StatJob { int32_t col; int32_t pad; int64_t row0; int64_t n_rows; };
constexpr int kStatWords = 5;     // per job: min, max, non-null rows, retracts, NaN seen
__global__ void k_pw_stats(const EncColumn *cols, const StatJob *jobs, int64_t *out /* [job][kStatWords] */) {
    const StatJob j = jobs[blockIdx.x];
    const EncColumn c = cols[j.col];
    const bool fp = c.type == PG_FLOAT || c.type == PG_DOUBLE;
    int64_t imin = INT64_MAX, imax = INT64_MIN;
    double dmin = INFINITY, dmax = -INFINITY;
    long long nn = 0, retr = 0;
    bool nan_seen = false;
    for (int64_t i = threadIdx.x; i < j.n_rows; i += blockDim.x) {
        const int64_t row = j.row0 + i;
        if (c.validity && !valid_bit(c.validity, row)) continue;
        nn++;
        if (c.width == 0) continue;
        if (fp) {
            double x = c.type == PG_FLOAT ? (double)((const float *)c.data)[row] : ((const double *)c.data)[row];
            if (x != x) { nan_seen = true; continue; }
            dmin = fmin(dmin, x); dmax = fmax(dmax, x);
        } else {
            int64_t x = sext(load_fixed(c.data, c.width, row), c.width);
            if (c.type == PG_BOOL) x = x != 0;
            imin = min(imin, x); imax = max(imax, x);
            if (c.type == PG_INT8 && (x == 1 || x == 3)) retr++;        // RowKind retracts, used for _VALUE_KIND
        }
    }
    __shared__ long long s_i[2], s_n[2];
    __shared__ double s_d[2];
    __shared__ int s_nan;
    if (threadIdx.x == 0) { s_i[0] = INT64_MAX; s_i[1] = INT64_MIN; s_d[0] = INFINITY; s_d[1] = -INFINITY; s_n[0] = s_n[1] = 0; s_nan = 0; }
    __syncthreads();
    if (fp) {
        // doubles: order-preserving via atomicMin/Max on the transformed bit pattern is overkill here: serialise
        // per warp leader through a CAS loop on the shared doubles
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            dmin = fmin(dmin, __shfl_xor_sync(0xffffffffu, dmin, d));
            dmax = fmax(dmax, __shfl_xor_sync(0xffffffffu, dmax, d));
        }
        if ((threadIdx.x & 31) == 0) {
            unsigned long long *pmin = (unsigned long long *)&s_d[0], *pmax = (unsigned long long *)&s_d[1];
            unsigned long long old = *pmin;
            while (dmin < __longlong_as_double((long long)old)) {
                unsigned long long prev = atomicCAS(pmin, old, (unsigned long long)__double_as_longlong(dmin));
                if (prev == old) break;
                old = prev;
            }
            old = *pmax;
            while (dmax > __longlong_as_double((long long)old)) {
                unsigned long long prev = atomicCAS(pmax, old, (unsigned long long)__double_as_longlong(dmax));
                if (prev == old) break;
                old = prev;
            }
        }
        if (nan_seen) s_nan = 1;
    } else {
        atomicMin(&s_i[0], (long long)imin);
        atomicMax(&s_i[1], (long long)imax);
    }
    atomicAdd((unsigned long long *)&s_n[0], (unsigned long long)nn);
    atomicAdd((unsigned long long *)&s_n[1], (unsigned long long)retr);
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t *o = out + kStatWords * (int64_t)blockIdx.x;
        if (fp) { o[0] = __double_as_longlong(s_d[0]); o[1] = __double_as_longlong(s_d[1]); }
        else { o[0] = s_i[0]; o[1] = s_i[1]; }
        o[2] = s_n[0];
        o[3] = s_n[1];
        o[4] = s_nan;
    }
}

// host-built pieces of the file (page headers, level prefixes, footer) -> their places in the device image
struct PatchJob { int64_t dst; int32_t src, len; };
__global__ void k_pw_patch(const PatchJob *jobs, int n, const uint8_t *bytes, uint8_t *file) {
    const int j = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (j >= n) return;
    const PatchJob pj = jobs[j];
    for (int i = lane; i < pj.len; i += 32) file[pj.dst + i] = bytes[pj.src + i];
}

// ------------------------------------------------------------------ zstd page compression
// The page bodies are written into a scratch image, every 128 KiB block of every body is compressed by one warp, the
// per-page frame sizes go back to the host (which lays out the file and writes the page headers), and a gather places
// the frames at their file offsets.

struct ZsBlockJob {
    int64_t src;                  // offset of the block in the body image
    int64_t out;                  // offset of its payload slot (n bytes)
    int64_t seq;                  // first sequence slot (n / 4 + 1 of them)
    int32_t n;                    // input bytes (<= 128 KiB)
    int32_t page;
};
struct ZsPage {
    int64_t raw;                  // body bytes
    int32_t first_block, n_blocks;
};

constexpr size_t kZsSmem = (sizeof(int32_t) << zs::kHashLog) + sizeof(zs::EncWork);

__global__ void __launch_bounds__(32)
k_zs_block(const ZsBlockJob *jobs, const uint8_t *img, uint8_t *out, zs::Seq *seqs, uint8_t *lits, int2 *res) {
    extern __shared__ __align__(16) uint8_t zs_smem[];
    int32_t *htab = (int32_t *)zs_smem;
    zs::EncWork &W = *(zs::EncWork *)(zs_smem + (sizeof(int32_t) << zs::kHashLog));
    const ZsBlockJob j = jobs[blockIdx.x];
    const zs::BlockOut r = zs::compress_block(img + j.src, j.n, out + j.out, htab, seqs + j.seq, lits + j.src, W);
    if (threadIdx.x == 0) res[blockIdx.x] = make_int2(r.type, r.size);
}

// per page: where each block's header goes inside the frame, and the frame size
__global__ void k_zs_page_sizes(const ZsPage *pages, int n_pages, const int2 *res, int32_t *boff, int64_t *frame_bytes) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pages) return;
    const ZsPage pg = pages[p];
    int64_t off = zs::frame_header_size((uint64_t)pg.raw);
    for (int b = 0; b < pg.n_blocks; b++) {
        boff[pg.first_block + b] = (int32_t)off;
        off += 3 + res[pg.first_block + b].y;
    }
    frame_bytes[p] = off;
}

// one CTA per block: frame header (first block of a page), block header, payload at the frame's file offset
__global__ void k_zs_gather(const ZsBlockJob *jobs, const ZsPage *pages, const int2 *res, const int32_t *boff,
                            const int64_t *frame_off, const uint8_t *img, const uint8_t *out, uint8_t *file) {
    const ZsBlockJob j = jobs[blockIdx.x];
    const ZsPage pg = pages[j.page];
    const int2 r = res[blockIdx.x];
    uint8_t *frame = file + frame_off[j.page];
    uint8_t *dst = frame + boff[blockIdx.x];
    if (threadIdx.x == 0) {
        if ((int)blockIdx.x == pg.first_block) zs::write_frame_header(frame, (uint64_t)pg.raw);
        zs::write_block_header(dst, (int)blockIdx.x == pg.first_block + pg.n_blocks - 1, r.x,
                               r.x == 2 ? (uint32_t)r.y : (uint32_t)j.n);
    }
    const uint8_t *pay = r.x == 0 ? img + j.src : out + j.out;
    for (int i = threadIdx.x; i < r.y; i += blockDim.x) dst[3 + i] = pay[i];
}

// ------------------------------------------------------------------ Thrift compact protocol writer

struct ThriftWriter {
    std::vector<uint8_t> b;
    std::vector<int> last{0};
    void varint(uint64_t v) { while (v >= 0x80) { b.push_back((uint8_t)(v | 0x80)); v >>= 7; } b.push_back((uint8_t)v); }
    void zigzag(int64_t v) { varint(((uint64_t)v << 1) ^ (uint64_t)(v >> 63)); }
    void field(int id, int type) {
        int d = id - last.back();
        if (d > 0 && d <= 15) b.push_back((uint8_t)((d << 4) | type));
        else { b.push_back((uint8_t)type); zigzag(id); }
        last.back() = id;
    }
    void i32(int id, int32_t v) { field(id, 5); zigzag(v); }
    void i64(int id, int64_t v) { field(id, 6); zigzag(v); }
    void bin(int id, const void *p, size_t n) { field(id, 8); varint(n); b.insert(b.end(), (const uint8_t *)p, (const uint8_t *)p + n); }
    void str(int id, const std::string &s) { bin(id, s.data(), s.size()); }
    void list(int id, int elem_type, size_t n) {
        field(id, 9);
        if (n < 15) b.push_back((uint8_t)((n << 4) | elem_type));
        else { b.push_back((uint8_t)(0xF0 | elem_type)); varint(n); }
    }
    void struct_field(int id) { field(id, 12); last.push_back(0); }
    void struct_elem() { last.push_back(0); }           // list element
    void end() { b.push_back(0); last.pop_back(); }
};

// ------------------------------------------------------------------ host orchestration

struct ColStats { int64_t min = 0, max = 0, null_count = 0; int has_minmax = 0; };

// the bits of a FLOAT / DOUBLE bound (held as a double), a zero of either sign replaced by `zero`
static int64_t zero_as(int64_t bits, double zero) {
    double x;
    memcpy(&x, &bits, 8);
    if (x == 0) memcpy(&bits, &zero, 8);
    return bits;
}

struct EncodedFile {
    unsigned char *d_file = nullptr;         // device image of the file (page bodies at their final offsets)
    int64_t file_bytes = 0;
    std::vector<std::pair<int64_t, std::vector<uint8_t>>> host_parts;   // (offset, bytes): headers, level prefixes, footer
    pg_file_meta meta{};
    std::vector<ColStats> stats;             // whole-file, per column
    bool image_complete = false;             // host_parts have been patched into d_file
    ~EncodedFile() { if (d_file) cudaFree(d_file); }
};
static Table<EncodedFile> g_enc(6);

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

static pg_status encode(uint64_t source, const char *const *names, int64_t row0, int64_t n_rows,
                        const pg_parquet_write_options *opt, int codec, uint64_t *out_file) {
    pg_status st = ensure_device();
    if (st) return st;
    BatchColumns batch;                                      // held until the encode below is done
    st = batch_columns(source, &batch);
    if (st) return st;
    const Schema *s = batch.schema.get();
    const std::vector<DevColumn> &dcols = batch.cols;
    for (int c = 0; c < s->n_cols() && batch.n_rows > 0; c++)
        if (!dcols[c].data && !dcols[c].offsets)
            return fail(PG_ERR_INVALID, "parquet encode: the batch was produced under a read-type projection and has no "
                                        "column " + std::to_string(c) + "; a data file needs every column");
    if (n_rows < 0) n_rows = batch.n_rows - row0;
    if (row0 < 0 || (row0 & 7) || row0 + n_rows > batch.n_rows)
        return fail(PG_ERR_INVALID, "parquet encode: row range outside the batch or not starting at a multiple of 8");
    const int nc = s->n_cols();
    int64_t page_rows = opt && opt->page_rows > 0 ? opt->page_rows : 32768;
    page_rows = (page_rows + 7) & ~(int64_t)7;
    int64_t group_rows = opt && opt->row_group_rows > 0 ? opt->row_group_rows : (int64_t)1 << 20;
    group_rows = ((group_rows + page_rows - 1) / page_rows) * page_rows;
    const int64_t n_groups = n_rows == 0 ? 0 : (n_rows + group_rows - 1) / group_rows;

    cudaEvent_t e0 = nullptr, e1 = nullptr;
    struct EvGuard { cudaEvent_t &a, &b; ~EvGuard() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); } } evg{e0, e1};
    PG_CUDA(cudaEventCreate(&e0));
    PG_CUDA(cudaEventCreate(&e1));
    PG_CUDA(cudaEventRecord(e0, 0));

    std::vector<EncColumn> cols(nc);
    for (int c = 0; c < nc; c++) {
        pg_field f = s->field(c);
        cols[c] = EncColumn{dcols[c].data, dcols[c].offsets, dcols[c].validity, f.type, type_width(f.type),
                            (f.nullable || dcols[c].validity) ? 1 : 0, 0};
    }
    // jobs: row group major, column, page
    std::vector<EncJob> jobs;
    std::vector<StatJob> sjobs;
    for (int64_t g = 0; g < n_groups; g++) {
        const int64_t g0 = row0 + g * group_rows, g1 = std::min(row0 + n_rows, g0 + group_rows);
        for (int c = 0; c < nc; c++) {
            sjobs.push_back(StatJob{c, 0, g0, g1 - g0});
            for (int64_t p0 = g0; p0 < g1; p0 += page_rows)
                jobs.push_back(EncJob{c, (int32_t)(std::min(g1, p0 + page_rows) - p0), p0, -1, 0});
        }
    }
    const size_t nj = jobs.size(), nsj = sjobs.size();
    std::vector<int64_t> counts(2 * nj + 2), stats(kStatWords * (nsj + 1));
    Scratch scratch(0);                                      // temporaries, released on every path out of this function
    EncColumn *d_cols = (EncColumn *)scratch.take(sizeof(EncColumn) * nc);
    EncJob *d_jobs = (EncJob *)scratch.take(sizeof(EncJob) * std::max<size_t>(nj, 1));
    StatJob *d_sjobs = (StatJob *)scratch.take(sizeof(StatJob) * std::max<size_t>(nsj, 1));
    int64_t *d_counts = (int64_t *)scratch.take(sizeof(int64_t) * (2 * nj + 2));
    int64_t *d_stats = (int64_t *)scratch.take(sizeof(int64_t) * kStatWords * (nsj + 1));
    if (!d_cols || !d_jobs || !d_sjobs || !d_counts || !d_stats)
        return fail(PG_ERR_CUDA, "parquet encode: out of device memory for the page tables");
    PG_CUDA(cudaMemcpy(d_cols, cols.data(), sizeof(EncColumn) * nc, cudaMemcpyHostToDevice));
    int launches = 0;
    if (nj) {
        PG_CUDA(cudaMemcpy(d_jobs, jobs.data(), sizeof(EncJob) * nj, cudaMemcpyHostToDevice));
        PG_CUDA(cudaMemcpy(d_sjobs, sjobs.data(), sizeof(StatJob) * nsj, cudaMemcpyHostToDevice));
        k_pw_count<<<(unsigned)nj, 256>>>(d_cols, d_jobs, d_counts);
        k_pw_stats<<<(unsigned)nsj, 256>>>(d_cols, d_sjobs, d_stats);
        launches += 2;
        PG_CUDA(cudaMemcpy(counts.data(), d_counts, sizeof(int64_t) * 2 * nj, cudaMemcpyDeviceToHost));
        PG_CUDA(cudaMemcpy(stats.data(), d_stats, sizeof(int64_t) * kStatWords * nsj, cudaMemcpyDeviceToHost));
    }

    // ---- page bodies: level prefix (host-built) + values, per page
    auto ef = std::make_unique<EncodedFile>();
    ef->stats.assign(nc, ColStats{});
    for (int c = 0; c < nc; c++) { ef->stats[c].min = INT64_MAX; ef->stats[c].max = INT64_MIN; }
    struct ChunkInfo { int64_t first_page, total_uncompressed, total_compressed, num_values, nn; size_t page0, page1; ColStats st; };
    struct PageInfo { std::vector<uint8_t> prefix; int64_t def_bytes, body, stored; };
    std::vector<ChunkInfo> chunks(nsj);
    std::vector<PageInfo> pages;
    pages.reserve(nj);
    std::vector<char> file_nan(nc, 0);                       // per column: a chunk holds a NaN
    size_t ji = 0;
    for (size_t sj = 0; sj < nsj; sj++) {
        const int c = sjobs[sj].col;
        const EncColumn &ec = cols[c];
        const int64_t *cs = &stats[kStatWords * sj];
        const bool fp = ec.type == PG_FLOAT || ec.type == PG_DOUBLE, nan = cs[4] != 0;
        ChunkInfo &ci = chunks[sj];
        ci.page0 = ji;
        ci.num_values = sjobs[sj].n_rows;
        ci.nn = cs[2];
        ci.st.null_count = ci.num_values - ci.nn;
        ci.st.has_minmax = ec.width > 0 && ci.nn > 0 && !nan;   // a chunk with a NaN has no min / max
        ci.st.min = cs[0];
        ci.st.max = cs[1];
        // parquet.thrift, Statistics: a zero min of a floating point column is written as -0.0, a zero max as +0.0,
        // so that min <= v <= max holds for both zeros in the order readers compare with (Double.compare: -0.0 <
        // +0.0).  The file-level merge below keeps the rule: the zero min it can take is -0.0, the zero max +0.0.
        if (fp && ci.st.has_minmax) { ci.st.min = zero_as(ci.st.min, -0.0); ci.st.max = zero_as(ci.st.max, 0.0); }
        file_nan[c] |= nan;
        ColStats &fs = ef->stats[c];
        fs.null_count += ci.st.null_count;
        if (ci.st.has_minmax) {
            if (!fs.has_minmax) { fs.min = ci.st.min; fs.max = ci.st.max; fs.has_minmax = 1; }
            else if (fp) {
                double a, b, x, y;
                memcpy(&a, &fs.min, 8); memcpy(&b, &fs.max, 8); memcpy(&x, &ci.st.min, 8); memcpy(&y, &ci.st.max, 8);
                a = std::min(a, x); b = std::max(b, y);
                memcpy(&fs.min, &a, 8); memcpy(&fs.max, &b, 8);
            } else { fs.min = std::min(fs.min, ci.st.min); fs.max = std::max(fs.max, ci.st.max); }
        }
        if (c == s->n_key + 1) ef->meta.delete_row_count += cs[3];
        for (; ji < nj && jobs[ji].col == c && jobs[ji].row0 >= sjobs[sj].row0 &&
               jobs[ji].row0 < sjobs[sj].row0 + sjobs[sj].n_rows; ji++) {
            EncJob &j = jobs[ji];
            const int64_t nn = counts[2 * ji], vb = counts[2 * ji + 1];
            std::vector<uint8_t> prefix;                       // [def length:int32][hybrid header varint]
            int64_t def_bytes = 0;
            if (ec.optional) {
                const int64_t groups = (j.n_rows + 7) / 8;
                ThriftWriter tw;
                tw.varint((uint64_t)(groups << 1) | 1);
                const uint32_t len = (uint32_t)(tw.b.size() + groups);
                prefix = {(uint8_t)len, (uint8_t)(len >> 8), (uint8_t)(len >> 16), (uint8_t)(len >> 24)};
                prefix.insert(prefix.end(), tw.b.begin(), tw.b.end());
                def_bytes = (int64_t)prefix.size() + groups;
            }
            int64_t val_bytes;
            if (ec.width == 0) val_bytes = 4 * nn + vb;
            else if (ec.type == PG_BOOL) val_bytes = (nn + 7) / 8;
            else val_bytes = nn * (ec.width == 8 ? 8 : 4);
            const int64_t body = def_bytes + val_bytes;
            if (body > 0x7fffffffLL) return fail(PG_ERR_UNSUPPORTED, "parquet encode: page larger than 2 GiB");
            pages.push_back(PageInfo{std::move(prefix), def_bytes, body, body});
        }
        ci.page1 = ji;
    }
    // A file with a NaN in a FLOAT / DOUBLE column has no min / max for that column, though its other chunks have
    // some: NaN sorts above every value (Double.compare), so a max taken around it would prune rows `x > max` matches.
    for (int c = 0; c < nc; c++)
        if (file_nan[c]) ef->stats[c] = ColStats{INT64_MAX, INT64_MIN, ef->stats[c].null_count, 0};
    const int n_pages = (int)pages.size();

    // ---- zstd: bodies into a scratch image, one frame per body; the frame sizes come back before the layout
    int launches_zs = 0;
    const bool zstd = codec == pq::C_ZSTD;
    std::vector<ZsBlockJob> bjobs;
    std::vector<ZsPage> zpages(zstd ? nj : 0);
    uint8_t *d_img = nullptr, *d_zout = nullptr;
    ZsBlockJob *d_bjobs = nullptr;
    ZsPage *d_zpages = nullptr;
    int2 *d_res = nullptr;
    int32_t *d_boff = nullptr;
    int64_t *d_frame = nullptr;
    if (zstd && nj) {
        std::vector<PatchJob> pjobs;
        std::vector<uint8_t> pbytes;
        int64_t img = 0, out = 0, seq = 0;
        for (size_t p = 0; p < nj; p++) {
            const PageInfo &pi = pages[p];
            if (!pi.prefix.empty()) {
                pjobs.push_back(PatchJob{img, (int32_t)pbytes.size(), (int32_t)pi.prefix.size()});
                pbytes.insert(pbytes.end(), pi.prefix.begin(), pi.prefix.end());
                jobs[p].def_off = img + (int64_t)pi.prefix.size();
            }
            jobs[p].val_off = img + pi.def_bytes;
            zpages[p] = ZsPage{pi.body, (int32_t)bjobs.size(), 0};
            for (int64_t b0 = 0; b0 == 0 || b0 < pi.body; b0 += zs::kMaxBlock) {
                const int32_t n = (int32_t)std::min<int64_t>(zs::kMaxBlock, pi.body - b0);
                bjobs.push_back(ZsBlockJob{img + b0, out, seq, n, (int32_t)p});
                out += n;
                seq += n / 4 + 1;
                zpages[p].n_blocks++;
            }
            img += pi.body;
        }
        const size_t nb = bjobs.size();
        d_img = (uint8_t *)scratch.take((size_t)img + 64);
        d_zout = (uint8_t *)scratch.take((size_t)out + 64);
        uint8_t *d_lits = (uint8_t *)scratch.take((size_t)img + 64);
        zs::Seq *d_seqs = (zs::Seq *)scratch.take(sizeof(zs::Seq) * (size_t)seq);
        d_bjobs = (ZsBlockJob *)scratch.take(sizeof(ZsBlockJob) * nb);
        d_zpages = (ZsPage *)scratch.take(sizeof(ZsPage) * nj);
        d_res = (int2 *)scratch.take(sizeof(int2) * nb);
        d_boff = (int32_t *)scratch.take(sizeof(int32_t) * nb);
        d_frame = (int64_t *)scratch.take(sizeof(int64_t) * nj);
        PatchJob *d_pjobs = (PatchJob *)scratch.take(sizeof(PatchJob) * pjobs.size() + 16);
        uint8_t *d_pbytes = (uint8_t *)scratch.take(pbytes.size() + 16);
        if (!d_img || !d_zout || !d_lits || !d_seqs || !d_bjobs || !d_zpages || !d_res || !d_boff || !d_frame || !d_pjobs || !d_pbytes)
            return fail(PG_ERR_CUDA, "parquet encode: out of device memory for the zstd page images");
        PG_CUDA(cudaMemsetAsync(d_img, 0, (size_t)img + 64, 0));
        PG_CUDA(cudaMemcpy(d_jobs, jobs.data(), sizeof(EncJob) * nj, cudaMemcpyHostToDevice));
        PG_CUDA(cudaMemcpy(d_bjobs, bjobs.data(), sizeof(ZsBlockJob) * nb, cudaMemcpyHostToDevice));
        PG_CUDA(cudaMemcpy(d_zpages, zpages.data(), sizeof(ZsPage) * nj, cudaMemcpyHostToDevice));
        k_pw_encode<<<(unsigned)nj, 256>>>(d_cols, d_jobs, d_img);
        launches_zs++;
        if (!pjobs.empty()) {
            PG_CUDA(cudaMemcpy(d_pjobs, pjobs.data(), sizeof(PatchJob) * pjobs.size(), cudaMemcpyHostToDevice));
            PG_CUDA(cudaMemcpy(d_pbytes, pbytes.data(), pbytes.size(), cudaMemcpyHostToDevice));
            k_pw_patch<<<(unsigned)((pjobs.size() * 32 + 127) / 128), 128>>>(d_pjobs, (int)pjobs.size(), d_pbytes, d_img);
            launches_zs++;
        }
        k_zs_block<<<(unsigned)nb, 32, kZsSmem>>>(d_bjobs, d_img, d_zout, d_seqs, d_lits, d_res);
        k_zs_page_sizes<<<(unsigned)((nj + 127) / 128), 128>>>(d_zpages, (int)nj, d_res, d_boff, d_frame);
        launches_zs += 2;
        std::vector<int64_t> frame_bytes(nj);
        SmallReads rd(0);
        if ((st = rd.add(frame_bytes.data(), d_frame, sizeof(int64_t) * nj))) return st;
        launches_zs++;
        if ((st = rd.finish())) return st;
        cudaError_t le = cudaGetLastError();
        if (le != cudaSuccess) return fail(PG_ERR_CUDA, std::string("parquet encode: ") + cudaGetErrorString(le));
        for (size_t p = 0; p < nj; p++) pages[p].stored = frame_bytes[p];
    }

    // ---- layout: page headers (Thrift), level prefixes (uncompressed), stored bodies
    int64_t pos = 4;                                         // after "PAR1"
    ef->host_parts.push_back({0, {'P', 'A', 'R', '1'}});
    std::vector<int64_t> frame_off(zstd ? nj : 0);
    for (size_t sj = 0; sj < nsj; sj++) {
        ChunkInfo &ci = chunks[sj];
        ci.first_page = pos;
        ci.total_uncompressed = ci.total_compressed = 0;
        for (size_t p = ci.page0; p < ci.page1; p++) {
            EncJob &j = jobs[p];
            const PageInfo &pi = pages[p];
            ThriftWriter ph;                                   // PageHeader
            ph.i32(1, pq::P_DATA);
            ph.i32(2, (int32_t)pi.body);
            ph.i32(3, (int32_t)pi.stored);
            ph.struct_field(5);                                // DataPageHeader
            ph.i32(1, j.n_rows);
            ph.i32(2, pq::E_PLAIN);
            ph.i32(3, pq::E_RLE);
            ph.i32(4, pq::E_RLE);
            ph.end();
            ph.end();
            ef->host_parts.push_back({pos, ph.b});
            pos += (int64_t)ph.b.size();
            if (zstd) frame_off[p] = pos;
            else {
                if (!pi.prefix.empty()) {
                    ef->host_parts.push_back({pos, pi.prefix});
                    j.def_off = pos + (int64_t)pi.prefix.size();
                }
                j.val_off = pos + pi.def_bytes;
            }
            pos += pi.stored;
            ci.total_uncompressed += (int64_t)ph.b.size() + pi.body;
            ci.total_compressed += (int64_t)ph.b.size() + pi.stored;
        }
    }
    const int64_t data_end = pos;

    // ---- footer
    ThriftWriter fw;
    fw.i32(1, 1);                                              // version
    fw.list(2, 12, (size_t)nc + 1);                            // schema
    fw.struct_elem();
    fw.str(4, "paimon_schema");
    fw.i32(5, nc);
    fw.end();
    for (int c = 0; c < nc; c++) {
        const EncColumn &ec = cols[c];
        fw.struct_elem();
        fw.i32(1, parquet_type_of(ec.type));
        fw.i32(3, ec.optional ? pq::R_OPTIONAL : pq::R_REQUIRED);
        fw.str(4, names && names[c] ? names[c] : ("c" + std::to_string(c)));
        if (ec.type == PG_STRING) fw.i32(6, 0);               // UTF8
        else if (ec.type == PG_INT8) fw.i32(6, 15);           // INT_8
        else if (ec.type == PG_INT16) fw.i32(6, 16);          // INT_16
        fw.end();
    }
    fw.i64(3, n_rows);
    fw.list(4, 12, (size_t)n_groups);
    for (int64_t g = 0; g < n_groups; g++) {
        fw.struct_elem();                                      // RowGroup
        fw.list(1, 12, (size_t)nc);
        int64_t group_bytes = 0;
        for (int c = 0; c < nc; c++) {
            const ChunkInfo &ci = chunks[(size_t)g * nc + c];
            const EncColumn &ec = cols[c];
            group_bytes += ci.total_uncompressed;
            fw.struct_elem();                                  // ColumnChunk
            fw.i64(2, ci.first_page);
            fw.struct_field(3);                                // ColumnMetaData
            fw.i32(1, parquet_type_of(ec.type));
            fw.list(2, 5, 2); fw.zigzag(pq::E_PLAIN); fw.zigzag(pq::E_RLE);
            fw.list(3, 8, 1);
            { std::string nm = names && names[c] ? names[c] : ("c" + std::to_string(c)); fw.varint(nm.size()); fw.b.insert(fw.b.end(), nm.begin(), nm.end()); }
            fw.i32(4, zstd ? pq::C_ZSTD : pq::C_UNCOMPRESSED);
            fw.i64(5, ci.num_values);
            fw.i64(6, ci.total_uncompressed);
            fw.i64(7, ci.total_compressed);
            fw.i64(9, ci.first_page);
            fw.struct_field(12);                               // Statistics
            fw.i64(3, ci.st.null_count);
            if (ci.st.has_minmax) {
                uint8_t mn[8], mx[8];
                size_t w = ec.width == 8 ? 8 : 4;
                if (ec.type == PG_FLOAT) {
                    double a, b; memcpy(&a, &ci.st.min, 8); memcpy(&b, &ci.st.max, 8);
                    float fa = (float)a, fb = (float)b; memcpy(mn, &fa, 4); memcpy(mx, &fb, 4);
                } else if (ec.type == PG_BOOL) {
                    w = 1; mn[0] = (uint8_t)ci.st.min; mx[0] = (uint8_t)ci.st.max;
                } else if (w == 4) {
                    int32_t a = (int32_t)ci.st.min, b = (int32_t)ci.st.max; memcpy(mn, &a, 4); memcpy(mx, &b, 4);
                } else { memcpy(mn, &ci.st.min, 8); memcpy(mx, &ci.st.max, 8); }
                fw.bin(5, mx, w);
                fw.bin(6, mn, w);
            }
            fw.end();
            fw.end();                                          // ColumnMetaData
            fw.end();                                          // ColumnChunk
        }
        fw.i64(2, group_bytes);
        fw.i64(3, std::min(row0 + n_rows, row0 + (g + 1) * group_rows) - (row0 + g * group_rows));
        fw.end();
    }
    fw.str(6, "paimon-b200 (libpaimon_gpu)");
    // column_orders: TYPE_ORDER (TypeDefinedOrder) for every column.  Readers take min_value / max_value only from a
    // file that declares the order they were computed in; without it parquet-cpp (pyarrow) ignores them.
    fw.list(7, 12, (size_t)nc);
    for (int c = 0; c < nc; c++) {
        fw.struct_elem();                                      // ColumnOrder (union)
        fw.struct_field(1);                                    // TYPE_ORDER: TypeDefinedOrder, no fields
        fw.end();
        fw.end();
    }
    fw.end();
    std::vector<uint8_t> tail = fw.b;
    const uint32_t flen = (uint32_t)fw.b.size();
    tail.insert(tail.end(), {(uint8_t)flen, (uint8_t)(flen >> 8), (uint8_t)(flen >> 16), (uint8_t)(flen >> 24), 'P', 'A', 'R', '1'});
    ef->host_parts.push_back({data_end, tail});
    ef->file_bytes = data_end + (int64_t)tail.size();

    // ---- page bodies on the device
    PG_CUDA(cudaMalloc(&ef->d_file, (size_t)ef->file_bytes + 64));
    PG_CUDA(cudaMemsetAsync(ef->d_file, 0, (size_t)ef->file_bytes + 64, 0));
    if (nj && zstd) {
        // (the frame sizes have been read: their buffer takes the frame offsets)
        PG_CUDA(cudaMemcpy(d_frame, frame_off.data(), sizeof(int64_t) * nj, cudaMemcpyHostToDevice));
        k_zs_gather<<<(unsigned)bjobs.size(), 256>>>(d_bjobs, d_zpages, d_res, d_boff, d_frame, d_img, d_zout, ef->d_file);
        launches += launches_zs + 1;
    } else if (nj) {
        PG_CUDA(cudaMemcpy(d_jobs, jobs.data(), sizeof(EncJob) * nj, cudaMemcpyHostToDevice));
        k_pw_encode<<<(unsigned)nj, 256>>>(d_cols, d_jobs, ef->d_file);
        launches++;
    }
    PG_CUDA(cudaEventRecord(e1, 0));
    PG_CUDA(cudaEventSynchronize(e1));
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaError_t le = cudaGetLastError();
    if (le != cudaSuccess) return fail(PG_ERR_CUDA, std::string("parquet encode: ") + cudaGetErrorString(le));

    ef->meta.n_rows = n_rows;
    ef->meta.file_bytes = ef->file_bytes;
    ef->meta.n_row_groups = (int32_t)n_groups;
    ef->meta.n_pages = n_pages;
    ef->meta.ms_encode = ms;
    ef->meta.launches = launches;
    const ColStats &sq = ef->stats[s->n_key];
    ef->meta.min_sequence_number = sq.has_minmax ? sq.min : 0;
    ef->meta.max_sequence_number = sq.has_minmax ? sq.max : 0;
    *out_file = g_enc.put(std::move(ef));
    return PG_OK;
}

}  // namespace pg

using namespace pg;

extern "C" {

pg_status pg_parquet_encode(uint64_t source, const char *const *column_names, int64_t row0, int64_t n_rows,
                            const pg_parquet_write_options *options, uint64_t *out_file) {
    if (!out_file) return fail(PG_ERR_INVALID, "null argument");
    return encode(source, column_names, row0, n_rows, options, pq::C_UNCOMPRESSED, out_file);
}

pg_status pg_parquet_encode_compressed(uint64_t source, const char *const *column_names, int64_t row0, int64_t n_rows,
                                       const pg_parquet_write_options *options, int32_t codec, int32_t level,
                                       uint64_t *out_file) {
    if (!out_file) return fail(PG_ERR_INVALID, "null argument");
    if (codec < pq::C_UNCOMPRESSED || codec > pq::C_LZ4_RAW)
        return fail(PG_ERR_INVALID, "parquet encode: codec " + std::to_string(codec) + " is not a Parquet CompressionCodec");
    if (codec != pq::C_UNCOMPRESSED && codec != pq::C_ZSTD)
        return fail(PG_ERR_UNSUPPORTED, "parquet encode: codec " + std::to_string(codec) +
                                            " is not written on the device (UNCOMPRESSED and ZSTD are)");
    if (codec == pq::C_ZSTD && (level == 0 || level > 1))
        return fail(PG_ERR_UNSUPPORTED, "parquet encode: file.compression.zstd-level " + std::to_string(level) +
                                            " is not written on the device (level 1 and the negative fast levels are)");
    return encode(source, column_names, row0, n_rows, options, codec, out_file);
}

pg_status pg_parquet_file_meta(uint64_t file, pg_file_meta *out) {
    std::shared_ptr<EncodedFile> ef = g_enc.get(file);
    if (!ef || !out) return fail(PG_ERR_INVALID, "unknown encoded file handle");
    *out = ef->meta;
    return PG_OK;
}

pg_status pg_parquet_file_column_stats(uint64_t file, int32_t column, int64_t *null_count, int32_t *has_min_max,
                                       void *min8, void *max8) {
    std::shared_ptr<EncodedFile> ef = g_enc.get(file);
    if (!ef) return fail(PG_ERR_INVALID, "unknown encoded file handle");
    if (column < 0 || column >= (int32_t)ef->stats.size()) return fail(PG_ERR_INVALID, "column out of range");
    const ColStats &cs = ef->stats[column];
    if (null_count) *null_count = cs.null_count;
    if (has_min_max) *has_min_max = cs.has_minmax;
    if (min8) memcpy(min8, &cs.min, 8);
    if (max8) memcpy(max8, &cs.max, 8);
    return PG_OK;
}

pg_status pg_parquet_file_fetch(uint64_t file, void *host_buffer, int64_t capacity) {
    std::shared_ptr<EncodedFile> ef = g_enc.get(file);
    if (!ef || !host_buffer) return fail(PG_ERR_INVALID, "unknown encoded file handle");
    if (capacity < ef->file_bytes) return fail(PG_ERR_INVALID, "buffer smaller than the file");
    pg_status st = ensure_device();
    if (st) return st;
    const auto &tail = ef->host_parts.back();
    PG_CUDA(cudaMemcpy(host_buffer, ef->d_file, (size_t)tail.first, cudaMemcpyDeviceToHost));
    for (const auto &p : ef->host_parts) memcpy((uint8_t *)host_buffer + p.first, p.second.data(), p.second.size());
    return PG_OK;
}

pg_status pg_parquet_file_device_image(uint64_t file, const uint8_t **device_bytes, int64_t *size) {
    std::shared_ptr<EncodedFile> ef = g_enc.get(file);
    if (!ef || !device_bytes || !size) return fail(PG_ERR_INVALID, "unknown encoded file handle");
    pg_status st = ensure_device();
    if (st) return st;
    if (!ef->image_complete) {
        std::vector<PatchJob> jobs;
        std::vector<uint8_t> bytes;
        for (const auto &p : ef->host_parts) {
            if (bytes.size() + p.second.size() > 0x7fffffffull) return fail(PG_ERR_UNSUPPORTED, "parquet encode: too many header bytes");
            jobs.push_back(PatchJob{p.first, (int32_t)bytes.size(), (int32_t)p.second.size()});
            bytes.insert(bytes.end(), p.second.begin(), p.second.end());
        }
        Scratch scratch(0);
        PatchJob *d_jobs = (PatchJob *)scratch.take(sizeof(PatchJob) * jobs.size() + 16);
        uint8_t *d_bytes = (uint8_t *)scratch.take(bytes.size() + 16);
        if (!d_jobs || !d_bytes) return fail(PG_ERR_CUDA, "parquet encode: out of device memory for the header patch");
        PG_CUDA(cudaMemcpy(d_jobs, jobs.data(), sizeof(PatchJob) * jobs.size(), cudaMemcpyHostToDevice));
        PG_CUDA(cudaMemcpy(d_bytes, bytes.data(), bytes.size(), cudaMemcpyHostToDevice));
        k_pw_patch<<<(unsigned)((jobs.size() * 32 + 127) / 128), 128>>>(d_jobs, (int)jobs.size(), d_bytes, ef->d_file);
        cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) return fail(PG_ERR_CUDA, std::string("parquet encode: ") + cudaGetErrorString(e));
        ef->image_complete = true;
    }
    *device_bytes = ef->d_file;
    *size = ef->file_bytes;
    return PG_OK;
}

pg_status pg_parquet_file_free(uint64_t file) {
    return g_enc.take(file) ? PG_OK : fail(PG_ERR_INVALID, "unknown encoded file handle");
}

}  // extern "C"
