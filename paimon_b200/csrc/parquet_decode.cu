// parquet_decode.cu — Parquet column-chunk decode on the device, one batch of launches per SECTION, feeding the
// merge without leaving HBM.
//
// Reference being replaced (paths under /root/reference/paimon-format/src/main/java/org/apache/paimon/format/):
//   parquet/ParquetReaderFactory.java:113-148          createReader (footer, schema clip by field NAME, vectors)
//   parquet/reader/VectorizedParquetRecordReader.java:178-241   nextBatch / row-group loop
//   parquet/reader/VectorizedColumnReader.java:143-383 page loop: V1 = [def RLE][values], V2 = separate levels
//   parquet/reader/VectorizedRleValuesReader.java:928-1019     RLE / bit-packed hybrid
//   parquet/reader/VectorizedPlainValuesReader.java:68-84,117-189,275-288   PLAIN booleans, fixed width, BYTE_ARRAY
//   parquet/reader/VectorizedDeltaBinaryPackedReader.java      DELTA_BINARY_PACKED
//   parquet/ParquetSchemaConverter.java:76-160         TINYINT/SMALLINT/INT/DATE -> INT32, BIGINT -> INT64, ...
// and, one level up, the way the files of a sorted run are concatenated into ONE merge input
//   paimon-core/.../mergetree/MergeTreeReaders.java:94-101 (readerForRun -> ConcatRecordReader of the run's files).
//
// The reference fills 1024-row ColumnVectors on one CPU thread per file.  Here a whole section (every file of every
// sorted run that overlaps one key interval) is decoded by ONE set of launches:
//   host    footers only (Thrift FileMetaData) -> a table of column chunks, ordered (run, column, file, row group)
//   walk    one thread per column chunk parses the Thrift page headers ON THE DEVICE (count pass, scan, fill pass)
//           -> one page table for the section
//   inflate Snappy / LZ4 / zstd / GZIP pages -> scratch images; DELTA_BINARY_PACKED pages -> PLAIN images
//   levels  one warp per page: definition levels -> the output validity bitmap (bit-packed runs are copied 32 bits
//           at a time), dictionary ids -> scratch, per-page non-null counts and var-len payload sizes
//   scan    per (run, var-len column): payload base of every page (files of a run continue each other's offsets)
//   walkba  one warp per PLAIN BYTE_ARRAY page: the serial [len][bytes] walk -> value start offsets
//   expand  one CTA per page: rank of every row under the validity bits -> values / dictionary lookups / offsets and
//           payload bytes at their final positions in the run's columns
// A file's rows land at its row offset inside its RUN: the k-way merge sees runs, not files.
// Anything the kernels do not implement is refused with PG_ERR_UNSUPPORTED (no CPU fallback).
#include <algorithm>
#include <cstring>
#include <memory>
#include <stdexcept>

#include "device_utils.cuh"
#include "parquet_meta.h"
#include "inflate_device.cuh"
#include "lz4_device.cuh"
#include "snappy_device.cuh"
#include "scan_kernels.cuh"
#include "zstd_device.cuh"

namespace pg {

enum : int { ENC_PLAIN = 0, ENC_DICT = 1, ENC_DELTA_BP = 2, ENC_RLE_BOOL = 3 };

// one column chunk of one file; host-built from the footer, counts and bases filled on the device
struct PqChunk {
    const uint8_t *base;      // device: first page header of the chunk
    int64_t avail;            // bytes from `base` to the end of the chunk (clipped to the file)
    int64_t num_values;
    int64_t row0;             // first row of the chunk inside its output run
    int32_t col, run, file, codec;
    int32_t max_def, phys, phys_width;
    int32_t cast;             // schema evolution: 0 none, 1 INT32 -> BIGINT (sign extension), 2 FLOAT -> DOUBLE
    // count pass
    int32_t n_pages, n_dicts;
    int64_t scratch_bytes;    // inflate / delta images this chunk needs
    int64_t dict_entries;     // BYTE_ARRAY dictionary entries
    int64_t ids_entries;      // dictionary ids / RLE booleans to materialise
    int64_t page_bytes;       // uncompressed page body bytes (the encoded bytes the decode stage reads)
    // chunk scan
    int32_t page_base, dict_base;
    int64_t scratch_base, dict_entry_base, ids_base;
};

struct PqPage {
    const uint8_t *src;       // page body as stored in the file
    const uint8_t *body;      // page body as the decode kernels read it (inflated / delta-expanded image)
    uint8_t *aux;             // DELTA_BINARY_PACKED: where the PLAIN image goes
    int32_t src_len, body_len;
    int32_t num_values, chunk;
    int8_t type, enc, compressed, bad;
    int32_t def_len;          // data page V2: bytes of definition levels in front of the values
    int64_t row0;             // first row inside the run
    // levels pass
    int32_t values_off, nnz;
    int64_t ids_base;         // first id of the page in the ids scratch
    int64_t payload_bytes;    // var-len: payload bytes of the page's values
    // page scan (var-len columns)
    int64_t payload_base;     // output byte offset of the page's first value
    int64_t vs_base;          // PLAIN BYTE_ARRAY: first entry of the page in the value-start scratch
    int32_t is_last, pad;
    int64_t entry_base;       // dictionary page of a BYTE_ARRAY column: first entry in dict_off / dict_len
};

// output column of one run: [run * n_cols + col]
struct PqOut {
    void *data;               // fixed width values, or the var-len payload (set after the size read-back)
    int32_t *offsets;
    uint32_t *validity;       // zeroed; bits are OR-ed in
    int32_t out_width;        // bytes of the output type, 0 for var-len
    int32_t is_bool;
};

// a (run, var-len column) pair: its chunks are contiguous in the chunk table, its pages in the page table
struct PqPair {
    int32_t run, col, chunk0, chunk1;
    int64_t vs_rows_base;     // rows of the pairs in front of this one (value-start scratch indexing)
    int32_t idx, pad;
};

// a run header of the RLE / bit-packed hybrid; `ok` is cleared when the stream ends inside it
__device__ __forceinline__ uint32_t pq_varint(const uint8_t *&p, const uint8_t *end, bool &ok) {
    uint32_t v = 0;
    int shift = 0;
    while (p < end) {
        uint8_t b = *p++;
        v |= (uint32_t)(b & 0x7f) << shift;
        if (!(b & 0x80)) return v;
        shift += 7;
    }
    ok = false;
    return v;
}

// ------------------------------------------------------------------ Thrift compact protocol, device side
//
// parquet-mr reads page headers with org.apache.parquet.format.Util.readPageHeader (Thrift compact protocol; the
// dependency is not under /root/reference, call site PQ3P/hadoop/ParquetFileReader.java:1345 Chunk.readAllPages).
// The encoding restated here is the public Thrift compact protocol + parquet.thrift field ids.

struct TRd {
    const uint8_t *p, *end;
    int bad;
    __host__ __device__ uint32_t byte() {
        if (p >= end) { bad = 1; return 0; }
        return *p++;
    }
    __host__ __device__ uint64_t varint() {
        uint64_t v = 0;
        for (int sh = 0; sh < 70; sh += 7) {
            const uint32_t b = byte();
            v |= (uint64_t)(b & 0x7f) << sh;
            if (!(b & 0x80)) return v;
        }
        bad = 1;
        return v;
    }
    __host__ __device__ int64_t zz() {
        const uint64_t v = varint();
        return (int64_t)(v >> 1) ^ -(int64_t)(v & 1);
    }
    // field header: returns the type (0 = STOP), updates the running field id
    __host__ __device__ int field(int &id) {
        const uint32_t h = byte();
        if (h == 0 || bad) return 0;
        const int d = (int)(h >> 4);
        if (d == 0) id = (int)zz(); else id += d;
        return (int)(h & 15);
    }
    __host__ __device__ void advance(uint64_t n) {
        if ((uint64_t)(end - p) < n) { bad = 1; p = end; } else p += n;
    }
    // anything but a struct
    __host__ __device__ void skip_flat(int t, bool in_container) {
        switch (t) {
            case 1: case 2: if (in_container) byte(); return;      // booleans live in the field header
            case 3: byte(); return;
            case 4: case 5: case 6: varint(); return;
            case 7: advance(8); return;
            case 8: advance(varint()); return;
            case 9: case 10: {
                const uint32_t h = byte();
                const int et = (int)(h & 15);
                uint64_t n = h >> 4;
                if (n == 15) n = varint();
                if (et == 9 || et == 10 || et == 11 || et == 12) { if (n) bad = 1; return; }   // nested containers: not in page headers
                for (uint64_t i = 0; i < n && !bad; i++) skip_flat(et, true);
                return;
            }
            case 11: { if (varint() != 0) bad = 1; return; }     // maps: not in page headers
            default: bad = 1; return;
        }
    }
    __host__ __device__ void skip(int t) {
        if (t != 12) { skip_flat(t, false); return; }
        int depth = 1;
        while (depth > 0 && !bad) {
            const uint32_t h = byte();
            if (h == 0) { depth--; continue; }
            if ((h >> 4) == 0) zz();
            const int ft = (int)(h & 15);
            if (ft == 12) depth++; else skip_flat(ft, false);
        }
    }
};

struct PqHeader {
    int type, unc, comp, nv, enc, def_enc, def_len, rep_len, is_compressed, hdr;
};

// parquet.thrift PageHeader {1 type, 2 uncompressed_page_size, 3 compressed_page_size, 5 DataPageHeader {1 num_values,
// 2 encoding, 3 definition_level_encoding}, 7 DictionaryPageHeader {1 num_values, 2 encoding}, 8 DataPageHeaderV2
// {1 num_values, 4 encoding, 5 definition_levels_byte_length, 6 repetition_levels_byte_length, 7 is_compressed}}
__host__ __device__ inline bool pq_parse_header(const uint8_t *p, const uint8_t *end, PqHeader &h) {
    TRd r{p, end, 0};
    h.type = -1; h.unc = 0; h.comp = 0; h.nv = 0; h.enc = 0; h.def_enc = pq::E_RLE; h.def_len = 0; h.rep_len = 0;
    h.is_compressed = 1;
    int id = 0, t;
    while ((t = r.field(id)) != 0 && !r.bad) {
        if (id == 1 && t == 5) h.type = (int)r.zz();
        else if (id == 2 && t == 5) h.unc = (int)r.zz();
        else if (id == 3 && t == 5) h.comp = (int)r.zz();
        else if ((id == 5 || id == 7 || id == 8) && t == 12) {
            const int outer = id;
            int i2 = 0, t2;
            while ((t2 = r.field(i2)) != 0 && !r.bad) {
                if (outer == 8) {
                    if (i2 == 1 && t2 == 5) h.nv = (int)r.zz();
                    else if (i2 == 4 && t2 == 5) h.enc = (int)r.zz();
                    else if (i2 == 5 && t2 == 5) h.def_len = (int)r.zz();
                    else if (i2 == 6 && t2 == 5) h.rep_len = (int)r.zz();
                    else if (i2 == 7 && (t2 == 1 || t2 == 2)) h.is_compressed = t2 == 1;
                    else r.skip(t2);
                } else {
                    if (i2 == 1 && t2 == 5) h.nv = (int)r.zz();
                    else if (i2 == 2 && t2 == 5) h.enc = (int)r.zz();
                    else if (i2 == 3 && t2 == 5 && outer == 5) h.def_enc = (int)r.zz();
                    else r.skip(t2);
                }
            }
        } else r.skip(t);
    }
    h.hdr = (int)(r.p - p);
    return !r.bad && h.type >= 0;
}

__device__ __forceinline__ void pq_err(int32_t *err, int code) { atomicCAS(err, KERR_NONE, code); }
__host__ __device__ __forceinline__ int64_t pq_al64(int64_t x) { return (x + 63) & ~(int64_t)63; }
__host__ __device__ __forceinline__ int64_t pq_min64(int64_t a, int64_t b) { return a < b ? a : b; }

// ------------------------------------------------------------------ page walk: one column chunk
//
// VectorizedColumnReader's page loop (:143-383) / ParquetFileReader.Chunk.readAllPages: header, body, next header.
// FILL = false counts (pages, dictionary entries, scratch bytes) into chunks[c]; FILL = true writes the page table.
// Returns the first KERR_* the chunk breaks (KERR_NONE when it is well formed).  k_pq_walk runs it on the device, one
// thread per chunk; pq_open runs the count pass on the host, so that pg_parquet_open refuses what the device would.
template <bool FILL>
__host__ __device__ inline int pq_walk_chunk(PqChunk *chunks, int c, PqPage *pages, PqPage *dicts, uint8_t *scratch) {
    const PqChunk ch = chunks[c];
    const uint8_t *p = ch.base, *end = ch.base + ch.avail;
    int64_t vals = 0, sc = 0, dict_entries = 0, page_bytes = 0;
    int n_pages = 0, n_dicts = 0;
    int code = KERR_NONE;
    bool needs_ids = false;
    const bool codec_on = ch.codec != pq::C_UNCOMPRESSED;
    while (vals < ch.num_values) {
        PqHeader h;
        if (p >= end || !pq_parse_header(p, end, h)) { code = KERR_PQ_HEADER; break; }
        const uint8_t *body = p + h.hdr;
        if (h.comp < 0 || h.unc < 0 || h.nv < 0 || (int64_t)(end - body) < (int64_t)h.comp) { code = KERR_PQ_HEADER; break; }
        if (h.type == pq::P_DICTIONARY) {
            if (n_dicts > 0 || n_pages > 0 || (h.enc != pq::E_PLAIN && h.enc != pq::E_PLAIN_DICTIONARY)) {
                code = KERR_PQ_ENCODING;
                break;
            }
            const int body_len = codec_on ? h.unc : h.comp;
            // fixed-width entries are looked up at body + id * width: every entry the header claims must be in the body
            // (BYTE_ARRAY entries are walked and bounded by k_pq_walk_dicts)
            if ((int64_t)h.nv * ch.phys_width > (int64_t)body_len) { code = KERR_BAD_PAGE; break; }
            if (FILL) {
                PqPage d;
                memset(&d, 0, sizeof(d));
                d.src = body; d.src_len = h.comp; d.body_len = body_len;
                d.body = codec_on ? scratch + ch.scratch_base + sc : body;
                d.num_values = h.nv; d.chunk = c; d.type = (int8_t)pq::P_DICTIONARY; d.compressed = codec_on;
                d.entry_base = ch.dict_entry_base;
                dicts[ch.dict_base] = d;
            }
            if (codec_on) sc += pq_al64((int64_t)h.unc + 16);
            if (ch.phys == pq::T_BYTE_ARRAY) dict_entries += h.nv;
            page_bytes += body_len;
            n_dicts++;
        } else if (h.type == pq::P_DATA || h.type == pq::P_DATA_V2) {
            int enc = -1;
            if (h.enc == pq::E_PLAIN) enc = ENC_PLAIN;
            else if (h.enc == pq::E_PLAIN_DICTIONARY || h.enc == pq::E_RLE_DICTIONARY) enc = ENC_DICT;
            else if (h.enc == pq::E_DELTA_BINARY_PACKED && (ch.phys == pq::T_INT32 || ch.phys == pq::T_INT64)) enc = ENC_DELTA_BP;
            else if (h.enc == pq::E_RLE && ch.phys == pq::T_BOOLEAN) enc = ENC_RLE_BOOL;
            if (enc < 0 || (enc == ENC_DICT && ch.phys == pq::T_BOOLEAN)) { code = KERR_PQ_ENCODING; break; }
            if (enc == ENC_DICT && n_dicts == 0) { code = KERR_PQ_NO_DICT; break; }
            const bool v2 = h.type == pq::P_DATA_V2;
            if ((v2 && h.rep_len != 0) || (!v2 && ch.max_def > 0 && h.def_enc != pq::E_RLE) || (v2 && h.def_len < 0)) {
                code = KERR_PQ_LEVELS;
                break;
            }
            const bool compressed = codec_on && (!v2 || h.is_compressed);
            const int body_len = compressed ? h.unc : h.comp;
            const int64_t unc_need = compressed ? pq_al64((int64_t)h.unc + 16) : 0;
            const int64_t aux_need = enc == ENC_DELTA_BP ? pq_al64((int64_t)body_len + (int64_t)h.nv * ch.phys_width + 16) : 0;
            if (FILL) {
                PqPage g;
                memset(&g, 0, sizeof(g));
                g.src = body; g.src_len = h.comp; g.body_len = body_len;
                g.body = compressed ? scratch + ch.scratch_base + sc : body;
                g.aux = aux_need ? scratch + ch.scratch_base + sc + unc_need : nullptr;
                g.num_values = h.nv; g.chunk = c; g.type = (int8_t)h.type; g.enc = (int8_t)enc; g.compressed = compressed;
                g.def_len = v2 ? h.def_len : 0;
                g.row0 = ch.row0 + vals;
                g.ids_base = ch.ids_base + vals;
                pages[ch.page_base + n_pages] = g;
            }
            sc += unc_need + aux_need;
            if (enc == ENC_DICT || enc == ENC_RLE_BOOL) needs_ids = true;
            page_bytes += body_len;
            vals += h.nv;
            n_pages++;
        }                                                // index pages are skipped
        p = body + h.comp;
    }
    if (code == KERR_NONE && vals != ch.num_values) code = KERR_PQ_ROWS;
    if (!FILL) {
        PqChunk &o = chunks[c];
        o.n_pages = n_pages; o.n_dicts = n_dicts; o.scratch_bytes = sc; o.dict_entries = dict_entries;
        o.ids_entries = needs_ids ? ch.num_values : 0;
        o.page_bytes = page_bytes;
    }
    return code;
}

template <bool FILL>
__global__ void k_pq_walk(PqChunk *chunks, int n_chunks, PqPage *pages, PqPage *dicts, uint8_t *scratch, int32_t *err) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chunks) return;
    const int code = pq_walk_chunk<FILL>(chunks, c, pages, dicts, scratch);
    if (code != KERR_NONE) pq_err(err, code);
}

// exclusive scans of the per-chunk counts -> bases; totals[0..5] = pages, dictionary pages, scratch bytes,
// dictionary entries, ids, page bytes
constexpr int kScanThreads = 512;
__global__ void __launch_bounds__(kScanThreads) k_pq_chunk_scan(PqChunk *chunks, int n, int64_t *totals) {
    __shared__ int64_t part[6][kScanThreads];
    const int per = (n + kScanThreads - 1) / kScanThreads;
    const int b = threadIdx.x * per, e = min(b + per, n);
    int64_t s[6] = {0, 0, 0, 0, 0, 0};
    for (int i = b; i < e; i++) {
        s[0] += chunks[i].n_pages; s[1] += chunks[i].n_dicts; s[2] += chunks[i].scratch_bytes;
        s[3] += chunks[i].dict_entries; s[4] += chunks[i].ids_entries; s[5] += chunks[i].page_bytes;
    }
    for (int q = 0; q < 6; q++) part[q][threadIdx.x] = s[q];
    __syncthreads();
    if (threadIdx.x < 6) {
        int64_t acc = 0;
        for (int i = 0; i < kScanThreads; i++) { const int64_t t = part[threadIdx.x][i]; part[threadIdx.x][i] = acc; acc += t; }
        totals[threadIdx.x] = acc;
    }
    __syncthreads();
    for (int q = 0; q < 6; q++) s[q] = part[q][threadIdx.x];
    for (int i = b; i < e; i++) {
        PqChunk &c = chunks[i];
        c.page_base = (int32_t)s[0]; c.dict_base = (int32_t)s[1]; c.scratch_base = s[2]; c.dict_entry_base = s[3];
        c.ids_base = s[4];
        s[0] += c.n_pages; s[1] += c.n_dicts; s[2] += c.scratch_bytes; s[3] += c.dict_entries; s[4] += c.ids_entries;
    }
}

// ------------------------------------------------------------------ Snappy / LZ4 page decompression
//
// Codec 1 (SNAPPY) pages are one Snappy stream (snappy_device.cuh): one warp per page parses the element stream in
// lock step and moves the bytes of a literal / copy lane-parallel.  Data page V2: the level bytes in front of the
// values are stored uncompressed and copied verbatim.
// Codec 5 (LZ4) pages are Hadoop-framed LZ4 blocks (lz4_device.cuh, the same warp-per-page shape); no length of a
// chunk's output is stored, so one warp walks a page's blocks in order.
__global__ void k_pq_snappy_lz4(const PqPage *pages, int n_pages, const PqPage *dicts, int n_dicts, const PqChunk *chunks,
                                int32_t *err) {
    const int w = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (w >= n_pages + n_dicts) return;
    const PqPage &pg = w < n_pages ? pages[w] : dicts[w - n_pages];
    const int codec = chunks[pg.chunk].codec;
    if (!pg.compressed || (codec != pq::C_SNAPPY && codec != pq::C_LZ4)) return;
    const int prefix = pg.type == pq::P_DATA_V2 ? pg.def_len : 0;
    uint8_t *out0 = const_cast<uint8_t *>(pg.body);
    const uint8_t *in0 = pg.src;
    if (prefix > pg.src_len || prefix > pg.body_len) { if (lane == 0) pq_err(err, KERR_BAD_PAGE); return; }
    for (int i = lane; i < prefix; i += 32) out0[i] = in0[i];
    const uint8_t *src = in0 + prefix;
    uint8_t *dst = out0 + prefix;
    const int n_src = pg.src_len - prefix, n_dst = pg.body_len - prefix;
    if (codec == pq::C_LZ4) {
        if (lz4::decode_hadoop(src, n_src, dst, n_dst) != n_dst && lane == 0) pq_err(err, KERR_BAD_PAGE);
        return;
    }
    if (snappy::decode(src, n_src, dst, n_dst) != n_dst && lane == 0) pq_err(err, KERR_BAD_PAGE);
}

// ------------------------------------------------------------------ Zstandard / GZIP page decompression
//
// zstd is Paimon's default codec (CoreOptions.java:318-321); gzip is parquet-mr's other general-purpose codec.  The
// decoders are zstd_device.cuh (RFC 8878) and inflate_device.cuh (RFC 1951 / 1952), written once for host and device;
// their host builds are pinned against libzstd / zlib by tests/test_zstd_cpu.py and tests/test_inflate_cpu.py.  A
// fixed grid of warps pulls pages off a counter: every warp owns one set of FSE / Huffman tables in shared memory and
// one 128 KiB literals buffer in global scratch; the lanes run the block decoder in lock step and move the bytes of
// literal / match copies lane-parallel.
constexpr int kZsWarps = 4;
__global__ void __launch_bounds__(kZsWarps * 32)
k_pq_zstd(const PqPage *pages, int n_pages, const PqPage *dicts, int n_dicts, const PqChunk *chunks, uint8_t *lit_scratch,
          int32_t *counter, int32_t *err) {
    __shared__ zs::Tables T[kZsWarps];                     // (the DEFLATE tables are smaller and overlay them)
    static_assert(sizeof(inflate::Tables) <= sizeof(zs::Tables), "tables overlay");
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t *lit = lit_scratch + ((size_t)blockIdx.x * kZsWarps + w) * (size_t)(zs::kMaxBlock + 64);
    while (true) {
        int j = 0;
        if (lane == 0) j = atomicAdd(counter, 1);
        j = __shfl_sync(0xffffffffu, j, 0);
        if (j >= n_pages + n_dicts) return;
        const PqPage &pg = j < n_pages ? pages[j] : dicts[j - n_pages];
        const int codec = chunks[pg.chunk].codec;
        if (!pg.compressed || (codec != pq::C_ZSTD && codec != pq::C_GZIP)) continue;
        const int prefix = pg.type == pq::P_DATA_V2 ? pg.def_len : 0;
        uint8_t *out0 = const_cast<uint8_t *>(pg.body);
        if (prefix > pg.src_len || prefix > pg.body_len) { if (lane == 0) pq_err(err, KERR_BAD_PAGE); continue; }
        for (int i = lane; i < prefix; i += 32) out0[i] = pg.src[i];
        const int64_t want = pg.body_len - prefix;
        const int64_t got = codec == pq::C_ZSTD
            ? zs::decode(pg.src + prefix, pg.src_len - prefix, out0 + prefix, want, lit, T[w])
            : inflate::inflate_gzip(pg.src + prefix, pg.src_len - prefix, out0 + prefix, want, *(inflate::Tables *)&T[w]);
        if (got != want && lane == 0) pq_err(err, KERR_BAD_PAGE);
        __syncwarp();
    }
}

// ------------------------------------------------------------------ DELTA_BINARY_PACKED
//
// VectorizedDeltaBinaryPackedReader.java; the layout restated here is the public Parquet encoding specification:
// <block size> <miniblocks per block> <total count> <first value> then per block <min delta> <bit width per
// miniblock> <bit-packed miniblocks>.  One warp per page expands the values into a PLAIN image behind a copy of the
// level bytes, and points the page at the image, so the PLAIN path reads the page afterwards.
__device__ __forceinline__ uint64_t dl_varint(const uint8_t *p, int n, int &pos) {
    uint64_t v = 0;
    for (int sh = 0; pos < n && sh < 70; sh += 7) {
        const uint8_t b = p[pos++];
        v |= (uint64_t)(b & 0x7f) << sh;
        if (!(b & 0x80)) break;
    }
    return v;
}
__global__ void k_pq_delta(PqPage *pages, int n_pages, const PqChunk *chunks, int32_t *err) {
    const int w = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (w >= n_pages) return;
    const PqPage pg = pages[w];
    if (pg.enc != ENC_DELTA_BP) return;
    const PqChunk &ch = chunks[pg.chunk];
    const int width = ch.phys_width;
    // level bytes in front of the values: V1 = 4-byte length + RLE levels (OPTIONAL only), V2 = def_len
    int prefix = 0;
    if (ch.max_def > 0) {
        if (pg.type == pq::P_DATA_V2) prefix = pg.def_len;
        else if (pg.body_len >= 4)
            prefix = 4 + (int)((uint32_t)pg.body[0] | ((uint32_t)pg.body[1] << 8) | ((uint32_t)pg.body[2] << 16) | ((uint32_t)pg.body[3] << 24));
        else prefix = -1;
    }
    if (prefix < 0 || prefix > pg.body_len) { if (lane == 0) { pq_err(err, KERR_BAD_PAGE); pages[w].bad = 1; } return; }
    for (int i = lane; i < prefix; i += 32) pg.aux[i] = pg.body[i];
    const uint8_t *p = pg.body + prefix;
    const int n = pg.body_len - prefix;
    uint8_t *out = pg.aux + prefix;
    int pos = 0;
    const int block_size = (int)dl_varint(p, n, pos);
    const int n_mini = (int)dl_varint(p, n, pos);
    const int64_t total = (int64_t)dl_varint(p, n, pos);
    const uint64_t zz = dl_varint(p, n, pos);
    uint64_t last = (zz >> 1) ^ (0 - (zz & 1));               // first value
    bool bad = n_mini <= 0 || block_size <= 0 || block_size % n_mini != 0 || total > pg.num_values || total < 0;
    const int mini = bad ? 1 : block_size / n_mini;
    if (!bad && total > 0 && lane == 0) {
        if (width == 8) memcpy(out, &last, 8); else { uint32_t x = (uint32_t)last; memcpy(out, &x, 4); }
    }
    int64_t done = 1;
    while (!bad && done < total) {
        const uint64_t mz = dl_varint(p, n, pos);
        const uint64_t min_delta = (mz >> 1) ^ (0 - (mz & 1));
        const int bw_pos = pos;
        pos += n_mini;
        if (pos > n) { bad = true; break; }
        for (int m = 0; m < n_mini && done < total; m++) {
            const int bw = p[bw_pos + m];
            if (bw > 64 || pos + (int64_t)mini * bw / 8 > n) { bad = true; break; }
            for (int v0 = 0; v0 < mini && done < total; v0 += 32) {
                const int v = v0 + lane;
                uint64_t d = 0;
                if (v < mini && bw > 0) {
                    const int64_t bit = (int64_t)v * bw;
                    const uint8_t *q = p + pos + (bit >> 3);
                    const int sh = (int)(bit & 7);
                    uint64_t lo = 0;                             // up to 9 bytes hold the value
                    const int nb = (sh + bw + 7) >> 3;
                    for (int b = 0; b < nb && b < 8; b++) lo |= (uint64_t)q[b] << (8 * b);
                    d = lo >> sh;
                    if (nb > 8) d |= (uint64_t)q[8] << (64 - sh);
                    if (bw < 64) d &= ((uint64_t)1 << bw) - 1;
                }
                uint64_t x = v < mini ? d + min_delta : 0;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {                // inclusive scan of the deltas over the warp
                    const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
                    if (lane >= o) x += y;
                }
                const uint64_t val = last + x;
                const int64_t idx = done + lane;
                if (v < mini && idx < total) {
                    if (width == 8) memcpy(out + idx * 8, &val, 8);
                    else { uint32_t t = (uint32_t)val; memcpy(out + idx * 4, &t, 4); }
                }
                const int cnt = min(32, mini - v0);
                last = __shfl_sync(0xffffffffu, val, cnt - 1);
                done += cnt;
            }
            pos += mini * bw / 8;
        }
    }
    if (lane == 0) {
        if (bad) { pq_err(err, KERR_BAD_PAGE); pages[w].bad = 1; }
        pages[w].body = pg.aux;
        pages[w].body_len = prefix + (int)(total > 0 && !bad ? total : 0) * width;
    }
}

// ------------------------------------------------------------------ levels, dictionary ids, page sizes
//
// Definition levels of a flat OPTIONAL column (bit width 1): the RLE / bit-packed hybrid stream
// (VectorizedRleValuesReader.java:928-1019) is turned straight into the run's Arrow validity bitmap at bit
// row0 + i.  A bit-packed run IS a bitmap: every lane moves 32 bits of it.  Returns the number of set bits; `ok` is
// cleared when the stream ends before `count` levels or inside a run (parquet-mr refuses such a page too).
__device__ int pq_def_to_bits(const uint8_t *p, const uint8_t *end, int count, uint32_t *bm, int64_t row0, bool &ok) {
    const int lane = threadIdx.x & 31;
    int pos = 0, nnz = 0;
    while (pos < count) {
        if (p >= end) { ok = false; break; }
        const uint32_t h = pq_varint(p, end, ok);
        const bool packed = h & 1;
        const int64_t span = packed ? (int64_t)(h >> 1) * 8 : (int64_t)(h >> 1);   // values the run stands for
        const int64_t run_bytes = packed ? (int64_t)(h >> 1) : 1;
        if (!ok || run_bytes > end - p) { ok = false; break; }
        const uint8_t *src = p;
        p += run_bytes;
        const int nv = (int)pq_min64(span, count - pos);
        const bool ones = !packed && (src[0] & 1);
        if (nv > 0 && (packed || ones)) {
            const int64_t d0 = row0 + pos, d1 = d0 + nv;
            for (int64_t w = (d0 >> 5) + lane; w <= ((d1 - 1) >> 5); w += 32) {
                const int64_t lo = max(d0, w * 32), hi = min(d1, w * 32 + 32);
                const int cnt = (int)(hi - lo);
                uint32_t bits = 0xffffffffu;
                if (packed) {
                    const int sbit = (int)(lo - d0);
                    const uint8_t *q = src + (sbit >> 3);
                    uint64_t v = 0;
#pragma unroll
                    for (int b = 0; b < 5; b++)
                        if (q + b < end) v |= (uint64_t)q[b] << (8 * b);
                    bits = (uint32_t)(v >> (sbit & 7));
                }
                if (cnt < 32) bits &= (1u << cnt) - 1;
                const uint32_t word = bits << (int)(lo - w * 32);
                if (cnt == 32) bm[w] = word;
                else if (word) atomicOr(&bm[w], word);
                nnz += __popc(word);
            }
        }
        pos += (int)pq_min64(span, (int64_t)count);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) nnz += __shfl_xor_sync(0xffffffffu, nnz, d);
    return nnz;
}

// Warp-cooperative RLE / bit-packed hybrid decode of `count` values of bit width bw: out(i, value).  Returns false
// (and stops before the run) when the stream ends before `count` values or a run's bytes reach past `end`.
template <typename Out>
__device__ bool pq_hybrid_decode(const uint8_t *p, const uint8_t *end, int bw, int count, Out out) {
    const int lane = threadIdx.x & 31;
    const uint32_t mask = bw >= 32 ? 0xffffffffu : ((1u << bw) - 1);
    int pos = 0;
    while (pos < count) {
        if (bw == 0) {                        // a zero-width stream encodes only zeros
            for (int i = pos + lane; i < count; i += 32) out(i, 0u);
            break;
        }
        if (p >= end) return false;
        bool ok = true;
        const uint32_t h = pq_varint(p, end, ok);
        if (!ok) return false;
        if (h & 1) {
            const int64_t groups = (int64_t)(h >> 1);
            const int64_t nvals = groups * 8;
            if (groups * bw > end - p) return false;
            for (int64_t i = lane; i < nvals && pos + i < count; i += 32) {
                const int64_t bit = i * bw;
                const uint8_t *q = p + (bit >> 3);
                uint64_t w = 0;
#pragma unroll
                for (int b = 0; b < 5; b++)
                    if (q + b < end) w |= (uint64_t)q[b] << (8 * b);
                out(pos + (int)i, (uint32_t)(w >> (bit & 7)) & mask);
            }
            p += groups * bw;
            pos = (int)pq_min64((int64_t)pos + nvals, (int64_t)count);
        } else {
            const int run = (int)(h >> 1);
            uint32_t v = 0;
            const int nb = (bw + 7) / 8;
            if (nb > end - p) return false;
            for (int b = 0; b < nb; b++) v |= (uint32_t)p[b] << (8 * b);
            p += nb;
            for (int i = lane; i < run && pos + i < count; i += 32) out(pos + i, v & mask);
            pos = (int)pq_min64((int64_t)pos + run, (int64_t)count);
        }
    }
    return true;
}

// one warp per data page
__global__ void k_pq_levels(PqPage *pages, int n_pages, const PqPage *dicts, const PqChunk *chunks, const PqOut *outs,
                            int n_cols, int32_t *ids, const int32_t *dict_len, int32_t *err) {
    const int j = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (j >= n_pages) return;
    const PqPage pg = pages[j];
    if (pg.bad) return;
    const PqChunk &ch = chunks[pg.chunk];
    const PqOut &out = outs[ch.run * n_cols + ch.col];
    const uint8_t *body = pg.body;
    const int nv = pg.num_values;
    int values_off = 0, nnz = nv;
    bool bad = false;
    if (ch.max_def > 0) {
        const uint8_t *dp = body;
        int dlen = pg.def_len;
        if (pg.type != pq::P_DATA_V2) {
            if (pg.body_len < 4) bad = true;
            else {
                dlen = (int)((uint32_t)body[0] | ((uint32_t)body[1] << 8) | ((uint32_t)body[2] << 16) | ((uint32_t)body[3] << 24));
                dp = body + 4;
                values_off = 4;
            }
        }
        if (!bad && (dlen < 0 || (int64_t)values_off + dlen > pg.body_len)) bad = true;
        if (!bad) {
            values_off += dlen;
            bool ok = true;
            nnz = pq_def_to_bits(dp, dp + dlen, nv, out.validity, pg.row0, ok);
            bad = !ok;
        }
    }
    else if (out.validity != nullptr) {
        // REQUIRED in this file, OPTIONAL in another file of the section: every row of the page is valid
        const int64_t d0 = pg.row0, d1 = pg.row0 + nv;
        for (int64_t w = (d0 >> 5) + lane; nv > 0 && w <= ((d1 - 1) >> 5); w += 32) {
            const int64_t lo = max(d0, w * 32), hi = min(d1, w * 32 + 32);
            const int cnt = (int)(hi - lo);
            const uint32_t word = (cnt < 32 ? (1u << cnt) - 1 : 0xffffffffu) << (int)(lo - w * 32);
            if (cnt == 32) out.validity[w] = word; else atomicOr(&out.validity[w], word);
        }
    }
    int64_t payload = 0;
    if (!bad) {
        const uint8_t *vp = body + values_off, *end = body + pg.body_len;
        const int64_t vbytes = pg.body_len - values_off;
        if (pg.enc == ENC_DICT) {
            const PqPage &dj = dicts[ch.dict_base];
            const uint32_t n_entries = (uint32_t)dj.num_values;
            const int bw = vp < end ? vp[0] : 0;
            int32_t *dst = ids + pg.ids_base;
            const bool ba = ch.phys == pq::T_BYTE_ARRAY;
            const int32_t *dl = dict_len + dj.entry_base;
            bool oob = false;
            // (the ids the stream does not cover would be whatever the ids scratch held: a short stream is refused)
            if (bw > 32 || (nnz > 0 && vp >= end)) bad = true;
            else bad = !pq_hybrid_decode(vp + 1, end, bw, nnz, [&](int i, uint32_t v) {
                if (v >= n_entries) { oob = true; v = 0; }
                dst[i] = (int32_t)v;
                if (ba && n_entries) payload += dl[v];
            });
            if (__any_sync(0xffffffffu, oob)) { if (lane == 0) pq_err(err, KERR_PQ_DICT_ID); bad = true; }
        } else if (pg.enc == ENC_RLE_BOOL) {
            // RLE-encoded BOOLEAN values: <length:4> <hybrid stream of bit width 1>
            int32_t *dst = ids + pg.ids_base;
            if (vbytes < 4) bad = nnz > 0;
            else bad = !pq_hybrid_decode(vp + 4, end, 1, nnz, [&](int i, uint32_t v) { dst[i] = (int32_t)v; });
        } else if (ch.phys == pq::T_BYTE_ARRAY) {
            const int64_t pb = vbytes - 4 * (int64_t)nnz;
            if (pb < 0) bad = true;
            payload = lane == 0 ? pb : 0;                  // (summed over the lanes below)
        } else if (ch.phys == pq::T_BOOLEAN) {
            if (vbytes < ((int64_t)nnz + 7) / 8) bad = true;
        } else {
            if (vbytes < (int64_t)nnz * ch.phys_width) bad = true;
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) payload += __shfl_xor_sync(0xffffffffu, payload, d);
    if (lane == 0) {
        PqPage &o = pages[j];
        o.values_off = values_off;
        o.nnz = nnz;
        o.payload_bytes = bad ? 0 : payload;
        if (bad) { o.bad = 1; pq_err(err, KERR_BAD_PAGE); }
    }
}

// one warp per (run, var-len column): payload base of every page; files of a run continue each other's offsets
__global__ void k_pq_scan_pages(PqPage *pages, const PqChunk *chunks, const PqPair *pairs, int n_pairs, int64_t *totals,
                                int32_t *err) {
    const int w = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (w >= n_pairs) return;
    const PqPair pr = pairs[w];
    int64_t carry = 0;
    if (pr.chunk1 > pr.chunk0) {
        const int first = chunks[pr.chunk0].page_base;
        const int last = chunks[pr.chunk1 - 1].page_base + chunks[pr.chunk1 - 1].n_pages;
        for (int base = first; base < last; base += 32) {
            const int i = base + lane;
            const int64_t x = i < last ? pages[i].payload_bytes : 0;
            int64_t incl = x;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int64_t y = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += y;
            }
            if (i < last) {
                pages[i].payload_base = carry + incl - x;
                pages[i].vs_base = pr.vs_rows_base + pages[i].row0 + i + pr.idx;
                pages[i].is_last = i == last - 1;
            }
            carry += __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    if (lane == 0) {
        totals[w] = carry;
        if (carry > 0x7fffffffLL) pq_err(err, KERR_OFFSET_OVERFLOW);
    }
}

// ------------------------------------------------------------------ PLAIN BYTE_ARRAY walk
//
// [len:4][bytes][len:4][bytes]... (VectorizedPlainValuesReader.java:275-288).  The lengths are embedded in the
// stream, so the walk itself is sequential; one warp per page stages the stream through shared memory in 2 KiB
// windows (coalesced 16-byte loads), lane 0 walks the window at shared-memory latency, and the results go out
// coalesced: emit(j, q, len) for value j whose length word sits at stream offset q.  Returns the stream offset
// behind the last value walked (-1: malformed).
constexpr int kWalkWindow = 2048;
constexpr int kWalkWarps = 8;

template <typename Emit>
__device__ int64_t pq_walk_stream(const uint8_t *stream, int64_t stream_len, int count, uint8_t *win, uint32_t *w_off,
                                  int32_t *w_len, Emit emit) {
    const int lane = threadIdx.x & 31;
    int done = 0;
    int64_t pos = 0;                                   // stream offset of the next length word
    while (done < count) {
        if (pos + 4 > stream_len) return -1;
        // window = [base, base + kWalkWindow + 16) clipped to the stream, base 16-byte aligned in memory
        const uint8_t *p = stream + pos;
        const uint8_t *base = (const uint8_t *)((uintptr_t)p & ~(uintptr_t)15);
        const int skip = (int)(p - base);
        const int avail = (int)min((int64_t)(stream + stream_len - base), (int64_t)(kWalkWindow + 16));
        for (int o = lane * 16; o < avail; o += 32 * 16) *(uint4 *)(win + o) = *(const uint4 *)(base + o);
        __syncwarp();
        int nfound = 0, q = skip;
        bool corrupt = false;
        if (lane == 0) {
            while (done + nfound < count && q + 4 <= avail && nfound < 256) {
                const int32_t len = (int32_t)((uint32_t)win[q] | ((uint32_t)win[q + 1] << 8) | ((uint32_t)win[q + 2] << 16) |
                                              ((uint32_t)win[q + 3] << 24));
                if (len < 0) { corrupt = true; break; }
                w_off[nfound] = (uint32_t)q;
                w_len[nfound] = len;
                nfound++;
                if ((int64_t)q + 4 + len > 0x7fffffff) { corrupt = true; break; }
                q += 4 + len;
            }
        }
        nfound = __shfl_sync(0xffffffffu, nfound, 0);
        q = __shfl_sync(0xffffffffu, q, 0);
        corrupt = __shfl_sync(0xffffffffu, (int)corrupt, 0);
        __syncwarp();
        const int64_t base_off = (int64_t)(base - stream);
        for (int i = lane; i < nfound; i += 32) emit(done + i, base_off + w_off[i], w_len[i]);
        __syncwarp();
        if (corrupt || nfound == 0) return -1;            // a length word straddles the stream end: malformed
        done += nfound;
        pos = base_off + q;
        if (pos > stream_len) return -1;
    }
    return pos;
}

// BYTE_ARRAY dictionary pages -> entry offsets / lengths: one warp per dictionary page (few, large pages).
__global__ void __launch_bounds__(kWalkWarps * 32)
k_pq_walk_dicts(const PqPage *dicts, int n_dicts, const PqChunk *chunks, int32_t *dict_off, int32_t *dict_len, int32_t *err) {
    __shared__ __align__(16) uint8_t s_win[kWalkWarps][kWalkWindow + 32];
    __shared__ uint32_t s_off[kWalkWarps][256];
    __shared__ int32_t s_len[kWalkWarps][256];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.x * kWalkWarps + w;
    if (t >= n_dicts) return;
    const PqPage dj = dicts[t];
    if (chunks[dj.chunk].phys != pq::T_BYTE_ARRAY) return;
    int32_t *doff = dict_off + dj.entry_base, *dlen = dict_len + dj.entry_base;
    const int64_t endq = pq_walk_stream(dj.body, dj.body_len, dj.num_values, s_win[w], s_off[w], s_len[w],
                                        [&](int j, int64_t q, int32_t len) { doff[j] = (int32_t)(q + 4); dlen[j] = len; });
    if (lane == 0 && endq < 0) pq_err(err, KERR_BAD_PAGE);
}

// PLAIN BYTE_ARRAY data pages -> value start offsets in the OUTPUT payload (vstart[vs_base + j], j <= nnz).
// The walk of one page is a dependent chain (every length word says where the next one is), so a page cannot be
// split; a section has tens of thousands of such pages, though, so every LANE walks its own page: 32 independent
// chains per warp instead of one lane working while 31 idle (the warp-per-page version was issue-bound).  Pages of a column chunk are neighbours in the page table, so the
// lanes of a warp walk streams of similar length.
// Reading the length words straight from global memory makes every lane miss a 32-byte sector on nearly every value
// (32 scattered sector fetches per warp step, one round trip each), so each lane's stream comes into shared memory
// through a RING of kWvRing chunks of kWvChunk bytes, loaded by the warp with coalesced 16-byte async copies (8 lanes
// per chunk).  The warp advances in uniform steps: every lane walks the length words inside its landed chunks (at most
// kWvCap values), then the warp refills the chunks the lanes have left and commits exactly one copy group, so every
// lane's group count stays the same and `cp.async.wait_group kWvLead` at the top of a step means "the chunks requested
// kWvLead + 1 steps ago have landed".  A lane never waits for a copy it has just issued: the round trip hides behind
// kWvLead steps of walking.  A small ring leaves the SMs' shared memory to the expansion beside the walk (1 KiB per
// lane held it back for about 4 ms of the C3 decode).
// Chunk k of a lane holds stream bytes [a0 + kWvChunk k, a0 + kWvChunk (k + 1)), a0 = the 16-byte boundary at or below
// the stream start, so the ring is plain modulo addressing.  Rows are XOR-swizzled per 16-byte unit (lanes walk their
// rows at similar offsets: without it every access is a 32-way bank conflict).
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async4(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
constexpr int kWvWarps = 1;
constexpr int kWvChunk = 128, kWvRing = 4, kWvLead = 1, kWvCap = 32;
constexpr int kWvRow = kWvChunk * kWvRing;                      // ring bytes per lane
static_assert(kWvCap == 32, "one lane's values of a step leave as one warp store");
static_assert((kWvRow & (kWvRow - 1)) == 0 && kWvChunk == 8 * 16 && kWvRow / 16 >= 16, "power-of-two ring, 8 units per chunk");

#ifdef PG_WALK_TIMING
// Cycle split of the value walk for every 4th warp (of the first 1024) that walks any value: per step, issuing the
// copies, waiting for them and walking; plus steps, values, the warp's start / end on the global timer (waves) and its
// SM.  Build with EXTRA_DEFS=-DPG_WALK_TIMING; every decode then synchronises and prints the split.
constexpr int kWtSlots = 256;
__device__ long long g_walk_ts[kWtSlots][8];
#define WT_DECL long long wt_t = 0, wt_acc[3] = {0, 0, 0}, wt_steps = 0, wt_g0 = 0; \
    const int wt_slot = (blockIdx.x % 4 == 0 && blockIdx.x < 4 * kWtSlots) ? (int)(blockIdx.x / 4) : -1; \
    if (wt_slot >= 0) { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(wt_g0)); wt_t = clock64(); }
#define WT_MARK(k) do { if (wt_slot >= 0) { const long long wt_n = clock64(); wt_acc[k] += wt_n - wt_t; wt_t = wt_n; \
    if ((k) == 2) wt_steps++; } } while (0)
#define WT_END(vals) do { if (wt_slot >= 0) { long long wt_v = (vals); \
    for (int d = 16; d > 0; d >>= 1) wt_v += __shfl_xor_sync(0xffffffffu, wt_v, d); \
    if ((threadIdx.x & 31) == 0 && wt_v > 0) { long long g1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g1)); \
        unsigned smid; asm("mov.u32 %0, %%smid;" : "=r"(smid)); long long *o = g_walk_ts[wt_slot]; \
        o[0] = wt_acc[0]; o[1] = wt_acc[1]; o[2] = wt_acc[2]; o[3] = wt_steps; o[4] = wt_v; o[5] = wt_g0; o[6] = g1; \
        o[7] = smid; } } } while (0)
#else
#define WT_DECL
#define WT_MARK(k) do {} while (0)
#define WT_END(vals) do {} while (0)
#endif

__global__ void __launch_bounds__(kWvWarps * 32)
k_pq_walk_values(PqPage *pages, int n_pages, const PqChunk *chunks, int32_t *vstart, int32_t *err) {
    __shared__ __align__(16) uint8_t s_ring[kWvWarps][32][kWvRow];
    // the step's copy requests, one per chunk: source, and (lane << 8 | slot << 4 | 16-byte units to load)
    __shared__ const uint8_t *s_req_src[kWvWarps][32 * kWvRing];
    __shared__ uint32_t s_req_dst[kWvWarps][32 * kWvRing];
    // the step's value starts of every lane, written out by the warp one lane's run at a time (one lane's stores are
    // one 128-byte run; storing straight from the walk would scatter every warp store over 32 lines)
    __shared__ int32_t s_vs[kWvWarps][32][kWvCap + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int t = blockIdx.x * (kWvWarps * 32) + threadIdx.x;
    WT_DECL
    bool done = true;
    PqPage pg;
    pg.nnz = 0;
    if (t < n_pages) {
        pg = pages[t];
        done = pg.bad || pg.enc != ENC_PLAIN || chunks[pg.chunk].phys != pq::T_BYTE_ARRAY;
    }
    const bool mine = !done;
    const uint8_t *stream = mine ? pg.body + pg.values_off : nullptr;
    const int32_t slen = mine ? pg.body_len - pg.values_off : 0;
    const int nnz = mine ? pg.nnz : 0;
    const uint8_t *a0 = (const uint8_t *)((uintptr_t)stream & ~(uintptr_t)15);
    // Positions are 32-bit offsets from a0 (a page body's size is an int32): p = the next length word, pend = the
    // stream end.  out(j) = payload_base + (offset of value j's length word in the stream) - 4 j = p_j + bias_j.
    const uint32_t off0 = (uint32_t)(stream - a0);
    uint32_t p = off0, pend = off0 + (uint32_t)max(slen, 0);
    uint32_t bias = mine ? (uint32_t)pg.payload_base - off0 : 0;
    int32_t *vs = mine ? vstart + pg.vs_base : nullptr;
    int j = 0;
    bool bad = slen < 0;
    if (nnz == 0 || bad) done = true;
    const int n_chunks = done ? 0 : (int)((pend + kWvChunk - 1) / kWvChunk);
    int next = 0;                                      // chunks [0, next) requested (or skipped)
    int hist[kWvLead + 1];                             // next after each of the last kWvLead + 1 steps' requests
#pragma unroll
    for (int i = 0; i <= kWvLead; i++) hist[i] = 0;
    uint8_t (*rows)[kWvRow] = s_ring[warp];
    const uint8_t *row = rows[lane];
    const int sw = lane & 15;
    while (true) {
        cp_async_wait<kWvLead>();
        __syncwarp();
        WT_MARK(1);
        // ---- walk the length words inside the landed chunks [p / kWvChunk, hist[0])
        const uint32_t lim = (uint32_t)hist[0] * kWvChunk;
        const int j0 = j;
        if (!done) {
            for (int c = 0; c < kWvCap; c++) {
                if (p + 4 > pend) { bad = true; break; }
                if (p + 4 > lim) break;
                // the length word: two aligned words of the (unit-swizzled) ring row, funnel-shifted
                const uint32_t wi = (p >> 2) & (kWvRow / 4 - 1), wj = (wi + 1) & (kWvRow / 4 - 1);
                const uint32_t lo = *(const uint32_t *)(row + ((((wi >> 2) ^ sw) << 4) | ((wi & 3) << 2)));
                const uint32_t hi = *(const uint32_t *)(row + ((((wj >> 2) ^ sw) << 4) | ((wj & 3) << 2)));
                const uint32_t len = __funnelshift_r(lo, hi, (p & 3) * 8);
                if (len > pend - p - 4) { bad = true; break; }
                s_vs[warp][lane][c] = (int32_t)(p + bias);
                bias -= 4;
                p += 4 + len;
                if (++j == nnz) break;
            }
            if (bad || j == nnz) done = true;
        }
        __syncwarp();
        for (unsigned m = __ballot_sync(0xffffffffu, j > j0); m != 0; m &= m - 1) {
            const int i = __ffs(m) - 1;
            const int n = __shfl_sync(0xffffffffu, j - j0, i);
            int32_t *dst = (int32_t *)__shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)(vs + j0), i);
            if (lane < n) dst[lane] = s_vs[warp][i][lane];
        }
        WT_MARK(2);
        if (__all_sync(0xffffffffu, done)) break;
        // ---- refill: chunks from `next` on, while the ring slot is free (its chunk was walked past, or a value skipped
        // it) and its previous occupant has landed (so two copies never target one slot)
        const int cur = (int)(p / kWvChunk);
        const int first = max(next, cur);
        const int nreq = done ? 0 : max(0, min(min(cur, hist[0]) + kWvRing, n_chunks) - first);
        next = first + nreq;
        int incl = nreq;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += y;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        for (int r = 0; r < nreq; r++) {
            const int k = first + r;
            const uint32_t units = min(8u, (pend - (uint32_t)k * kWvChunk + 15) / 16);   // (<= 15 bytes past the page)
            s_req_src[warp][incl - nreq + r] = a0 + (size_t)k * kWvChunk;
            s_req_dst[warp][incl - nreq + r] = (uint32_t)lane << 8 | (uint32_t)(k % kWvRing) << 4 | units;
        }
        __syncwarp();
        for (int e = lane >> 3; e < total; e += 4) {
            const uint32_t d = s_req_dst[warp][e], u = lane & 7;
            if (u < (d & 15)) {
                const int owner = (int)(d >> 8), unit = (int)(((d >> 4) & 15) * 8 + u);
                cp_async16(&rows[owner][(unit ^ (owner & 15)) << 4], s_req_src[warp][e] + 16 * u);
            }
        }
        cp_async_commit();
#pragma unroll
        for (int i = 0; i < kWvLead; i++) hist[i] = hist[i + 1];
        hist[kWvLead] = next;
        WT_MARK(0);
    }
    cp_async_wait<0>();
    WT_END(nnz);
    if (mine) {
        if (bad || (nnz > 0 && p != pend) || (nnz == 0 && slen != 0)) { pq_err(err, KERR_BAD_PAGE); pages[t].bad = 1; return; }
        vs[nnz] = (int32_t)(p + bias);
    }
}

// ------------------------------------------------------------------ expand: one CTA per data page
//
// Null cells occupy no space in the value stream (VectorizedRleValuesReader.java:260-289): the value of row r is the
// rank(r)-th value of the page, rank = number of set validity bits in front of r inside the page.  The page's rows are
// walked in windows of 256 validity words (aligned to the run's 32-row words, so pages that start in the middle of a
// word mask their neighbours' bits out); a block scan of the word popcounts gives every word its rank base.
constexpr int kExpThreads = 256;
constexpr int kPayIn = 8 * 1024, kPayOut = 7 * 1024;      // staging of a batch of kExpThreads PLAIN BYTE_ARRAY values
constexpr int kPayBatches = 1023;                          // batch boundaries kept per page (pages beyond: direct path)


__device__ __forceinline__ uint64_t pq_load_unaligned(const uint8_t *p, int w) {
    if (w == 8) {
        const uintptr_t a = (uintptr_t)p;
        const uint64_t *q = (const uint64_t *)(a & ~(uintptr_t)7);
        const int sh = (int)(a & 7) * 8;
        const uint64_t lo = q[0];
        return sh ? (lo >> sh) | (q[1] << (64 - sh)) : lo;
    }
    const uintptr_t a = (uintptr_t)p;
    const uint32_t *q = (const uint32_t *)(a & ~(uintptr_t)3);
    const int sh = (int)(a & 3) * 8;
    const uint32_t lo = q[0];
    return sh ? (uint64_t)((lo >> sh) | (q[1] << (32 - sh))) : (uint64_t)lo;
}

// Shared-memory staging of the PLAIN BYTE_ARRAY payload copy.  Only the instantiation that expands those pages has it:
// without its 29 KB, the expansion of the other pages fits on an SM beside the value walk's windows.
template <bool kPlainStrings> struct PqPlainStage {
    int vs[2][kExpThreads + 4];
    int bnd[kPayBatches + 1];
    alignas(16) uint8_t in[2][kPayIn];
    alignas(16) uint8_t out[kPayOut];
};
template <> struct PqPlainStage<false> {};

// kPlainStrings: the PLAIN BYTE_ARRAY pages (after the value walk), else every other page
template <bool kPlainStrings>
__global__ void __launch_bounds__(kExpThreads, 6)
k_pq_expand(const PqPage *pages, const PqPage *dicts, const PqChunk *chunks, const PqOut *outs, int n_cols,
            const int32_t *ids, const int32_t *vstart, const int32_t *dict_off, const int32_t *dict_len) {
    __shared__ uint32_t s_bits[kExpThreads];
    __shared__ int s_rank[kExpThreads];
    __shared__ int s_wlen[kExpThreads];
    __shared__ int s_ws[34];
    __shared__ PqPlainStage<kPlainStrings> stage;
    const PqPage pg = pages[blockIdx.x];
    if (pg.bad || pg.num_values == 0) return;
    const PqChunk ch = chunks[pg.chunk];
    if (kPlainStrings != (ch.phys == pq::T_BYTE_ARRAY && pg.enc == ENC_PLAIN)) return;
    const PqOut out = outs[ch.run * n_cols + ch.col];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t row0 = pg.row0, row1 = pg.row0 + pg.num_values;
    const int64_t g0 = row0 & ~(int64_t)31;
    const int n_words = (int)((row1 - g0 + 31) >> 5);
    const uint8_t *values = pg.body + pg.values_off;
    const int pw = ch.phys_width;
    const bool varlen = ch.phys == pq::T_BYTE_ARRAY;
    const bool is_dict = pg.enc == ENC_DICT;
    const PqPage *dj = is_dict ? &dicts[ch.dict_base] : nullptr;
    const uint8_t *dbody = is_dict ? dj->body : nullptr;
    const int64_t ebase = is_dict ? dj->entry_base : 0;
    const int32_t *pids = ids + pg.ids_base;
    const int32_t *vs = vstart + pg.vs_base;
    uint8_t *payload = varlen ? (uint8_t *)out.data : nullptr;
    int carry_rank = 0;
    int64_t carry_bytes = pg.payload_base;
    for (int w0 = 0; w0 < n_words; w0 += kExpThreads) {
        // this thread's validity word, masked to the page's rows
        const int jw = w0 + tid;
        uint32_t bits = 0;
        if (jw < n_words) {
            const int64_t wrow = g0 + 32 * (int64_t)jw;
            const int lo = wrow < row0 ? (int)(row0 - wrow) : 0;
            const int64_t hi = pq_min64(32, row1 - wrow);
            const uint32_t mask = (hi >= 32 ? 0xffffffffu : ((1u << hi) - 1)) & ~((1u << lo) - 1);
            bits = out.validity ? (out.validity[wrow >> 5] & mask) : mask;
        }
        int tot = 0;
        const int excl = block_scan_excl(__popc(bits), s_ws, &tot);
        s_bits[tid] = bits;
        s_rank[tid] = carry_rank + excl;
        __syncthreads();
        const int nw = min(kExpThreads, n_words - w0);
        if (varlen && is_dict) {
            // dictionary strings: lengths per row -> offsets need a second scan level (bytes per word)
            for (int jj = warp; jj < nw; jj += kExpThreads / 32) {
                const uint32_t b = s_bits[jj];
                int len = 0;
                if ((b >> lane) & 1) len = dict_len[ebase + pids[s_rank[jj] + __popc(b & ((1u << lane) - 1))]];
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) len += __shfl_xor_sync(0xffffffffu, len, d);
                if (lane == 0) s_wlen[jj] = len;
            }
            __syncthreads();
            int wtot = 0;
            const int wl = tid < nw ? s_wlen[tid] : 0;
            const int wex = block_scan_excl(wl, s_ws, &wtot);
            s_wlen[tid] = wex;
            __syncthreads();
            for (int jj = warp; jj < nw; jj += kExpThreads / 32) {
                const uint32_t b = s_bits[jj];
                const int64_t row = g0 + 32 * (int64_t)(w0 + jj) + lane;
                const bool inpage = row >= row0 && row < row1;
                int len = 0;
                const uint8_t *src = nullptr;
                if ((b >> lane) & 1) {
                    const int id = pids[s_rank[jj] + __popc(b & ((1u << lane) - 1))];
                    len = dict_len[ebase + id];
                    src = dbody + dict_off[ebase + id];
                }
                const int incl = warp_scan_incl(len);
                const int64_t off = carry_bytes + s_wlen[jj] + incl - len;
                if (inpage) out.offsets[row] = (int32_t)off;
                // payload: 8 lanes per row, 4 rows at a time
                for (int r8 = 0; r8 < 32; r8 += 4) {
                    const int sl = r8 + (lane >> 3);
                    const int64_t o2 = __shfl_sync(0xffffffffu, off, sl);
                    const int l2 = __shfl_sync(0xffffffffu, len, sl);
                    const uint8_t *s2 = (const uint8_t *)__shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)src, sl);
                    for (int bb = lane & 7; bb < l2; bb += 8) payload[o2 + bb] = s2[bb];
                }
            }
            carry_bytes += wtot;
        } else {
            // every thread keeps kExpUnroll independent loads in flight (one validity word = one warp step; a warp
            // takes words warp, warp + 8, ...): with a single load per thread the 64 resident warps of an SM cover
            // ~8 KB of the ~40 KB that have to be in flight per SM to fill the HBM pipe.
            constexpr int kExpUnroll = 4, kStep = kExpThreads / 32;
            const int fmode = varlen ? 0 : pg.enc == ENC_RLE_BOOL ? 1 : ch.phys == pq::T_BOOLEAN ? 2 : is_dict ? 3 : 4;
            if (fmode == 4 && pw == 8 && out.out_width == 8 && ch.cast == 0) {
                // the common case (PLAIN INT64 / DOUBLE into an 8-byte column): two rows per lane and one 16-byte store,
                // a warp step covers two validity words; kPairUnroll steps in flight
                constexpr int kPairUnroll = 2;
                const int half = lane >> 4, p0 = 2 * (lane & 15);
                const uintptr_t a0 = (uintptr_t)values;
                const int sh = (int)(a0 & 7) * 8;
                const uint64_t *q0 = (const uint64_t *)(a0 & ~(uintptr_t)7);
                uint64_t *od = (uint64_t *)out.data;
                for (int j0 = 2 * warp; j0 < nw; j0 += 2 * kStep * kPairUnroll) {
                    int64_t row[kPairUnroll];
                    bool in0[kPairUnroll], in1[kPairUnroll];
                    uint64_t l0[kPairUnroll], h0[kPairUnroll], l1[kPairUnroll], h1[kPairUnroll];
#pragma unroll
                    for (int u = 0; u < kPairUnroll; u++) {
                        const int jj = j0 + 2 * kStep * u + half;
                        const uint32_t b = jj < nw ? s_bits[jj] : 0;
                        const int rk = jj < nw ? s_rank[jj] + __popc(b & ((1u << p0) - 1)) : 0;
                        const bool v0 = (b >> p0) & 1, v1 = (b >> (p0 + 1)) & 1;
                        row[u] = g0 + 32 * (int64_t)(w0 + jj) + p0;
                        in0[u] = jj < nw && row[u] >= row0 && row[u] < row1;
                        in1[u] = jj < nw && row[u] + 1 >= row0 && row[u] + 1 < row1;
                        const int r1 = rk + (v0 ? 1 : 0);
                        l0[u] = v0 ? q0[rk] : 0;                        // (bits outside the page are masked out above)
                        h0[u] = (v0 && sh) ? q0[rk + 1] : 0;
                        l1[u] = v1 ? q0[r1] : 0;
                        h1[u] = (v1 && sh) ? q0[r1 + 1] : 0;
                    }
#pragma unroll
                    for (int u = 0; u < kPairUnroll; u++) {
                        const uint64_t x0 = sh ? (l0[u] >> sh) | (h0[u] << (64 - sh)) : l0[u];
                        const uint64_t x1 = sh ? (l1[u] >> sh) | (h1[u] << (64 - sh)) : l1[u];
                        if (in0[u] && in1[u]) *(ulonglong2 *)(od + row[u]) = make_ulonglong2(x0, x1);
                        else if (in0[u]) od[row[u]] = x0;
                        else if (in1[u]) od[row[u] + 1] = x1;
                    }
                }
            } else
            for (int j0 = warp; j0 < nw; j0 += kStep * kExpUnroll) {
                int64_t row[kExpUnroll];
                int rank[kExpUnroll];
                bool inpage[kExpUnroll], valid[kExpUnroll];
#pragma unroll
                for (int u = 0; u < kExpUnroll; u++) {
                    const int jj = j0 + u * kStep;
                    const uint32_t b = jj < nw ? s_bits[jj] : 0;
                    row[u] = g0 + 32 * (int64_t)(w0 + jj) + lane;
                    inpage[u] = jj < nw && row[u] >= row0 && row[u] < row1;
                    valid[u] = (b >> lane) & 1;
                    rank[u] = jj < nw ? s_rank[jj] + __popc(b & ((1u << lane) - 1)) : 0;
                }
                if (fmode == 0) {
                    int32_t o[kExpUnroll];
#pragma unroll
                    for (int u = 0; u < kExpUnroll; u++) o[u] = inpage[u] ? vs[rank[u]] : 0;   // a NULL row starts where the next value starts
#pragma unroll
                    for (int u = 0; u < kExpUnroll; u++) if (inpage[u]) out.offsets[row[u]] = o[u];
                    continue;
                }
                uint64_t v[kExpUnroll];
                if (fmode == 4) {
                    if (pw == 8) {
                        const uintptr_t a0 = (uintptr_t)values;
                        const int sh = (int)(a0 & 7) * 8;
                        const uint64_t *q0 = (const uint64_t *)(a0 & ~(uintptr_t)7);
                        uint64_t lo[kExpUnroll], hi[kExpUnroll];
#pragma unroll
                        for (int u = 0; u < kExpUnroll; u++) {
                            const bool ld = inpage[u] && valid[u];
                            lo[u] = ld ? q0[rank[u]] : 0;
                            hi[u] = (ld && sh) ? q0[rank[u] + 1] : 0;
                        }
#pragma unroll
                        for (int u = 0; u < kExpUnroll; u++) v[u] = sh ? (lo[u] >> sh) | (hi[u] << (64 - sh)) : lo[u];
                    } else {
                        const uintptr_t a0 = (uintptr_t)values;
                        const int sh = (int)(a0 & 3) * 8;
                        const uint32_t *q0 = (const uint32_t *)(a0 & ~(uintptr_t)3);
                        uint32_t lo[kExpUnroll], hi[kExpUnroll];
#pragma unroll
                        for (int u = 0; u < kExpUnroll; u++) {
                            const bool ld = inpage[u] && valid[u];
                            lo[u] = ld ? q0[rank[u]] : 0;
                            hi[u] = (ld && sh) ? q0[rank[u] + 1] : 0;
                        }
#pragma unroll
                        for (int u = 0; u < kExpUnroll; u++) v[u] = __funnelshift_r(lo[u], hi[u], sh);
                    }
                } else if (fmode == 3) {
                    int32_t id[kExpUnroll];
#pragma unroll
                    for (int u = 0; u < kExpUnroll; u++) id[u] = (inpage[u] && valid[u]) ? pids[rank[u]] : -1;
#pragma unroll
                    for (int u = 0; u < kExpUnroll; u++) v[u] = id[u] >= 0 ? pq_load_unaligned(dbody + (int64_t)id[u] * pw, pw) : 0;
                } else {
#pragma unroll
                    for (int u = 0; u < kExpUnroll; u++) {
                        v[u] = 0;
                        if (inpage[u] && valid[u])
                            v[u] = fmode == 1 ? (uint64_t)(pids[rank[u]] & 1) : (uint64_t)((values[rank[u] >> 3] >> (rank[u] & 7)) & 1);
                    }
                }
#pragma unroll
                for (int u = 0; u < kExpUnroll; u++) {
                    if (!inpage[u]) continue;
                    uint64_t x = valid[u] ? v[u] : 0;
                    // a file written before the column was widened (SchemaEvolutionUtil / CastExecutors on the
                    // Java side, DataFileRecordReader.java:55-57): INT -> BIGINT, FLOAT -> DOUBLE are exact
                    if (valid[u] && ch.cast == 1) x = (uint64_t)(int64_t)(int32_t)(uint32_t)x;
                    else if (valid[u] && ch.cast == 2) x = (uint64_t)__double_as_longlong((double)__uint_as_float((uint32_t)x));
                    store_fixed(out.data, out.out_width, row[u], x);    // narrowing keeps the low bytes (INT32 -> TINYINT)
                }
            }
        }
        carry_rank += tot;
        __syncthreads();
    }
    if (varlen) {
        if constexpr (kPlainStrings) {
            auto &s_vs = stage.vs;
            auto &s_bnd = stage.bnd;
            auto &s_in = stage.in;
            auto &s_out = stage.out;
            // PLAIN: the page's payload is its value stream with the 4-byte length words squeezed out.  Batches of
            // kExpThreads values: the batch's stretch of the stream comes into shared memory with 16-byte async copies
            // (the NEXT batch is in flight while this one is worked on), every thread moves ONE value byte by byte
            // inside shared memory (all 32 lanes busy, no global latency), and the batch's contiguous output range
            // leaves with 16-byte stores.  (8 lanes per value straight on global memory spent many warp
            // instructions per value and stalled on the gathers.)  Batches that do not fit the staging buffers
            // (long values) and pages with more batches than the boundary table holds take the direct path.
            const int nnz = pg.nnz;
            const int64_t pb = pg.payload_base;
            const int nb = (nnz + kExpThreads - 1) / kExpThreads;
            const bool staged_page = nb <= kPayBatches;
            __syncthreads();
            if (staged_page) for (int i = tid; i <= nb; i += kExpThreads) s_bnd[i] = vs[min(i * kExpThreads, nnz)];
            __syncthreads();
            // batch b: values [b T, b T + jn), output bytes [s_bnd[b], s_bnd[b + 1]), stream bytes from value b T's length word
            auto batch_src = [&](int b2) -> const uint8_t * { return values + ((int64_t)s_bnd[b2] - pb) + 4 * (int64_t)b2 * kExpThreads; };
            auto batch_fits = [&](int b2) -> bool {
                const int jn = min(kExpThreads, nnz - b2 * kExpThreads);
                const int out_len = s_bnd[b2 + 1] - s_bnd[b2];
                const int iskew = (int)((uintptr_t)batch_src(b2) & 15), oskew = (int)((uintptr_t)(payload + s_bnd[b2]) & 15);
                return iskew + out_len + 4 * jn <= kPayIn && oskew + out_len <= kPayOut;
            };
            auto prefetch = [&](int b2) {
                const int jn = min(kExpThreads, nnz - b2 * kExpThreads);
                int *dv = s_vs[b2 & 1];
                for (int i = tid; i <= jn; i += kExpThreads) cp_async4(dv + i, vs + b2 * kExpThreads + i);
                if (batch_fits(b2)) {
                    const uint8_t *src0 = batch_src(b2);
                    const int iskew = (int)((uintptr_t)src0 & 15);
                    const int n16 = (iskew + (s_bnd[b2 + 1] - s_bnd[b2]) + 4 * jn + 15) >> 4;
                    uint8_t *di = s_in[b2 & 1];
                    for (int i = tid; i < n16; i += kExpThreads) cp_async16(di + 16 * i, src0 - iskew + 16 * i);   // (<= 15 bytes past the page)
                }
                cp_async_commit();
            };
            if (staged_page && nb > 0) prefetch(0);
            for (int b2 = 0; b2 < nb; b2++) {
                const int j0 = b2 * kExpThreads, jn = min(kExpThreads, nnz - j0);
                if (!staged_page) {
                    for (int t = tid >> 3; t < jn; t += kExpThreads / 8) {
                        const int st = vs[j0 + t], len = vs[j0 + t + 1] - st;
                        const uint8_t *src = values + ((int64_t)st - pb) + 4 * (int64_t)(j0 + t + 1);
                        for (int b3 = tid & 7; b3 < len; b3 += 8) payload[(int64_t)st + b3] = src[b3];
                    }
                    continue;
                }
                if (b2 + 1 < nb) { prefetch(b2 + 1); cp_async_wait<1>(); } else cp_async_wait<0>();
                __syncthreads();                                            // batch b2 has landed for every thread
                const int *cvs = s_vs[b2 & 1];
                const int out0 = s_bnd[b2], out_len = s_bnd[b2 + 1] - out0;
                if (batch_fits(b2)) {
                    const uint8_t *src0 = batch_src(b2);
                    const int iskew = (int)((uintptr_t)src0 & 15), oskew = (int)((uintptr_t)(payload + out0) & 15);
                    if (tid < jn) {
                        const int o = cvs[tid] - out0, len = cvs[tid + 1] - cvs[tid];
                        const uint8_t *sp = s_in[b2 & 1] + iskew + o + 4 * (tid + 1);
                        uint8_t *dp = s_out + oskew + o;
                        for (int b3 = 0; b3 < len; b3++) dp[b3] = sp[b3];
                    }
                    __syncthreads();
                    // s_out[oskew + i] is output byte out0 + i: whole 16-byte chunks as vectors, the edges byte-wise
                    uint8_t *dst16 = payload + out0 - oskew;                // 16-byte aligned
                    const int end = oskew + out_len;
                    for (int c = tid; c * 16 < end; c += kExpThreads) {
                        const int c0 = c * 16;
                        if (c0 >= oskew && c0 + 16 <= end) *(uint4 *)(dst16 + c0) = *(const uint4 *)(s_out + c0);
                        else for (int b3 = max(c0, oskew); b3 < min(c0 + 16, end); b3++) dst16[b3] = s_out[b3];
                    }
                } else {
                    for (int t = tid >> 3; t < jn; t += kExpThreads / 8) {
                        const int st = cvs[t], len = cvs[t + 1] - st;
                        const uint8_t *src = values + ((int64_t)st - pb) + 4 * (int64_t)(j0 + t + 1);
                        for (int b3 = tid & 7; b3 < len; b3 += 8) payload[(int64_t)st + b3] = src[b3];
                    }
                }
                __syncthreads();                                            // s_out / the buffers of batch b2 are free again
            }
        }
        if (pg.is_last && tid == 0) out.offsets[row1] = (int32_t)(pg.payload_base + pg.payload_bytes);
    }
}

// an empty run still needs offsets[0] = 0 for its var-len columns
__global__ void k_pq_zero_first_offset(const PqOut *outs, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && outs[i].offsets) outs[i].offsets[0] = 0;
}

// ------------------------------------------------------------------ host side

// ParquetSchemaConverter.java:76-160 — which physical type a Paimon column has in the file.  Returns the cast the
// decoder applies (0 = none), or -1 when the file type does not map to the read type.  Besides the exact mapping, the
// widenings Paimon's schema evolution allows without rewriting files are accepted: INT-family -> BIGINT, FLOAT -> DOUBLE.
static int phys_cast(int pg_t, int phys) {
    switch (pg_t) {
        case PG_INT8: case PG_INT16: case PG_INT32: return phys == pq::T_INT32 ? 0 : -1;
        case PG_INT64: return phys == pq::T_INT64 ? 0 : (phys == pq::T_INT32 ? 1 : -1);
        case PG_FLOAT: return phys == pq::T_FLOAT ? 0 : -1;
        case PG_DOUBLE: return phys == pq::T_DOUBLE ? 0 : (phys == pq::T_FLOAT ? 2 : -1);
        case PG_BOOL: return phys == pq::T_BOOLEAN ? 0 : -1;
        case PG_STRING: case PG_BINARY: return phys == pq::T_BYTE_ARRAY ? 0 : -1;
        default: return -1;
    }
}
static int phys_width_of(int phys) {
    return phys == pq::T_INT32 || phys == pq::T_FLOAT ? 4 : (phys == pq::T_INT64 || phys == pq::T_DOUBLE ? 8 : 0);
}

// A file of run `run` against the read schema [_KEY_*, _SEQUENCE_NUMBER, _VALUE_KIND, value...]: a flat schema, whose
// columns b.add_file resolves, with physical types that map to the read types and codecs the device decodes.
static pg_status map_file_schema(RunBuilder &b, const pq::FileMetaData &m, int run) {
    if (m.schema.empty()) return fail(PG_ERR_FORMAT, "parquet: empty schema");
    const int nleaf = (int)m.schema.size() - 1;
    if (m.schema[0].num_children != nleaf)
        return fail(PG_ERR_UNSUPPORTED, "parquet: nested columns are not decoded on device (flat KeyValue file schemas are)");
    std::vector<std::string> cols(nleaf);
    for (int i = 1; i <= nleaf; i++) {
        if (m.schema[i].num_children != 0 || m.schema[i].repetition == pq::R_REPEATED)
            return fail(PG_ERR_UNSUPPORTED, "parquet: nested / repeated column " + m.schema[i].name);
        cols[i - 1] = m.schema[i].name;
    }
    { pg_status st = b.add_file(run, m.num_rows, cols); if (st) return st; }
    for (int c = 0; c < b.nc; c++) {
        const int fc = b.file_col.back()[c];
        if (fc < 0) continue;
        const pq::SchemaElement &e = m.schema[fc + 1];
        if (phys_cast(b.schema->field(c).type, e.type) < 0)
            return fail(PG_ERR_UNSUPPORTED, "parquet: column " + e.name + " has a physical type the device decoder "
                                            "does not map to the table type");
    }
    for (const pq::RowGroup &g : m.row_groups) {
        if ((int)g.columns.size() != nleaf) return fail(PG_ERR_FORMAT, "parquet: row group with a different column count");
        for (const pq::ColumnChunk &cc : g.columns)
            if (cc.codec != pq::C_UNCOMPRESSED && cc.codec != pq::C_SNAPPY && cc.codec != pq::C_ZSTD && cc.codec != pq::C_GZIP &&
                cc.codec != pq::C_LZ4)
                return fail(PG_ERR_UNSUPPORTED, "parquet: compression codec " + std::to_string(cc.codec) +
                                                " is not decoded on device (UNCOMPRESSED, SNAPPY, ZSTD, GZIP and Hadoop-framed LZ4 = 5 are); write with "
                                                "'file.compression'='zstd' / 'snappy' / 'gzip' / 'lz4' / 'none' or let the Java side decompress");
    }
    return PG_OK;
}

// the chunk table, ordered (run, column, file, row group) so that the pages of a (run, column) end up contiguous, and
// the (run, var-len column) pairs
struct ChunkTables {
    std::vector<PqChunk> chunks;
    std::vector<PqPair> pairs;
    bool any_snappy = false, any_lz4 = false, any_delta = false, any_zstd = false;
    int64_t pair_rows = 0;
};

static pg_status build_chunk_tables(const Schema *s, const pg_file_desc *files, const std::vector<const uint8_t *> &d_file,
                                    const std::vector<const pq::FileMetaData *> &meta, const RunBuilder &b, ChunkTables &t) {
    const int nc = s->n_cols();
    const int n_runs = (int)b.run_rows.size();
    std::vector<std::vector<int>> run_files(n_runs);
    for (int f = 0; f < (int)meta.size(); f++) run_files[files[f].run].push_back(f);
    for (int r = 0; r < n_runs; r++) {
        for (int c = 0; c < nc; c++) {
            if (!b.read[c]) continue;
            const int chunk0 = (int)t.chunks.size();
            for (int f : run_files[r]) {
                const pq::FileMetaData &m = *meta[f];
                const int fc = b.file_col[f][c];
                int64_t rg_row0 = 0;
                int64_t rows = 0;
                if (fc < 0) continue;
                for (const pq::RowGroup &g : m.row_groups) {
                    const pq::ColumnChunk &cc = g.columns[fc];
                    const int64_t start = cc.start();
                    if (cc.num_values != g.num_rows) return fail(PG_ERR_FORMAT, "parquet: page row counts do not add up");
                    if (cc.num_values == 0) continue;            // an empty row group has no pages (and no valid offsets)
                    if (start < 4 || start >= files[f].size) return fail(PG_ERR_FORMAT, "parquet: page offset out of range");
                    PqChunk ch;
                    memset(&ch, 0, sizeof(ch));
                    ch.base = d_file[f] + start;
                    ch.avail = std::min<int64_t>(cc.total_compressed_size > 0 ? cc.total_compressed_size : files[f].size,
                                                 files[f].size - start);
                    ch.num_values = cc.num_values;
                    ch.row0 = b.file_row0[f] + rg_row0;
                    ch.col = c; ch.run = r; ch.file = f; ch.codec = cc.codec;
                    ch.max_def = m.schema[fc + 1].repetition == pq::R_OPTIONAL ? 1 : 0;
                    ch.phys = cc.type;
                    ch.phys_width = phys_width_of(cc.type);
                    ch.cast = phys_cast(s->field(c).type, cc.type);
                    if (cc.type != m.schema[fc + 1].type) return fail(PG_ERR_FORMAT, "parquet: column chunk type differs from the schema");
                    if (cc.codec == pq::C_SNAPPY) t.any_snappy = true;
                    if (cc.codec == pq::C_LZ4) t.any_lz4 = true;
                    if (cc.codec == pq::C_ZSTD || cc.codec == pq::C_GZIP) t.any_zstd = true;
                    for (int32_t e : cc.encodings) if (e == pq::E_DELTA_BINARY_PACKED) t.any_delta = true;
                    if (cc.num_values > 0) t.chunks.push_back(ch);
                    rg_row0 += g.num_rows;
                    rows += g.num_rows;
                }
                if (rows != m.num_rows) return fail(PG_ERR_FORMAT, "parquet: row group row counts do not add up");
            }
            if (is_varlen(s->field(c).type)) {
                PqPair pr{r, c, chunk0, (int)t.chunks.size(), t.pair_rows, (int)t.pairs.size(), 0};
                t.pairs.push_back(pr);
                t.pair_rows += b.run_rows[r];
            }
        }
    }
    return PG_OK;
}

#ifdef PG_WALK_TIMING
// prints the sampled warps' split (synchronises: a timing build only) and clears the samples
static void walk_timing_dump() {
    static long long h[kWtSlots][8];
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(h, g_walk_ts, sizeof(h));
    double acc[3] = {0, 0, 0}, steps = 0, vals = 0, steps_max = 0;
    long long g_lo = LLONG_MAX, g_hi = 0;
    int n = 0;
    for (int s = 0; s < kWtSlots; s++) {
        if (h[s][4] == 0) continue;
        n++;
        for (int k = 0; k < 3; k++) acc[k] += (double)h[s][k];
        steps += (double)h[s][3];
        steps_max = std::max(steps_max, (double)h[s][3]);
        vals += (double)h[s][4];
        g_lo = std::min(g_lo, h[s][5]);
        g_hi = std::max(g_hi, h[s][6]);
    }
    if (n == 0) return;
    const double tot = acc[0] + acc[1] + acc[2];
    fprintf(stderr, "[walk timing] %d warps: cycles per step issue %.0f wait %.0f walk %.0f (%.1f / %.1f / %.1f %%); "
                    "steps per warp %.1f (max %.0f), values per lane-step %.2f, span %.3f ms\n",
            n, acc[0] / steps, acc[1] / steps, acc[2] / steps, 100 * acc[0] / tot, 100 * acc[1] / tot, 100 * acc[2] / tot,
            steps / n, steps_max, vals / (32.0 * steps), (g_hi - g_lo) * 1e-6);
    // start times in tenths of the span: how the CTAs fall into waves
    int hist[10] = {0};
    double busy = 0;
    for (int s = 0; s < kWtSlots; s++) {
        if (h[s][4] == 0) continue;
        hist[std::min(9, (int)(10.0 * (h[s][5] - g_lo) / (double)(g_hi - g_lo + 1)))]++;
        busy += (double)(h[s][6] - h[s][5]);
    }
    fprintf(stderr, "[walk timing] warp start by tenth of the span:");
    for (int i = 0; i < 10; i++) fprintf(stderr, " %d", hist[i]);
    fprintf(stderr, "; mean warp lifetime %.3f ms\n", busy / n * 1e-6);
    static long long z[kWtSlots][8];
    cudaMemcpyToSymbol(g_walk_ts, z, sizeof(z));
}
#endif

// The side stream of the calling thread's decodes, and its fork / join events.  Highest priority: the value walk's few,
// long-running CTAs must get their slots before the expansion's 250 k short ones fill every SM — otherwise the walk
// only starts when the expansion drains.
struct SideStream {
    cudaStream_t s = nullptr;
    cudaEvent_t fork = nullptr, tables = nullptr, join = nullptr;
};
static pg_status side_stream(SideStream **out) {
    static thread_local SideStream side;
    if (!side.s) {
        int prio_lo = 0, prio_hi = 0;
        cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
        PG_CUDA(cudaStreamCreateWithPriority(&side.s, cudaStreamNonBlocking, prio_hi));
        PG_CUDA(cudaEventCreateWithFlags(&side.fork, cudaEventDisableTiming));
        PG_CUDA(cudaEventCreateWithFlags(&side.tables, cudaEventDisableTiming));
        PG_CUDA(cudaEventCreateWithFlags(&side.join, cudaEventDisableTiming));
    }
    *out = &side;
    return PG_OK;
}

// Synchronises the side stream when a decode returns, before the frame's Scratch synchronises the main stream and
// gives the buffers back: an error found by read-back 2 returns while the value walk may still run there.
struct SideSync {
    cudaStream_t s = nullptr;
    ~SideSync() { if (s) cudaStreamSynchronize(s); }
};

// footer0: the footer of files[0], already parsed (the single-file reader), or NULL
static pg_status decode_section(const std::shared_ptr<const Schema> &s, const pg_file_desc *files, int nf, int n_runs,
                                const char *const *names, const uint8_t *read_cols, uint64_t *out_runs,
                                pg_section_info *info, const pq::FileMetaData *footer0 = nullptr) {
    const int nc = s->n_cols();
    SectionFrame fr(s, n_runs, "parquet");
    SideSync side_sync;                                  // (destroyed before fr: the side stream first)
    PG_HOST_MARKS("parquet decode_section");
    RunBuilder &b = fr.b;
    cudaStream_t sm = fr.stream;
    { pg_status st = fr.start(read_cols, names); if (st) return st; }

    // ---- file bytes on the device, footers on the host (those of device-resident files through small reads)
    { pg_status st = fr.place(files, nf); if (st) return st; }
    std::vector<pq::FileMetaData> own_meta(nf);
    std::vector<const pq::FileMetaData *> meta(nf, nullptr);
    if (footer0) meta[0] = footer0;
    DeviceRanges rd(sm, files, nf);
    try {
        if (!rd.files.empty()) {
            std::vector<pq::FileMetaData> m = pq::read_footers(rd, rd.sizes);
            for (size_t i = 0; i < rd.files.size(); i++) own_meta[rd.files[i]] = std::move(m[i]);
        }
        for (int f = 0; f < nf; f++) {
            if (meta[f]) continue;
            if (files[f].mem == PG_MEM_HOST) own_meta[f] = pq::parse_footer(files[f].bytes, files[f].size);
            meta[f] = &own_meta[f];
        }
    } catch (const std::exception &e) {
        return rd.st ? rd.st : fail(PG_ERR_FORMAT, e.what());
    }
    PG_HOST_MARK("footers");
    std::vector<uint8_t> any_optional(nc, 0);
    for (int f = 0; f < nf; f++) {
        pg_status st = map_file_schema(b, *meta[f], files[f].run);
        if (st) return st;
        for (int c = 0; c < nc; c++) {
            const int fc = b.file_col[f][c];
            if (fc == -1 || (fc >= 0 && meta[f]->schema[fc + 1].repetition == pq::R_OPTIONAL)) any_optional[c] = 1;
        }
    }
    { pg_status st = b.check_runs(); if (st) return st; }
    ChunkTables ct;
    { pg_status st = build_chunk_tables(s.get(), files, fr.d_file, meta, b, ct); if (st) return st; }
    const int n_chunks = (int)ct.chunks.size(), n_pairs = (int)ct.pairs.size();
    PG_HOST_MARK("chunk_tables");

    // ---- output columns (the rows of files that lack a column stay NULL and get defined contents)
    { pg_status st = b.alloc(any_optional, b.missing); if (st) return st; }
    std::vector<PqOut> outs((size_t)n_runs * nc);
    auto fill_outs = [&] {
        for (size_t i = 0; i < outs.size(); i++) {
            const int t = s->field((int)(i % nc)).type;
            outs[i] = PqOut{b.out[i].data, b.out[i].offsets, b.out[i].validity, type_width(t), t == PG_BOOL};
        }
    };
    fill_outs();
    const bool any_empty = std::find(b.run_rows.begin(), b.run_rows.end(), 0) != b.run_rows.end();

    // ---- tables to the device, page count pass
    // (two output tables: the second one adds the var-len payload pointers, known only after read-back 2)
    PqChunk *d_chunks;
    PqOut *d_outs, *d_outs2;
    PqPair *d_pairs;
    int64_t *d_totals;               // [0..5] chunk totals, [6] error word, [7] zstd ticket, [8..] pair totals
    auto carve_tables = [&](void *base) {
        Carver cv(base);
        d_chunks = cv.take<PqChunk>((size_t)std::max(n_chunks, 1));
        d_outs = cv.take<PqOut>(outs.size());
        d_outs2 = cv.take<PqOut>(outs.size());
        d_pairs = cv.take<PqPair>((size_t)std::max(n_pairs, 1));
        d_totals = cv.take<int64_t>(8 + (size_t)n_pairs);
        return cv.bytes();
    };
    const size_t tb_bytes = carve_tables(nullptr);
    void *tb = fr.scratch.take(tb_bytes);
    if (!tb) return oom("parquet", "the chunk tables", tb_bytes);
    carve_tables(tb);
    int32_t *d_err = (int32_t *)(d_totals + 6);
    PG_CUDA(cudaMemsetAsync(d_totals, 0, sizeof(int64_t) * (8 + (size_t)n_pairs), sm));
    // (tables go through small_h2d: a kernel reads them out of mapped host memory, so they do not queue behind an
    // asynchronous upload of the next section on the copy engine)
    if (n_chunks) { pg_status ts = small_h2d(d_chunks, ct.chunks.data(), sizeof(PqChunk) * n_chunks, sm); if (ts) return ts; }
    { pg_status ts = small_h2d(d_outs, outs.data(), sizeof(PqOut) * outs.size(), sm); if (ts) return ts; }
    if (n_pairs) { pg_status ts = small_h2d(d_pairs, ct.pairs.data(), sizeof(PqPair) * n_pairs, sm); if (ts) return ts; }
    int64_t h_tot[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    PG_HOST_MARK("tables");
    if (n_chunks) {
        k_pq_walk<false><<<(n_chunks + 63) / 64, 64, 0, sm>>>(d_chunks, n_chunks, nullptr, nullptr, nullptr, d_err);
        k_pq_chunk_scan<<<1, kScanThreads, 0, sm>>>(d_chunks, n_chunks, d_totals);
        fr.launches += 2;
        {
            SmallReads rb(sm);                           // read-back 1: how many pages the section has
            pg_status rs = rb.add(h_tot, d_totals, sizeof(int64_t) * 8);
            if (!rs) rs = rb.finish();
            if (!rs) rs = kernel_error((int)(h_tot[6] & 0xffffffff), "parquet");
            if (rs) return rs;
        }
    }
    const int64_t n_pages = h_tot[0], n_dicts = h_tot[1], sc_bytes = h_tot[2], dict_entries = h_tot[3],
                  ids_entries = h_tot[4];
    fr.page_bytes = h_tot[5];
    PG_HOST_MARK("readback1");
    if (n_pages > 0x7fffffffLL) return fail(PG_ERR_UNSUPPORTED, "parquet: too many pages in one section");

    // ---- page table + scratch, fill pass, inflate
    int zs_ctas = 0;
    if (ct.any_zstd) {
        int dev = 0, sms = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        zs_ctas = (int)std::min<int64_t>((int64_t)sms * 5, (n_pages + n_dicts + kZsWarps - 1) / kZsWarps);
    }
    PqPage *d_pages, *d_dicts;
    uint8_t *d_sc, *d_zs_lit;
    int32_t *d_dict_off, *d_dict_len, *d_ids, *d_vstart;
    auto carve_pages = [&](void *base) {
        Carver cv(base);
        d_pages = cv.take<PqPage>((size_t)std::max<int64_t>(n_pages, 1));
        d_dicts = cv.take<PqPage>((size_t)std::max<int64_t>(n_dicts, 1));
        d_sc = cv.take<uint8_t>((size_t)sc_bytes + kReadPast);
        d_dict_off = cv.take<int32_t>((size_t)dict_entries + 1);
        d_dict_len = cv.take<int32_t>((size_t)dict_entries + 1);
        d_ids = cv.take<int32_t>((size_t)ids_entries + 1);
        d_vstart = cv.take<int32_t>((size_t)(ct.pair_rows + n_pages + n_pairs + 2));
        d_zs_lit = cv.take<uint8_t>((size_t)zs_ctas * kZsWarps * (size_t)(zs::kMaxBlock + 64));
        return cv.bytes();
    };
    const size_t sb_bytes = carve_pages(nullptr);
    void *sbuf = fr.scratch.take(sb_bytes);
    if (!sbuf) return oom("parquet", "the page table and scratch", sb_bytes);
    carve_pages(sbuf);
    const int np = (int)n_pages, nd = (int)n_dicts;
    std::vector<int64_t> pair_tot(std::max(n_pairs, 1), 0);
    if (np > 0) {
        k_pq_walk<true><<<(n_chunks + 63) / 64, 64, 0, sm>>>(d_chunks, n_chunks, d_pages, d_dicts, d_sc, d_err);
        fr.launches++;
        if (ct.any_snappy || ct.any_lz4) {
            const int64_t th = (int64_t)(np + nd) * 32;
            k_pq_snappy_lz4<<<(unsigned)((th + 127) / 128), 128, 0, sm>>>(d_pages, np, d_dicts, nd, d_chunks, d_err);
            fr.launches++;
        }
        if (ct.any_zstd && zs_ctas > 0) {
            k_pq_zstd<<<zs_ctas, kZsWarps * 32, 0, sm>>>(d_pages, np, d_dicts, nd, d_chunks, d_zs_lit, (int32_t *)(d_totals + 7), d_err);
            fr.launches++;
        }
        if (ct.any_delta) {
            k_pq_delta<<<(unsigned)(((int64_t)np * 32 + 127) / 128), 128, 0, sm>>>(d_pages, np, d_chunks, d_err);
            fr.launches++;
        }
        if (dict_entries > 0) {
            k_pq_walk_dicts<<<(nd + kWalkWarps - 1) / kWalkWarps, kWalkWarps * 32, 0, sm>>>(
                d_dicts, nd, d_chunks, d_dict_off, d_dict_len, d_err);
            fr.launches++;
        }
        k_pq_levels<<<(unsigned)(((int64_t)np * 32 + 127) / 128), 128, 0, sm>>>(d_pages, np, d_dicts, d_chunks, d_outs, nc,
                                                                            d_ids, d_dict_len, d_err);
        fr.launches++;
        if (n_pairs) {
            k_pq_scan_pages<<<(n_pairs * 32 + 127) / 128, 128, 0, sm>>>(d_pages, d_chunks, d_pairs, n_pairs, d_totals + 8, d_err);
            fr.launches++;
        }
    }

    // ---- the value walk and the expansion.  With var-len columns the value walk (one lane per page: latency-bound at
    // low occupancy) and the PLAIN BYTE_ARRAY pages that need it run on a side stream beside the expansion of all other
    // pages.  Read-back 2 (the exact payload sizes) is issued first, and the walk and the main-stream expansion are
    // enqueued before the host waits for it: neither needs the payload buffers, so the device keeps working through
    // the wait, the payload allocation and the upload of the second output table.  Only dictionary-encoded strings,
    // which the main-stream expansion copies, make it wait for the payload buffers.
    if (n_pairs == 0) {
        if (np > 0) {
            k_pq_expand<false><<<np, kExpThreads, 0, sm>>>(d_pages, d_dicts, d_chunks, d_outs, nc, d_ids, d_vstart,
                                                           d_dict_off, d_dict_len);
            fr.launches++;
        }
    } else {
        SmallReads rb(sm);                               // read-back 2: exact payload sizes of the var-len columns
        pg_status rs = rb.add(pair_tot.data(), d_totals + 8, sizeof(int64_t) * n_pairs);
        if (!rs) rs = rb.add(h_tot, d_totals, sizeof(int64_t) * 8);
        if (rs) return rs;
        SideStream *side = nullptr;
        { pg_status st = side_stream(&side); if (st) return st; }
        side_sync.s = side->s;
        PG_CUDA(cudaEventRecord(side->fork, sm));        // (behind read-back 2: its event)
        const bool main_early = dict_entries == 0;
        if (np > 0) {
            PG_CUDA(cudaStreamWaitEvent(side->s, side->fork, 0));
            k_pq_walk_values<<<(np + kWvWarps * 32 - 1) / (kWvWarps * 32), kWvWarps * 32, 0, side->s>>>(
                d_pages, np, d_chunks, d_vstart, d_err);
            fr.launches++;
            if (main_early) {
                k_pq_expand<false><<<np, kExpThreads, 0, sm>>>(d_pages, d_dicts, d_chunks, d_outs, nc, d_ids, d_vstart,
                                                               d_dict_off, d_dict_len);
                fr.launches++;
            }
        }
        PG_HOST_MARK("enqueue");
        rs = rb.finish(side->fork);
        if (!rs) rs = kernel_error((int)(h_tot[6] & 0xffffffff), "parquet");
        if (rs) return rs;
        PG_HOST_MARK("readback2");
        // ---- var-len payload buffers (one per run), in a second output table: the first one is being read
        std::vector<int64_t> payload((size_t)n_runs * nc, 0);
        for (const PqPair &pr : ct.pairs) payload[(size_t)pr.run * nc + pr.col] = pair_tot[pr.idx];
        { pg_status st = b.alloc_payload(payload); if (st) return st; }
        fill_outs();
        if (main_early) {
            pg_status ts = small_h2d(d_outs2, outs.data(), sizeof(PqOut) * outs.size(), side->s);
            if (ts) return ts;
        } else {
            pg_status ts = small_h2d(d_outs2, outs.data(), sizeof(PqOut) * outs.size(), sm);
            if (ts) return ts;
            PG_CUDA(cudaEventRecord(side->tables, sm));
            PG_CUDA(cudaStreamWaitEvent(side->s, side->tables, 0));
            if (np > 0) {
                k_pq_expand<false><<<np, kExpThreads, 0, sm>>>(d_pages, d_dicts, d_chunks, d_outs2, nc, d_ids, d_vstart,
                                                               d_dict_off, d_dict_len);
                fr.launches++;
            }
        }
        if (np > 0) {
            // the PLAIN BYTE_ARRAY pages follow their walk on the side stream
            k_pq_expand<true><<<np, kExpThreads, 0, side->s>>>(d_pages, d_dicts, d_chunks, d_outs2, nc, d_ids, d_vstart,
                                                               d_dict_off, d_dict_len);
            fr.launches++;
        }
        PG_CUDA(cudaEventRecord(side->join, side->s));
        PG_CUDA(cudaStreamWaitEvent(sm, side->join, 0));
#ifdef PG_WALK_TIMING
        if (np > 0) walk_timing_dump();
#endif
        PG_HOST_MARK("payload");
    }
    if (any_empty && n_pairs) {
        k_pq_zero_first_offset<<<(n_runs * nc + 127) / 128, 128, 0, sm>>>(d_outs, n_runs * nc);
        fr.launches++;
    }
    // (the parsed footers go while the expansions run, not between the decode and the merge that follows it)
    meta.clear();
    std::vector<pq::FileMetaData>().swap(own_meta);
    { pg_status st = fr.finish(d_err, out_runs, info); if (st) return st; }
    if (info) {
        info->n_chunks = n_chunks;
        info->n_data_pages = np;
        info->n_dictionary_pages = nd;
    }
    return PG_OK;
}

// ---- the single-file reader (FormatReaderFactory.createReader + readBatch): a section of one file

struct PqReader {
    std::shared_ptr<const Schema> schema;
    pq::FileMetaData meta;
    std::vector<uint8_t> file;             // host copy: pg_parquet_open's caller may free its buffer
    int64_t n_rows = 0;
    int n_data_pages = 0, n_dict_pages = 0;
    float ms_decode = 0;
    int launches = 0;
};

static Table<PqReader> g_pq(5);

// open = footer + schema check + the page walk's count pass on the host, so that files the device walk would refuse
// are refused here, before any device work (and on a box without a GPU)
static pg_status pq_open(uint64_t schema, const uint8_t *bytes, int64_t size, uint64_t *out) {
    std::shared_ptr<Schema> s = g_schemas.get(schema);
    if (!s || !bytes || !out) return fail(PG_ERR_INVALID, "bad schema handle or null argument");
    auto rd = std::make_unique<PqReader>();
    rd->schema = s;
    try {
        rd->meta = pq::parse_footer(bytes, size);
    } catch (const std::exception &e) {
        return fail(PG_ERR_FORMAT, e.what());
    }
    Scratch scratch(nullptr);                          // (stays empty: the columns are resolved by position on the host)
    RunBuilder b(s, 1, scratch, "parquet");
    pg_status st = map_file_schema(b, rd->meta, 0);
    if (st) return st;
    // the chunk table and the count pass of the section decode, over the host bytes
    const pg_file_desc file{bytes, size, PG_MEM_HOST, 0};
    ChunkTables ct;
    st = build_chunk_tables(s.get(), &file, {bytes}, {&rd->meta}, b, ct);
    if (st) return st;
    for (int c = 0; c < (int)ct.chunks.size(); c++) {
        st = kernel_error(pq_walk_chunk<false>(ct.chunks.data(), c, nullptr, nullptr, nullptr), "parquet");
        if (st) return st;
        rd->n_data_pages += ct.chunks[c].n_pages;
        rd->n_dict_pages += ct.chunks[c].n_dicts;
    }
    rd->n_rows = rd->meta.num_rows;
    rd->file.assign(bytes, bytes + size);
    *out = g_pq.put(std::move(rd));
    return PG_OK;
}

static pg_status pq_read_run(PqReader *rd, uint64_t *out_run) {
    const pg_file_desc file{rd->file.data(), (int64_t)rd->file.size(), PG_MEM_HOST, 0};
    pg_section_info info;
    pg_status st = decode_section(rd->schema, &file, 1, 1, nullptr, nullptr, out_run, &info, &rd->meta);
    if (st) return st;
    rd->ms_decode = info.ms_decode;
    rd->launches = info.launches;
    return PG_OK;
}


// ------------------------------------------------------------------ deletion vectors
//
// ApplyDeletionVectorReader (paimon-core/.../deletionvectors/ApplyDeletionVectorReader.java:31-54) skips the rows of
// a data file whose position is marked in the file's deletion vector.  Here: a device run minus the marked rows.

__global__ void k_dv_keep(const uint8_t *deleted, int64_t n_bits, int64_t n, int32_t *keep) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool del = i < n_bits && ((deleted[i >> 3] >> (i & 7)) & 1);
    keep[i] = del ? 0 : 1;
}
// src[j] = input row of output row j (incl = inclusive scan of keep)
__global__ void k_dv_sources(const int32_t *incl, int64_t n, int32_t *src) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t cur = incl[i], prev = i ? incl[i - 1] : 0;
    if (cur != prev) src[cur - 1] = (int32_t)i;
}
__global__ void k_dv_gather_fixed(const void *in, int width, const int32_t *src, int64_t m, void *out) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    store_fixed(out, width, j, load_fixed(in, width, src[j]));
}
__global__ void k_dv_gather_bits(const uint8_t *in, const int32_t *src, int64_t m, uint32_t *out) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool v = j < m && valid_bit(in, src[j]);
    const unsigned w = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && j < m) out[j >> 5] = w;
}
__global__ void k_dv_lengths(const int32_t *offs, const int32_t *src, int64_t m, int32_t *out_offsets) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j == 0) out_offsets[0] = 0;
    if (j >= m) return;
    out_offsets[1 + j] = offs[src[j] + 1] - offs[src[j]];
}
__global__ void k_dv_copy_bytes(const uint8_t *data, const int32_t *offs, const int32_t *src, const int32_t *out_offsets,
                                uint8_t *out, int64_t m) {
    int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    if (row >= m) return;
    const uint8_t *s = data + offs[src[row]];
    const int o0 = out_offsets[row], o1 = out_offsets[row + 1];
    for (int b = o0 + (threadIdx.x & 7); b < o1; b += 8) out[b] = s[b - o0];
}

static pg_status apply_deletion_vector(uint64_t run_h, const uint8_t *deleted, int64_t n_bits, uint64_t *out_run) {
    std::shared_ptr<Run> in = g_runs.get(run_h);
    if (!in || !out_run || (n_bits > 0 && !deleted)) return fail(PG_ERR_INVALID, "unknown run handle or null argument");
    pg_status st = ensure_device();
    if (st) return st;
    const Schema *s = in->schema.get();
    const int nc = s->n_cols();
    const int64_t n = in->n_rows;
    if (n_bits < 0) return fail(PG_ERR_INVALID, "negative deletion vector size");
    cudaStream_t sm = 0;
    Scratch scratch(sm);                               // temporaries, and the new run until it is registered
    // ---- kept rows
    const int64_t nb = std::max<int64_t>((n + 4095) / 4096, 1);
    uint8_t *d_del = (uint8_t *)scratch.take((size_t)(n_bits + 7) / 8 + 16);
    int32_t *d_incl = (int32_t *)scratch.take(sizeof(int32_t) * (size_t)(n + 1));
    int64_t *d_sums = (int64_t *)scratch.take(sizeof(int64_t) * (size_t)nb);     // (also the offsets scans: m <= n)
    int32_t *d_err = (int32_t *)scratch.take(16);
    if (!d_del || !d_incl || !d_sums || !d_err) return oom("deletion vector", "the row scan", sizeof(int32_t) * (size_t)n);
    PG_CUDA(cudaMemsetAsync(d_err, 0, 4, sm));
    if (n_bits > 0) PG_CUDA(cudaMemcpyAsync(d_del, deleted, (size_t)(n_bits + 7) / 8, cudaMemcpyHostToDevice, sm));
    int64_t m = 0;
    if (n > 0) {
        k_dv_keep<<<(int)((n + 255) / 256), 256, 0, sm>>>(d_del, n_bits, n, d_incl);
        launch_inclusive_scan(d_incl, n, d_sums, d_err, sm);
        int32_t last = 0;
        PG_CUDA(cudaMemcpyAsync(&last, d_incl + n - 1, 4, cudaMemcpyDeviceToHost, sm));
        PG_CUDA(cudaStreamSynchronize(sm));
        m = last;
    }
    int32_t *d_src = (int32_t *)scratch.take(sizeof(int32_t) * (size_t)std::max<int64_t>(m, 1));
    if (!d_src) return oom("deletion vector", "the row sources", sizeof(int32_t) * (size_t)m);
    if (n > 0) k_dv_sources<<<(int)((n + 255) / 256), 256, 0, sm>>>(d_incl, n, d_src);
    // ---- the kept rows of the columns the input has, with the bitmaps the input has
    RunBuilder b(in->schema, 1, scratch, "deletion vector");
    b.place_file(0, m);
    std::vector<uint8_t> bitmap(nc), no_zero(nc, 0);
    for (int c = 0; c < nc; c++) {
        b.read[c] = in->cols[c].data || in->cols[c].offsets;
        bitmap[c] = in->cols[c].validity != nullptr;
    }
    st = b.alloc(bitmap, no_zero);
    if (st) return st;
    const int gm = (int)((std::max<int64_t>(m, 1) + 255) / 256);
    for (int c = 0; c < nc; c++) {
        if (!b.read[c]) continue;
        const DevColumn &ic = in->cols[c];
        const OutColumn &oc = b.out[c];
        if (oc.validity && m > 0) k_dv_gather_bits<<<gm, 256, 0, sm>>>(ic.validity, d_src, m, oc.validity);
        if (!is_varlen(s->field(c).type)) {
            if (m > 0) k_dv_gather_fixed<<<gm, 256, 0, sm>>>(ic.data, type_width(s->field(c).type), d_src, m, oc.data);
        } else {
            k_dv_lengths<<<gm, 256, 0, sm>>>(ic.offsets, d_src, m, oc.offsets);
            launch_offsets_scan(oc.offsets, m, d_sums, d_err, sm);
        }
    }
    // payload sizes: one read-back for all var-len columns
    std::vector<int32_t> totals(nc, 0);
    for (int c = 0; c < nc; c++)
        if (b.out[c].offsets && m > 0)
            PG_CUDA(cudaMemcpyAsync(&totals[c], b.out[c].offsets + m, 4, cudaMemcpyDeviceToHost, sm));
    int32_t herr = 0;
    PG_CUDA(cudaMemcpyAsync(&herr, d_err, 4, cudaMemcpyDeviceToHost, sm));
    PG_CUDA(cudaStreamSynchronize(sm));
    st = b.alloc_payload(std::vector<int64_t>(totals.begin(), totals.end()));
    if (st) return st;
    for (int c = 0; c < nc; c++)
        if (b.out[c].offsets && m > 0)
            k_dv_copy_bytes<<<(int)((m * 8 + 255) / 256), 256, 0, sm>>>((const uint8_t *)in->cols[c].data, in->cols[c].offsets,
                                                                        d_src, b.out[c].offsets, (uint8_t *)b.out[c].data, m);
    PG_CUDA(cudaStreamSynchronize(sm));
    PG_CUDA(cudaGetLastError());
    st = kernel_error(herr, "deletion vector");
    if (st) return st;
    b.finish(out_run, 0, nullptr);
    return PG_OK;
}


}  // namespace pg

using namespace pg;

extern "C" {

pg_status pg_parquet_open(uint64_t schema, const uint8_t *file_bytes, int64_t size, uint64_t *out_reader) {
    return pq_open(schema, file_bytes, size, out_reader);
}

pg_status pg_parquet_describe(uint64_t reader, pg_parquet_info *out) {
    std::shared_ptr<PqReader> rd = g_pq.get(reader);
    if (!rd || !out) return fail(PG_ERR_INVALID, "unknown parquet reader handle");
    out->n_rows = rd->n_rows;
    out->n_row_groups = (int32_t)rd->meta.row_groups.size();
    out->n_columns = rd->schema->n_cols();
    out->n_data_pages = rd->n_data_pages;
    out->n_dictionary_pages = rd->n_dict_pages;
    out->ms_decode = rd->ms_decode;
    out->launches = rd->launches;
    return PG_OK;
}

pg_status pg_parquet_read_run(uint64_t reader, uint64_t *out_run) {
    std::shared_ptr<PqReader> rd = g_pq.get(reader);
    if (!rd || !out_run) return fail(PG_ERR_INVALID, "unknown parquet reader handle");
    pg_status st = ensure_device();           // fails loudly without pg_init / a CUDA device: no CPU fallback
    if (st) return st;
    return pq_read_run(rd.get(), out_run);
}

pg_status pg_parquet_read_section(uint64_t schema, const pg_file_desc *files, int32_t n_files, int32_t n_runs,
                                  const char *const *column_names, const uint8_t *read_columns, uint64_t *out_runs,
                                  pg_section_info *info) {
    std::shared_ptr<const Schema> s;
    pg_status st = check_section_args(schema, files, n_files, n_runs, out_runs, &s);
    if (st || n_runs == 0) return st;
    st = ensure_device();
    if (st) return st;
    return decode_section(s, files, n_files, n_runs, column_names, read_columns, out_runs, info);
}

pg_status pg_run_apply_deletion_vector(uint64_t run, const uint8_t *deleted_bitmap, int64_t n_bits, uint64_t *out_run) {
    return apply_deletion_vector(run, deleted_bitmap, n_bits, out_run);
}

pg_status pg_parquet_free(uint64_t reader) {
    return g_pq.take(reader) ? PG_OK : fail(PG_ERR_INVALID, "unknown parquet reader handle");
}

}  // extern "C"
