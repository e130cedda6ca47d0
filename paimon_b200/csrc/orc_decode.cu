// orc_decode.cu — ORC stripe decode on the device behind the same format seam as the Parquet decoder
// (SURVEY.md §8 rows a25 / f3).
//
// Reference being replaced: paimon-format/src/main/java/org/apache/paimon/format/orc/OrcReaderFactory.java:98-163
// (createReader: orc-core RecordReader over the projected TypeDescription, batches of VectorizedRowBatch) and the
// vector adapters in orc/reader/*; the decode arithmetic itself is orc-core 1.9.2 (not under /root/reference; restated
// from the public ORC specification in orc_meta.cc / orc_device.cuh).
//
// One call decodes a whole SECTION like pg_parquet_read_section: the files of a sorted run are concatenated into one
// device run.  The file bytes may be host memory (copied to the device) or device memory (used in place).  Host: file
// tails (protobuf footers, inflated on the host; those of device-resident files read back in at most three rounds of
// small reads) -> a plan of streams and (stripe, column) tasks.  Device: k_orc_walk + k_orc_scan (one thread per
// stream: the compression chunk headers -> the stream's bound of inflated bytes -> its place in the scratch; one
// read-back of the total), k_orc_inflate (one warp per stream: compression chunks -> contiguous bytes with the shared
// DEFLATE / zstd / LZ4 decoders), k_orc_task<0> (one thread per task: PRESENT -> validity, values / lengths), an offsets
// scan per var-len column, k_orc_task<1> (payload bytes).  The stream decoders are the host-pinned orc_device.cuh.
#include <algorithm>
#include <cstring>
#include <memory>
#include <stdexcept>

#include "orc_device.cuh"
#include "orc_meta.h"
#include "scan_kernels.cuh"
#include "zstd_device.cuh"

namespace pg {

struct OrcStream {
    const uint8_t *src;        // device: the stream as stored in the file
    int64_t dst_off;           // compressed files: the inflated stream's place in the scratch (k_orc_scan)
    int64_t length, bound;     // bound: of the inflated bytes (k_orc_walk)
    int32_t codec;             // orc::Compression of the stream's file (files of a section may differ)
    int32_t block_size;        // compression block size of that file
    const uint8_t *bytes;      // result: contiguous decoded bytes
    int64_t n;
};

struct OrcTaskRef {            // stream table indexes of a task (-1 = absent)
    int32_t s_present, s_data, s_length, s_dict, s_secondary;
};

// the words a section decode's kernels report in, cleared by one memset
struct OrcWords {
    int32_t err;               // the kernel error word
    int32_t counter;           // k_orc_inflate's stream ticket
    int64_t sc_total;          // k_orc_scan: bytes of the stream scratch
};

// one thread per stream: the bound of the bytes its compression chunks inflate to, from the chunk headers (0 for the
// streams of uncompressed files, which are read in place); a chunk cut off by the stream's end sets *err
__global__ void k_orc_walk(OrcStream *streams, int n_streams, int32_t *err) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_streams) return;
    const OrcStream &st = streams[i];
    int64_t b = 0;
    if (st.codec != orc::C_NONE) {
        b = orcdev::chunk_bound(st.src, st.length, st.codec, st.block_size);
        if (b < 0) { atomicCAS(err, KERR_NONE, KERR_BAD_PAGE); b = 0; }
    }
    streams[i].bound = b;
}

// one CTA: each compressed stream's scratch offset, 64-byte aligned with 64 bytes of slack behind it (the exclusive
// scan of the bounds, in stream order); *total = the scratch bytes
constexpr int kOrcScanThreads = 1024;
__global__ void __launch_bounds__(kOrcScanThreads) k_orc_scan(OrcStream *streams, int n_streams, int64_t *total) {
    __shared__ int64_t part[kOrcScanThreads];
    const int per = (n_streams + kOrcScanThreads - 1) / kOrcScanThreads;
    const int b = threadIdx.x * per, e = min(b + per, n_streams);
    auto need = [&](int i) -> int64_t {
        return streams[i].codec == orc::C_NONE ? 0 : (streams[i].bound + 64 + 63) & ~(int64_t)63;
    };
    int64_t s = 0;
    for (int i = b; i < e; i++) s += need(i);
    part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t acc = 0;
        for (int i = 0; i < kOrcScanThreads; i++) { const int64_t t = part[i]; part[i] = acc; acc += t; }
        *total = acc;
    }
    __syncthreads();
    s = part[threadIdx.x];
    for (int i = b; i < e; i++) { streams[i].dst_off = s; s += need(i); }
}

constexpr int kOrcWarps = 4;
// the grid launches at most 4 CTAs per SM; the bound caps the registers (128) so that all 4 stay resident, which
// the decoders alone would not (153 registers leave room for 3)
__global__ void __launch_bounds__(kOrcWarps * 32, 4)
k_orc_inflate(OrcStream *streams, int n_streams, uint8_t *scratch, uint8_t *lit_scratch, int32_t *counter, int32_t *err) {
    __shared__ zs::Tables ZT[kOrcWarps];               // (the DEFLATE tables are smaller and overlay them)
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t *lit = lit_scratch + ((size_t)blockIdx.x * kOrcWarps + w) * (size_t)(zs::kMaxBlock + 64);
    while (true) {
        int j = 0;
        if (lane == 0) j = atomicAdd(counter, 1);
        j = __shfl_sync(0xffffffffu, j, 0);
        if (j >= n_streams) return;
        OrcStream st = streams[j];
        if (st.codec == orc::C_NONE) {
            if (lane == 0) { streams[j].bytes = st.src; streams[j].n = st.length; }
            continue;
        }
        uint8_t *dst = scratch + st.dst_off;
        const int64_t out = orcdev::inflate_chunks(st.src, st.length, st.codec, st.block_size, dst, st.bound, ZT[w], lit);
        if (lane == 0) {
            if (out < 0) atomicCAS(err, KERR_NONE, KERR_BAD_PAGE);
            streams[j].bytes = dst;
            streams[j].n = out < 0 ? 0 : out;
        }
    }
}

// one thread per (stripe, column); PHASE 0 = validity / values / lengths, PHASE 1 = var-len payload
template <int PHASE>
__global__ void k_orc_task(orcdev::Task *tasks, const OrcTaskRef *refs, const OrcStream *streams, int n_tasks, int32_t *err) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_tasks) return;
    orcdev::Task t = tasks[i];
    if (PHASE == 0) {
        const OrcTaskRef r = refs[i];
        auto bind = [&](int idx, const uint8_t *&p, int64_t &n) {
            if (idx >= 0) { p = streams[idx].bytes; n = streams[idx].n; } else { p = nullptr; n = 0; }
        };
        bind(r.s_present, t.present, t.present_n);
        bind(r.s_data, t.data, t.data_n);
        bind(r.s_length, t.length, t.length_n);
        bind(r.s_dict, t.dict_data, t.dict_data_n);
        bind(r.s_secondary, t.secondary, t.secondary_n);
        orcdev::decode_task_a(t);
    } else {
        orcdev::decode_task_b(t);
    }
    if (t.bad) atomicCAS(err, KERR_NONE, KERR_BAD_PAGE);
    tasks[i] = t;
}

// var-len output column: the payload pointer reaches the tasks after the size read-back
__global__ void k_orc_set_payload(orcdev::Task *tasks, int n_tasks, const int32_t *task_out, uint8_t *const *payload_of_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_tasks && tasks[i].out_width == 0) tasks[i].out_payload = payload_of_out[task_out[i]];
}

// OrcTypeUtil (paimon-format/.../orc/OrcTypeUtil.java convertToOrcType): which ORC type a Paimon column has in the file;
// the integer / float widenings schema evolution allows are accepted (orc-core's SchemaEvolution does the same)
static bool orc_type_ok(int pg_t, const orc::Type &ty) {
    const int k = ty.kind;
    switch (pg_t) {
        case PG_BOOL: return k == orc::K_BOOLEAN;
        case PG_INT8: return k == orc::K_BYTE;
        case PG_INT16: return k == orc::K_SHORT || k == orc::K_BYTE;
        case PG_INT32: return k == orc::K_INT || k == orc::K_SHORT || k == orc::K_BYTE || k == orc::K_DATE;
        case PG_INT64: return k == orc::K_LONG || k == orc::K_INT || k == orc::K_SHORT || k == orc::K_BYTE ||
                              (k == orc::K_DECIMAL && ty.precision <= 18);
        case PG_FLOAT: return k == orc::K_FLOAT;
        case PG_DOUBLE: return k == orc::K_DOUBLE || k == orc::K_FLOAT;
        case PG_STRING: return k == orc::K_STRING || k == orc::K_VARCHAR || k == orc::K_CHAR;
        case PG_BINARY: return k == orc::K_BINARY;
        default: return false;
    }
}

static pg_status orc_decode_section(const std::shared_ptr<const Schema> &s, const pg_file_desc *files, int nf, int n_runs,
                                    const char *const *names, const uint8_t *read_cols, uint64_t *out_runs,
                                    pg_section_info *info) {
    const int nc = s->n_cols();
    SectionFrame fr(s, n_runs, "orc");
    RunBuilder &b = fr.b;
    cudaStream_t sm = fr.stream;
    { pg_status st = fr.start(read_cols, names); if (st) return st; }

    // ---- file tails on the host (those of device-resident files through small reads), column resolution, plans,
    // file bytes on the device
    std::vector<orc::FileTail> tails(nf);
    std::vector<orc::Plan> plans(nf);
    bool any_compressed = false, any_zstd = false;
    // (a codec or type this decoder does not cover is a refusal, not a malformed file)
    auto parse_error = [](const std::exception &e) {
        const bool refusal = strstr(e.what(), "is not decoded") != nullptr || strstr(e.what(), "not supported") != nullptr;
        return fail(refusal ? PG_ERR_UNSUPPORTED : PG_ERR_FORMAT, e.what());
    };
    DeviceRanges rd(sm, files, nf);
    if (!rd.files.empty()) {
        try {
            std::vector<orc::FileTail> t = orc::read_tails(rd, rd.sizes);
            for (size_t i = 0; i < rd.files.size(); i++) tails[rd.files[i]] = std::move(t[i]);
        } catch (const std::exception &e) {
            return rd.st ? rd.st : parse_error(e);
        }
    }
    for (int f = 0; f < nf; f++) {
        try {
            if (files[f].mem == PG_MEM_HOST) tails[f] = orc::parse_file(files[f].bytes, files[f].size);
            const orc::FileTail &t = tails[f];
            if (t.types.empty() || t.types[0].kind != orc::K_STRUCT) return fail(PG_ERR_UNSUPPORTED, "orc: the root type is not a struct");
            if (t.compression != orc::C_NONE && t.compression != orc::C_ZLIB && t.compression != orc::C_ZSTD &&
                t.compression != orc::C_LZ4)
                return fail(PG_ERR_UNSUPPORTED, "orc: compression kind " + std::to_string(t.compression) +
                                                " is not decoded on device (NONE, ZLIB, LZ4 and ZSTD are)");
            if (t.compression != orc::C_NONE) any_compressed = true;
            if (t.compression == orc::C_ZSTD) any_zstd = true;
            if (t.block_size > (1u << 30)) return fail(PG_ERR_UNSUPPORTED, "orc: compression block size above 1 GiB");
            const orc::Type &root = t.types[0];
            if (root.field_names.size() != root.subtypes.size())
                return fail(PG_ERR_FORMAT, "orc: the root struct's field names do not match its fields");
            { pg_status st = b.add_file(files[f].run, (int64_t)t.rows, root.field_names); if (st) return st; }
            const std::vector<int> &file_col = b.file_col[f];
            for (int c = 0; c < nc; c++) {
                if (file_col[c] < 0) continue;
                const uint32_t tid = root.subtypes[file_col[c]];
                if (tid >= t.types.size() || !orc_type_ok(s->field(c).type, t.types[tid]))
                    return fail(PG_ERR_UNSUPPORTED, "orc: column " + std::to_string(c) + " has an ORC type the device decoder does "
                                                    "not map to the table type (timestamps, DECIMAL(p > 18), nested types: Java side)");
            }
            plans[f] = orc::plan_file(t, files[f].size, file_col);
        } catch (const std::exception &e) {
            return parse_error(e);
        }
    }
    { pg_status st = fr.place(files, nf); if (st) return st; }
    { pg_status st = b.check_runs(); if (st) return st; }

    // ---- output columns.  ORC columns are nullable by format: every column the read schema calls nullable gets a
    // bitmap.  Var-len lengths are scanned in place: rows nobody writes must read 0; missing columns are all NULL.
    {
        std::vector<uint8_t> bitmap(nc), zero((size_t)n_runs * nc);
        for (int c = 0; c < nc; c++) bitmap[c] = s->field(c).nullable;
        for (size_t i = 0; i < zero.size(); i++) zero[i] = is_varlen(s->field((int)(i % nc)).type) || b.missing[i];
        pg_status st = b.alloc(bitmap, zero);
        if (st) return st;
    }

    // ---- stream and task tables
    std::vector<OrcStream> h_streams;
    std::vector<orcdev::Task> h_tasks;
    std::vector<OrcTaskRef> h_refs;
    std::vector<int32_t> h_task_out;
    uint64_t dict_entries = 0;
    for (int f = 0; f < nf; f++) dict_entries += plans[f].dict_entries;
    int32_t *d_dict_off = (int32_t *)fr.scratch.take(4 * (size_t)(dict_entries + 1) + 256);
    if (!d_dict_off) return oom("orc", "the dictionary offsets", 4 * (size_t)(dict_entries + 1));
    uint64_t dict_base = 0;
    for (int f = 0; f < nf; f++) {
        const int s0 = (int)h_streams.size();
        for (const orc::PlanStream &ps : plans[f].streams) {
            OrcStream st{};
            st.src = fr.d_file[f] + ps.offset;
            st.length = (int64_t)ps.length;
            st.codec = tails[f].compression;
            st.block_size = (int32_t)tails[f].block_size;
            h_streams.push_back(st);
            fr.page_bytes += (int64_t)ps.length;
        }
        auto idx = [&](int i) { return i < 0 ? -1 : s0 + i; };
        for (const orc::PlanTask &p : plans[f].tasks) {
            const int r = files[f].run;
            const OutColumn &o = b.out[(size_t)r * nc + p.col];
            orcdev::Task k;
            memset(&k, 0, sizeof(k));
            k.row0 = b.file_row0[f] + p.row0;
            k.rows = p.rows;
            k.kind = p.kind; k.enc = p.enc; k.dict_size = (int32_t)p.dict_size; k.scale = p.scale;
            k.out_width = type_width(s->field(p.col).type);
            k.out_data = o.data;
            k.out_offsets = o.offsets;
            k.out_validity = o.validity;
            k.dict_off = d_dict_off + dict_base + p.dict_off_base;
            h_tasks.push_back(k);
            h_refs.push_back(OrcTaskRef{idx(p.s_present), idx(p.s_data), idx(p.s_length), idx(p.s_dict), idx(p.s_secondary)});
            h_task_out.push_back(r * nc + p.col);
        }
        dict_base += plans[f].dict_entries;
    }
    const int n_streams = (int)h_streams.size(), n_tasks = (int)h_tasks.size();
    int sms = 132, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int inflate_ctas = !any_compressed ? std::max(1, std::min(sms, (n_streams + kOrcWarps - 1) / kOrcWarps))
                                                  : std::max(1, std::min(sms * 4, (n_streams + kOrcWarps - 1) / kOrcWarps));
    OrcStream *d_streams;
    orcdev::Task *d_tasks;
    OrcTaskRef *d_refs;
    int32_t *d_task_out;
    uint8_t **d_payload;
    uint8_t *d_lit;                                      // the zstd literal scratch of each inflate warp
    OrcWords *d_words;
    auto carve = [&](void *base) {
        Carver cv(base);
        d_streams = cv.take<OrcStream>((size_t)std::max(n_streams, 1));
        d_tasks = cv.take<orcdev::Task>((size_t)std::max(n_tasks, 1));
        d_refs = cv.take<OrcTaskRef>((size_t)std::max(n_tasks, 1));
        d_task_out = cv.take<int32_t>((size_t)std::max(n_tasks, 1));
        d_payload = cv.take<uint8_t *>(b.out.size());
        d_lit = cv.take<uint8_t>(any_zstd ? (size_t)inflate_ctas * kOrcWarps * (size_t)(zs::kMaxBlock + 64) : 0);
        d_words = cv.take<OrcWords>(1);
        return cv.bytes();
    };
    const size_t tb_bytes = carve(nullptr);
    void *tb = fr.scratch.take(tb_bytes);
    if (!tb) return oom("orc", "the stream and task tables", tb_bytes);
    carve(tb);
    int32_t *d_err = &d_words->err;
    PG_CUDA(cudaMemsetAsync(d_words, 0, sizeof(OrcWords), sm));
    // (tables go through small_h2d: a kernel reads them out of mapped host memory, so they do not queue behind an
    // asynchronous upload of the next section on the copy engine)
    if (n_streams) { pg_status ts = small_h2d(d_streams, h_streams.data(), sizeof(OrcStream) * n_streams, sm); if (ts) return ts; }
    if (n_tasks) {
        pg_status ts = small_h2d(d_tasks, h_tasks.data(), sizeof(orcdev::Task) * n_tasks, sm);
        if (!ts) ts = small_h2d(d_refs, h_refs.data(), sizeof(OrcTaskRef) * n_tasks, sm);
        if (!ts) ts = small_h2d(d_task_out, h_task_out.data(), 4 * (size_t)n_tasks, sm);
        if (ts) return ts;
    }
    // ---- compressed sections: the chunk walk sizes the stream scratch (one read-back)
    uint8_t *d_sc = nullptr;
    if (any_compressed && n_streams) {
        k_orc_walk<<<(n_streams + 127) / 128, 128, 0, sm>>>(d_streams, n_streams, d_err);
        k_orc_scan<<<1, kOrcScanThreads, 0, sm>>>(d_streams, n_streams, &d_words->sc_total);
        fr.launches += 2;
        int32_t herr = 0;
        int64_t sc_bytes = 0;
        {
            SmallReads rb(sm);
            pg_status rs = rb.add(&herr, d_err, 4);
            if (!rs) rs = rb.add(&sc_bytes, &d_words->sc_total, 8);
            if (!rs) rs = rb.finish();
            if (!rs) rs = kernel_error(herr, "orc");
            if (rs) return rs;
        }
        d_sc = (uint8_t *)fr.scratch.take((size_t)sc_bytes + 256);
        if (!d_sc) return oom("orc", "the stream scratch", (size_t)sc_bytes);
    }
    if (n_streams) {
        k_orc_inflate<<<inflate_ctas, kOrcWarps * 32, 0, sm>>>(d_streams, n_streams, d_sc, d_lit, &d_words->counter, d_err);
        fr.launches++;
    }
    if (n_tasks) {
        k_orc_task<0><<<(n_tasks + 31) / 32, 32, 0, sm>>>(d_tasks, d_refs, d_streams, n_tasks, d_err);
        fr.launches++;
    }
    // ---- var-len columns: lengths -> offsets, exact payload sizes (one read-back), payload
    std::vector<int32_t> totals(b.out.size(), 0);          // per (run, column)
    if (std::any_of(b.out.begin(), b.out.end(), [](const OutColumn &o) { return o.offsets != nullptr; })) {
        const int64_t max_n = *std::max_element(b.run_rows.begin(), b.run_rows.end());
        int64_t *d_sums = (int64_t *)fr.scratch.take(8 * (size_t)(max_n / 4096 + 4));
        if (!d_sums) return oom("orc", "the offsets scan", 8 * (size_t)(max_n / 4096 + 4));
        SmallReads rb(sm);                                 // the read-back: exact payload sizes
        for (size_t i = 0; i < b.out.size(); i++) {
            const OutColumn &o = b.out[i];
            if (!o.offsets) continue;
            const int64_t n = b.run_rows[i / nc];
            launch_offsets_scan(o.offsets, n, d_sums, d_err, sm);
            fr.launches += n > 0 ? 3 : 0;
            { pg_status rs = rb.add(&totals[i], o.offsets + n, 4); if (rs) return rs; }
        }
        int32_t herr = 0;
        { pg_status rs = rb.add(&herr, d_err, 4); if (!rs) rs = rb.finish(); if (!rs) rs = kernel_error(herr, "orc"); if (rs) return rs; }
        { pg_status st = b.alloc_payload(std::vector<int64_t>(totals.begin(), totals.end())); if (st) return st; }
        std::vector<uint8_t *> h_payload(b.out.size());   // (k_orc_set_payload reads the var-len entries only)
        for (size_t i = 0; i < b.out.size(); i++) h_payload[i] = (uint8_t *)b.out[i].data;
        { pg_status ts = small_h2d(d_payload, h_payload.data(), sizeof(void *) * h_payload.size(), sm); if (ts) return ts; }
        if (n_tasks) {
            k_orc_set_payload<<<(n_tasks + 127) / 128, 128, 0, sm>>>(d_tasks, n_tasks, d_task_out, d_payload);
            k_orc_task<1><<<(n_tasks + 31) / 32, 32, 0, sm>>>(d_tasks, d_refs, d_streams, n_tasks, d_err);
            fr.launches += 2;
        }
    }
    { pg_status st = fr.finish(d_err, out_runs, info); if (st) return st; }
    if (info) {
        info->n_chunks = n_tasks;
        info->n_data_pages = n_streams;
    }
    return PG_OK;
}

}  // namespace pg

using namespace pg;

extern "C" pg_status pg_orc_read_section(uint64_t schema, const pg_file_desc *files, int32_t n_files, int32_t n_runs,
                                         const char *const *column_names, const uint8_t *read_columns, uint64_t *out_runs,
                                         pg_section_info *info) {
    std::shared_ptr<const Schema> s;
    pg_status st = check_section_args(schema, files, n_files, n_runs, out_runs, &s);
    if (st || n_runs == 0) return st;
    st = ensure_device();
    if (st) return st;
    return orc_decode_section(s, files, n_files, n_runs, column_names, read_columns, out_runs, info);
}
