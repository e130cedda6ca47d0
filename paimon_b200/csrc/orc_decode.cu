// orc_decode.cu — ORC stripe decode on the device behind the same format seam as the Parquet decoder
// (SURVEY.md §8 rows a25 / f3).
//
// Reference being replaced: paimon-format/src/main/java/org/apache/paimon/format/orc/OrcReaderFactory.java:98-163
// (createReader: orc-core RecordReader over the projected TypeDescription, batches of VectorizedRowBatch) and the
// vector adapters in orc/reader/*; the decode arithmetic itself is orc-core 1.9.2 (not under /root/reference; restated
// from the public ORC specification in orc_meta.cc / orc_device.cuh).
//
// One call decodes a whole SECTION like pg_parquet_read_section: the files of a sorted run are concatenated into one
// device run.  Host: file tails (protobuf footers, inflated on the host) -> a plan of streams and (stripe, column)
// tasks.  Device: k_orc_inflate (one warp per stream: compression chunks -> contiguous bytes with the shared
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
    uint8_t *dst;              // scratch image (compressed files)
    int64_t length, bound;
    int32_t codec;             // orc::Compression of the stream's file (files of a section may differ)
    int32_t block_size;        // compression block size of that file
    const uint8_t *bytes;      // result: contiguous decoded bytes
    int64_t n;
};

struct OrcTaskRef {            // stream table indexes of a task (-1 = absent)
    int32_t s_present, s_data, s_length, s_dict, s_secondary;
};

constexpr int kOrcWarps = 4;
// the grid launches at most 4 CTAs per SM; the bound caps the registers (128) so that all 4 stay resident, which
// the decoders alone would not (153 registers leave room for 3)
__global__ void __launch_bounds__(kOrcWarps * 32, 4)
k_orc_inflate(OrcStream *streams, int n_streams, uint8_t *lit_scratch, int32_t *counter, int32_t *err) {
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
        const int64_t out = orcdev::inflate_chunks(st.src, st.length, st.codec, st.block_size, st.dst, st.bound, ZT[w], lit);
        if (lane == 0) {
            if (out < 0) atomicCAS(err, KERR_NONE, KERR_BAD_PAGE);
            streams[j].bytes = st.dst;
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
    cudaStream_t sm = copy_stream();
    Scratch scratch(sm);                               // file images, tables, scratch and the runs until registered
    RunBuilder b(s, n_runs, scratch, "orc");
    SectionTimer tm;
    PG_CUDA(cudaEventCreate(&tm.e0));
    PG_CUDA(cudaEventCreate(&tm.e1));
    PG_CUDA(cudaEventRecord(tm.e0, sm));
    { pg_status st = b.read_columns(read_cols, names); if (st) return st; }

    // ---- file tails, column resolution, plans
    std::vector<orc::FileTail> tails(nf);
    std::vector<orc::Plan> plans(nf);
    std::vector<const uint8_t *> d_file(nf, nullptr);
    int64_t file_bytes = 0, page_bytes = 0;
    bool any_compressed = false, any_zstd = false;
    for (int f = 0; f < nf; f++) {
        if (files[f].mem != PG_MEM_HOST)
            return fail(PG_ERR_UNSUPPORTED, "orc: the file bytes must be host memory (the footers and chunk headers are walked on the host)");
        try {
            tails[f] = orc::parse_file(files[f].bytes, files[f].size);
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
            plans[f] = orc::plan_file(t, files[f].bytes, files[f].size, file_col);
        } catch (const std::exception &e) {
            // (a codec or type this decoder does not cover is a refusal, not a malformed file)
            const bool refusal = strstr(e.what(), "is not decoded") != nullptr || strstr(e.what(), "not supported") != nullptr;
            return fail(refusal ? PG_ERR_UNSUPPORTED : PG_ERR_FORMAT, e.what());
        }
        file_bytes += files[f].size;
        { pg_status st = file_image(scratch, files[f].bytes, files[f].size, "orc", &d_file[f]); if (st) return st; }
    }
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
    uint64_t sc_bytes = 0, dict_entries = 0;
    for (int f = 0; f < nf; f++) { sc_bytes += plans[f].scratch_bytes; dict_entries += plans[f].dict_entries; }
    uint8_t *d_sc = !any_compressed ? nullptr : (uint8_t *)scratch.take((size_t)sc_bytes + 256);
    if (any_compressed && !d_sc) return oom("orc", "the stream scratch", (size_t)sc_bytes);
    int32_t *d_dict_off = (int32_t *)scratch.take(4 * (size_t)(dict_entries + 1) + 256);
    if (!d_dict_off) return oom("orc", "the dictionary offsets", 4 * (size_t)(dict_entries + 1));
    uint64_t sc_base = 0, dict_base = 0;
    for (int f = 0; f < nf; f++) {
        const int s0 = (int)h_streams.size();
        for (const orc::PlanStream &ps : plans[f].streams) {
            OrcStream st{};
            st.src = d_file[f] + ps.offset;
            st.length = (int64_t)ps.length;
            st.bound = (int64_t)ps.out_bound;
            st.codec = tails[f].compression;
            st.block_size = (int32_t)tails[f].block_size;
            st.dst = d_sc ? d_sc + sc_base + ps.out_off : nullptr;
            h_streams.push_back(st);
            page_bytes += (int64_t)ps.length;
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
        sc_base += plans[f].scratch_bytes;
        dict_base += plans[f].dict_entries;
    }
    const int n_streams = (int)h_streams.size(), n_tasks = (int)h_tasks.size();
    const size_t tb_s = align256(sizeof(OrcStream) * (size_t)std::max(n_streams, 1)), tb_t = align256(sizeof(orcdev::Task) * (size_t)std::max(n_tasks, 1));
    const size_t tb_r = align256(sizeof(OrcTaskRef) * (size_t)std::max(n_tasks, 1)), tb_o = align256(4 * (size_t)std::max(n_tasks, 1));
    const size_t tb_p = align256(sizeof(void *) * b.out.size());
    int sms = 132, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int inflate_ctas = !any_compressed ? std::max(1, std::min(sms, (n_streams + kOrcWarps - 1) / kOrcWarps))
                                                  : std::max(1, std::min(sms * 4, (n_streams + kOrcWarps - 1) / kOrcWarps));
    const size_t tb_lit = any_zstd ? align256((size_t)inflate_ctas * kOrcWarps * (size_t)(zs::kMaxBlock + 64)) : 256;
    unsigned char *tb = (unsigned char *)scratch.take(tb_s + tb_t + tb_r + tb_o + tb_p + tb_lit + 1024);
    if (!tb) return oom("orc", "the stream and task tables", tb_s + tb_t + tb_r + tb_o + tb_p + tb_lit);
    OrcStream *d_streams = (OrcStream *)tb;
    orcdev::Task *d_tasks = (orcdev::Task *)(tb + tb_s);
    OrcTaskRef *d_refs = (OrcTaskRef *)(tb + tb_s + tb_t);
    int32_t *d_task_out = (int32_t *)(tb + tb_s + tb_t + tb_r);
    uint8_t **d_payload = (uint8_t **)(tb + tb_s + tb_t + tb_r + tb_o);
    uint8_t *d_lit = tb + tb_s + tb_t + tb_r + tb_o + tb_p;
    int32_t *d_err = (int32_t *)(d_lit + tb_lit);
    int32_t *d_counter = d_err + 4;
    PG_CUDA(cudaMemsetAsync(d_err, 0, 64, sm));
    int launches = 0;
    if (n_streams) PG_CUDA(cudaMemcpyAsync(d_streams, h_streams.data(), sizeof(OrcStream) * n_streams, cudaMemcpyHostToDevice, sm));
    if (n_tasks) {
        PG_CUDA(cudaMemcpyAsync(d_tasks, h_tasks.data(), sizeof(orcdev::Task) * n_tasks, cudaMemcpyHostToDevice, sm));
        PG_CUDA(cudaMemcpyAsync(d_refs, h_refs.data(), sizeof(OrcTaskRef) * n_tasks, cudaMemcpyHostToDevice, sm));
        PG_CUDA(cudaMemcpyAsync(d_task_out, h_task_out.data(), 4 * (size_t)n_tasks, cudaMemcpyHostToDevice, sm));
    }
    if (n_streams) {
        k_orc_inflate<<<inflate_ctas, kOrcWarps * 32, 0, sm>>>(d_streams, n_streams, d_lit, d_counter, d_err);
        launches++;
    }
    if (n_tasks) {
        k_orc_task<0><<<(n_tasks + 31) / 32, 32, 0, sm>>>(d_tasks, d_refs, d_streams, n_tasks, d_err);
        launches++;
    }
    // ---- var-len columns: lengths -> offsets, exact payload sizes (one read-back), payload
    std::vector<int32_t> totals(b.out.size(), 0);          // per (run, column)
    int32_t herr = 0;
    if (std::any_of(b.out.begin(), b.out.end(), [](const OutColumn &o) { return o.offsets != nullptr; })) {
        const int64_t max_n = *std::max_element(b.run_rows.begin(), b.run_rows.end());
        int64_t *d_sums = (int64_t *)scratch.take(8 * (size_t)(max_n / 4096 + 4));
        if (!d_sums) return oom("orc", "the offsets scan", 8 * (size_t)(max_n / 4096 + 4));
        for (size_t i = 0; i < b.out.size(); i++) {
            const OutColumn &o = b.out[i];
            if (!o.offsets) continue;
            const int64_t n = b.run_rows[i / nc];
            launch_offsets_scan(o.offsets, n, d_sums, d_err, sm);
            launches += n > 0 ? 3 : 0;
            PG_CUDA(cudaMemcpyAsync(&totals[i], o.offsets + n, 4, cudaMemcpyDeviceToHost, sm));
        }
        PG_CUDA(cudaMemcpyAsync(&herr, d_err, 4, cudaMemcpyDeviceToHost, sm));
        PG_CUDA(cudaStreamSynchronize(sm));               // the read-back: exact payload sizes
        if (herr != KERR_NONE)
            return fail(herr == KERR_OFFSET_OVERFLOW ? PG_ERR_INTERNAL : PG_ERR_FORMAT,
                        herr == KERR_OFFSET_OVERFLOW ? "orc: a var-len column exceeds 2 GiB of payload"
                                                     : "orc: a stream does not decode (malformed file or unsupported encoding)");
        { pg_status st = b.alloc_payload(std::vector<int64_t>(totals.begin(), totals.end())); if (st) return st; }
        std::vector<uint8_t *> h_payload(b.out.size());   // (k_orc_set_payload reads the var-len entries only)
        for (size_t i = 0; i < b.out.size(); i++) h_payload[i] = (uint8_t *)b.out[i].data;
        PG_CUDA(cudaMemcpyAsync(d_payload, h_payload.data(), sizeof(void *) * h_payload.size(), cudaMemcpyHostToDevice, sm));
        if (n_tasks) {
            k_orc_set_payload<<<(n_tasks + 127) / 128, 128, 0, sm>>>(d_tasks, n_tasks, d_task_out, d_payload);
            k_orc_task<1><<<(n_tasks + 31) / 32, 32, 0, sm>>>(d_tasks, d_refs, d_streams, n_tasks, d_err);
            launches += 2;
        }
        PG_CUDA(cudaStreamSynchronize(sm));               // (h_payload is a local)
    }
    PG_CUDA(cudaEventRecord(tm.e1, sm));
    PG_CUDA(cudaMemcpyAsync(&herr, d_err, 4, cudaMemcpyDeviceToHost, sm));
    PG_CUDA(cudaStreamSynchronize(sm));
    PG_CUDA(cudaGetLastError());
    if (herr != KERR_NONE) return fail(PG_ERR_FORMAT, "orc: a stream does not decode (malformed file or unsupported encoding)");
    b.finish(out_runs, file_bytes, info);
    if (info) {
        info->file_bytes = file_bytes;
        info->page_bytes = page_bytes;
        info->n_files = nf;
        info->n_chunks = n_tasks;
        info->n_data_pages = n_streams;
        info->launches = launches;
        info->ms_decode = tm.ms();
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
