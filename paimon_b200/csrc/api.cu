// api.cu — host side of libpaimon_gpu.so: handle tables, plan-time validation of merge specs,
// device descriptors, and the launch sequence of one merge (partition levels -> plan -> scan ->
// emit).  Everything the Java side sees goes through the extern "C" functions at the bottom
// (include/paimon_gpu.h).  There is no CPU fallback anywhere in this file: a spec the kernels do not
// implement is refused with PG_ERR_UNSUPPORTED.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <queue>

#include "pg_internal.h"

namespace pg {

static thread_local std::string g_last_error;
void set_error(const std::string &msg) { g_last_error = msg; }
pg_status fail(pg_status code, const std::string &msg) {
    g_last_error = msg;
    return code;
}

static int g_device = -1;

// grow-only device allocation, carved by its user (Carver)
struct Arena {
    unsigned char *base = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (base) cudaFree(base);
        base = nullptr;
        cap = 0;
        cudaError_t e = cudaMalloc((void **)&base, bytes);
        if (e == cudaSuccess) cap = bytes;
        return e;
    }
    void release() {
        if (base) cudaFree(base);
        base = nullptr;
        cap = 0;
    }
    ~Arena() { release(); }
};

// the device descriptors of a merge handle, carved from one allocation (Merge::d_desc)
struct MergeDesc {
    const void **key_ptrs;              // [run * n_key + field]
    const int32_t **key_offs;
    const int64_t **seq_ptrs;           // [k]
    const int8_t **kind_ptrs;           // [k]
    const void **data;                  // ColPtrs: [col * k + run]
    const int32_t **offsets;
    const uint32_t **validity;
    int64_t *run_rows;                  // [k]
    ColDesc *cols;                      // [n_cols]
    pg_out_column *out_cols;            // [n_cols]
    int64_t *totals;                    // [1 + n_varlen]
    int32_t *err;
    int32_t *tile_counter;
    int32_t *col_order;                 // the emit kernel's pass list
    int32_t *varlen_cols;               // [n_varlen]
    SeqGroups *groups;                  // NULL on the device without sequence groups
    ColPtrs ptrs() const { return ColPtrs{data, offsets, validity}; }
    // the layout, for k runs, nk key fields, nc columns and nv var-len columns: returns its bytes
    size_t carve(void *base, int k, int nk, int nc, int nv) {
        Carver cv(base);
        key_ptrs = cv.take<const void *>((size_t)k * nk);
        key_offs = cv.take<const int32_t *>((size_t)k * nk);
        seq_ptrs = cv.take<const int64_t *>(k);
        kind_ptrs = cv.take<const int8_t *>(k);
        data = cv.take<const void *>((size_t)k * nc);
        offsets = cv.take<const int32_t *>((size_t)k * nc);
        validity = cv.take<const uint32_t *>((size_t)k * nc);
        run_rows = cv.take<int64_t>(k);
        cols = cv.take<ColDesc>(nc);
        out_cols = cv.take<pg_out_column>(nc);
        totals = cv.take<int64_t>(nv + 1);
        err = cv.take<int32_t>(1);
        tile_counter = cv.take<int32_t>(1);
        col_order = cv.take<int32_t>(2 * (size_t)nc + 2);
        varlen_cols = cv.take<int32_t>(nv + 1);
        groups = cv.take<SeqGroups>(1);
        return cv.bytes();
    }
};

struct Merge {
    std::shared_ptr<const Spec> spec;
    std::vector<std::shared_ptr<const Run>> runs;  // from the bind until an execute has merged them (see execute)
    std::vector<std::weak_ptr<const Run>> bound;   // the same runs, for a re-execute
    std::vector<int64_t> row0;          // per run: first row that takes part (pg_merge_rebind), else 0
    int k = 0;
    int64_t n_in = 0;
    size_t desc_cap = 0;                // bytes allocated behind d_desc
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    std::vector<int64_t> varlen_bound;     // per var-len column: sum of the runs' payload bytes
    KeyDesc key{};
    SeqFields seq{};
    MergeFlags flags{};
    std::vector<ColDesc> cols;
    std::vector<int32_t> varlen_cols;
    std::vector<uint8_t> emit;          // per column: part of the merged batch (read-type projection)
    // persistent device descriptors
    void *d_desc = nullptr;            // one allocation holding all descriptor arrays
    MergeDesc desc{};                  // ... carved into them
    int n_passes = 0;
    bool has_group_aggs = false;
    // pinned host mirror of totals + err
    int64_t *h_totals = nullptr;
    int32_t *h_err = nullptr;
    // output of the last execute
    std::vector<pg_out_column> out_cols;
    Arena work;                        // temporaries of one execute (bounds, sample keys, plan, ...)
    Arena outbuf;                      // the output batch
    int64_t n_out = 0;
    bool has_batch = false;
    pg_stats stats{};
    // may run on a thread that never bound the device; the arenas, runs and spec are released after this body
    ~Merge() {
        if (g_device >= 0) cudaSetDevice(g_device);
        if (stream) cudaStreamSynchronize(stream);
        if (d_desc) cudaFree(d_desc);
        if (h_totals) cudaFreeHost(h_totals);
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
        if (stream) cudaStreamDestroy(stream);
    }
};

// ------------------------------------------------------------------ handle tables

Table<Schema> g_schemas(1);
static Table<Spec> g_specs(2);
Table<Run> g_runs(3);
static Table<Merge> g_merges(4);

pg_status ensure_device() {
    if (g_device < 0) return fail(PG_ERR_INVALID, "pg_init has not been called");
    PG_CUDA(cudaSetDevice(g_device));
    return PG_OK;
}

// Many small copies (one per column buffer) in one driver call: cudaMemcpyBatchAsync where the driver has it,
// else one cudaMemcpyAsync per buffer.  A wide table has hundreds of buffers per run and the per-call cost
// of the copy API would otherwise bound a reader that streams small key ranges.
static pg_status copy_batch(std::vector<void *> &dsts, std::vector<void *> &srcs, std::vector<size_t> &sizes,
                            cudaMemcpyKind kind, cudaStream_t stream) {
    if (dsts.empty()) return PG_OK;
    static bool batch_ok = true;
    if (batch_ok && dsts.size() > 1) {
        cudaMemcpyAttributes attr{};
        attr.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
        size_t attr_idx = 0, fail_idx = 0;
        cudaError_t e = cudaMemcpyBatchAsync(dsts.data(), srcs.data(), sizes.data(), dsts.size(), &attr, &attr_idx, 1,
                                             &fail_idx, stream);
        if (e == cudaSuccess) return PG_OK;
        cudaGetLastError();
        batch_ok = false;                               // not supported here: fall back for good
    }
    for (size_t i = 0; i < dsts.size(); i++) PG_CUDA(cudaMemcpyAsync(dsts[i], srcs[i], sizes[i], kind, stream));
    return PG_OK;
}
// ---- the recycled-buffer cache (pg_internal.h): free buffers keyed by size, up to PG_RUN_CACHE_BYTES in all
static std::mutex g_buf_mu;
static std::multimap<size_t, void *> g_free_bufs;
static size_t g_free_bytes = 0;
static size_t buf_cache_limit() {
    static size_t lim = [] {
        const char *e = getenv("PG_RUN_CACHE_BYTES");
        return e ? (size_t)strtoull(e, nullptr, 10) : ((size_t)16 << 30);
    }();
    return lim;
}
static void buf_trim(size_t keep_bytes) {
    std::vector<void *> drop;
    {
        std::lock_guard<std::mutex> g(g_buf_mu);
        while (g_free_bytes > keep_bytes && !g_free_bufs.empty()) {
            auto it = std::prev(g_free_bufs.end());
            drop.push_back(it->second);
            g_free_bytes -= it->first;
            g_free_bufs.erase(it);
        }
    }
    for (void *p : drop) cudaFree(p);
}
void *buf_take(size_t bytes, size_t *got) {
    {
        std::lock_guard<std::mutex> g(g_buf_mu);
        auto it = g_free_bufs.lower_bound(bytes);
        if (it != g_free_bufs.end() && it->first <= bytes + bytes / 2 + (1 << 20)) {
            void *p = it->second;
            *got = it->first;
            g_free_bytes -= it->first;
            g_free_bufs.erase(it);
            return p;
        }
    }
    void *p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) {
        cudaGetLastError();
        buf_trim(0);                                  // give the cached buffers back and retry once
        if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
    }
    *got = bytes;
    return p;
}
void buf_give(void *p, size_t bytes) {
    {
        std::lock_guard<std::mutex> g(g_buf_mu);
        if (g_free_bytes + bytes <= buf_cache_limit()) {
            g_free_bufs.emplace(bytes, p);
            g_free_bytes += bytes;
            return;
        }
    }
    cudaFree(p);
}
cudaStream_t copy_stream() {                          // one non-blocking copy stream per calling thread
    static thread_local cudaStream_t st = nullptr;
    if (!st) cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    return st;
}

pg_status batch_columns(uint64_t handle, BatchColumns *out) {
    if (std::shared_ptr<Merge> m = g_merges.get(handle)) {
        if (!m->has_batch) return fail(PG_ERR_INVALID, "no batch: call pg_merge_execute first");
        if (m->stream) PG_CUDA(cudaStreamSynchronize(m->stream));
        out->schema = m->spec->schema;
        out->n_rows = m->n_out;
        for (const pg_out_column &oc : m->out_cols) out->cols.push_back(DevColumn{oc.data, oc.offsets, oc.validity});
        out->merge = std::move(m);
        return PG_OK;
    }
    std::shared_ptr<Run> r = g_runs.get(handle);
    if (!r) return fail(PG_ERR_INVALID, "unknown run / merge handle");
    out->schema = r->schema;
    out->n_rows = r->n_rows;
    out->cols = r->cols;
    out->run = std::move(r);
    return PG_OK;
}

// ------------------------------------------------------------------ decoded runs (pg_internal.h: RunBuilder)

pg_status oom(const char *who, const char *what, size_t bytes) {
    size_t fr = 0, tot = 0;
    cudaMemGetInfo(&fr, &tot);
    cudaGetLastError();
    return fail(PG_ERR_CUDA, std::string(who) + ": out of device memory for " + what + " (" + std::to_string(bytes >> 20) +
                                 " MiB wanted, " + std::to_string(fr >> 20) + " of " + std::to_string(tot >> 20) + " MiB free)");
}

pg_status check_file_desc(const pg_file_desc &f) {
    if (f.mem != PG_MEM_HOST && f.mem != PG_MEM_DEVICE)
        return fail(PG_ERR_INVALID, "file descriptor: memory kind " + std::to_string(f.mem) + " is neither host nor device");
    if (f.size < 0) return fail(PG_ERR_INVALID, "file descriptor: negative size");
    if (f.size > 0 && !f.bytes) return fail(PG_ERR_INVALID, "file descriptor: no bytes for a file of " + std::to_string(f.size) + " bytes");
    return PG_OK;
}

pg_status check_section_args(uint64_t schema, const pg_file_desc *files, int n_files, int n_runs, const uint64_t *out_runs,
                             std::shared_ptr<const Schema> *s) {
    *s = g_schemas.get(schema);
    if (!*s || !out_runs || n_files < 0 || n_runs < 0 || (n_files > 0 && !files))
        return fail(PG_ERR_INVALID, "bad schema handle or null argument");
    for (int i = 0; i < n_files; i++) {
        pg_status st = check_file_desc(files[i]);
        if (st) return st;
        if (files[i].run < 0 || files[i].run >= n_runs)
            return fail(PG_ERR_INVALID, "file descriptor: run index " + std::to_string(files[i].run) + " out of range");
    }
    return PG_OK;
}

pg_status file_image(Scratch &scratch, const uint8_t *bytes, int64_t size, const char *who, const uint8_t **out) {
    uint8_t *d = (uint8_t *)scratch.take((size_t)size + 64);
    if (!d) return oom(who, "a file image", (size_t)size);
    PG_CUDA(cudaMemcpyAsync(d, bytes, (size_t)size, cudaMemcpyHostToDevice, scratch.stream));
    *out = d;
    return PG_OK;
}

pg_status RunBuilder::read_columns(const uint8_t *read_cols, const char *const *column_names) {
    names = column_names;
    if (names)
        for (int c = 0; c < nc; c++)
            if (!names[c]) return fail(PG_ERR_INVALID, std::string(who) + ": column name " + std::to_string(c) + " is NULL");
    if (!read_cols) return PG_OK;
    for (int c = 0; c < schema->n_key + 2; c++)
        if (!read_cols[c]) return fail(PG_ERR_INVALID, std::string(who) + ": key, sequence number and kind columns are always read");
    for (int c = 0; c < nc; c++) read[c] = read_cols[c] != 0;
    return PG_OK;
}

pg_status RunBuilder::add_file(int run, int64_t rows, const std::vector<std::string> &cols) {
    if (!names && (int)cols.size() != nc)
        return fail(PG_ERR_UNSUPPORTED, std::string(who) + ": the file has " + std::to_string(cols.size()) + " columns and the "
                                        "read schema " + std::to_string(nc) + " (pass the field names)");
    std::unordered_map<std::string, int> by_name;
    if (names) for (int i = 0; i < (int)cols.size(); i++) by_name.emplace(cols[i], i);
    std::vector<int> fc(nc, -2);
    for (int c = 0; c < nc; c++) {
        if (!read[c]) continue;
        fc[c] = c;
        if (names) {
            auto it = by_name.find(names[c]);               // (of two equal names in a file, the first counts)
            fc[c] = it == by_name.end() ? -1 : it->second;
        }
        if (fc[c] == -1 && (c < schema->n_key + 2 || !schema->field(c).nullable))
            return fail(PG_ERR_UNSUPPORTED, std::string(who) + ": the file has no column '" + names[c] + "' and the read "
                                            "schema does not allow NULL for it");
        const size_t i = (size_t)run * nc + c;
        if (fc[c] == -1) missing[i] = 1;
        if (rows > 0) with_rows[i] |= fc[c] == -1 ? 2 : 1;
    }
    file_col.push_back(std::move(fc));
    file_row0.push_back(place_file(run, rows));
    return PG_OK;
}

pg_status RunBuilder::check_runs() const {
    for (int64_t n : run_rows)
        if (n > 0x7fffffffLL) return fail(PG_ERR_UNSUPPORTED, std::string(who) + ": more than 2^31 rows in one run");
    for (size_t i = 0; i < with_rows.size(); i++)
        if (with_rows[i] == 3 && is_varlen(schema->field((int)(i % nc)).type))
            return fail(PG_ERR_UNSUPPORTED, std::string(who) + ": a var-len column exists in some files with rows of a sorted "
                                            "run only (mixed table schemas inside one run: not decoded on device)");
    return PG_OK;
}

pg_status RunBuilder::alloc(const std::vector<uint8_t> &bitmap, const std::vector<uint8_t> &zero) {
    const int n_runs = (int)run_rows.size();
    scratch.runs.resize(n_runs);
    out.assign((size_t)n_runs * nc, OutColumn());
    for (int r = 0; r < n_runs; r++) {
        const int64_t n = run_rows[r];
        OutColumn *o = &out[(size_t)r * nc];
        // values, or int32 offsets
        auto main_bytes = [&](int c) { const int w = type_width(schema->field(c).type); return w ? (size_t)n * w : 4 * (size_t)(n + 1); };
        size_t vspan = 0;                                // the bitmaps: [0, vspan)
        auto carve = [&](void *base) {
            Carver cv(base);
            for (int c = 0; c < nc; c++)
                if (read[c] && bitmap[c]) o[c].validity = cv.take<uint32_t>((size_t)(n + 31) / 32 + kReadPast / 4);
            vspan = cv.bytes();
            for (int c = 0; c < nc; c++) {
                if (!read[c]) continue;
                if (type_width(schema->field(c).type)) o[c].data = cv.take<uint8_t>(main_bytes(c) + kReadPast);
                else o[c].offsets = cv.take<int32_t>((size_t)n + 1 + kReadPast / 4);
            }
            return cv.bytes();
        };
        const size_t total = carve(nullptr);
        scratch.runs[r] = std::make_unique<Run>(schema, n);
        scratch.runs[r]->bufs.emplace_back(total);
        unsigned char *base = scratch.runs[r]->bufs.back().get();
        if (!base) return oom(who, "the columns of a run", total);
        carve(base);
        if (vspan) PG_CUDA(cudaMemsetAsync(base, 0, vspan, scratch.stream));
        for (int c = 0; c < nc; c++) {
            if (!read[c]) continue;
            if (bitmap[c]) decoded_bytes += (n + 7) / 8;
            decoded_bytes += (int64_t)main_bytes(c);
            void *values = type_width(schema->field(c).type) ? o[c].data : (void *)o[c].offsets;
            if (zero[(size_t)r * nc + c]) PG_CUDA(cudaMemsetAsync(values, 0, main_bytes(c), scratch.stream));
        }
    }
    return PG_OK;
}

pg_status RunBuilder::alloc_payload(const std::vector<int64_t> &payload) {
    bool any = false;
    for (int c = 0; c < nc; c++) any |= read[c] && is_varlen(schema->field(c).type);
    if (!any) return PG_OK;
    for (int r = 0; r < (int)run_rows.size(); r++) {
        OutColumn *o = &out[(size_t)r * nc];
        const int64_t *bytes = &payload[(size_t)r * nc];
        auto carve = [&](void *base) {
            Carver cv(base);
            for (int c = 0; c < nc; c++)
                if (read[c] && is_varlen(schema->field(c).type)) o[c].data = cv.take<uint8_t>((size_t)bytes[c] + kReadPast);
            return cv.bytes();
        };
        const size_t total = carve(nullptr);
        Run &run = *scratch.runs[r];
        run.bufs.emplace_back(total);
        unsigned char *pl = run.bufs.back().get();
        if (!pl) return oom(who, "the var-len payload of a run", total);
        carve(pl);
        for (int c = 0; c < nc; c++) {
            if (!read[c] || !is_varlen(schema->field(c).type)) continue;
            run.varlen_bytes[c] = bytes[c];
            decoded_bytes += bytes[c];
        }
    }
    return PG_OK;
}

void RunBuilder::finish(uint64_t *out_runs, int64_t bytes_h2d, pg_section_info *info) {
    const int n_runs = (int)run_rows.size();
    for (int r = 0; r < n_runs; r++) {
        Run &run = *scratch.runs[r];
        for (int c = 0; c < nc; c++) {
            const OutColumn &o = out[(size_t)r * nc + c];
            if (read[c]) run.cols[c] = DevColumn{o.data ? o.data : run.bufs[0].get(), o.offsets, (const uint8_t *)o.validity};
        }
        run.bytes_h2d = r == 0 ? bytes_h2d : 0;
        out_runs[r] = g_runs.put(std::move(scratch.runs[r]));
    }
    if (info) {
        memset(info, 0, sizeof(*info));
        for (int64_t n : run_rows) info->n_rows += n;
        info->n_runs = n_runs;
        info->decoded_bytes = decoded_bytes;
    }
}

SectionFrame::SectionFrame(std::shared_ptr<const Schema> s, int n_runs, const char *who)
    : stream(copy_stream()), scratch(stream), b(std::move(s), n_runs, scratch, who) {}

pg_status SectionFrame::start(const uint8_t *read_cols, const char *const *names) {
    PG_CUDA(cudaEventCreate(&tm.e0));
    PG_CUDA(cudaEventCreate(&tm.e1));
    PG_CUDA(cudaEventRecord(tm.e0, stream));
    return b.read_columns(read_cols, names);
}

pg_status SectionFrame::place(const pg_file_desc *files, int n_files) {
    d_file.assign(n_files, nullptr);
    for (int f = 0; f < n_files; f++) {
        file_bytes += files[f].size;
        if (files[f].mem == PG_MEM_DEVICE) { d_file[f] = files[f].bytes; continue; }
        { pg_status st = file_image(scratch, files[f].bytes, files[f].size, b.who, &d_file[f]); if (st) return st; }
        h2d += files[f].size;
    }
    return PG_OK;
}

pg_status SectionFrame::finish(const int32_t *d_err, uint64_t *out_runs, pg_section_info *info) {
    PG_CUDA(cudaEventRecord(tm.e1, stream));
    int32_t herr = 0;
    SmallReads rb(stream);
    { pg_status rs = rb.add(&herr, d_err, 4); if (!rs) rs = rb.finish(); if (rs) return rs; }
    PG_CUDA(cudaGetLastError());
    { pg_status st = kernel_error(herr, b.who); if (st) return st; }
    b.finish(out_runs, h2d, info);
    if (info) {
        info->file_bytes = file_bytes;
        info->page_bytes = page_bytes;
        info->n_files = (int32_t)d_file.size();
        info->launches = launches;
        info->ms_decode = tm.ms();
    }
    return PG_OK;
}

// drop the current batch; the arena itself is kept for the next execute unless `release_memory`
static void free_outputs(Merge *m, bool release_memory = false) {
    m->out_cols.clear();
    m->has_batch = false;
    if (release_memory) {
        if (m->stream) cudaStreamSynchronize(m->stream);
        m->outbuf.release();
    }
}

// ------------------------------------------------------------------ plan-time validation

static bool agg_supports_retract(int agg) {
    return agg == PG_AGG_SUM || agg == PG_AGG_PRODUCT || agg == PG_AGG_LAST_VALUE ||
           agg == PG_AGG_LAST_NON_NULL_VALUE || agg == PG_AGG_PRIMARY_KEY;
}

static pg_status build_descriptors(Merge *m) {
    const Schema *s = m->spec->schema.get();
    const Spec *sp = m->spec.get();
    // primary key: a 64-bit order-preserving prefix lives in shared memory; keys that do not fit it exactly
    // (strings, binaries, composites wider than 8 bytes) fall back to a full comparison on prefix ties
    if (s->n_key < 1 || s->n_key > PG_MAX_KEY_FIELDS)
        return fail(PG_ERR_UNSUPPORTED, "more than 4 primary-key fields are not implemented on the device");
    m->key = KeyDesc{};
    m->key.n_fields = s->n_key;
    int key_bytes = 0;
    bool all_fixed = true;
    for (int f = 0; f < s->n_key; f++) {
        int t = s->key_fields[f].type;
        if (t == PG_FLOAT || t == PG_DOUBLE)
            return fail(PG_ERR_UNSUPPORTED, "FLOAT / DOUBLE primary keys are not implemented on the device "
                                            "(the reference's comparator treats NaN as equal to everything)");
        m->key.type[f] = t;
        m->key.width[f] = type_width(t);
        if (is_varlen(t)) all_fixed = false;
        key_bytes += type_width(t);
    }
    m->key.exact = all_fixed && key_bytes <= 8;
    // 'sequence.field': fixed-width value fields compared before _SEQUENCE_NUMBER
    m->seq = SeqFields{};
    if (sp->seq_fields.size() > 4)
        return fail(PG_ERR_UNSUPPORTED, "more than 4 'sequence.field' columns are not implemented on the device");
    for (size_t i = 0; i < sp->seq_fields.size(); i++) {
        int vf = sp->seq_fields[i];
        if (vf < 0 || vf >= s->n_val) return fail(PG_ERR_INVALID, "sequence.field index out of range");
        int t = s->val_fields[vf].type;
        if (is_varlen(t))
            return fail(PG_ERR_UNSUPPORTED, "var-len 'sequence.field' columns are not implemented on the device");
        m->seq.col[i] = s->n_key + 2 + vf;
        m->seq.type[i] = t;
        m->seq.width[i] = type_width(t);
    }
    m->seq.n = (int32_t)sp->seq_fields.size();
    m->seq.ascending = sp->seq_ascending ? 1 : 0;
    m->flags = MergeFlags{sp->engine, sp->ignore_delete, sp->remove_record_on_delete, sp->drop_delete};

    const int nc = s->n_cols();
    m->cols.assign(nc, ColDesc{});
    m->varlen_cols.clear();
    m->emit.assign(nc, 1);
    for (int c = s->n_key + 2; c < nc; c++)
        if (!sp->read_fields.empty() && !sp->read_fields[c - s->n_key - 2]) m->emit[c] = 0;
    // columns the kernels read: everything that is emitted, plus what the plan kernel compares
    std::vector<uint8_t> needed = m->emit;
    for (int32_t vf : sp->seq_fields) if (vf >= 0 && vf < s->n_val) needed[s->n_key + 2 + vf] = 1;
    for (int32_t vf : sp->group_seq_fields) if (vf >= 0 && vf < s->n_val) needed[s->n_key + 2 + vf] = 1;
    for (int r = 0; r < m->k; r++)
        for (int c = 0; c < nc; c++)
            if (needed[c] && m->runs[r]->n_rows > 0 && !m->runs[r]->cols[c].data && !m->runs[r]->cols[c].offsets)
                return fail(PG_ERR_INVALID, "run " + std::to_string(r) + " has no buffers for column " + std::to_string(c) +
                                            ", which the merge reads (read-type projection dropped a field the merge "
                                            "function compares or emits)");
    for (int c = 0; c < nc; c++) {
        pg_field f = s->field(c);
        ColDesc &cd = m->cols[c];
        cd.type = f.type;
        cd.width = type_width(f.type);
        cd.nullable = f.nullable;
        cd.agg = PG_AGG_NONE;
        cd.retract = RT_OK;
        cd.varlen_index = -1;
        cd.decimal = 0;
        if (is_varlen(f.type) && m->emit[c]) {
            cd.varlen_index = (int)m->varlen_cols.size();
            m->varlen_cols.push_back(c);
        }
        if (c < s->n_key) { cd.mode = CM_KEY; cd.nullable = 0; }
        else if (c == s->n_key) { cd.mode = CM_SEQ; cd.nullable = 0; }
        else if (c == s->n_key + 1) { cd.mode = CM_KIND; cd.nullable = 0; }
        else {
            int vi = c - s->n_key - 2;
            int agg = sp->agg.empty() ? PG_AGG_NONE : sp->agg[vi];
            bool ign = !sp->ignore_retract.empty() && sp->ignore_retract[vi];
            // DECIMAL(p, s) of the field for sum / product (the only aggregators whose result depends on it)
            const int32_t dec = sp->decimal.empty() ? 0 : sp->decimal[vi];
            const int32_t fold_dec = agg == PG_AGG_SUM || agg == PG_AGG_PRODUCT ? dec : 0;
            if (sp->engine == PG_ENGINE_AGGREGATE) {
                if (agg == PG_AGG_NONE) agg = PG_AGG_LAST_NON_NULL_VALUE;   // AggregateMergeFunction.java:199-202
                bool numeric = f.type == PG_INT8 || f.type == PG_INT16 || f.type == PG_INT32 ||
                               f.type == PG_INT64 || f.type == PG_FLOAT || f.type == PG_DOUBLE;
                if ((agg == PG_AGG_SUM || agg == PG_AGG_PRODUCT) && !numeric)
                    return fail(PG_ERR_INVALID, "sum/product need a numeric column");
                if ((agg == PG_AGG_BOOL_AND || agg == PG_AGG_BOOL_OR) && f.type != PG_BOOL)
                    return fail(PG_ERR_INVALID, "bool_and/bool_or need a BOOLEAN column");
                if ((agg == PG_AGG_MAX || agg == PG_AGG_MIN) && f.type == PG_BOOL)
                    return fail(PG_ERR_INVALID, "Incomparable type: BOOLEAN");
                if (agg < PG_AGG_SUM || agg > PG_AGG_PRIMARY_KEY)
                    return fail(PG_ERR_UNSUPPORTED, "aggregate function not implemented on the device");
                cd.mode = CM_FOLD;
                cd.agg = agg;
                cd.decimal = fold_dec;
                // an aggregator can produce NULL from non-null inputs (retract of last_value, ignored
                // retracts only, ...) and AggregateMergeFunction does not re-check NOT NULL: the output of a
                // folded column always carries a validity bitmap
                cd.nullable = 1;
                cd.retract = ign ? RT_IGNORE : (agg_supports_retract(agg) ? RT_OK : RT_ERROR);
            } else {
                const bool in_group = sp->n_groups() > 0 && sp->field_group[vi] >= 0;
                if (sp->engine == PG_ENGINE_PARTIAL_UPDATE && !in_group && agg != PG_AGG_NONE &&
                    agg != PG_AGG_LAST_NON_NULL_VALUE && agg != PG_AGG_PRIMARY_KEY)
                    return fail(PG_ERR_INVALID, "Must use sequence group for aggregation functions");
                cd.mode = CM_SELECT;
                if (sp->n_groups() > 0 && sp->field_group[vi] >= 0) {
                    const int g = sp->field_group[vi];
                    bool is_seq = false;
                    for (int j = sp->group_seq_start[g]; j < sp->group_seq_start[g + 1]; j++)
                        if (sp->group_seq_fields[j] == vi) is_seq = true;
                    cd.mode = is_seq ? CM_GSEQ : CM_GVAL;
                    cd.agg = g;
                    cd.nullable = 1;                // a retract NULLs the group's fields whatever the schema says
                    if (!is_seq && agg != PG_AGG_NONE) {
                        // a group field with an aggregate function (PartialUpdateMergeFunction.java:228-244)
                        cd.mode = CM_GAGG;
                        cd.agg = agg;
                        cd.decimal = fold_dec;
                        cd.group = g;
                        cd.retract = ign ? RT_IGNORE : (agg_supports_retract(agg) ? RT_OK : RT_ERROR);
                        m->has_group_aggs = true;
                    }
                }
            }
        }
    }

    // one device allocation for all descriptor arrays, filled through a host mirror of the same layout
    const int k = m->k, nk = s->n_key, nv = (int)m->varlen_cols.size();
    MergeDesc h;
    const size_t total = h.carve(nullptr, k, nk, nc, nv);
    std::vector<unsigned char> host(total, 0);
    h.carve(host.data(), k, nk, nc, nv);
    m->varlen_bound.assign(nv, 0);
    for (int r = 0; r < k; r++) {
        const Run *run = m->runs[r].get();
        for (int f = 0; f < nk; f++) {
            h.key_ptrs[r * nk + f] = run->cols[f].data;
            h.key_offs[r * nk + f] = run->cols[f].offsets;
        }
        h.seq_ptrs[r] = (const int64_t *)run->cols[nk].data;
        h.kind_ptrs[r] = (const int8_t *)run->cols[nk + 1].data;
        for (int c = 0; c < nc; c++) {
            h.data[(size_t)c * k + r] = run->cols[c].data;
            h.offsets[(size_t)c * k + r] = run->cols[c].offsets;
            h.validity[(size_t)c * k + r] = (const uint32_t *)run->cols[c].validity;
            if (m->cols[c].varlen_index >= 0) m->varlen_bound[m->cols[c].varlen_index] += run->varlen_bytes[c];
        }
        h.run_rows[r] = run->n_rows;
    }
    memcpy(h.cols, m->cols.data(), sizeof(ColDesc) * nc);
    {
        // the emit kernel's pass list: var-len columns first (their cross-tile look-back then happens while the CTAs of
        // a wave are still close together in time), then everything else; columns the read type leaves out are skipped
        int n = 0;
        for (int c = 0; c < nc; c++) if (m->emit[c] && m->cols[c].width == 0) h.col_order[n++] = c;
        for (int c = 0; c < nc; c++) if (m->emit[c] && m->cols[c].width != 0) h.col_order[n++] = c;
        m->n_passes = n;
        for (int v = 0; v < nv; v++) h.varlen_cols[v] = m->varlen_cols[v];
    }
    if (sp->n_groups() > 0) {
        SeqGroups *sg = h.groups;
        sg->n = sp->n_groups();
        for (int g = 0; g <= sg->n; g++) sg->start[g] = sp->group_seq_start[g];
        for (int j = 0; j < sp->group_seq_start[sg->n]; j++) {
            const int vf = sp->group_seq_fields[j];
            sg->col[j] = s->n_key + 2 + vf;
            sg->type[j] = s->val_fields[vf].type;
            sg->width[j] = type_width(s->val_fields[vf].type);
        }
        for (int g = 0; g < sg->n; g++) sg->partial_delete[g] = sp->group_partial_delete[g];
    }
    if (!m->d_desc || total > m->desc_cap) {
        if (m->d_desc) cudaFree(m->d_desc);
        m->d_desc = nullptr;
        PG_CUDA(cudaMalloc(&m->d_desc, total));
        m->desc_cap = total;
    }
    { pg_status ts = small_h2d(m->d_desc, host.data(), total, m->stream); if (ts) return ts; }
    PG_CUDA(cudaStreamSynchronize(m->stream));
    m->desc.carve(m->d_desc, k, nk, nc, nv);
    if (sp->n_groups() == 0) m->desc.groups = nullptr;        // (the plan kernel's test for sequence groups)
    if (!m->h_totals) PG_CUDA(cudaMallocHost((void **)&m->h_totals, sizeof(int64_t) * (nv + 1) + 16));
    m->h_err = (int32_t *)(m->h_totals + nv + 1);
    return PG_OK;
}

pg_status kernel_error(int code, const char *who) {
    static const struct { int code; pg_status st; const char *msg; } kErrors[] = {
        // what the Java merge functions throw, verbatim
        {KERR_PU_DELETE, PG_ERR_MERGE_FUNCTION,
         "By default, Partial update can not accept delete records, you can choose one of the "
         "following solutions:\n1. Configure 'ignore-delete' to ignore delete records.\n"
         "2. Configure 'partial-update.remove-record-on-delete' to remove the whole row when "
         "receiving delete records.\n3. Configure 'sequence-group's to retract partial columns. "
         "Also configure 'partial-update.remove-record-on-sequence-group' to remove the whole "
         "row when receiving deleted records of `specified sequence group`."},
        {KERR_FIRST_ROW_RETRACT, PG_ERR_MERGE_FUNCTION,
         "By default, First row merge engine can not accept DELETE/UPDATE_BEFORE records.\n"
         "You can config 'ignore-delete' to ignore the DELETE/UPDATE_BEFORE records."},
        {KERR_AGG_RETRACT, PG_ERR_MERGE_FUNCTION,
         "Aggregate function does not support retraction, If you allow this function to ignore "
         "retraction messages, you can configure 'fields.${field_name}.ignore-retract'='true'."},
        {KERR_DIV_ZERO, PG_ERR_MERGE_FUNCTION, "ArithmeticException: / by zero"},
        {KERR_DEC_DIV_ZERO, PG_ERR_MERGE_FUNCTION, "ArithmeticException: Division by zero"},
        {KERR_DEC_DIV_UNDEFINED, PG_ERR_MERGE_FUNCTION, "ArithmeticException: Division undefined"},
        {KERR_DEC_NON_TERMINATING, PG_ERR_MERGE_FUNCTION,
         "ArithmeticException: Non-terminating decimal expansion; no exact representable decimal result."},
        // limits of the device path
        {KERR_TILE_OVERFLOW, PG_ERR_INTERNAL,
         "a merge tile overflowed (does a run contain duplicate keys? SortMergeReader.java:37 requires unique keys per reader)"},
        {KERR_OFFSET_OVERFLOW, PG_ERR_INTERNAL, "a var-len column exceeds 2 GiB of payload"},
        // file bytes
        {KERR_BAD_PAGE, PG_ERR_FORMAT, "a page or stream does not decode (malformed file or unsupported encoding)"},
        {KERR_PQ_HEADER, PG_ERR_FORMAT, "malformed or truncated page header"},
        {KERR_PQ_NO_DICT, PG_ERR_FORMAT, "dictionary-encoded page without dictionary"},
        {KERR_PQ_ROWS, PG_ERR_FORMAT, "page row counts do not add up"},
        {KERR_PQ_DICT_ID, PG_ERR_FORMAT, "dictionary id outside the dictionary"},
        {KERR_PQ_ENCODING, PG_ERR_UNSUPPORTED,
         "a page uses a value encoding the device decoder does not implement (PLAIN, dictionary, DELTA_BINARY_PACKED "
         "integers and RLE booleans are decoded)"},
        {KERR_PQ_LEVELS, PG_ERR_UNSUPPORTED, "repetition levels / BIT_PACKED definition levels are not decoded on device"},
    };
    if (code == KERR_NONE) return PG_OK;
    for (const auto &e : kErrors)
        if (e.code == code) return fail(e.st, e.st == PG_ERR_MERGE_FUNCTION ? std::string(e.msg) : std::string(who) + ": " + e.msg);
    return fail(PG_ERR_INTERNAL, std::string(who) + ": unknown kernel error " + std::to_string(code));
}

// ------------------------------------------------------------------ one merge

static pg_status execute(Merge *m) {
    pg_status st = ensure_device();
    if (st) return st;
    cudaStream_t sm = m->stream;
    PG_HOST_MARKS("merge execute");
    free_outputs(m);
    for (size_t r = m->runs.size(); r < m->bound.size(); r++)     // a re-execute takes the merged runs back
        if (!m->runs.emplace_back(m->bound[r].lock())) {
            m->runs.clear();
            return fail(PG_ERR_INVALID, "a run of this merge has been freed since it was merged: rebind first");
        }
    const Schema *s = m->spec->schema.get();
    const int k = m->k, nc = s->n_cols(), nv = (int)m->varlen_cols.size();
    m->stats = pg_stats{};
    m->stats.rows_in = m->n_in;
    int launches = 0;

    // ---- level sizes
    const int S = kSampleStride;
    const int q = kPlanTile / S - 2 * k;
    if (q < 1) return fail(PG_ERR_UNSUPPORTED, "too many runs for one merge call");
    std::vector<LevelView> views;
    std::vector<int64_t> level_total;
    {
        int64_t stride = 1;
        while (true) {
            LevelView lv{};
            lv.stride = stride;
            int64_t tot = 0;
            for (int r = 0; r < k; r++) {
                lv.row0[r] = m->row0[r];
                lv.count[r] = (m->runs[r]->n_rows - m->row0[r]) / stride;
                tot += lv.count[r];
            }
            views.push_back(lv);
            level_total.push_back(tot);
            if (tot <= kPlanTile) break;
            stride *= S;
        }
    }
    const int top = (int)views.size() - 1;
    std::vector<int> n_tiles(top + 1);
    n_tiles[top] = 1;
    for (int l = top - 1; l >= 0; l--) n_tiles[l] = (int)((level_total[l + 1] + q - 1) / q);
    m->stats.n_levels = top;
    m->stats.n_tiles = n_tiles[0];

    PG_CUDA(cudaMemsetAsync(m->desc.err, 0, sizeof(int32_t), sm));
    PG_CUDA(cudaEventRecord(m->ev[0], sm));

    MergeLaunch ml{k, m->key, KeySrc{m->desc.key_ptrs, m->desc.key_offs}, sm, m->desc.err, nullptr};
    // Workspace: one grow-only device allocation per merge handle.  Its size depends only on the input shapes, so a
    // reader that is executed repeatedly (or a pool of readers of one bucket layout) never goes back to the driver
    // allocator.  The plan-sized arrays are indexed by sums of absolute rows (N counts the rows a rebind skips) and
    // keep 16 bytes behind their last entry.
    const int T = n_tiles[0];
    int64_t N = m->n_in;
    for (int r = 0; r < k; r++) N += m->row0[r];
    int *d_skip = nullptr;
    std::vector<int64_t *> bounds(top + 1);
    std::vector<uint64_t *> sk(top + 1), sref(top + 1);   // level l > 0: its sorted keys, and the rows they came from
    uint16_t *plan = nullptr;
    uint32_t *gplan = nullptr, *gagg = nullptr;
    int32_t *tile_rows = nullptr;
    int64_t *tmp_seq = nullptr, *row_base = nullptr;
    int8_t *tmp_kind = nullptr;
    uint64_t *vl_state = nullptr;
    const size_t vl_words = (size_t)T * std::max(nv, 1);
    auto carve_work = [&](void *base) {
        Carver cv(base);
        if (!m->key.exact) d_skip = cv.take<int>(1);
        for (int l = top; l >= 0; l--) {
            bounds[l] = cv.take<int64_t>((size_t)(n_tiles[l] + 1) * k);
            if (l > 0) {
                sk[l] = cv.take<uint64_t>((size_t)std::max<int64_t>(level_total[l], 1));
                sref[l] = cv.take<uint64_t>((size_t)std::max<int64_t>(level_total[l], 1));
            }
        }
        plan = cv.take<uint16_t>((size_t)N + 8);
        if (m->desc.groups) gplan = cv.take<uint32_t>((size_t)N + 4);
        if (m->has_group_aggs) gagg = cv.take<uint32_t>((size_t)N + 4);
        tile_rows = cv.take<int32_t>(T);
        tmp_seq = cv.take<int64_t>((size_t)N + 2);
        tmp_kind = cv.take<int8_t>((size_t)N + 16);
        row_base = cv.take<int64_t>(T);
        vl_state = cv.take<uint64_t>(vl_words);
        return cv.bytes();
    };
    PG_CUDA(m->work.reserve(carve_work(nullptr)));
    carve_work(m->work.base);

    if (!m->key.exact) {
        // window keys start behind the prefix all keys share (strings like "user_0000123", wide composites)
        launch_key_lcp(ml, views[0], d_skip);
        ml.skip = d_skip;
        launches++;
    }
    for (int l = top; l >= 0; l--) {
        // the sorted sample keys of the level above split this one
        launch_partition(ml, views[l], l < top ? sk[l + 1] : nullptr, l < top ? sref[l + 1] : nullptr, q, n_tiles[l],
                         bounds[l]);
        launches++;
        if (l > 0) {
            launch_merge_keys(ml, views[l], bounds[l], n_tiles[l], sk[l], sref[l]);
            launches++;
        }
    }
    PG_CUDA(cudaEventRecord(m->ev[1], sm));

    // ---- plan + scan
    PG_CUDA(cudaMemsetAsync(vl_state, 0, sizeof(uint64_t) * vl_words, sm));
    PG_CUDA(cudaMemsetAsync(m->desc.tile_counter, 0, sizeof(int32_t), sm));

    PlanArgs pa{};
    pa.bounds = bounds[0];
    pa.n_tiles = T;
    pa.seq_ptrs = m->desc.seq_ptrs;
    pa.kind_ptrs = m->desc.kind_ptrs;
    pa.flags = m->flags;
    pa.seq = m->seq;
    pa.ptrs = m->desc.ptrs();
    pa.plan = plan;
    pa.tile_rows = tile_rows;
    pa.tmp_seq = tmp_seq;
    pa.tmp_kind = tmp_kind;
    pa.groups = m->desc.groups;
    pa.gplan = gplan;
    pa.gagg = gagg;
    launch_plan(ml, pa);
    launch_scan(sm, tile_rows, T, row_base, m->desc.totals);
    launches += 2;
    PG_CUDA(cudaEventRecord(m->ev[2], sm));
    PG_HOST_MARK("enqueue");
    {
        SmallReads rb(sm);                   // the one size read-back: output buffers are sized exactly
        pg_status rs = rb.add(m->h_totals, m->desc.totals, sizeof(int64_t));
        if (!rs) rs = rb.add(m->h_err, m->desc.err, sizeof(int32_t));
        if (!rs) rs = rb.finish();
        if (rs) return rs;
    }
    if (*m->h_err != KERR_NONE) return kernel_error(*m->h_err, "merge");
    PG_HOST_MARK("size_readback");

    // ---- output buffers
    const int64_t n_out = m->h_totals[0];
    m->n_out = n_out;
    m->out_cols.assign(nc, pg_out_column{});
    // output arena (grow-only, reused until pg_merge_release): the validity bitmaps first and contiguous, so that one
    // memset clears them all, then per column its values, or its var-len payload and offsets.  The exact payload size
    // is only known after the emit kernel's look-back; every output cell is one input cell, so the runs' payload bytes
    // bound it.
    size_t vspan = 0;                                    // the bitmaps: [0, vspan)
    int64_t bytes_out = 0;
    auto carve_out = [&](void *base) {
        Carver cv(base);
        bytes_out = 0;
        for (int c = 0; c < nc; c++)
            if (m->cols[c].nullable && m->emit[c]) {
                m->out_cols[c].validity = cv.take<uint8_t>((size_t)((n_out + 31) / 32) * 4 + kReadPast);
                bytes_out += (n_out + 7) / 8;
            }
        vspan = cv.bytes();
        for (int c = 0; c < nc; c++) {
            const ColDesc &cd = m->cols[c];
            pg_out_column &oc = m->out_cols[c];
            if (!m->emit[c]) continue;                       // not part of the read type: the batch has no such column
            if (cd.width > 0) {
                oc.data_bytes = n_out * cd.width;
                oc.data = cv.take<uint8_t>((size_t)oc.data_bytes + kReadPast);
                bytes_out += oc.data_bytes;
            } else {
                oc.data_bytes = m->varlen_bound[cd.varlen_index];
                oc.data = cv.take<uint8_t>((size_t)oc.data_bytes + kReadPast);
                oc.offsets = cv.take<int32_t>((size_t)n_out + 1 + kReadPast / 4);
                bytes_out += 4 * (n_out + 1);
            }
        }
        return cv.bytes();
    };
    PG_CUDA(m->outbuf.reserve(carve_out(nullptr)));
    carve_out(m->outbuf.base);
    if (vspan) PG_CUDA(cudaMemsetAsync(m->outbuf.base, 0, vspan, sm));
    m->stats.bytes_out = bytes_out;
    { pg_status ts = small_h2d(m->desc.out_cols, m->out_cols.data(), sizeof(pg_out_column) * nc, sm); if (ts) return ts; }

    // ---- emit
    EmitArgs ea{};
    ea.bounds = bounds[0];
    ea.n_tiles = (T + 1) / 2;
    ea.n_plan_tiles = T;
    ea.tile_rows = tile_rows;
    ea.k = k;
    ea.plan = plan;
    ea.row_base = row_base;
    ea.tmp_seq = tmp_seq;
    ea.tmp_kind = tmp_kind;
    ea.gplan = gplan;
    ea.gagg = gagg;
    ea.cols = m->desc.cols;
    ea.col_order = m->desc.col_order;
    ea.n_passes = m->n_passes;
    ea.varlen_cols = m->desc.varlen_cols;
    ea.ptrs = m->desc.ptrs();
    ea.run_rows = m->desc.run_rows;
    ea.n_cols = nc;
    ea.n_varlen = nv;
    ea.out_cols = m->desc.out_cols;
    ea.totals = m->desc.totals;
    ea.vl_state = vl_state;
    ea.tile_counter = m->desc.tile_counter;
    ea.err = m->desc.err;
    ea.stream = sm;
    PG_CUDA(cudaEventRecord(m->ev[4], sm));
    launch_emit(ea);
    launches++;
    PG_CUDA(cudaEventRecord(m->ev[3], sm));
    PG_HOST_MARK("alloc_emit");
    {
        SmallReads rb(sm);
        pg_status rs = rb.add(m->h_err, m->desc.err, sizeof(int32_t));
        if (!rs) rs = rb.add(m->h_totals, m->desc.totals, sizeof(int64_t) * (nv + 1));
        if (!rs) rs = rb.finish();
        if (rs) return rs;
    }
    PG_CUDA(cudaGetLastError());
    PG_HOST_MARK("emit_readback");
    m->has_batch = true;
    if (*m->h_err != KERR_NONE) {
        free_outputs(m);
        return kernel_error(*m->h_err, "merge");
    }
    for (int c = 0; c < nc; c++)
        if (m->cols[c].width == 0 && m->emit[c]) {
            m->out_cols[c].data_bytes = m->h_totals[1 + m->cols[c].varlen_index];
            m->stats.bytes_out += m->out_cols[c].data_bytes;
        }
    m->stats.rows_out = n_out;
    m->stats.launches = launches;
    cudaEventElapsedTime(&m->stats.ms_partition, m->ev[0], m->ev[1]);
    cudaEventElapsedTime(&m->stats.ms_plan, m->ev[1], m->ev[2]);
    cudaEventElapsedTime(&m->stats.ms_alloc, m->ev[2], m->ev[4]);
    cudaEventElapsedTime(&m->stats.ms_emit, m->ev[4], m->ev[3]);
    cudaEventElapsedTime(&m->stats.ms_total, m->ev[0], m->ev[3]);
    // The read-back above waited for the kernels, so the runs may go: a reader that frees them before it decodes the
    // next section gets their buffers back at once, instead of holding two sections' runs per merge handle.
    m->runs.clear();
    return PG_OK;
}

}  // namespace pg

// ====================================================================== C ABI

using namespace pg;

extern "C" {

const char *pg_last_error(void) { return g_last_error.c_str(); }
int32_t pg_abi_version(void) { return PG_ABI_VERSION; }

pg_status pg_init(int32_t device_ordinal) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(PG_ERR_CUDA, std::string("no CUDA device: libpaimon_gpu has no CPU fallback (") +
                                     cudaGetErrorString(e) + ")");
    if (device_ordinal < 0 || device_ordinal >= n) return fail(PG_ERR_INVALID, "bad device ordinal");
    if (g_device >= 0 && g_device != device_ordinal)
        return fail(PG_ERR_INVALID, "pg_init: this process is already bound to device " + std::to_string(g_device) +
                                    " (one process per GPU: handles, streams and cached buffers belong to it)");
    PG_CUDA(cudaSetDevice(device_ordinal));
    g_device = device_ordinal;
    cudaMemPool_t pool;
    PG_CUDA(cudaDeviceGetDefaultMemPool(&pool, device_ordinal));
    uint64_t thr = UINT64_MAX;                 // keep freed blocks cached: steady-state merges do not hit the driver
    PG_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    return PG_OK;
}

pg_status pg_shutdown(void) {
    if (g_device >= 0) {
        cudaSetDevice(g_device);
        cudaDeviceSynchronize();
        buf_trim(0);
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, g_device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
    }
    return PG_OK;
}

pg_status pg_schema_create(const pg_schema_desc *desc, uint64_t *out_schema) {
    if (!desc || !out_schema) return fail(PG_ERR_INVALID, "null argument");
    if (desc->n_key < 1 || desc->n_val < 0 || desc->n_key + 2 + desc->n_val > kMaxCols)
        return fail(PG_ERR_INVALID, "bad field counts");
    auto s = std::make_unique<Schema>();
    s->n_key = desc->n_key;
    s->n_val = desc->n_val;
    for (int i = 0; i < desc->n_key; i++) {
        if (!type_ok(desc->key_fields[i].type)) return fail(PG_ERR_INVALID, "bad key field type");
        s->key_fields.push_back(pg_field{desc->key_fields[i].type, 0});
    }
    for (int i = 0; i < desc->n_val; i++) {
        if (!type_ok(desc->val_fields[i].type)) return fail(PG_ERR_INVALID, "bad value field type");
        s->val_fields.push_back(desc->val_fields[i]);
    }
    *out_schema = g_schemas.put(std::move(s));
    return PG_OK;
}

pg_status pg_schema_info(uint64_t schema, int32_t *n_key, int32_t *n_val) {
    std::shared_ptr<Schema> s = g_schemas.get(schema);
    if (!s) return fail(PG_ERR_INVALID, "unknown schema handle");
    if (n_key) *n_key = s->n_key;
    if (n_val) *n_val = s->n_val;
    return PG_OK;
}

pg_status pg_schema_free(uint64_t schema) {
    return g_schemas.take(schema) ? PG_OK : fail(PG_ERR_INVALID, "unknown schema handle");
}

pg_status pg_merge_spec_create(uint64_t schema, const pg_merge_spec *spec, uint64_t *out_spec) {
    std::shared_ptr<Schema> s = g_schemas.get(schema);
    if (!s || !spec || !out_spec) return fail(PG_ERR_INVALID, "bad schema handle or null argument");
    if (spec->engine < PG_ENGINE_DEDUPLICATE || spec->engine > PG_ENGINE_FIRST_ROW)
        return fail(PG_ERR_INVALID, "Unsupported merge engine");
    if (spec->n_sequence_groups < 0 || (spec->n_sequence_groups > 0 && (!spec->group_seq_start ||
                                                                         !spec->group_seq_fields || !spec->field_group)))
        return fail(PG_ERR_INVALID, "bad sequence group description");
    if (spec->n_sequence_groups > 0 && spec->engine != PG_ENGINE_PARTIAL_UPDATE)
        return fail(PG_ERR_INVALID, "sequence groups belong to the partial-update merge engine");
    if (spec->n_sequence_groups > PG_MAX_SEQ_GROUPS)
        return fail(PG_ERR_UNSUPPORTED, "more than 16 sequence groups are not implemented on the device");
    auto sp = std::make_unique<Spec>();
    sp->schema = s;
    sp->engine = spec->engine;
    sp->ignore_delete = spec->ignore_delete != 0;
    sp->remove_record_on_delete = spec->remove_record_on_delete != 0;
    sp->drop_delete = spec->drop_delete != 0;
    sp->seq_ascending = spec->seq_ascending;
    if (spec->n_seq_fields < 0 || (spec->n_seq_fields > 0 && !spec->seq_fields))
        return fail(PG_ERR_INVALID, "bad sequence.field description");
    for (int i = 0; i < spec->n_seq_fields; i++) {
        if (spec->seq_fields[i] < 0 || spec->seq_fields[i] >= s->n_val) return fail(PG_ERR_INVALID, "sequence.field index out of range");
        sp->seq_fields.push_back(spec->seq_fields[i]);
    }
    if (spec->agg) sp->agg.assign(spec->agg, spec->agg + s->n_val);
    if (spec->ignore_retract) sp->ignore_retract.assign(spec->ignore_retract, spec->ignore_retract + s->n_val);
    if (spec->read_fields) sp->read_fields.assign(spec->read_fields, spec->read_fields + s->n_val);
    if (spec->decimal) {
        sp->decimal.assign(spec->decimal, spec->decimal + s->n_val);
        for (int f = 0; f < s->n_val; f++) {
            const int32_t d = sp->decimal[f];
            if (d == 0) continue;
            const int p = d >> 8, sc = d & 0xff;
            if (p > 18)
                return fail(PG_ERR_UNSUPPORTED, "DECIMAL(p > 18) is not implemented on the device (field " +
                                                    std::to_string(f) + ")");
            if (p < 1 || sc > p || s->val_fields[f].type != PG_INT64)
                return fail(PG_ERR_INVALID, "bad DECIMAL description of value field " + std::to_string(f) +
                                                " (precision 1..18, scale <= precision, an INT64 column)");
        }
    }
    if (spec->n_sequence_groups > 0) {
        const int ng = spec->n_sequence_groups;
        sp->group_seq_start.assign(spec->group_seq_start, spec->group_seq_start + ng + 1);
        sp->group_seq_fields.assign(spec->group_seq_fields, spec->group_seq_fields + sp->group_seq_start[ng]);
        sp->field_group.assign(spec->field_group, spec->field_group + s->n_val);
        sp->group_partial_delete.assign(ng, 0);
        for (int g = 0; g < ng; g++) {
            const int n = sp->group_seq_start[g + 1] - sp->group_seq_start[g];
            if (n < 1) return fail(PG_ERR_INVALID, "a sequence group needs a sequence field");
            if (n > 4)
                return fail(PG_ERR_UNSUPPORTED, "more than 4 sequence fields in one sequence group are not "
                                                "implemented on the device");
            for (int j = sp->group_seq_start[g]; j < sp->group_seq_start[g + 1]; j++) {
                const int f = sp->group_seq_fields[j];
                if (f < 0 || f >= s->n_val) return fail(PG_ERR_INVALID, "sequence group field out of range");
                if (is_varlen(s->val_fields[f].type))
                    return fail(PG_ERR_UNSUPPORTED, "var-len sequence-group fields are not implemented on the device");
                if (spec->group_partial_delete && spec->group_partial_delete[f]) sp->group_partial_delete[g] = 1;
            }
        }
        for (int f = 0; f < s->n_val; f++) {
            if (sp->field_group[f] < -1 || sp->field_group[f] >= ng)
                return fail(PG_ERR_INVALID, "field_group out of range");
            if (sp->field_group[f] >= 0 && !sp->agg.empty() && sp->agg[f] != PG_AGG_NONE) {
                const int agg = sp->agg[f], t = s->val_fields[f].type;
                if (is_varlen(t))
                    return fail(PG_ERR_UNSUPPORTED, "aggregate functions on var-len fields inside a sequence group "
                                                    "are not implemented on the device");
                if (agg < PG_AGG_SUM || agg > PG_AGG_PRIMARY_KEY)
                    return fail(PG_ERR_UNSUPPORTED, "aggregate function not implemented on the device");
                const bool numeric = t == PG_INT8 || t == PG_INT16 || t == PG_INT32 || t == PG_INT64 ||
                                     t == PG_FLOAT || t == PG_DOUBLE;
                if ((agg == PG_AGG_SUM || agg == PG_AGG_PRODUCT) && !numeric)
                    return fail(PG_ERR_INVALID, "sum/product need a numeric column");
                if ((agg == PG_AGG_BOOL_AND || agg == PG_AGG_BOOL_OR) && t != PG_BOOL)
                    return fail(PG_ERR_INVALID, "bool_and/bool_or need a BOOLEAN column");
            }
        }
    }
    if (sp->engine == PG_ENGINE_PARTIAL_UPDATE && sp->ignore_delete && sp->remove_record_on_delete)
        return fail(PG_ERR_INVALID, "ignore-delete and partial-update.remove-record-on-delete have conflicting "
                                    "behavior so should not be enabled at the same time.");
    *out_spec = g_specs.put(std::move(sp));
    return PG_OK;
}

pg_status pg_merge_spec_free(uint64_t spec) {
    return g_specs.take(spec) ? PG_OK : fail(PG_ERR_INVALID, "unknown spec handle");
}

pg_status pg_trim(void) {
    buf_trim(0);
    return PG_OK;
}

pg_status pg_run_open(uint64_t schema, const pg_run_desc *desc, int32_t mem, uint64_t *out_run) {
    std::shared_ptr<Schema> s = g_schemas.get(schema);
    if (!s || !desc || !out_run) return fail(PG_ERR_INVALID, "bad schema handle or null argument");
    if (desc->n_rows < 0 || desc->n_rows > 0x7fffffffLL) return fail(PG_ERR_INVALID, "bad row count");
    pg_status st = ensure_device();
    if (st) return st;
    auto run = std::make_unique<Run>(s, desc->n_rows);
    const int nc = s->n_cols();
    const int64_t n = desc->n_rows;
    if (mem == PG_MEM_DEVICE) {
        for (int c = 0; c < nc; c++) {
            const pg_column &pc = desc->cols[c];
            if ((((uintptr_t)pc.data) | ((uintptr_t)pc.offsets) | ((uintptr_t)pc.validity)) & 15)
                return fail(PG_ERR_INVALID, "device column buffers must be 16-byte aligned");
            run->cols[c] = DevColumn{pc.data, pc.offsets, pc.validity};
            if (is_varlen(s->field(c).type) && n > 0) {
                if (!pc.offsets) return fail(PG_ERR_INVALID, "var-len column without offsets");
                // offsets may start anywhere, `data` is byte 0 of their space: one read of offsets[0] and offsets[n]
                int32_t b[2] = {0, 0};
                PG_CUDA(cudaMemcpy2D(b, sizeof(int32_t), pc.offsets, sizeof(int32_t) * (size_t)n, sizeof(int32_t), 2,
                                     cudaMemcpyDeviceToHost));
                if (b[1] < b[0]) return fail(PG_ERR_INVALID, "decreasing offsets");
                run->varlen_base[c] = b[0];
                run->varlen_bytes[c] = b[1] - b[0];
            }
        }
    } else if (mem == PG_MEM_HOST) {
        // one device allocation per run, columns sub-allocated at 256-byte boundaries
        std::vector<size_t> o_data(nc), o_off(nc), o_val(nc), b_data(nc), b_off(nc), b_val(nc);
        size_t total = 0;
        for (int c = 0; c < nc; c++) {
            pg_field f = s->field(c);
            const pg_column &pc = desc->cols[c];
            if (is_varlen(f.type)) {
                if (n > 0 && !pc.offsets) return fail(PG_ERR_INVALID, "var-len column without offsets");
                b_off[c] = sizeof(int32_t) * (size_t)(n + 1);
                // offsets may start anywhere (a slice of a longer run): only [offsets[0], offsets[n]) is copied
                if (n > 0 && pc.offsets[n] < pc.offsets[0]) return fail(PG_ERR_INVALID, "decreasing offsets");
                b_data[c] = n > 0 ? (size_t)(pc.offsets[n] - pc.offsets[0]) : 0;
                run->varlen_base[c] = n > 0 ? pc.offsets[0] : 0;
            } else {
                b_off[c] = 0;
                b_data[c] = (size_t)n * type_width(f.type);
            }
            b_val[c] = pc.validity ? (size_t)((n + 7) / 8) : 0;
            o_data[c] = total; total += align256(b_data[c] + 16);
            o_off[c] = total; total += align256(b_off[c]);
            o_val[c] = total; total += align256(b_val[c] + 8);
        }
        cudaStream_t cs = copy_stream();
        Scratch scratch(cs);                          // the run's buffer until its copies are done
        unsigned char *d = (unsigned char *)scratch.take(total + 256);
        if (!d) return fail(PG_ERR_CUDA, "out of device memory for a run");
        std::vector<void *> cp_dst, cp_src;
        std::vector<size_t> cp_size;
        auto add_copy = [&](void *dst, const void *src, size_t bytes) {
            cp_dst.push_back(dst); cp_src.push_back(const_cast<void *>(src)); cp_size.push_back(bytes);
        };
        for (int c = 0; c < nc; c++) {
            const pg_column &pc = desc->cols[c];
            DevColumn dc;
            // var-len: `data` stays the address of byte 0 of the offsets' space
            dc.data = d + o_data[c] - run->varlen_base[c];
            if (b_data[c]) add_copy(d + o_data[c], (const unsigned char *)pc.data + run->varlen_base[c], b_data[c]);
            if (b_off[c]) {
                dc.offsets = (const int32_t *)(d + o_off[c]);
                if (n >= 0 && pc.offsets) add_copy(d + o_off[c], pc.offsets, b_off[c]);
            }
            if (b_val[c]) {
                dc.validity = d + o_val[c];
                add_copy(d + o_val[c], pc.validity, b_val[c]);
            }
            run->bytes_h2d += (int64_t)(b_data[c] + b_off[c] + b_val[c]);
            if (is_varlen(s->field(c).type)) run->varlen_bytes[c] = (int64_t)b_data[c];
            run->cols[c] = dc;
        }
        pg_status cst = copy_batch(cp_dst, cp_src, cp_size, cudaMemcpyHostToDevice, cs);
        if (cst) return cst;
        PG_CUDA(cudaStreamSynchronize(cs));
        run->bufs.swap(scratch.bufs);
    } else {
        return fail(PG_ERR_INVALID, "bad memory kind");
    }
    *out_run = g_runs.put(std::move(run));
    return PG_OK;
}

pg_status pg_run_free(uint64_t run) {
    return g_runs.take(run) ? PG_OK : fail(PG_ERR_INVALID, "unknown run handle");
}

pg_status pg_run_layout(uint64_t run, int64_t *n_rows, int64_t *data_bytes, int32_t *has_validity, int32_t n_cols) {
    std::shared_ptr<Run> r = g_runs.get(run);
    if (!r || !n_rows) return fail(PG_ERR_INVALID, "unknown run handle");
    const int nc = r->schema->n_cols();
    if (n_cols != nc) return fail(PG_ERR_INVALID, "column count mismatch");
    *n_rows = r->n_rows;
    for (int c = 0; c < nc; c++) {
        pg_field f = r->schema->field(c);
        const bool absent = !r->cols[c].data && !r->cols[c].offsets;      // not decoded (read-type projection)
        if (data_bytes) data_bytes[c] = absent ? -1 : (is_varlen(f.type) ? r->varlen_bytes[c] : r->n_rows * type_width(f.type));
        if (has_validity) has_validity[c] = r->cols[c].validity != nullptr;
    }
    return PG_OK;
}

pg_status pg_run_fetch(uint64_t run, const pg_out_column *host_cols, int32_t n_cols) {
    std::shared_ptr<Run> r = g_runs.get(run);
    if (!r || !host_cols) return fail(PG_ERR_INVALID, "unknown run handle");
    const int nc = r->schema->n_cols();
    if (n_cols != nc) return fail(PG_ERR_INVALID, "column count mismatch");
    pg_status st = ensure_device();
    if (st) return st;
    const int64_t n = r->n_rows;
    for (int c = 0; c < nc && n > 0; c++) {
        pg_field f = r->schema->field(c);
        const DevColumn &dc = r->cols[c];
        const pg_out_column &hc = host_cols[c];
        size_t db = is_varlen(f.type) ? (size_t)r->varlen_bytes[c] : (size_t)n * type_width(f.type);
        if (!dc.data && !dc.offsets) continue;           // column not decoded (read-type projection)
        if (db && hc.data && (size_t)hc.data_bytes < db)
            return fail(PG_ERR_INVALID, "pg_run_fetch: data buffer of column " + std::to_string(c) + " is too small");
        if (db && hc.data)
            PG_CUDA(cudaMemcpy(hc.data, (const unsigned char *)dc.data + (c < (int)r->varlen_base.size() ? r->varlen_base[c] : 0),
                               db, cudaMemcpyDeviceToHost));
        if (dc.offsets && hc.offsets)
            PG_CUDA(cudaMemcpy(hc.offsets, dc.offsets, sizeof(int32_t) * (size_t)(n + 1), cudaMemcpyDeviceToHost));
        if (dc.validity && hc.validity)
            PG_CUDA(cudaMemcpy(hc.validity, dc.validity, (size_t)((n + 7) / 8), cudaMemcpyDeviceToHost));
    }
    return PG_OK;
}

}  // extern "C"

// a view of rows [row_lo & ~127, row_hi) of a run or of a merge handle's batch: no copy, the columns point into the
// source's buffers (128 rows keep every buffer 16-byte aligned: 1-byte values, 4-byte offsets, 1-bit validity)
static pg_status make_slice(uint64_t source, int64_t row_lo, int64_t row_hi, uint64_t *out_run, int64_t *start_row) {
    BatchColumns batch;
    pg_status st = batch_columns(source, &batch);
    if (st) return st;
    if (row_lo < 0 || row_hi < row_lo || row_hi > batch.n_rows) return fail(PG_ERR_INVALID, "slice outside the source");
    const int64_t lo = row_lo & ~(int64_t)127;
    auto run = std::make_unique<Run>(batch.schema, row_hi - lo);
    run->source = batch.run;
    const int nc = batch.schema->n_cols();
    for (int c = 0; c < nc; c++) {
        const pg_field f = batch.schema->field(c);
        DevColumn dc = batch.cols[c];
        if (is_varlen(f.type)) {
            if (dc.offsets && run->n_rows > 0) {
                int32_t b[2] = {0, 0};
                PG_CUDA(cudaMemcpy(&b[0], dc.offsets + lo, 4, cudaMemcpyDeviceToHost));
                PG_CUDA(cudaMemcpy(&b[1], dc.offsets + row_hi, 4, cudaMemcpyDeviceToHost));
                run->varlen_base[c] = b[0];
                run->varlen_bytes[c] = b[1] - b[0];
            }
            if (dc.offsets) dc.offsets += lo;             // `data` stays the address of byte 0 of the offsets' space
        } else if (dc.data) {
            dc.data = (const unsigned char *)dc.data + lo * type_width(f.type);
        }
        if (dc.validity) dc.validity += lo / 8;
        run->cols[c] = dc;
    }
    if (start_row) *start_row = row_lo - lo;
    *out_run = g_runs.put(std::move(run));
    return PG_OK;
}

extern "C" {

pg_status pg_run_slice(uint64_t source, int64_t row_lo, int64_t row_hi, uint64_t *out_run, int64_t *start_row) {
    if (!out_run) return fail(PG_ERR_INVALID, "null argument");
    pg_status st = ensure_device();
    if (st) return st;
    return make_slice(source, row_lo, row_hi, out_run, start_row);
}

pg_status pg_thread_stream(void **out_cuda_stream) {
    if (!out_cuda_stream) return fail(PG_ERR_INVALID, "null argument");
    pg_status st = ensure_device();
    if (st) return st;
    *out_cuda_stream = (void *)copy_stream();
    return PG_OK;
}

// (re)binds a merge handle to k runs; runs without rows to merge are dropped (exhausted readers are legal,
// SortMergeReaderTestBase.java:53-56)
static pg_status bind_runs(Merge *m, const uint64_t *runs, int32_t k, const int64_t *row0) {
    const Spec *sp = m->spec.get();
    m->runs.clear();
    m->bound.clear();
    m->row0.clear();
    m->k = 0;                                    // a failed bind merges nothing: the descriptors may be stale
    m->n_in = 0;
    m->stats = pg_stats{};
    for (int i = 0; i < k; i++) {
        std::shared_ptr<Run> r = g_runs.get(runs[i]);
        if (!r) return fail(PG_ERR_INVALID, "unknown run handle");
        if (r->schema != sp->schema) {           // different handles are fine as long as the schemas are equal
            const Schema *a = r->schema.get(), *b = sp->schema.get();
            bool same = a->n_key == b->n_key && a->n_val == b->n_val;
            for (int c = 0; same && c < a->n_cols(); c++)
                same = a->field(c).type == b->field(c).type && a->field(c).nullable == b->field(c).nullable;
            if (!same) return fail(PG_ERR_INVALID, "run and spec use different schemas");
        }
        const int64_t skip = row0 ? row0[i] : 0;
        if (skip < 0 || skip > r->n_rows) return fail(PG_ERR_INVALID, "start row outside the run");
        m->stats.bytes_h2d += r->bytes_h2d;
        if (r->n_rows - skip == 0) continue;
        m->runs.push_back(r);
        m->bound.push_back(r);
        m->row0.push_back(skip);
        m->n_in += r->n_rows - skip;
    }
    m->k = (int)m->runs.size();
    pg_status st = m->k > 0 ? build_descriptors(m) : PG_OK;
    if (st) m->k = 0;
    return st;
}

pg_status pg_merge_open(uint64_t spec, const uint64_t *runs, int32_t k, uint64_t *out_merge) {
    std::shared_ptr<Spec> sp = g_specs.get(spec);
    if (!sp || !out_merge || (k > 0 && !runs)) return fail(PG_ERR_INVALID, "bad spec handle or null argument");
    if (k < 0) return fail(PG_ERR_INVALID, "negative run count");
    if (k > PG_MAX_RUNS)
        return fail(PG_ERR_UNSUPPORTED, "more than PG_MAX_RUNS runs in one merge call");
    pg_status st = ensure_device();
    if (st) return st;
    std::unique_ptr<Merge> m(new Merge());
    m->spec = std::move(sp);
    PG_CUDA(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
    for (auto &e : m->ev) PG_CUDA(cudaEventCreate(&e));
    st = bind_runs(m.get(), runs, k, nullptr);
    if (st) return st;
    *out_merge = g_merges.put(std::move(m));
    return PG_OK;
}

pg_status pg_merge_rebind(uint64_t merge, const uint64_t *runs, int32_t k, const int64_t *start_rows) {
    std::shared_ptr<Merge> m = g_merges.get(merge);
    if (!m || (k > 0 && !runs)) return fail(PG_ERR_INVALID, "unknown merge handle or null argument");
    if (k < 0 || k > PG_MAX_RUNS) return fail(PG_ERR_INVALID, "bad run count");
    pg_status st = ensure_device();
    if (st) return st;
    PG_HOST_MARKS("merge rebind");
    PG_CUDA(cudaStreamSynchronize(m->stream));
    free_outputs(m.get());
    PG_HOST_MARK("sync");
    st = bind_runs(m.get(), runs, k, start_rows);
    PG_HOST_MARK("bind");
    return st;
}

pg_status pg_merge_execute(uint64_t merge) {
    std::shared_ptr<Merge> m = g_merges.get(merge);
    if (!m) return fail(PG_ERR_INVALID, "unknown merge handle");
    if (m->k == 0 || m->n_in == 0) {
        // no input rows: one empty batch
        free_outputs(m.get());
        m->n_out = 0;
        m->out_cols.assign(m->spec->schema->n_cols(), pg_out_column{});
        m->has_batch = true;
        m->stats = pg_stats{};
        return PG_OK;
    }
    int64_t h2d = m->stats.bytes_h2d;
    pg_status st = execute(m.get());
    m->stats.bytes_h2d = h2d;
    return st;
}

pg_status pg_merge_device_batch(uint64_t merge, pg_batch *out) {
    std::shared_ptr<Merge> m = g_merges.get(merge);
    if (!m || !out) return fail(PG_ERR_INVALID, "unknown merge handle");
    if (!m->has_batch) return fail(PG_ERR_INVALID, "no batch: call pg_merge_execute first");
    out->n_rows = m->n_out;
    out->n_cols = (int32_t)m->out_cols.size();
    out->cols = m->out_cols.data();
    return PG_OK;
}

pg_status pg_merge_fetch(uint64_t merge, const pg_out_column *host_cols, int32_t n_cols) {
    std::shared_ptr<Merge> m = g_merges.get(merge);
    if (!m || !host_cols) return fail(PG_ERR_INVALID, "unknown merge handle");
    if (!m->has_batch) return fail(PG_ERR_INVALID, "no batch: call pg_merge_execute first");
    if (n_cols != (int32_t)m->out_cols.size()) return fail(PG_ERR_INVALID, "column count mismatch");
    pg_status st = ensure_device();
    if (st) return st;
    const int64_t n = m->n_out;
    int64_t bytes = 0;
    std::vector<void *> cp_dst, cp_src;
    std::vector<size_t> cp_size;
    for (int c = 0; c < n_cols && n > 0; c++) {
        const pg_out_column &oc = m->out_cols[c];
        const pg_out_column &hc = host_cols[c];
        if (oc.data_bytes && hc.data) {
            if (hc.data_bytes < oc.data_bytes)
                return fail(PG_ERR_INVALID, "pg_merge_fetch: data buffer of column " + std::to_string(c) + " holds " +
                                            std::to_string(hc.data_bytes) + " bytes, the batch needs " + std::to_string(oc.data_bytes));
            cp_dst.push_back(hc.data); cp_src.push_back(oc.data); cp_size.push_back((size_t)oc.data_bytes);
            bytes += oc.data_bytes;
        }
        if (oc.offsets && hc.offsets) {
            cp_dst.push_back(hc.offsets); cp_src.push_back(oc.offsets); cp_size.push_back(sizeof(int32_t) * (size_t)(n + 1));
            bytes += 4 * (n + 1);
        }
        if (oc.validity && hc.validity) {
            cp_dst.push_back(hc.validity); cp_src.push_back(oc.validity); cp_size.push_back((size_t)((n + 7) / 8));
            bytes += (n + 7) / 8;
        }
    }
    st = copy_batch(cp_dst, cp_src, cp_size, cudaMemcpyDeviceToHost, m->stream);
    if (st) return st;
    PG_CUDA(cudaStreamSynchronize(m->stream));
    m->stats.bytes_d2h = bytes;
    return PG_OK;
}

pg_status pg_merge_release(uint64_t merge) {
    std::shared_ptr<Merge> m = g_merges.get(merge);
    if (!m) return fail(PG_ERR_INVALID, "unknown merge handle");
    if (ensure_device() == PG_OK) free_outputs(m.get(), true);
    return PG_OK;
}

pg_status pg_merge_stats(uint64_t merge, pg_stats *out) {
    std::shared_ptr<Merge> m = g_merges.get(merge);
    if (!m || !out) return fail(PG_ERR_INVALID, "unknown merge handle");
    *out = m->stats;
    return PG_OK;
}

pg_status pg_merge_stream(uint64_t merge, void **out_cuda_stream) {
    std::shared_ptr<Merge> m = g_merges.get(merge);
    if (!m || !out_cuda_stream) return fail(PG_ERR_INVALID, "unknown merge handle");
    *out_cuda_stream = (void *)m->stream;
    return PG_OK;
}

pg_status pg_merge_free(uint64_t merge) {
    return g_merges.take(merge) ? PG_OK : fail(PG_ERR_INVALID, "unknown merge handle");
}

// IntervalPartition.partition(), paimon-core/.../mergetree/compact/IntervalPartition.java:67-125.
// Host logic: it only looks at file key bounds (SURVEY §8a row a13: "negligible; stays on host").
pg_status pg_interval_partition(int32_t n_files, const int64_t *min_key, const int64_t *max_key,
                                int32_t *section_of, int32_t *run_of, int32_t *n_sections) {
    if (n_files < 0 || (n_files > 0 && (!min_key || !max_key || !section_of || !run_of)) || !n_sections)
        return fail(PG_ERR_INVALID, "null argument");
    std::vector<int> order(n_files);
    for (int i = 0; i < n_files; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
        if (min_key[a] != min_key[b]) return min_key[a] < min_key[b];
        return max_key[a] < max_key[b];
    });
    int sections = 0;
    size_t begin = 0;
    auto close_section = [&](size_t b, size_t e) {
        // runs ordered by the max key of their last file; the smallest takes the next file if it fits
        using Item = std::pair<int64_t, int>;                 // (last max key, run id)
        std::priority_queue<Item, std::vector<Item>, std::greater<Item>> heap;
        int n_runs = 0;
        for (size_t i = b; i < e; i++) {
            int f = order[i];
            if (!heap.empty() && min_key[f] > heap.top().first) {
                Item top = heap.top();
                heap.pop();
                run_of[f] = top.second;
                heap.push(Item(max_key[f], top.second));
            } else {
                run_of[f] = n_runs;
                heap.push(Item(max_key[f], n_runs++));
            }
            section_of[f] = sections;
        }
        sections++;
    };
    int64_t bound = 0;
    for (size_t i = 0; i < (size_t)n_files; i++) {
        int f = order[i];
        if (i > begin && min_key[f] > bound) {
            close_section(begin, i);
            begin = i;
        }
        if (i == begin || max_key[f] > bound) bound = max_key[f];
    }
    if ((size_t)n_files > begin) close_section(begin, n_files);
    *n_sections = sections;
    return PG_OK;
}

}  // extern "C"
