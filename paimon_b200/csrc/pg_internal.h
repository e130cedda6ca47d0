// Internal declarations shared by the translation units of libpaimon_gpu.so.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <chrono>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "device_layout.h"
#include "paimon_gpu.h"
#include "range_reader.h"

namespace pg {

constexpr int kPlanTile = 2048;      // rows merged by one plan / merge-keys CTA (shared-memory tile)
constexpr int kTileMax = 2 * kPlanTile;   // rows of one emit CTA: two consecutive plan tiles (fewer, fatter
                                     // column passes in the emit kernel; more CTAs per SM in the plan kernel)
constexpr int kSampleStride = 16;    // S: every S-th key of a level is a sample of the next level
constexpr int kThreads = 256;        // plan / merge-keys CTAs (4 per SM)
constexpr int kMaxCols = 256;

// ---- plan entry (one uint16 per merged input position) ----
// bits 0..11 slot inside the tile (source order: run-major), bits 12..13 member op,
// bit 14 group emits an output row (on the head), bit 15 first member of a key group
constexpr uint16_t kPlanSlotMask = 0x0FFF;
constexpr int kPlanOpShift = 12;
constexpr uint16_t kPlanEmit = 0x4000;
constexpr uint16_t kPlanHead = 0x8000;
enum : int { OP_NOOP = 0, OP_UPD = 1, OP_SET = 2, OP_RETRACT = 3 };

// error codes raised by kernels (first one wins); kernel_error turns them into statuses
enum : int {
    KERR_NONE = 0,
    KERR_TILE_OVERFLOW = 1,          // internal: a tile exceeded kTileMax (duplicate keys inside a run?)
    KERR_PU_DELETE = 2,              // PartialUpdateMergeFunction.java:155-164
    KERR_FIRST_ROW_RETRACT = 3,      // FirstRowMergeFunction.java:56-60
    KERR_AGG_RETRACT = 4,            // FieldAggregator.java:47-54
    KERR_OFFSET_OVERFLOW = 5,        // a var-len output column exceeds int32 offsets
    KERR_DIV_ZERO = 6,               // FieldProductAgg retract: integer division by zero
    KERR_BAD_PAGE = 7,               // a compressed Parquet page does not decompress to its declared size
    KERR_PQ_HEADER = 8,              // malformed / truncated Thrift page header, or page sizes that leave the chunk
    KERR_PQ_ENCODING = 9,            // a page uses an encoding the device decoder does not implement
    KERR_PQ_NO_DICT = 10,            // dictionary-encoded page in a chunk without dictionary page
    KERR_PQ_ROWS = 11,               // the pages of a chunk do not add up to the chunk's value count
    KERR_PQ_DICT_ID = 12,            // dictionary id outside the dictionary
    KERR_PQ_LEVELS = 13,             // repetition levels / unsupported level encoding
    KERR_DEC_DIV_ZERO = 14,          // FieldProductAgg retract on DECIMAL: BigDecimal.divide by zero
    KERR_DEC_DIV_UNDEFINED = 15,     // the same with a zero dividend (0 / 0)
    KERR_DEC_NON_TERMINATING = 16    // the same when the exact quotient has no finite decimal expansion
};

struct Schema {
    int n_key = 0, n_val = 0;
    std::vector<pg_field> key_fields, val_fields;
    int n_cols() const { return n_key + 2 + n_val; }
    pg_field field(int c) const {
        if (c < n_key) return key_fields[c];
        if (c == n_key) return pg_field{PG_INT64, 0};
        if (c == n_key + 1) return pg_field{PG_INT8, 0};
        return val_fields[c - n_key - 2];
    }
};

struct Spec {
    std::shared_ptr<const Schema> schema;
    int engine = 0, ignore_delete = 0, remove_record_on_delete = 0, drop_delete = 0;
    std::vector<int32_t> seq_fields;
    int seq_ascending = 1;
    std::vector<int32_t> agg;            // per value field
    std::vector<uint8_t> ignore_retract;
    // partial-update sequence groups
    std::vector<int32_t> group_seq_start, group_seq_fields, field_group;
    std::vector<uint8_t> group_partial_delete;      // per group
    std::vector<uint8_t> read_fields;               // per value field: part of the read type (empty = all)
    std::vector<int32_t> decimal;                   // per value field: precision << 8 | scale, 0 (empty = none)
    int n_groups() const { return group_seq_start.empty() ? 0 : (int)group_seq_start.size() - 1; }
};

struct DevColumn {
    const void *data = nullptr;
    const int32_t *offsets = nullptr;
    const uint8_t *validity = nullptr;
};

// ---- recycled device buffers (api.cu): a reader that streams a bucket through the device opens and frees runs at a
// high rate, and cudaMalloc / cudaFree would serialise the pipeline.  Runs, uploads and the temporaries of a decode, a
// deletion vector or an encode come from this cache; only the merge handles' arenas and descriptors and an encoded
// file's image are allocated directly.
void *buf_take(size_t bytes, size_t *got);     // NULL when the device is out of memory (after trimming the cache)
void buf_give(void *p, size_t bytes);

// One buffer from the cache (pointer and granted size), given back when destroyed.  The owner guarantees that no
// queued work still touches it by then (see Scratch).
class DeviceBuffer {
 public:
    DeviceBuffer() = default;
    explicit DeviceBuffer(size_t bytes) { p_ = buf_take(bytes, &n_); }
    DeviceBuffer(DeviceBuffer &&o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
    DeviceBuffer &operator=(DeviceBuffer &&o) noexcept {
        std::swap(p_, o.p_);
        std::swap(n_, o.n_);
        return *this;
    }
    DeviceBuffer(const DeviceBuffer &) = delete;
    DeviceBuffer &operator=(const DeviceBuffer &) = delete;
    ~DeviceBuffer() { if (p_) buf_give(p_, n_); }
    unsigned char *get() const { return (unsigned char *)p_; }
    explicit operator bool() const { return p_ != nullptr; }

 private:
    void *p_ = nullptr;
    size_t n_ = 0;
};

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

struct Run {
    Run(std::shared_ptr<const Schema> s, int64_t rows)
        : schema(std::move(s)), n_rows(rows), cols(schema->n_cols()), varlen_bytes(schema->n_cols(), 0),
          varlen_base(schema->n_cols(), 0) {}
    Run(const Run &) = delete;
    Run &operator=(const Run &) = delete;
    std::shared_ptr<const Schema> schema;
    int64_t n_rows;
    std::vector<DevColumn> cols;
    std::vector<int64_t> varlen_bytes;   // per column: payload bytes of a var-len column (offsets[n_rows] - offsets[0])
    std::vector<int64_t> varlen_base;    // per column: offsets[0] (data points at byte 0 of the offsets' space)
    std::vector<DeviceBuffer> bufs;      // device memory the run owns (none for device-memory runs and slices)
    std::shared_ptr<const Run> source;   // a slice of a run: that run (a slice of a merge batch holds no merge: no cycle)
    int64_t bytes_h2d = 0;
};

// The device buffers of one call: its temporaries, and what it builds (runs, uploads) until that is registered under a
// handle.
// Ordering invariant: no buffer goes back to the cache while work queued on `stream` may still touch it.  The destructor
// synchronises the stream before the members release anything, so every early return is safe whatever was queued.  A
// call that builds runs keeps them in `runs` until it registers them, so the run buffers a failed call drops are
// covered by the same synchronisation.
struct Scratch {
    explicit Scratch(cudaStream_t s) : stream(s) {}
    ~Scratch() { if (!bufs.empty() || !runs.empty()) cudaStreamSynchronize(stream); }
    void *take(size_t bytes) {                     // NULL when the device is out of memory
        DeviceBuffer b(bytes ? bytes : 256);
        if (!b) return nullptr;
        bufs.push_back(std::move(b));
        return bufs.back().get();
    }
    cudaStream_t stream;
    std::vector<DeviceBuffer> bufs;
    std::vector<std::unique_ptr<Run>> runs;
};

// PG_ERR_CUDA "<who>: out of device memory for <what> (N MiB wanted, F of T MiB free)"
pg_status oom(const char *who, const char *what, size_t bytes);

// where a decoder writes column c of run r: RunBuilder::out[r * n_cols + c]
struct OutColumn {
    void *data = nullptr;            // fixed-width values, or the var-len payload (set by alloc_payload)
    int32_t *offsets = nullptr;
    uint32_t *validity = nullptr;
};

// The arguments of a section read, checked before any device work (api.cu), PG_ERR_INVALID when wrong.  A file
// descriptor: PG_MEM_HOST or PG_MEM_DEVICE, size >= 0, bytes when size > 0.  A section: the schema handle (*s receives
// its lease), out_runs, the counts, and every file's descriptor with 0 <= run < n_runs.
pg_status check_file_desc(const pg_file_desc &f);
pg_status check_section_args(uint64_t schema, const pg_file_desc *files, int n_files, int n_runs, const uint64_t *out_runs,
                             std::shared_ptr<const Schema> *s);
// *out = a device copy of a host file in scratch, size + 64 bytes (the readers look past a page's end)
pg_status file_image(Scratch &scratch, const uint8_t *bytes, int64_t size, const char *who, const uint8_t **out);

// The runs a section decode or a deletion vector builds (api.cu), in the layout of DESIGN.md §3: per run one buffer
// with the validity bitmaps first and contiguous (one memset clears them), then the values or int32 offsets of each
// read column; after the caller's read-back of the exact sizes, one payload buffer per run for its var-len columns.
// The runs stay in scratch.runs until finish() registers them.  `who` prefixes the error messages.
struct RunBuilder {
    RunBuilder(std::shared_ptr<const Schema> s, int n_runs, Scratch &scratch, const char *who)
        : schema(std::move(s)), nc(schema->n_cols()), scratch(scratch), who(who), read(nc, 1), run_rows(n_runs, 0),
          missing((size_t)n_runs * nc, 0), with_rows((size_t)n_runs * nc, 0) {}
    // read[c] from a read-column mask (NULL = every column); the key, sequence number and kind columns are always read.
    // names: the names the read schema's columns have in the files (NULL = by position), none of them NULL
    pg_status read_columns(const uint8_t *read_cols, const char *const *names);
    // The next file of the section: `rows` rows of run `run`, top-level columns `cols`.  Resolves the read columns in it
    // by the `column_names` rule of paimon_gpu.h (file_col.back()) and places its rows (file_row0.back()).
    pg_status add_file(int run, int64_t rows, const std::vector<std::string> &cols);
    // the rows of a file land behind those of the files in front of it in its run: returns its first row
    int64_t place_file(int run, int64_t rows) {
        const int64_t row0 = run_rows[run];
        run_rows[run] += rows;
        return row0;
    }
    // after the last add_file: no run holds more than 2^31 rows, and no var-len column is in some of the files with rows
    // of a run but not in others (the offsets of the other files' rows would have to be filled)
    pg_status check_runs() const;
    // one buffer per run (validity cleared); bitmap[c]: a read column carries validity, zero[r * nc + c]: clear the
    // values / offsets of that column of that run as well
    pg_status alloc(const std::vector<uint8_t> &bitmap, const std::vector<uint8_t> &zero);
    // payload[r * nc + c]: exact payload bytes of each var-len read column
    pg_status alloc_payload(const std::vector<int64_t> &payload);
    // registers the runs; *info (if any) is zeroed but for n_rows, n_runs and decoded_bytes
    void finish(uint64_t *out_runs, int64_t bytes_h2d, pg_section_info *info);

    const std::shared_ptr<const Schema> schema;
    const int nc;
    Scratch &scratch;
    const char *who;
    std::vector<uint8_t> read;       // per column: part of the read type (a run has no buffers for the others)
    const char *const *names = nullptr;
    std::vector<int64_t> run_rows;
    std::vector<std::vector<int>> file_col;  // per file and column: the file's column, -1 = absent (NULL rows), -2 = not read
    std::vector<int64_t> file_row0;          // per file: its first row in its run
    std::vector<uint8_t> missing;    // per (run, column): some file of the run lacks the column
    std::vector<uint8_t> with_rows;  // per (run, column), bits: 1 = a file with rows has the column, 2 = one lacks it
    std::vector<OutColumn> out;
    int64_t decoded_bytes = 0;       // validity (n + 7) / 8, values n * width, offsets 4 (n + 1), payload bytes
};

// Host phase times of a call, in a timing build only (EXTRA_DEFS=-DPG_HOST_TIMING; compiled out by default): a call
// opens PG_HOST_MARKS(who), marks the end of each host phase with PG_HOST_MARK(phase), and prints on return one line
// "[host timing] <who>: <phase> <ms> ..." to stderr, so that each idle gap of a device trace has a named host phase.
#ifdef PG_HOST_TIMING
struct HostMarks {
    explicit HostMarks(const char *who) : who(who), t0(std::chrono::steady_clock::now()), last(t0) {}
    void mark(const char *phase) {
        const auto t = std::chrono::steady_clock::now();
        line += std::string(" ") + phase + " " + std::to_string(std::chrono::duration<double, std::milli>(t - last).count());
        last = t;
    }
    ~HostMarks() {
        mark("rest");
        fprintf(stderr, "[host timing] %s:%s total %.4f\n", who, line.c_str(),
                std::chrono::duration<double, std::milli>(last - t0).count());
    }
    const char *who;
    std::chrono::steady_clock::time_point t0, last;
    std::string line;
};
#define PG_HOST_MARKS(who) pg::HostMarks pg_host_marks_(who)
#define PG_HOST_MARK(phase) pg_host_marks_.mark(phase)
#else
#define PG_HOST_MARKS(who) do {} while (0)
#define PG_HOST_MARK(phase) do {} while (0)
#endif

// the two events ms_decode is measured between
struct SectionTimer {
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    ~SectionTimer() {
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
    }
    float ms() const {
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        return ms;
    }
};

// The host frame of one section decode (api.cu), shared by the Parquet and ORC decoders: the calling thread's copy
// stream, the call's Scratch and RunBuilder, the ms_decode events, the launch count and the section's files on the
// device.  The format decoder builds its tables and launches its kernels between start() and finish().
struct SectionFrame {
    SectionFrame(std::shared_ptr<const Schema> s, int n_runs, const char *who);
    // records the first event of ms_decode, then RunBuilder::read_columns
    pg_status start(const uint8_t *read_cols, const char *const *names);
    // d_file[f]: the bytes of file f on the device, a copy (file_image) of a host file, a device file in place
    pg_status place(const pg_file_desc *files, int n_files);
    // after the last launch: records the second event, reads the error word d_err back (one SmallReads) and turns it
    // into a status, registers the runs, and fills *info (if any) but for the format's own counts: n_chunks,
    // n_data_pages and n_dictionary_pages
    pg_status finish(const int32_t *d_err, uint64_t *out_runs, pg_section_info *info);

    const cudaStream_t stream;
    Scratch scratch;                 // file images, tables, scratch and the runs until registered
    RunBuilder b;
    SectionTimer tm;
    int launches = 0;
    std::vector<const uint8_t *> d_file;
    int64_t file_bytes = 0, h2d = 0, page_bytes = 0;     // (page_bytes: set by the format decoder)
};

// ---- handle tables: one per handle kind.  A handle carries its kind's tag in the top byte (1 schema, 2 merge spec,
// 3 run, 4 merge; 5 Parquet reader, 6 encoded Parquet or ORC file, 7 upload), so a handle of one kind is never found by
// another kind's entry points.
// The table holds one reference to each object; get() hands out a lease that an entry point holds until it returns, and
// objects hold leases on what they use, so freeing a handle never frees an object in use.  No object holds a lease on
// a Merge.  Scratch's ordering rule holds wherever a last lease is dropped: a lease may be dropped when its call
// returns, because the call's device work is finished by then (every entry point synchronises before it returns).
template <typename T>
class Table {
 public:
    explicit Table(uint64_t tag) : tag_(tag << 56) {}
    uint64_t put(std::shared_ptr<T> p) {
        std::lock_guard<std::mutex> g(mu_);
        const uint64_t h = tag_ | next_++;
        map_[h] = std::move(p);
        return h;
    }
    std::shared_ptr<T> get(uint64_t h) {     // NULL = unknown handle
        std::lock_guard<std::mutex> g(mu_);
        auto it = map_.find(h);
        return it == map_.end() ? nullptr : it->second;
    }
    std::shared_ptr<T> take(uint64_t h) {    // removes the handle: the table's reference, NULL = unknown handle
        std::lock_guard<std::mutex> g(mu_);
        auto node = map_.extract(h);
        return node.empty() ? nullptr : std::move(node.mapped());
    }

 private:
    std::mutex mu_;
    std::unordered_map<uint64_t, std::shared_ptr<T>> map_;
    uint64_t next_ = 1;
    const uint64_t tag_;
};
extern Table<Schema> g_schemas;      // api.cu
extern Table<Run> g_runs;

// ---- the rest of api.cu that the format readers and writers use
pg_status ensure_device();           // pg_init has been called; binds the calling thread to the device
cudaStream_t copy_stream();          // the calling thread's non-blocking stream
// the columns of a merge handle's current batch, or of a run, with leases on the schema and on the source that the
// caller keeps for its whole call
struct Merge;
struct BatchColumns {
    std::shared_ptr<const Schema> schema;
    std::vector<DevColumn> cols;
    int64_t n_rows = 0;
    std::shared_ptr<const Run> run;      // the source: a run,
    std::shared_ptr<Merge> merge;        // or a merge handle
};
pg_status batch_columns(uint64_t handle, BatchColumns *out);

// ---- device-side descriptors (copied to device memory once per merge handle) ----

// column descriptor used by the emit kernel; 32 bytes (the kernel keeps 64 of them in shared memory, and a larger
// static footprint would cost a second resident CTA per SM at some run counts)
struct ColDesc {
    int32_t type;        // pg_type
    int32_t width;       // bytes, 0 for var-len
    int16_t nullable;    // output carries a validity bitmap
    int16_t retract;     // RT_*
    int32_t mode;        // CM_*
    int32_t agg;         // PG_AGG_* for CM_FOLD
    int32_t varlen_index;// index among var-len columns, -1 otherwise
    int32_t group;       // CM_GAGG: the sequence group of the field
    int32_t decimal;     // DECIMAL value field: precision << 8 | scale (sum / product use decimal_arith), else 0
};
static_assert(sizeof(ColDesc) == 32, "ColDesc is staged in shared memory by the emit kernel");
// CM_GVAL / CM_GSEQ: field / sequence field of partial-update sequence group `agg`: the cell of the member the
// plan kernel marked for the group (verbatim, NULL included), NULL when no member is marked
// CM_GAGG: field of a sequence group with an aggregate function (`agg`): folded over the members the plan kernel
// marked as taking part, in order or reversed (PartialUpdateMergeFunction.java:228-244), retracts included
enum : int { CM_SELECT = 0, CM_FOLD = 1, CM_KEY = 2, CM_SEQ = 3, CM_KIND = 4, CM_GVAL = 5, CM_GSEQ = 6, CM_GAGG = 7 };
enum : int { RT_OK = 0, RT_IGNORE = 1, RT_ERROR = 2 };

struct MergeFlags {
    int32_t engine, ignore_delete, remove_record_on_delete, drop_delete;
};

// key normalisation: how to build the order-preserving uint64 of a row
struct KeyDesc {
    int32_t n_fields;
    int32_t exact;                      // the 64-bit prefix IS the key (fixed-width fields, <= 8 bytes in total)
    int32_t type[PG_MAX_KEY_FIELDS];
    int32_t width[PG_MAX_KEY_FIELDS];   // bytes; 0 = var-len (CHAR / VARCHAR / BINARY)
};

// key columns of the runs: [run * n_fields + field]
struct KeySrc {
    const void *const *data;
    const int32_t *const *offsets;      // var-len fields, else NULL entries
};

inline int type_width(int t) {
    switch (t) {
        case PG_INT8: case PG_BOOL: return 1;
        case PG_INT16: return 2;
        case PG_INT32: case PG_FLOAT: return 4;
        case PG_INT64: case PG_DOUBLE: return 8;
        default: return 0;
    }
}
static bool type_ok(int t) { return t >= PG_INT8 && t <= PG_BINARY; }
inline bool is_varlen(int t) { return t == PG_STRING || t == PG_BINARY; }

void set_error(const std::string &msg);
pg_status fail(pg_status code, const std::string &msg);
// The status of a kernel error word (api.cu): PG_OK for KERR_NONE.  What a merge function raises is
// PG_ERR_MERGE_FUNCTION with the message Java throws; the rest is a format, unsupported or internal status with a
// message behind "<who>: ".
pg_status kernel_error(int code, const char *who);

#define PG_CUDA(expr)                                                                      \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess)                                                             \
            return pg::fail(PG_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)

// ---- kernel launchers (merge.cu) ----

struct LevelView {             // keys of level l of run r: key(row = row0 + (j + 1) * stride - 1), j < count
    int64_t count[PG_MAX_RUNS];
    int64_t row0[PG_MAX_RUNS]; // first row of the run that takes part in the merge (rows before it are skipped)
    int64_t stride;
};

struct MergeLaunch {
    int k;
    KeyDesc key;
    KeySrc ks;                         // device: [k][n_key] key column data / offsets pointers
    cudaStream_t stream;
    int32_t *err;                      // device error word
    const int *skip;                   // device: key-stream bytes all rows share (NULL for exact keys = 0)
};

// B[(t) * k + r] for t in [0, n_tiles]: tile boundaries per run at this level.
void launch_partition(const MergeLaunch &ml, const LevelView &lv, const uint64_t *splitter_keys,
                      const uint64_t *splitter_refs, int q, int n_tiles, int64_t *bounds);
void launch_key_lcp(const MergeLaunch &ml, const LevelView &lv0, int *skip);
void launch_merge_keys(const MergeLaunch &ml, const LevelView &lv, const int64_t *bounds, int n_tiles,
                       uint64_t *sorted_keys, uint64_t *sorted_refs);

// per-column, per-run input pointers, transposed for coalesced access: [col * k + run]
struct ColPtrs {
    const void *const *data;
    const int32_t *const *offsets;
    const uint32_t *const *validity;   // bitmaps read as 32-bit words
};

// 'sequence.field': user defined sequence fields (file column indexes), compared before _SEQUENCE_NUMBER
struct SeqFields {
    int32_t n;
    int32_t ascending;
    int32_t col[4];
    int32_t type[4];
    int32_t width[4];
};

// partial-update sequence groups, as the plan kernel needs them (device memory)
struct SeqGroups {
    int32_t n;
    int32_t start[PG_MAX_SEQ_GROUPS + 1];            // CSR into col / type / width
    int32_t col[PG_MAX_SEQ_GROUPS * 4];              // file column of a group's sequence field
    int32_t type[PG_MAX_SEQ_GROUPS * 4];
    int32_t width[PG_MAX_SEQ_GROUPS * 4];
    int32_t partial_delete[PG_MAX_SEQ_GROUPS];       // 'partial-update.remove-record-on-sequence-group'
};

struct PlanArgs {
    const int64_t *bounds;             // level-0 tile bounds [(n_tiles+1) * k]
    int n_tiles;
    SeqFields seq;
    ColPtrs ptrs;
    const int64_t *const *seq_ptrs;    // device [k]
    const int8_t *const *kind_ptrs;    // device [k]
    MergeFlags flags;
    // outputs
    uint16_t *plan;                    // [N]
    int32_t *tile_rows;                // [n_tiles]
    int64_t *tmp_seq;                  // [N]  result sequence number per (tile in_base + out idx)
    int8_t *tmp_kind;                  // [N]
    const SeqGroups *groups;           // device; NULL without sequence groups
    uint32_t *gplan;                   // [N] per merged position: bit g = value source of group g, bit 16+g = its
                                       // sequence-field source
    uint32_t *gagg;                    // [N] (only with aggregates inside groups) bit g = the member's group-g
                                       // fields are aggregated in order, bit 16+g = reversed (older group sequence)
};
void launch_plan(const MergeLaunch &ml, const PlanArgs &pa);

// exclusive scan of tile_rows into int64 row offsets; totals[0] = output rows
void launch_scan(cudaStream_t stream, const int32_t *tile_rows, int n_tiles, int64_t *row_base, int64_t *totals);

struct EmitArgs {
    const int64_t *bounds;             // plan-tile bounds [(n_plan_tiles + 1) * k]
    int n_tiles;                       // emit tiles = ceil(n_plan_tiles / 2)
    int n_plan_tiles;
    const int32_t *tile_rows;          // output rows per plan tile
    int k;
    const uint16_t *plan;
    const int64_t *row_base;           // [n_plan_tiles]
    const int64_t *tmp_seq;
    const int8_t *tmp_kind;
    const uint32_t *gplan;             // sequence-group marks (see PlanArgs), NULL without groups
    const uint32_t *gagg;
    const ColDesc *cols;
    const int32_t *col_order;          // device [n_passes]: the emit kernel's pass list (column indexes)
    int n_passes;
    const int32_t *varlen_cols;        // device [n_varlen]: column of var-len index v
    ColPtrs ptrs;
    const int64_t *run_rows;           // device [k] rows per run
    int n_cols;
    int n_varlen;
    const pg_out_column *out_cols;     // device [n_cols]
    int64_t *totals;                   // device [1 + n_varlen]: [0] rows (in), [1+v] var-len bytes (out)
    uint64_t *vl_state;                // [n_varlen * n_tiles] decoupled look-back state, zeroed per launch
    int32_t *tile_counter;             // ticket counter, zeroed per launch
    int32_t *err;
    cudaStream_t stream;
};
void launch_emit(const EmitArgs &ea);

// readback.cu: small device -> host reads through device-mapped page-locked memory (a kernel stores them), so that
// they do not queue behind another thread's large copies on the device -> host copy engine.  add() enqueues on the
// stream, finish() synchronises the stream and delivers the bytes.  finish(ev) waits for an event the caller recorded on
// the stream behind the last add() instead, so that work enqueued after it keeps the device busy meanwhile.  One object
// per synchronisation point, per thread.
pg_status small_h2d(void *dev_dst, const void *host_src, size_t n, cudaStream_t stream);   // tables / descriptors

class SmallReads {
 public:
    explicit SmallReads(cudaStream_t s) : stream_(s) {}
    pg_status add(void *host_dst, const void *dev_src, size_t n);
    pg_status finish(cudaEvent_t after = nullptr);

 private:
    struct Item { void *dst; size_t off, n; };
    cudaStream_t stream_;
    std::vector<Item> items_;
    size_t used_ = 0;
};

// The byte ranges of the device-resident files of a section through SmallReads (orc::read_tails, pq::read_footers).
// files[i] is the index in the section of the i-th device-resident file, sizes[i] its size.  flush() throws when a
// read-back fails; st then holds its status (the message is set).
struct DeviceRanges : RangeReader {
    DeviceRanges(cudaStream_t s, const pg_file_desc *section, int n_files);
    void read(int file, uint64_t off, uint64_t n, uint8_t *dst) override;
    void flush() override;
    const pg_file_desc *section;
    std::vector<int> files;
    std::vector<uint64_t> sizes;
    SmallReads rb;
    pg_status st = PG_OK;
};

}  // namespace pg
