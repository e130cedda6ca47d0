// Internal declarations shared by the translation units of libpaimon_gpu.so.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "paimon_gpu.h"

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

// error codes raised by kernels (first one wins), decoded in api.cu
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
    uint64_t schema_h = 0;
    const Schema *schema = nullptr;
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
    Run(const Schema &s, int64_t rows)
        : schema(&own_schema), own_schema(s), n_rows(rows), cols(s.n_cols()), varlen_bytes(s.n_cols(), 0),
          varlen_base(s.n_cols(), 0) {}
    Run(const Run &) = delete;
    Run &operator=(const Run &) = delete;
    const Schema *schema;
    Schema own_schema;                   // copy: a run may outlive the schema handle it was opened with
    int64_t n_rows;
    std::vector<DevColumn> cols;
    std::vector<int64_t> varlen_bytes;   // per column: payload bytes of a var-len column (offsets[n_rows] - offsets[0])
    std::vector<int64_t> varlen_base;    // per column: offsets[0] (data points at byte 0 of the offsets' space)
    std::vector<DeviceBuffer> bufs;      // device memory the run owns (none for device-memory runs and slices)
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

// ---- handle tables: one per handle kind.  A handle carries its kind's tag in the top byte (1 schema, 2 merge spec,
// 3 run, 4 merge; 5 Parquet reader, 6 encoded Parquet file, 7 upload), so a handle of one kind is never found by
// another kind's entry points.
template <typename T>
class Table {
 public:
    explicit Table(uint64_t tag) : tag_(tag << 56) {}
    uint64_t put(std::unique_ptr<T> p) {
        std::lock_guard<std::mutex> g(mu_);
        const uint64_t h = tag_ | next_++;
        map_[h] = std::move(p);
        return h;
    }
    T *get(uint64_t h) {
        std::lock_guard<std::mutex> g(mu_);
        auto it = map_.find(h);
        return it == map_.end() ? nullptr : it->second.get();
    }
    // fn(T &) with the table locked, so that a concurrent take() cannot free the object meanwhile; false = unknown
    template <typename F>
    bool with(uint64_t h, F &&fn) {
        std::lock_guard<std::mutex> g(mu_);
        auto it = map_.find(h);
        if (it == map_.end()) return false;
        fn(*it->second);
        return true;
    }
    std::unique_ptr<T> take(uint64_t h) {
        std::lock_guard<std::mutex> g(mu_);
        auto it = map_.find(h);
        if (it == map_.end()) return nullptr;
        std::unique_ptr<T> p = std::move(it->second);
        map_.erase(it);
        return p;
    }

 private:
    std::mutex mu_;
    std::unordered_map<uint64_t, std::unique_ptr<T>> map_;
    uint64_t next_ = 1;
    const uint64_t tag_;
};
extern Table<Schema> g_schemas;      // api.cu
extern Table<Run> g_runs;

// ---- the rest of api.cu that the format readers and writers use
pg_status ensure_device();           // pg_init has been called; binds the calling thread to the device
cudaStream_t copy_stream();          // the calling thread's non-blocking stream
// the columns of a merge handle's current batch, or of a run
pg_status batch_columns(uint64_t handle, const Schema **schema, std::vector<DevColumn> *cols, int64_t *n_rows);

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
// stream, finish() synchronises the stream and delivers the bytes.  One object per synchronisation point, per thread.
pg_status small_h2d(void *dev_dst, const void *host_src, size_t n, cudaStream_t stream);   // tables / descriptors

class SmallReads {
 public:
    explicit SmallReads(cudaStream_t s) : stream_(s) {}
    pg_status add(void *host_dst, const void *dev_src, size_t n);
    pg_status finish();

 private:
    struct Item { void *dst; size_t off, n; };
    cudaStream_t stream_;
    std::vector<Item> items_;
    size_t used_ = 0;
};

}  // namespace pg
