// encoded_file.h — the back end the compaction output encoders (parquet_encode.cu, orc_encode.cu) share, in
// encoded_file.cu: the source-batch checks, k_pw_stats and the file statistics fold, zstd framing of a list of bodies,
// the patch of host-built parts, and the handles behind pg_parquet_file_meta / _column_stats / _fetch / _device_image
// / _free, which serve Parquet and ORC files alike.
#pragma once

#include <string.h>

#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "pg_internal.h"

namespace pg {

// one column of the batch being encoded
struct EncColumn {
    const void *data;
    const int32_t *offsets;
    const uint8_t *validity;     // NULL = no nulls
    int32_t type;                // pg_type
    int32_t width;               // bytes in memory, 0 = var-len
    int32_t optional;            // OPTIONAL in the file (definition levels are written)
    int32_t pad;
};

// k_pw_stats: per job, min / max of the non-null values of a fixed-width numeric column, as int64 / double bit patterns
// (FLOAT / DOUBLE: of the non-NaN values), non-null rows, RowKind retracts (TINYINT), whether a non-null value is NaN
struct StatJob { int32_t col; int32_t pad; int64_t row0; int64_t n_rows; };
constexpr int kStatWords = 5;     // per job: min, max, non-null rows, retracts, NaN seen
void launch_pw_stats(const EncColumn *cols, const StatJob *jobs, int n_jobs, int64_t *out /* [job][kStatWords] */);

// whole-file statistics of one column, as pg_parquet_file_column_stats reports them
struct ColStats { int64_t min = 0, max = 0, null_count = 0; int has_minmax = 0; };

// the bits of a FLOAT / DOUBLE bound (held as a double), a zero of either sign replaced by `zero`
inline int64_t zero_as(int64_t bits, double zero) {
    double x;
    memcpy(&x, &bits, 8);
    if (x == 0) memcpy(&bits, &zero, 8);
    return bits;
}

// The statistics of a piece of `rows` rows from its k_pw_stats words: no min / max if var-len, all null or holding a
// NaN; a FLOAT / DOUBLE zero min as -0.0, a zero max as +0.0 (parquet.thrift), so both zeros lie inside.
ColStats piece_stats(const EncColumn &ec, const int64_t *sw, int64_t rows);

using Part = std::pair<int64_t, std::vector<uint8_t>>;  // a host-built piece of the file: (offset, bytes)

struct EncodedFile {
    unsigned char *d_file = nullptr;         // device image of the file (the bodies at their final offsets)
    int64_t file_bytes = 0;
    int64_t data_end = 0;                    // end of the data the device wrote, where the host-built tail starts
    std::vector<Part> host_parts;            // headers, footers, file tail
    pg_file_meta meta{};
    std::vector<ColStats> stats;             // whole-file, per column
    bool image_complete = false;             // host_parts have been patched into d_file
    ~EncodedFile() { if (d_file) cudaFree(d_file); }
    pg_status alloc_image() {                // d_file: file_bytes + 64 bytes, zeroed
        PG_CUDA(cudaMalloc(&d_file, (size_t)file_bytes + 64));
        PG_CUDA(cudaMemsetAsync(d_file, 0, (size_t)file_bytes + 64, 0));
        return PG_OK;
    }
};

// The columns of `source` for rows [row0, row0 + *n_rows) (*n_rows < 0: to the batch's end), leased by *out; `who`
// prefixes the refusal of a batch under a read-type projection or a range outside it or not starting at a multiple of 8.
pg_status encode_source(uint64_t source, const char *who, int64_t row0, int64_t *n_rows, BatchColumns *out);

// ms_encode runs from start_encode to finish_encode, which waits for the encode, sets meta.file_bytes, ms_encode and
// launches, and registers the file under *out_file.
pg_status start_encode(SectionTimer &tm);
pg_status finish_encode(SectionTimer &tm, std::unique_ptr<EncodedFile> ef, int launches, const char *who,
                        uint64_t *out_file);

// Copies host-built parts into the device image `dst` with one launch, none when there are no parts.  The staging
// buffers come from `scratch`; `what` names them when the device is out of memory.
pg_status patch(Scratch &scratch, const std::vector<Part> &parts, uint8_t *dst, const char *what);

// The file statistics of pg_parquet_file_column_stats and pg_file_meta, folded from the k_pw_stats words of the pieces
// of each column (a Parquet column chunk, or one column of an ORC stripe).
struct FileStats {
    explicit FileStats(const Schema &s);
    // Folds in a piece of `rows` rows of column `col` and returns its piece_stats.
    ColStats add(int col, const EncColumn &ec, const int64_t *sw, int64_t rows);
    // ef.stats, with no min / max where any piece held a NaN (NaN sorts above every value under Double.compare);
    // delete_row_count (the retracts of the _VALUE_KIND column) and min / max_sequence_number
    void finish(EncodedFile &ef);
 private:
    const int n_key_;
    std::vector<ColStats> cols_;
    std::vector<char> nan_;       // per column: a piece held a NaN
    int64_t deletes_ = 0;
};

// zstd framing of bodies in a device image: every block of at most 128 KiB of a body is compressed by one warp
// (k_zs_block) and each body becomes one frame.
struct ZsBlockJob; struct ZsBody;  // encoded_file.cu
class ZstdFrames {
 public:
    struct Body { int64_t off, bytes; };   // offset in the image, bytes
    explicit ZstdFrames(const char *who) : who_(who) {}
    // Compresses `bodies` of `img` and reads each body's frame size back into *frame_bytes.  The buffers come from
    // `scratch`, which has to outlive gather().
    pg_status compress(Scratch &scratch, const uint8_t *img, const std::vector<Body> &bodies,
                       std::vector<int64_t> *frame_bytes, int *launches);
    // Places body i at file + dst_off[i]: its frame, or where raw[i] is set its bytes as they are (an empty `raw`:
    // every body as its frame).
    pg_status gather(const std::vector<int64_t> &dst_off, const std::vector<uint8_t> &raw, uint8_t *file, int *launches);
 private:
    const char *who_;
    const uint8_t *img_ = nullptr;
    uint8_t *out_ = nullptr, *raw_ = nullptr;
    ZsBlockJob *jobs_ = nullptr;
    ZsBody *bodies_ = nullptr;
    int2 *res_ = nullptr;
    int32_t *boff_ = nullptr;
    int64_t *frame_ = nullptr;    // the frame sizes, then the destination offsets
    size_t n_blocks_ = 0, n_bodies_ = 0;
};

}  // namespace pg
