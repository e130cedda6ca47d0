// encoded_file.h — what the compaction output encoders (parquet_encode.cu, orc_encode.cu) share: the encoded-file
// handle table behind pg_parquet_file_meta / _column_stats / _fetch / _device_image / _free, the column and statistics
// jobs of k_pw_stats, and the zstd block jobs of k_zs_block.
#pragma once

#include <string.h>

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
};
extern Table<EncodedFile> g_enc;             // parquet_encode.cu; Parquet and ORC files alike

// Copies host-built parts into the device image `dst` with one launch, none when there are no parts.  The staging
// buffers come from `scratch`; `what` names them when the device is out of memory.
pg_status patch(Scratch &scratch, const std::vector<Part> &parts, uint8_t *dst, const char *what);

// ---- zstd: every block of at most 128 KiB of a body is compressed by one warp (k_zs_block); a body is one frame
struct ZsBlockJob {
    int64_t src;                  // offset of the block in the body image
    int64_t out;                  // offset of its payload slot (n bytes)
    int64_t seq;                  // first sequence slot (n / 4 + 1 of them)
    int32_t n;                    // input bytes (<= 128 KiB)
    int32_t page;                 // its body
};
struct ZsPage {
    int64_t raw;                  // body bytes
    int32_t first_block, n_blocks;
};
// k_zs_block over n_blocks jobs (res[j] = block type, payload bytes), then per body the offset of each block's header
// inside its frame (boff) and the frame size (frame_bytes)
void launch_zs_compress(const ZsBlockJob *jobs, int n_blocks, const ZsPage *pages, int n_pages, const uint8_t *img,
                        uint8_t *out, void *seqs, uint8_t *lits, int2 *res, int32_t *boff, int64_t *frame_bytes);
// the bytes of the sequence slots of a job table that needs `seq` of them
size_t zs_seq_bytes(int64_t seq);

}  // namespace pg
