// Host build of the Parquet footer reader (parquet_meta.cc: parse_footer and read_footers, the path
// pg_parquet_read_section takes for the footers of device-resident files).  tests/test_parquet_device_tail_cpu.py
// drives read_footers through a reader that records every byte range it is asked for, and compares its parse with
// parse_footer's.
#include <string.h>

#include <stdexcept>
#include <string>
#include <vector>

#include "parquet_meta.h"

namespace {

struct Recorder : pq::RangeReader {
    const unsigned char *const *files;
    const long long *sizes;
    std::vector<long long> ranges;               // (file, offset, length, round) per range
    long long round = 0;
    void read(int f, uint64_t off, uint64_t n, uint8_t *dst) override {
        ranges.insert(ranges.end(), {(long long)f, (long long)off, (long long)n, round});
        if (f >= 0 && off <= (uint64_t)sizes[f] && n <= (uint64_t)sizes[f] - off) memcpy(dst, files[f] + off, n);
        else memset(dst, 0, n);
    }
    void flush() override { round++; }
};

// every field the decoder uses, as text: two parses are equal when their dumps are
std::string dump(const pq::FileMetaData &m) {
    std::string o = "v" + std::to_string(m.version) + " r" + std::to_string(m.num_rows) + " " + m.created_by;
    for (const pq::SchemaElement &e : m.schema)
        o += "\nE" + e.name + " t" + std::to_string(e.type) + " l" + std::to_string(e.type_length) + " r" +
             std::to_string(e.repetition) + " n" + std::to_string(e.num_children) + " c" + std::to_string(e.converted_type);
    for (const pq::RowGroup &g : m.row_groups) {
        o += "\nG" + std::to_string(g.num_rows) + " " + std::to_string(g.total_byte_size) + ":";
        for (const pq::ColumnChunk &c : g.columns) {
            o += " (" + std::to_string(c.type) + "," + std::to_string(c.codec) + "," + std::to_string(c.num_values) + "," +
                 std::to_string(c.total_uncompressed_size) + "," + std::to_string(c.total_compressed_size) + "," +
                 std::to_string(c.data_page_offset) + "," + std::to_string(c.dictionary_page_offset) + " e";
            for (int32_t e : c.encodings) o += std::to_string(e) + ".";
            for (const std::string &p : c.path) o += "/" + p;
            o += ")";
        }
    }
    return o;
}

std::string g_dump, g_err;
std::vector<long long> g_ranges;

}  // namespace

extern "C" {

const char *pq_tail_error() { return g_err.c_str(); }

// The footers of n files read through the recorder (from_ranges = 1) or parsed whole by parse_footer (0).  Returns the
// number of reader rounds (0 for parse_footer), or -1 with pq_tail_error; pq_tail_dump() has the files' dumps,
// pq_tail_ranges() the recorded ranges of the last call either way.
int pq_tail_read(const unsigned char *const *files, const long long *sizes, int n, int from_ranges) {
    g_dump.clear();
    g_ranges.clear();
    Recorder rec;
    rec.files = files;
    rec.sizes = sizes;
    try {
        std::vector<pq::FileMetaData> m;
        if (from_ranges) {
            std::vector<uint64_t> sz(sizes, sizes + n);
            m = pq::read_footers(rec, sz);
        } else {
            for (int f = 0; f < n; f++) m.push_back(pq::parse_footer(files[f], sizes[f]));
        }
        for (const pq::FileMetaData &x : m) g_dump += dump(x) + "\n=\n";
    } catch (const std::exception &e) {
        g_err = e.what();
        g_ranges = rec.ranges;
        return -1;
    }
    g_ranges = rec.ranges;
    return (int)rec.round;
}
const char *pq_tail_dump() { return g_dump.c_str(); }
long long pq_tail_ranges(const long long **out) { *out = g_ranges.data(); return (long long)g_ranges.size() / 4; }

}  // extern "C"
