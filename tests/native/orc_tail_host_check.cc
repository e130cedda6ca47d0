// Host build of the ORC tail reader (orc_meta.cc: parse_file and read_tails, the path pg_orc_read_section takes for
// the file tails of device-resident files).  tests/test_orc_device_tail_cpu.py drives read_tails through a reader that
// records every byte range it is asked for, and compares its parse with parse_file's.
#include <string.h>

#include <stdexcept>
#include <string>
#include <vector>

#include "orc_meta.h"

// ---- the file tails of a section's device-resident files, as the section decoder reads them: orc::read_tails through
// a reader that records every range it is asked for (and copies only ranges inside their file)
namespace {

struct Recorder : orc::RangeReader {
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
std::string dump(const orc::FileTail &t) {
    std::string o = "c" + std::to_string(t.compression) + " b" + std::to_string(t.block_size) + " r" + std::to_string(t.rows) + " v";
    for (uint32_t v : t.version) o += std::to_string(v) + ".";
    for (const orc::Type &ty : t.types) {
        o += "\nT" + std::to_string(ty.kind) + " p" + std::to_string(ty.precision) + " s" + std::to_string(ty.scale) + " [";
        for (uint32_t s : ty.subtypes) o += std::to_string(s) + ",";
        o += "] [";
        for (const std::string &n : ty.field_names) o += n + ",";
        o += "]";
    }
    for (size_t i = 0; i < t.stripes.size(); i++) {
        const orc::StripeInfo &si = t.stripes[i];
        o += "\nS" + std::to_string(si.offset) + " " + std::to_string(si.index_length) + " " + std::to_string(si.data_length) +
             " " + std::to_string(si.footer_length) + " " + std::to_string(si.rows) + ":";
        for (const orc::StreamInfo &st : t.stripe_footers[i].streams)
            o += " (" + std::to_string(st.kind) + "," + std::to_string(st.column) + "," + std::to_string(st.length) + "@" +
                 std::to_string(st.offset) + ")";
        o += " |";
        for (const orc::ColumnEncoding &e : t.stripe_footers[i].columns)
            o += " " + std::to_string(e.kind) + "/" + std::to_string(e.dictionary_size);
    }
    return o;
}

std::string g_dump, g_err;
std::vector<long long> g_ranges;

}  // namespace

extern "C" {

const char *orc_tail_error() { return g_err.c_str(); }

// The tails of n files read through the recorder (from_ranges = 1) or parsed whole by parse_file (0).  Returns the
// number of reader rounds (0 for parse_file), or -1 with orc_tail_error; orc_tail_dump() has the files' dumps,
// orc_tail_ranges() the recorded ranges of the last call either way.
int orc_tail_read(const unsigned char *const *files, const long long *sizes, int n, int from_ranges) {
    g_dump.clear();
    g_ranges.clear();
    Recorder rec;
    rec.files = files;
    rec.sizes = sizes;
    try {
        std::vector<orc::FileTail> t;
        if (from_ranges) {
            std::vector<uint64_t> sz(sizes, sizes + n);
            t = orc::read_tails(rec, sz);
        } else {
            for (int f = 0; f < n; f++) t.push_back(orc::parse_file(files[f], sizes[f]));
        }
        for (const orc::FileTail &x : t) g_dump += dump(x) + "\n=\n";
    } catch (const std::exception &e) {
        g_err = e.what();
        g_ranges = rec.ranges;
        return -1;
    }
    g_ranges = rec.ranges;
    return (int)rec.round;
}
const char *orc_tail_dump() { return g_dump.c_str(); }
long long orc_tail_ranges(const long long **out) { *out = g_ranges.data(); return (long long)g_ranges.size() / 4; }

}  // extern "C"
