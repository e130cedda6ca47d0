// Host build of the section footer parse (parquet_meta.cc: parse_footers, which pg_parquet_read_section runs on the
// footers of a section's device-resident files).  tests/test_parquet_footers_cpu.py compares its dumps and its errors
// with those of parse_footer run on the files one after another.
#include "parquet_tail_host_check.cc"      // (its dump of a FileMetaData)

namespace {
std::string g_fdump, g_ferr;
}

extern "C" {

const char *pq_footers_dump() { return g_fdump.c_str(); }
const char *pq_footers_error() { return g_ferr.c_str(); }

// The footers of n whole files: parse_footers over their Thrift footers (parallel = 1), or parse_footer file by file
// (0).  Returns 0, or -1 with pq_footers_error.  The files' framing (magic, footer length) must be sound.
int pq_footers_read(const unsigned char *const *files, const long long *sizes, int n, int parallel) {
    g_fdump.clear();
    g_ferr.clear();
    try {
        std::vector<pq::FileMetaData> m;
        if (parallel) {
            std::vector<pq::FooterBytes> spans;
            for (int f = 0; f < n; f++) {
                const unsigned char *t = files[f] + sizes[f] - 8;
                const long long flen = (long long)t[0] | ((long long)t[1] << 8) | ((long long)t[2] << 16) | ((long long)t[3] << 24);
                spans.push_back(pq::FooterBytes{files[f] + sizes[f] - 8 - flen, flen});
            }
            m = pq::parse_footers(spans);
        } else {
            for (int f = 0; f < n; f++) m.push_back(pq::parse_footer(files[f], sizes[f]));
        }
        for (const pq::FileMetaData &x : m) g_fdump += dump(x) + "\n=\n";
    } catch (const std::exception &e) {
        g_ferr = e.what();
        return -1;
    }
    return 0;
}

}  // extern "C"
