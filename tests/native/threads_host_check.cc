// Host build of the file metadata parsers under many threads at once: pq::parse_footer and pq::parse_footers
// (parquet_meta.cc), orc::parse_file and orc::read_tails (orc_meta.cc, whose compressed metadata inflates through
// per-thread zstd tables).  The section decoders run these on whatever thread calls them, so several reader threads
// parse at the same time.  tests/test_host_threads_cpu.py builds this driver with ThreadSanitizer and runs it as a child
// process.
//
// stdin: records of [kind:1 (0 Parquet, 1 ORC)][size:8 LE][the whole file].  The driver parses every file once on the
// main thread, then kThreads threads parse all of them kRounds times each, starting together: every thread every file
// in its own order (shared inputs), then thread t the files i with i % kThreads == t, once per round (distinct inputs).
// Each parse is compared with the sequential one.  stdout: one line "files F parses P mismatches M"; exit status 1 when
// a parse differs (the first difference on stderr).
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <condition_variable>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "orc_dump.h"
#include "orc_meta.h"
#include "parquet_dump.h"
#include "parquet_meta.h"

namespace {

constexpr int kThreads = 8, kRounds = 2;

struct File {
    int kind;
    std::vector<uint8_t> bytes;
};

// the ORC tails of one file through read_tails, from memory (the ranges the device path would read back)
struct Memory : orc::RangeReader {
    const std::vector<uint8_t> *f;
    void read(int, uint64_t off, uint64_t n, uint8_t *dst) override {
        if (off > f->size() || n > f->size() - off) throw std::runtime_error("range outside the file");
        memcpy(dst, f->data() + off, n);
    }
    void flush() override {}
};

// every parse of one file, as text (an error is its message)
std::string parse(const File &f) {
    try {
        const uint8_t *p = f.bytes.data();
        const int64_t n = (int64_t)f.bytes.size();
        if (f.kind == 0) {
            std::string o = dump(pq::parse_footer(p, n));
            const int64_t flen = (int64_t)p[n - 8] | ((int64_t)p[n - 7] << 8) | ((int64_t)p[n - 6] << 16) | ((int64_t)p[n - 5] << 24);
            std::vector<pq::FooterBytes> one{pq::FooterBytes{p + n - 8 - flen, flen}, pq::FooterBytes{p + n - 8 - flen, flen}};
            for (const pq::FileMetaData &m : pq::parse_footers(one)) o += "\n|" + dump(m);
            return o;
        }
        std::string o = dump(orc::parse_file(p, n));
        Memory rd;
        rd.f = &f.bytes;
        for (const orc::FileTail &t : orc::read_tails(rd, {(uint64_t)n})) o += "\n|" + dump(t);
        return o;
    } catch (const std::exception &e) {
        return std::string("error: ") + e.what();
    }
}

struct Start {                      // every thread begins its round together
    std::mutex mu;
    std::condition_variable cv;
    int waiting = 0, generation = 0;
    void arrive() {
        std::unique_lock<std::mutex> g(mu);
        const int gen = generation;
        if (++waiting == kThreads) {
            waiting = 0;
            generation++;
            cv.notify_all();
        } else {
            cv.wait(g, [&] { return generation != gen; });
        }
    }
};

}  // namespace

int main() {
    std::vector<File> files;
    for (;;) {
        uint8_t kind;
        int64_t size;
        if (fread(&kind, 1, 1, stdin) != 1) break;
        if (fread(&size, 8, 1, stdin) != 1 || size < 12) { fprintf(stderr, "bad record\n"); return 2; }
        File f{kind, std::vector<uint8_t>((size_t)size)};
        if (fread(f.bytes.data(), 1, (size_t)size, stdin) != (size_t)size) { fprintf(stderr, "short record\n"); return 2; }
        files.push_back(std::move(f));
    }
    const int nf = (int)files.size();
    std::vector<std::string> want(nf);
    for (int i = 0; i < nf; i++) want[i] = parse(files[i]);

    Start start;
    std::atomic<long long> parses{0}, mismatches{0};
    std::mutex first_mu;
    std::string first;
    auto check = [&](int t, int i) {
        parses++;
        if (parse(files[i]) == want[i]) return;
        if (mismatches++ == 0) {
            std::lock_guard<std::mutex> g(first_mu);
            first = "thread " + std::to_string(t) + ", file " + std::to_string(i) + ": the parse differs from the sequential one";
        }
    };
    std::vector<std::thread> th;
    for (int t = 0; t < kThreads; t++)
        th.emplace_back([&, t] {
            for (int r = 0; r < kRounds; r++) {
                start.arrive();
                for (int j = 0; j < nf; j++) check(t, (j + t * 7 + r) % nf);        // shared: every file
                start.arrive();
                for (int i = t; i < nf; i += kThreads) check(t, i);                // distinct: this thread's files
            }
        });
    for (std::thread &x : th) x.join();
    printf("files %d parses %lld mismatches %lld\n", nf, parses.load(), mismatches.load());
    if (mismatches) {
        fprintf(stderr, "%s\n", first.c_str());
        return 1;
    }
    return 0;
}
