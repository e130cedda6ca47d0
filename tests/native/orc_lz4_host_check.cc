// Host build of the ORC decode path with every compression kind the device decodes: orc_meta.cc (metadata + plan),
// inflate_device.cuh / lz4_device.cuh / zstd_device.cuh (compression chunks) and orc_device.cuh (stream decoders, task
// phases A and B) — the same sources the device path compiles — driven serially on the host.  The same C entry points
// as orc_host_check.cc (tests/orc_util.decode drives either), with LZ4 chunks (CompressionKind 4) beside ZLIB and
// ZSTD; tests/test_lz4_files_cpu.py pins LZ4 files against pyarrow.orc without a GPU.  Flat schemas; the caller names
// the output width of every column (0 = var-len).
#include <stdlib.h>
#include <string.h>

#include <stdexcept>
#include <string>
#include <vector>

#include "inflate_device.cuh"
#include "lz4_device.cuh"
#include "orc_device.cuh"
#include "orc_meta.h"
#include "zstd_device.cuh"

namespace {

struct Result {
    std::vector<std::vector<uint8_t>> data;       // fixed: values, var-len: payload
    std::vector<std::vector<int32_t>> offsets;
    std::vector<std::vector<uint32_t>> validity;
    int64_t rows = 0;
    std::string error;
    std::vector<int> kinds;
};

// a stream stored as compression chunks -> contiguous bytes
int64_t inflate_stream(const uint8_t *p, uint64_t n, int codec, uint64_t block, uint8_t *dst, uint64_t cap) {
    if (codec == orc::C_NONE) { memcpy(dst, p, n); return (int64_t)n; }
    inflate::Tables it;
    static zs::Tables zt;
    std::vector<uint8_t> lit(zs::kMaxBlock + 64);
    uint64_t pos = 0, out = 0;
    while (pos < n) {
        const uint32_t h = p[pos] | (p[pos + 1] << 8) | (p[pos + 2] << 16);
        const uint32_t len = h >> 1;
        pos += 3;
        if (h & 1) { if (out + len > cap) return -1; memcpy(dst + out, p + pos, len); out += len; }
        else {
            const int64_t lim = (int64_t)std::min<uint64_t>(block, cap - out);
            const int64_t got = codec == orc::C_ZLIB  ? inflate::inflate_raw(p + pos, len, dst + out, lim, it, nullptr)
                                : codec == orc::C_LZ4 ? lz4::decode_block(p + pos, len, dst + out, lim)
                                                      : zs::decode(p + pos, len, dst + out, lim, lit.data(), zt);
            if (got < 0) return -1;
            out += got;
        }
        pos += len;
    }
    return (int64_t)out;
}

}  // namespace

extern "C" {

// out_widths[c]: bytes of the output type of column c (0 = var-len).  Returns an opaque result (or NULL, see orc_host_error).
static std::string g_err;
const char *orc_host_error() { return g_err.c_str(); }

void *orc_host_decode(const unsigned char *file, long long size, int n_cols, const int *out_widths) {
    auto res = new Result();
    try {
        orc::FileTail t = orc::parse_file(file, size);
        std::vector<int> cols(n_cols);
        for (int c = 0; c < n_cols; c++) cols[c] = c;
        if (t.types[0].subtypes.size() != (size_t)n_cols) throw std::runtime_error("column count mismatch");
        orc::Plan pl = orc::plan_file(t, file, size, cols);
        std::vector<uint8_t> scratch(pl.scratch_bytes + 64);
        std::vector<int64_t> slen(pl.streams.size());
        for (size_t i = 0; i < pl.streams.size(); i++) {
            const orc::PlanStream &ps = pl.streams[i];
            slen[i] = inflate_stream(file + ps.offset, ps.length, t.compression, t.block_size, scratch.data() + ps.out_off, ps.out_bound);
            if (slen[i] < 0) throw std::runtime_error("a stream does not inflate");
        }
        const int64_t n = (int64_t)t.rows;
        res->rows = n;
        res->data.resize(n_cols); res->offsets.resize(n_cols); res->validity.resize(n_cols); res->kinds.resize(n_cols);
        for (int c = 0; c < n_cols; c++) {
            res->validity[c].assign((size_t)(n + 31) / 32 + 2, 0);
            if (out_widths[c]) res->data[c].assign((size_t)n * out_widths[c] + 16, 0);
            else res->offsets[c].assign((size_t)n + 2, 0);
        }
        std::vector<int32_t> dict_off(pl.dict_entries + 1);
        std::vector<orcdev::Task> tasks(pl.tasks.size());
        auto sp = [&](int idx) -> const uint8_t * { return idx < 0 ? nullptr : scratch.data() + pl.streams[idx].out_off; };
        auto sn = [&](int idx) -> int64_t { return idx < 0 ? 0 : slen[idx]; };
        for (size_t i = 0; i < pl.tasks.size(); i++) {
            const orc::PlanTask &p = pl.tasks[i];
            orcdev::Task &k = tasks[i];
            memset(&k, 0, sizeof(k));
            k.present = sp(p.s_present); k.present_n = sn(p.s_present);
            k.data = sp(p.s_data); k.data_n = sn(p.s_data);
            k.length = sp(p.s_length); k.length_n = sn(p.s_length);
            k.dict_data = sp(p.s_dict); k.dict_data_n = sn(p.s_dict);
            k.secondary = sp(p.s_secondary); k.secondary_n = sn(p.s_secondary);
            k.row0 = p.row0; k.rows = p.rows; k.kind = p.kind; k.enc = p.enc; k.dict_size = (int32_t)p.dict_size; k.scale = p.scale;
            k.out_width = out_widths[p.col];
            k.out_data = out_widths[p.col] ? res->data[p.col].data() : nullptr;
            k.out_offsets = out_widths[p.col] ? nullptr : res->offsets[p.col].data();
            k.out_validity = res->validity[p.col].data();
            k.dict_off = dict_off.data() + p.dict_off_base;
            res->kinds[p.col] = p.kind;
            orcdev::decode_task_a(k);
            if (k.bad) throw std::runtime_error("task (stripe " + std::to_string(p.stripe) + ", column " + std::to_string(p.col) + ") is malformed");
        }
        for (int c = 0; c < n_cols; c++) {
            if (out_widths[c]) continue;
            int64_t acc = 0;
            std::vector<int32_t> &o = res->offsets[c];
            o[0] = 0;
            for (int64_t r = 0; r < n; r++) { acc += o[r + 1]; o[r + 1] = (int32_t)acc; }
            res->data[c].assign((size_t)acc + 16, 0);
        }
        for (size_t i = 0; i < pl.tasks.size(); i++) {
            orcdev::Task &k = tasks[i];
            if (k.out_width) continue;
            k.out_payload = res->data[pl.tasks[i].col].data();
            orcdev::decode_task_b(k);
            if (k.bad) throw std::runtime_error("task payload is malformed");
        }
    } catch (const std::exception &e) {
        g_err = e.what();
        delete res;
        return nullptr;
    }
    return res;
}
long long orc_host_rows(void *r) { return ((Result *)r)->rows; }
const void *orc_host_data(void *r, int c, long long *bytes) { auto &v = ((Result *)r)->data[c]; *bytes = (long long)v.size(); return v.data(); }
const void *orc_host_offsets(void *r, int c) { return ((Result *)r)->offsets[c].data(); }
const void *orc_host_validity(void *r, int c) { return ((Result *)r)->validity[c].data(); }
void orc_host_free(void *r) { delete (Result *)r; }

}  // extern "C"
