// Host build of the ORC encode path: orc_encode_device.cuh (integer RLE v2, byte RLE, PRESENT bytes) and orc_meta.cc
// (stripe footers, statistics, file tail, zstd chunks) — the sources the device encoder compiles — driven serially on
// the host to write whole files.  tests/test_orc_encode_cpu.py reads them back with pyarrow.orc and with the host build
// of the project's ORC decoder, and checks the footers' statistics against tests/orc_stats_reference.py.
// The statistics computed here follow the rules orc_encode.cu applies; the model in Python is independent of both.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <stdexcept>
#include <string>
#include <vector>

#include "orc_encode_device.cuh"
#include "orc_meta.h"

namespace {

std::vector<uint8_t> g_file;
std::string g_err;

struct Col {
    int kind, precision, scale, max_length;
    int width;                    // bytes per value in memory, 0 = var-len
    const uint8_t *data;
    const int32_t *offsets;
    const uint8_t *valid;         // one byte per row, NULL = no nulls
};

int64_t value_of(const Col &c, int64_t r) {
    switch (c.width) {
        case 1: return (int8_t)c.data[r];
        case 2: { int16_t v; memcpy(&v, c.data + 2 * r, 2); return v; }
        case 4: { int32_t v; memcpy(&v, c.data + 4 * r, 4); return v; }
        default: { int64_t v; memcpy(&v, c.data + 8 * r, 8); return v; }
    }
}

void byte_rle(const std::vector<uint8_t> &v, std::vector<uint8_t> &out) {
    for (size_t i = 0; i < v.size(); i += orcdev::kByteGroup) {
        const int n = (int)std::min<size_t>(orcdev::kByteGroup, v.size() - i);
        const size_t at = out.size();
        out.resize(at + orcdev::brle_size(v.data() + i, n));
        orcdev::brle_write(v.data() + i, n, out.data() + at);
    }
}
void int_rle(const std::vector<int64_t> &v, int is_signed, std::vector<uint8_t> &out) {
    for (size_t i = 0; i < v.size(); i += orcdev::kRunValues) {
        const int n = (int)std::min<size_t>(orcdev::kRunValues, v.size() - i);
        const orcdev::Rle2Plan p = orcdev::rle2_plan(v.data() + i, n, is_signed);
        const size_t at = out.size();
        out.resize(at + p.size);
        orcdev::rle2_write(v.data() + i, n, is_signed, p, out.data() + at);
    }
}

bool fits_int64(__int128 v) { return v >= (__int128)INT64_MIN && v <= (__int128)INT64_MAX; }
bool is_int(int k) { return k == orc::K_BYTE || k == orc::K_SHORT || k == orc::K_INT || k == orc::K_LONG; }

}  // namespace

extern "C" {

const char *orc_enc_host_error() { return g_err.c_str(); }
const unsigned char *orc_enc_host_bytes() { return g_file.data(); }

// types: 4 ints per column (kind, precision, scale, max_length).  Returns the file size, or -1 (orc_enc_host_error).
long long orc_enc_host_write(int n_cols, const int *types, const int *widths, const void *const *data,
                             const int32_t *const *offsets, const uint8_t *const *valid, const char *const *names,
                             long long n_rows, long long stripe_rows, int codec, long long block) {
    try {
        std::vector<Col> cols(n_cols);
        std::vector<orc::OutType> otypes(n_cols);
        std::vector<std::string> onames(n_cols);
        std::vector<int> enc(n_cols + 1, orc::E_DIRECT);
        for (int c = 0; c < n_cols; c++) {
            cols[c] = Col{types[4 * c], types[4 * c + 1], types[4 * c + 2], types[4 * c + 3], widths[c],
                          (const uint8_t *)data[c], offsets[c], valid[c]};
            otypes[c].kind = cols[c].kind;
            otypes[c].precision = (uint32_t)cols[c].precision;
            otypes[c].scale = (uint32_t)cols[c].scale;
            otypes[c].max_length = (uint32_t)cols[c].max_length;
            onames[c] = names[c];
            const int k = cols[c].kind;
            if (k != orc::K_BYTE && k != orc::K_BOOLEAN && k != orc::K_FLOAT && k != orc::K_DOUBLE) enc[c + 1] = orc::E_DIRECT_V2;
        }
        stripe_rows = (stripe_rows + 7) & ~7LL;
        std::vector<uint8_t> file = {'O', 'R', 'C'};
        std::vector<orc::OutStripe> stripes;
        std::vector<orc::ColumnStats> fstats(n_cols + 1);
        fstats[0].values = (uint64_t)n_rows;
        for (long long g0 = 0; g0 < n_rows; g0 += stripe_rows) {
            const long long rows = std::min(stripe_rows, n_rows - g0);
            orc::OutStripe sp;
            sp.offset = file.size();
            sp.rows = (uint64_t)rows;
            sp.stats.resize(n_cols + 1);
            sp.stats[0].values = (uint64_t)rows;
            std::vector<orc::OutStream> list;
            for (int c = 0; c < n_cols; c++) {
                const Col &col = cols[c];
                const int k = col.kind;
                auto ok = [&](long long r) { return !col.valid || col.valid[r]; };
                std::vector<uint8_t> present, data_s, second;
                std::vector<int64_t> ints, lens;
                std::vector<uint8_t> bytes;
                orc::ColumnStats st;
                bool nan = false;
                uint64_t nn = 0;
                double dmin = INFINITY, dmax = -INFINITY;
                for (long long r = g0; r < g0 + rows; r++) {
                    if (!ok(r)) continue;
                    nn++;
                    if (col.width == 0) {
                        const int32_t s = col.offsets[r], l = col.offsets[r + 1] - s;
                        data_s.insert(data_s.end(), col.data + s, col.data + s + l);
                        lens.push_back(l);
                        st.bytes += l;
                        continue;
                    }
                    const int64_t x = value_of(col, r);
                    if (k == orc::K_FLOAT || k == orc::K_DOUBLE) {
                        double d;
                        if (k == orc::K_FLOAT) { float f; memcpy(&f, col.data + 4 * r, 4); d = f; data_s.insert(data_s.end(), col.data + 4 * r, col.data + 4 * r + 4); }
                        else { memcpy(&d, col.data + 8 * r, 8); data_s.insert(data_s.end(), col.data + 8 * r, col.data + 8 * r + 8); }
                        if (d != d) nan = true;
                        else { dmin = std::min(dmin, d); dmax = std::max(dmax, d); }
                        continue;
                    }
                    if (!st.has_minmax) { st.imin = st.imax = x; st.has_minmax = true; }
                    st.imin = std::min(st.imin, x);
                    st.imax = std::max(st.imax, x);
                    if (k == orc::K_BOOLEAN) { st.trues += x != 0; bytes.push_back(x != 0); st.has_minmax = false; }
                    else if (k == orc::K_BYTE) { bytes.push_back((uint8_t)x); st.sum += x; }
                    else if (k == orc::K_DECIMAL) {
                        st.sum += x;
                        orcdev::Out o{nullptr, 0};
                        orcdev::put_varint(o, orcdev::zigzag(x));
                        const size_t at = data_s.size();
                        data_s.resize(at + o.n);
                        orcdev::Out w{data_s.data() + at, 0};
                        orcdev::put_varint(w, orcdev::zigzag(x));
                        lens.push_back(col.scale);
                    } else { ints.push_back(x); if (k != orc::K_DATE) st.sum += x; }
                }
                st.values = nn;
                st.has_null = nn < (uint64_t)rows;
                if (nn == 0) st = orc::ColumnStats{0, true};
                else if (k == orc::K_FLOAT || k == orc::K_DOUBLE) {
                    st.has_minmax = true;
                    if (nan) { st.dmin = -INFINITY; st.dmax = NAN; }
                    else { st.dmin = dmin == 0 ? -0.0 : dmin; st.dmax = dmax == 0 ? 0.0 : dmax; }
                } else st.has_sum = k == orc::K_DECIMAL || (is_int(k) && fits_int64(st.sum));
                sp.stats[c + 1] = st;
                // file statistics: the merge of the stripes'
                orc::ColumnStats &f = fstats[c + 1];
                if (stripes.empty()) f = st;
                else {
                    f.values += st.values; f.has_null |= st.has_null; f.trues += st.trues; f.bytes += st.bytes; f.sum += st.sum;
                    f.has_sum = k == orc::K_DECIMAL || (is_int(k) && fits_int64(f.sum));
                    if (st.has_minmax) {
                        if (!f.has_minmax) { f.has_minmax = true; f.imin = st.imin; f.imax = st.imax; f.dmin = st.dmin; f.dmax = st.dmax; }
                        else {
                            f.imin = std::min(f.imin, st.imin); f.imax = std::max(f.imax, st.imax);
                            if (isnan(f.dmax) || isnan(st.dmax)) { f.dmin = -INFINITY; f.dmax = NAN; }
                            else { f.dmin = std::min(f.dmin, st.dmin); f.dmax = std::max(f.dmax, st.dmax); }
                        }
                    }
                }
                // streams
                auto emit = [&](int kind, const std::vector<uint8_t> &raw) {
                    const std::vector<uint8_t> s = orc::compress_section(raw, codec, (uint64_t)block);
                    file.insert(file.end(), s.begin(), s.end());
                    list.push_back(orc::OutStream{kind, (uint32_t)(c + 1), (uint64_t)s.size()});
                };
                if (nn < (uint64_t)rows) {
                    std::vector<uint8_t> pb((size_t)(rows + 7) / 8, 0);
                    for (long long r = 0; r < rows; r++)
                        if (ok(g0 + r)) pb[r >> 3] |= (uint8_t)(0x80 >> (r & 7));
                    byte_rle(pb, present);
                    emit(orc::S_PRESENT, present);
                }
                std::vector<uint8_t> out;
                if (k == orc::K_BYTE) byte_rle(bytes, out);
                else if (k == orc::K_BOOLEAN) {
                    std::vector<uint8_t> pb((bytes.size() + 7) / 8, 0);
                    for (size_t i = 0; i < bytes.size(); i++)
                        if (bytes[i]) pb[i >> 3] |= (uint8_t)(0x80 >> (i & 7));
                    byte_rle(pb, out);
                } else if (k == orc::K_SHORT || k == orc::K_INT || k == orc::K_LONG || k == orc::K_DATE) int_rle(ints, 1, out);
                else out = data_s;
                emit(orc::S_DATA, out);
                if (col.width == 0 || k == orc::K_DECIMAL) {
                    int_rle(lens, k == orc::K_DECIMAL ? 1 : 0, second);
                    emit(k == orc::K_DECIMAL ? orc::S_SECONDARY : orc::S_LENGTH, second);
                }
            }
            sp.data_length = file.size() - sp.offset;
            const std::vector<uint8_t> foot = orc::compress_section(orc::stripe_footer(list, enc), codec, (uint64_t)block);
            sp.footer_length = foot.size();
            file.insert(file.end(), foot.begin(), foot.end());
            stripes.push_back(std::move(sp));
        }
        if (stripes.empty())
            for (int c = 0; c < n_cols; c++) fstats[c + 1] = orc::ColumnStats{};
        const std::vector<uint8_t> tail = orc::file_tail(otypes, onames, stripes, fstats, (uint64_t)n_rows, file.size(), codec,
                                                         (uint64_t)block);
        file.insert(file.end(), tail.begin(), tail.end());
        g_file = std::move(file);
        return (long long)g_file.size();
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
}

// one integer RLE v2 run as the encoder plans and writes it: returns its size; *form, *width: the plan
int orc_enc_host_rle2(const int64_t *v, int n, int is_signed, unsigned char *dst, int *form, int *width) {
    const orcdev::Rle2Plan p = orcdev::rle2_plan(v, n, is_signed);
    orcdev::rle2_write(v, n, is_signed, p, dst);
    *form = p.form;
    *width = p.width;
    return p.size;
}

}  // extern "C"
