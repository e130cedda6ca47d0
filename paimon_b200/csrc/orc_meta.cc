// orc_meta.cc — protobuf wire reader + ORC file tail / stripe footers (see orc_meta.h).
#include "orc_meta.h"

#include <string.h>

#include <algorithm>
#include <memory>
#include <stdexcept>

#include "orc_device.cuh"
#include "zstd_encode_device.cuh"

namespace orc {

namespace {

struct Pb {
    const uint8_t *p, *end;
    Pb(const uint8_t *b, size_t n) : p(b), end(b + n) {}
    bool done() const { return p >= end; }
    uint64_t varint() {
        uint64_t v = 0;
        for (int sh = 0; sh < 70; sh += 7) {
            if (p >= end) throw std::runtime_error("orc: truncated protobuf varint");
            const uint8_t b = *p++;
            v |= (uint64_t)(b & 0x7f) << sh;
            if (!(b & 0x80)) return v;
        }
        throw std::runtime_error("orc: bad protobuf varint");
    }
    // next field: returns false at the end; wire types 0 varint, 1 fixed64, 2 length-delimited, 5 fixed32
    bool next(uint32_t &field, int &wire) {
        if (p >= end) return false;
        const uint64_t key = varint();
        field = (uint32_t)(key >> 3);
        wire = (int)(key & 7);
        return true;
    }
    Pb bytes() {
        const uint64_t n = varint();
        if ((uint64_t)(end - p) < n) throw std::runtime_error("orc: truncated protobuf field");
        Pb sub(p, (size_t)n);
        p += n;
        return sub;
    }
    void skip(int wire) {
        switch (wire) {
            case 0: varint(); return;
            case 1: if (end - p < 8) throw std::runtime_error("orc: truncated protobuf"); p += 8; return;
            case 2: bytes(); return;
            case 5: if (end - p < 4) throw std::runtime_error("orc: truncated protobuf"); p += 4; return;
            default: throw std::runtime_error("orc: unsupported protobuf wire type");
        }
    }
    // a repeated uint32 that may be packed (wire 2) or not (wire 0)
    void repeated_u32(int wire, std::vector<uint32_t> &out) {
        if (wire == 0) { out.push_back((uint32_t)varint()); return; }
        Pb sub = bytes();
        while (!sub.done()) out.push_back((uint32_t)sub.varint());
    }
};

// a metadata section stored as compression chunks
std::vector<uint8_t> inflate_section(const uint8_t *p, uint64_t n, int codec, uint64_t block_size) {
    if (codec == C_NONE) return std::vector<uint8_t>(p, p + n);
    if (codec != C_ZLIB && codec != C_ZSTD && codec != C_LZ4)
        throw std::runtime_error("orc: compression kind " + std::to_string(codec) + " is not decoded (NONE, ZLIB, LZ4 and ZSTD are)");
    const int64_t bound = orcdev::chunk_bound(p, (int64_t)n, codec, (int64_t)block_size);
    if (bound < 0) throw std::runtime_error("orc: truncated compression chunk");
    std::vector<uint8_t> out((size_t)bound), lit(zs::kMaxBlock + 64);
    static thread_local zs::Tables *zt = nullptr;
    if (!zt) zt = new zs::Tables();
    const int64_t got = orcdev::inflate_chunks(p, (int64_t)n, codec, (int64_t)block_size, out.data(), bound, *zt, lit.data());
    if (got < 0) throw std::runtime_error("orc: a metadata compression chunk does not inflate");
    out.resize((size_t)got);
    return out;
}

Type read_type(Pb pb) {
    Type t;
    uint32_t f;
    int w;
    while (pb.next(f, w)) {
        if (f == 1 && w == 0) t.kind = (int)pb.varint();
        else if (f == 2) pb.repeated_u32(w, t.subtypes);
        else if (f == 3 && w == 2) { Pb s = pb.bytes(); t.field_names.emplace_back((const char *)s.p, (size_t)(s.end - s.p)); }
        else if (f == 5 && w == 0) t.precision = (uint32_t)pb.varint();
        else if (f == 6 && w == 0) t.scale = (uint32_t)pb.varint();
        else pb.skip(w);
    }
    return t;
}

StripeInfo read_stripe_info(Pb pb) {
    StripeInfo s;
    uint32_t f;
    int w;
    while (pb.next(f, w)) {
        if (w != 0) { pb.skip(w); continue; }
        const uint64_t v = pb.varint();
        if (f == 1) s.offset = v;
        else if (f == 2) s.index_length = v;
        else if (f == 3) s.data_length = v;
        else if (f == 4) s.footer_length = v;
        else if (f == 5) s.rows = v;
    }
    return s;
}

StripeFooter read_stripe_footer(Pb pb) {
    StripeFooter sf;
    uint32_t f;
    int w;
    while (pb.next(f, w)) {
        if (f == 1 && w == 2) {
            Pb s = pb.bytes();
            StreamInfo si;
            uint32_t f2;
            int w2;
            while (s.next(f2, w2)) {
                if (w2 != 0) { s.skip(w2); continue; }
                const uint64_t v = s.varint();
                if (f2 == 1) si.kind = (int)v;
                else if (f2 == 2) si.column = (uint32_t)v;
                else if (f2 == 3) si.length = v;
            }
            sf.streams.push_back(si);
        } else if (f == 2 && w == 2) {
            Pb s = pb.bytes();
            ColumnEncoding ce;
            uint32_t f2;
            int w2;
            while (s.next(f2, w2)) {
                if (w2 != 0) { s.skip(w2); continue; }
                const uint64_t v = s.varint();
                if (f2 == 1) ce.kind = (int)v;
                else if (f2 == 2) {
                    if (v > 0xffffffffull) throw std::runtime_error("orc: dictionarySize outside uint32");
                    ce.dictionary_size = (uint32_t)v;
                }
            }
            sf.columns.push_back(ce);
        } else pb.skip(w);
    }
    return sf;
}

void check_magic(const uint8_t *head, uint64_t size) {
    if (size < 4 || head[0] != 'O' || head[1] != 'R' || head[2] != 'C') throw std::runtime_error("orc: missing ORC magic");
}

}  // namespace

uint64_t parse_tail(const uint8_t *tail, uint64_t n, uint64_t size, FileTail &t) {
    const uint64_t ps_len = tail[n - 1];
    if (ps_len + 1 > size) throw std::runtime_error("orc: bad postscript length");
    t = FileTail();
    uint64_t footer_len = 0;
    {
        Pb pb(tail + n - 1 - ps_len, (size_t)ps_len);
        uint32_t f;
        int w;
        while (pb.next(f, w)) {
            if (f == 1 && w == 0) footer_len = pb.varint();
            else if (f == 2 && w == 0) t.compression = (int)pb.varint();
            else if (f == 3 && w == 0) t.block_size = pb.varint();
            else if (f == 4) pb.repeated_u32(w, t.version);
            else pb.skip(w);
        }
    }
    if (footer_len > size - ps_len - 1) throw std::runtime_error("orc: bad footer length");
    const uint64_t need = footer_len + ps_len + 1;
    if (need > n) return need;
    const std::vector<uint8_t> footer = inflate_section(tail + n - need, footer_len, t.compression, t.block_size);
    {
        Pb pb(footer.data(), footer.size());
        uint32_t f;
        int w;
        while (pb.next(f, w)) {
            if (f == 3 && w == 2) t.stripes.push_back(read_stripe_info(pb.bytes()));
            else if (f == 4 && w == 2) t.types.push_back(read_type(pb.bytes()));
            else if (f == 6 && w == 0) t.rows = pb.varint();
            else pb.skip(w);
        }
    }
    t.stripe_footers.resize(t.stripes.size());
    return 0;
}

uint64_t stripe_footer_offset(const FileTail &t, size_t i, uint64_t size) {
    const StripeInfo &si = t.stripes[i];
    uint64_t end = si.offset;                            // (each step is checked: corrupt lengths must not wrap)
    for (const uint64_t len : {si.index_length, si.data_length, si.footer_length}) {
        if (end > size || len > size - end) throw std::runtime_error("orc: stripe footer outside the file");
        end += len;
    }
    return end - si.footer_length;
}

void parse_stripe_footer(FileTail &t, size_t i, const uint8_t *stored) {
    const StripeInfo &si = t.stripes[i];
    const std::vector<uint8_t> raw = inflate_section(stored, si.footer_length, t.compression, t.block_size);
    StripeFooter sf = read_stripe_footer(Pb(raw.data(), raw.size()));
    const uint64_t fo = si.offset + si.index_length + si.data_length;      // (stripe_footer_offset checked the sum)
    uint64_t off = si.offset;
    for (StreamInfo &s : sf.streams) {
        if (s.length > fo - off) throw std::runtime_error("orc: stream lengths exceed the stripe");
        s.offset = off;
        off += s.length;
    }
    t.stripe_footers[i] = std::move(sf);
}

FileTail parse_file(const uint8_t *file, int64_t size) {
    check_magic(file, (uint64_t)size);
    FileTail t;
    parse_tail(file, (uint64_t)size, (uint64_t)size, t);
    for (size_t i = 0; i < t.stripes.size(); i++) parse_stripe_footer(t, i, file + stripe_footer_offset(t, i, (uint64_t)size));
    return t;
}

std::vector<FileTail> read_tails(RangeReader &rd, const std::vector<uint64_t> &sizes) {
    const size_t nf = sizes.size();
    std::vector<FileTail> t(nf);
    std::vector<std::vector<uint8_t>> tail(nf);
    std::vector<uint8_t> head(4 * nf);
    // round 1: the magic and the last min(size, 16 KiB) bytes of every file
    for (size_t f = 0; f < nf; f++) {
        if (sizes[f] < 4) throw std::runtime_error("orc: missing ORC magic");
        tail[f].resize((size_t)std::min(sizes[f], kTailRead));
        rd.read((int)f, 0, 3, &head[4 * f]);
        rd.read((int)f, sizes[f] - tail[f].size(), tail[f].size(), tail[f].data());
    }
    rd.flush();
    // round 2: the rest of each Footer that begins in front of its file's tail
    std::vector<uint64_t> need(nf, 0);
    std::vector<std::vector<uint8_t>> full(nf);
    bool more = false;
    for (size_t f = 0; f < nf; f++) {
        check_magic(&head[4 * f], sizes[f]);
        need[f] = parse_tail(tail[f].data(), tail[f].size(), sizes[f], t[f]);
        if (!need[f]) continue;
        const uint64_t have = tail[f].size();
        full[f].resize((size_t)need[f]);
        memcpy(full[f].data() + (need[f] - have), tail[f].data(), (size_t)have);
        rd.read((int)f, sizes[f] - need[f], need[f] - have, full[f].data());
        more = true;
    }
    if (more) rd.flush();
    for (size_t f = 0; f < nf; f++) {
        if (need[f] && parse_tail(full[f].data(), need[f], sizes[f], t[f]) != 0)
            throw std::runtime_error("orc: the footer does not fit the length its postscript gives");
        full[f] = std::vector<uint8_t>();
    }
    // round 3: every stripe footer of every file
    std::vector<std::vector<std::vector<uint8_t>>> stored(nf);
    bool any = false;
    for (size_t f = 0; f < nf; f++) {
        stored[f].resize(t[f].stripes.size());
        uint64_t total = 0;                              // (the stripe footers of a file are disjoint parts of it: this
        for (size_t i = 0; i < t[f].stripes.size(); i++) {   // bounds the host memory a corrupt Footer can claim)
            const uint64_t off = stripe_footer_offset(t[f], i, sizes[f]);
            total += t[f].stripes[i].footer_length;
            if (total > sizes[f]) throw std::runtime_error("orc: the stripe footers are larger than the file");
            stored[f][i].resize((size_t)t[f].stripes[i].footer_length);
            rd.read((int)f, off, stored[f][i].size(), stored[f][i].data());
            any = true;
        }
    }
    if (any) rd.flush();
    for (size_t f = 0; f < nf; f++)
        for (size_t i = 0; i < t[f].stripes.size(); i++) parse_stripe_footer(t[f], i, stored[f][i].data());
    return t;
}

Plan plan_file(const FileTail &t, int64_t size, const std::vector<int> &file_col_of) {
    Plan pl;
    if (t.types.empty() || t.types[0].kind != K_STRUCT) throw std::runtime_error("orc: the root type is not a struct");
    int64_t row0 = 0;
    for (size_t si = 0; si < t.stripes.size(); si++) {
        const StripeFooter &sf = t.stripe_footers[si];
        for (size_t c = 0; c < file_col_of.size(); c++) {
            if (file_col_of[c] < 0) continue;
            if ((size_t)file_col_of[c] >= t.types[0].subtypes.size()) throw std::runtime_error("orc: column outside the file schema");
            const uint32_t tid = t.types[0].subtypes[file_col_of[c]];
            if (tid >= t.types.size() || tid >= sf.columns.size()) throw std::runtime_error("orc: type id outside the footer");
            PlanTask task;
            task.stripe = (int)si;
            task.col = (int)c;
            task.type_id = (int)tid;
            task.kind = t.types[tid].kind;
            task.scale = (int)t.types[tid].scale;
            task.enc = sf.columns[tid].kind;
            task.dict_size = sf.columns[tid].dictionary_size;
            task.row0 = row0;
            task.rows = (int64_t)t.stripes[si].rows;
            for (const StreamInfo &s : sf.streams) {
                if (s.column != tid || s.length == 0) continue;
                int *slot = nullptr;
                if (s.kind == S_PRESENT) slot = &task.s_present;
                else if (s.kind == S_DATA) slot = &task.s_data;
                else if (s.kind == S_LENGTH) slot = &task.s_length;
                else if (s.kind == S_DICTIONARY_DATA) slot = &task.s_dict;
                else if (s.kind == S_SECONDARY) slot = &task.s_secondary;
                if (!slot) continue;                      // row indexes, bloom filters
                if (s.offset + s.length > (uint64_t)size) throw std::runtime_error("orc: stream outside the file");
                PlanStream ps;
                ps.offset = s.offset;
                ps.length = s.length;
                *slot = (int)pl.streams.size();
                pl.streams.push_back(ps);
            }
            if (task.enc == E_DICTIONARY || task.enc == E_DICTIONARY_V2) {
                // a dictionary holds distinct values of the stripe's rows: a larger claim is a corrupt footer, refused
                // before the offsets scratch is sized from it
                if (task.dict_size > (uint64_t)task.rows)
                    throw std::runtime_error("orc: stripe " + std::to_string(si) + " claims a dictionary of " +
                                             std::to_string(task.dict_size) + " entries for " + std::to_string(task.rows) + " rows");
                task.dict_off_base = pl.dict_entries;
                pl.dict_entries += (uint64_t)task.dict_size + 1;
            }
            pl.tasks.push_back(task);
        }
        row0 += (int64_t)t.stripes[si].rows;
    }
    return pl;
}

Plan plan_file(const FileTail &t, const uint8_t *file, int64_t size, const std::vector<int> &file_col_of) {
    Plan pl = plan_file(t, size, file_col_of);
    for (PlanStream &ps : pl.streams) {
        if (t.compression == C_NONE) ps.out_bound = ps.length;
        else {
            const int64_t bound = orcdev::chunk_bound(file + ps.offset, (int64_t)ps.length, t.compression, (int64_t)t.block_size);
            if (bound < 0) throw std::runtime_error("orc: truncated compression chunk");
            ps.out_bound = (uint64_t)bound;
        }
        ps.out_off = pl.scratch_bytes;
        pl.scratch_bytes += (ps.out_bound + 64 + 63) & ~(uint64_t)63;
    }
    return pl;
}

// ---------------------------------------------------------------- writer

void PbWriter::varint(uint64_t v) {
    while (v >= 0x80) { b.push_back((uint8_t)(v | 0x80)); v >>= 7; }
    b.push_back((uint8_t)v);
}
void PbWriter::f64(uint32_t field, double v) {
    key(field, 1);
    uint8_t x[8];
    memcpy(x, &v, 8);
    b.insert(b.end(), x, x + 8);
}
void PbWriter::bytes(uint32_t field, const void *p, size_t n) {
    key(field, 2);
    varint(n);
    b.insert(b.end(), (const uint8_t *)p, (const uint8_t *)p + n);
}

std::string decimal_string(__int128 v, int scale) {
    const bool neg = v < 0;
    unsigned __int128 u = neg ? (unsigned __int128)0 - (unsigned __int128)v : (unsigned __int128)v;
    std::string digits;
    do { digits.insert(digits.begin(), (char)('0' + (int)(u % 10))); u /= 10; } while (u);
    if (scale > 0) {
        if ((int)digits.size() <= scale) digits.insert(digits.begin(), (size_t)(scale + 1 - digits.size()), '0');
        digits.insert(digits.end() - scale, '.');
    }
    return neg ? "-" + digits : digits;
}

std::vector<uint8_t> column_statistics(const OutType &t, const ColumnStats &s) {
    PbWriter w;
    w.u64(1, s.values);
    if (s.values > 0) {
        PbWriter m;
        switch (t.kind) {
            case K_BYTE: case K_SHORT: case K_INT: case K_LONG:
                if (s.has_minmax) { m.s64(1, s.imin); m.s64(2, s.imax); }
                if (s.has_sum) m.s64(3, (int64_t)s.sum);
                w.msg(2, m);
                break;
            case K_FLOAT: case K_DOUBLE:
                if (s.has_minmax) { m.f64(1, s.dmin); m.f64(2, s.dmax); }
                w.msg(3, m);
                break;
            case K_STRING: case K_VARCHAR:
                m.s64(3, s.bytes);
                w.msg(4, m);
                break;
            case K_BOOLEAN: {
                PbWriter packed;
                packed.varint(s.trues);
                m.bytes(1, packed.b.data(), packed.b.size());
                w.msg(5, m);
                break;
            }
            case K_DECIMAL:
                if (s.has_minmax) { m.str(1, decimal_string(s.imin, (int)t.scale)); m.str(2, decimal_string(s.imax, (int)t.scale)); }
                if (s.has_sum) m.str(3, decimal_string(s.sum, (int)t.scale));
                w.msg(6, m);
                break;
            case K_DATE:
                if (s.has_minmax) { m.s64(1, s.imin); m.s64(2, s.imax); }
                w.msg(7, m);
                break;
            case K_BINARY:
                m.s64(1, s.bytes);
                w.msg(8, m);
                break;
            default:
                break;                                   // the root struct: the counts only
        }
    }
    w.u64(10, s.has_null ? 1 : 0);
    return std::move(w.b);
}

std::vector<uint8_t> stripe_footer(const std::vector<OutStream> &streams, const std::vector<int> &encodings) {
    PbWriter w;
    for (const OutStream &s : streams) {
        PbWriter m;
        m.u64(1, (uint64_t)s.kind);
        m.u64(2, s.column);
        m.u64(3, s.length);
        w.msg(1, m);
    }
    for (int e : encodings) {
        PbWriter m;
        m.u64(1, (uint64_t)e);
        w.msg(2, m);
    }
    return std::move(w.b);
}

std::vector<uint8_t> compress_section(const std::vector<uint8_t> &raw, int codec, uint64_t block_size) {
    if (codec == C_NONE) return raw;
    if (codec != C_ZSTD) throw std::runtime_error("orc: compression kind " + std::to_string(codec) + " is not written");
    std::vector<int32_t> htab((size_t)1 << zs::kHashLog);
    std::vector<zs::Seq> seqs(zs::kMaxBlock / 4 + 1);
    std::vector<uint8_t> lits(zs::kMaxBlock), blk(zs::kMaxBlock), frame;
    std::unique_ptr<zs::EncWork> W(new zs::EncWork());
    std::vector<uint8_t> out;
    for (size_t pos = 0; pos < raw.size(); pos += block_size) {
        const size_t n = std::min<size_t>(block_size, raw.size() - pos);
        frame.resize((size_t)zs::frame_bound((int64_t)n));
        const int64_t f = zs::compress_frame(raw.data() + pos, (int64_t)n, frame.data(), (int64_t)frame.size(), htab.data(),
                                             seqs.data(), lits.data(), blk.data(), *W);
        const bool original = f < 0 || (uint64_t)f >= n;
        const uint32_t len = original ? (uint32_t)n : (uint32_t)f;
        const uint32_t h = len << 1 | (original ? 1u : 0u);
        out.push_back((uint8_t)h); out.push_back((uint8_t)(h >> 8)); out.push_back((uint8_t)(h >> 16));
        if (original) out.insert(out.end(), raw.begin() + pos, raw.begin() + pos + n);
        else out.insert(out.end(), frame.begin(), frame.begin() + f);
    }
    return out;
}

std::vector<uint8_t> row_index(const OutType &t, const std::vector<std::vector<uint64_t>> &positions,
                               const std::vector<ColumnStats> &stats) {
    PbWriter w;
    for (size_t e = 0; e < stats.size(); e++) {
        PbWriter entry;
        if (!positions[e].empty()) {
            PbWriter packed;
            for (uint64_t p : positions[e]) packed.varint(p);
            entry.bytes(1, packed.b.data(), packed.b.size());
        }
        const std::vector<uint8_t> cs = column_statistics(t, stats[e]);
        entry.bytes(2, cs.data(), cs.size());
        w.msg(1, entry);
    }
    return std::move(w.b);
}

std::vector<uint8_t> bloom_filter_index(int k, const uint64_t *words, size_t n_words, size_t n_filters) {
    PbWriter w;
    std::vector<uint8_t> le(8 * n_words);
    for (size_t f = 0; f < n_filters; f++) {
        for (size_t i = 0; i < n_words; i++)
            for (int b = 0; b < 8; b++) le[8 * i + b] = (uint8_t)(words[f * n_words + i] >> (8 * b));
        PbWriter m;
        m.u64(1, (uint64_t)k);
        m.bytes(3, le.data(), le.size());
        w.msg(1, m);
    }
    return std::move(w.b);
}

std::vector<uint8_t> file_tail(const std::vector<OutType> &types, const std::vector<std::string> &names,
                               const std::vector<OutStripe> &stripes, const std::vector<ColumnStats> &file_stats,
                               uint64_t rows, uint64_t content_length, int codec, uint64_t block_size,
                               uint64_t row_index_stride) {
    std::vector<OutType> all(1);
    all[0].kind = K_STRUCT;
    all.insert(all.end(), types.begin(), types.end());
    PbWriter meta;                                       // Metadata: per stripe, the statistics of every column
    for (const OutStripe &s : stripes) {
        PbWriter ss;
        for (size_t c = 0; c < all.size(); c++) {
            const std::vector<uint8_t> cs = column_statistics(all[c], s.stats[c]);
            ss.bytes(1, cs.data(), cs.size());
        }
        meta.msg(1, ss);
    }
    PbWriter f;                                          // Footer
    f.u64(1, 3);
    f.u64(2, content_length);
    for (const OutStripe &s : stripes) {
        PbWriter m;
        m.u64(1, s.offset);
        m.u64(2, s.index_length);
        m.u64(3, s.data_length);
        m.u64(4, s.footer_length);
        m.u64(5, s.rows);
        f.msg(3, m);
    }
    for (size_t c = 0; c < all.size(); c++) {
        PbWriter m;
        m.u64(1, (uint64_t)all[c].kind);
        if (c == 0) {
            PbWriter sub;
            for (size_t k = 1; k < all.size(); k++) sub.varint(k);
            m.bytes(2, sub.b.data(), sub.b.size());
            for (const std::string &n : names) m.str(3, n);
        }
        if (all[c].kind == K_VARCHAR) m.u64(4, all[c].max_length);
        if (all[c].kind == K_DECIMAL) { m.u64(5, all[c].precision); m.u64(6, all[c].scale); }
        f.msg(4, m);
    }
    f.u64(6, rows);
    for (size_t c = 0; c < all.size(); c++) {
        const std::vector<uint8_t> cs = column_statistics(all[c], file_stats[c]);
        f.bytes(7, cs.data(), cs.size());
    }
    f.u64(8, row_index_stride);                          // rowIndexStride, 0 = no row indexes
    const std::vector<uint8_t> meta_c = compress_section(meta.b, codec, block_size);
    const std::vector<uint8_t> foot_c = compress_section(f.b, codec, block_size);
    PbWriter ps;                                         // PostScript
    ps.u64(1, foot_c.size());
    ps.u64(2, (uint64_t)codec);
    ps.u64(3, block_size);
    const uint8_t version[2] = {0, 12};
    ps.bytes(4, version, 2);
    ps.u64(5, meta_c.size());
    ps.u64(6, 9);                                        // writerVersion ORC_14
    ps.str(8000, "ORC");
    std::vector<uint8_t> out = meta_c;
    out.insert(out.end(), foot_c.begin(), foot_c.end());
    out.insert(out.end(), ps.b.begin(), ps.b.end());
    out.push_back((uint8_t)ps.b.size());
    return out;
}

}  // namespace orc
