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

}  // namespace

FileTail parse_file(const uint8_t *file, int64_t size) {
    if (size < 4 || file[0] != 'O' || file[1] != 'R' || file[2] != 'C') throw std::runtime_error("orc: missing ORC magic");
    const uint64_t ps_len = file[size - 1];
    if ((int64_t)ps_len + 1 > size) throw std::runtime_error("orc: bad postscript length");
    FileTail t;
    uint64_t footer_len = 0;
    {
        Pb pb(file + size - 1 - ps_len, (size_t)ps_len);
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
    if (footer_len + ps_len + 1 > (uint64_t)size) throw std::runtime_error("orc: bad footer length");
    const std::vector<uint8_t> footer = inflate_section(file + size - 1 - ps_len - footer_len, footer_len, t.compression, t.block_size);
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
    for (const StripeInfo &si : t.stripes) {
        const uint64_t fo = si.offset + si.index_length + si.data_length;
        if (fo + si.footer_length > (uint64_t)size) throw std::runtime_error("orc: stripe footer outside the file");
        const std::vector<uint8_t> raw = inflate_section(file + fo, si.footer_length, t.compression, t.block_size);
        StripeFooter sf = read_stripe_footer(Pb(raw.data(), raw.size()));
        uint64_t off = si.offset;
        for (StreamInfo &s : sf.streams) {
            s.offset = off;
            off += s.length;
        }
        if (off > fo) throw std::runtime_error("orc: stream lengths exceed the stripe");
        t.stripe_footers.push_back(std::move(sf));
    }
    return t;
}

Plan plan_file(const FileTail &t, const uint8_t *file, int64_t size, const std::vector<int> &file_col_of) {
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
                if (t.compression == C_NONE) ps.out_bound = s.length;
                else {
                    const int64_t bound = orcdev::chunk_bound(file + s.offset, (int64_t)s.length, t.compression,
                                                              (int64_t)t.block_size);
                    if (bound < 0) throw std::runtime_error("orc: truncated compression chunk");
                    ps.out_bound = (uint64_t)bound;
                }
                ps.out_off = pl.scratch_bytes;
                pl.scratch_bytes += (ps.out_bound + 64 + 63) & ~(uint64_t)63;
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

std::vector<uint8_t> file_tail(const std::vector<OutType> &types, const std::vector<std::string> &names,
                               const std::vector<OutStripe> &stripes, const std::vector<ColumnStats> &file_stats,
                               uint64_t rows, uint64_t content_length, int codec, uint64_t block_size) {
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
        m.u64(2, 0);
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
    f.u64(8, 0);                                         // rowIndexStride: no row indexes
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
