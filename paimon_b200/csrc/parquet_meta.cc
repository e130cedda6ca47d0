// parquet_meta.cc — Thrift compact protocol reader + Parquet footer parse (see parquet_meta.h).
#include "parquet_meta.h"

#include <algorithm>
#include <stdexcept>

namespace pq {

namespace {

struct Reader {
    const uint8_t *p, *end;
    Reader(const uint8_t *b, int64_t n) : p(b), end(b + n) {}

    uint8_t byte() {
        if (p >= end) throw std::runtime_error("parquet: truncated thrift data");
        return *p++;
    }
    uint64_t varint() {
        if (p < end && !(*p & 0x80)) return *p++;      // (most varints of a footer are one byte)
        uint64_t v = 0;
        int shift = 0;
        while (true) {
            uint8_t b = byte();
            v |= (uint64_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) return v;
            shift += 7;
            if (shift > 63) throw std::runtime_error("parquet: bad varint");
        }
    }
    int64_t zigzag() {
        uint64_t v = varint();
        return (int64_t)(v >> 1) ^ -(int64_t)(v & 1);
    }
    std::string binary() {
        uint64_t n = varint();
        if ((uint64_t)(end - p) < n) throw std::runtime_error("parquet: truncated binary");
        std::string s((const char *)p, (size_t)n);
        p += n;
        return s;
    }
    void skip_binary() {
        uint64_t n = varint();
        if ((uint64_t)(end - p) < n) throw std::runtime_error("parquet: truncated binary");
        p += n;
    }
    // returns false at STOP; otherwise sets field id and type
    bool field(int16_t &last_id, int &type) {
        uint8_t h = byte();
        if (h == CT_STOP) return false;
        int delta = h >> 4;
        type = h & 0x0f;
        if (delta == 0) last_id = (int16_t)zigzag();
        else last_id = (int16_t)(last_id + delta);
        return true;
    }
    void list_header(int &elem_type, uint32_t &size) {
        uint8_t h = byte();
        elem_type = h & 0x0f;
        size = h >> 4;
        if (size == 15) size = (uint32_t)varint();
    }
    void skip(int type) {
        switch (type) {
            case CT_TRUE: case CT_FALSE: return;
            case CT_BYTE: byte(); return;
            case CT_I16: case CT_I32: case CT_I64: varint(); return;
            case CT_DOUBLE: if (end - p < 8) throw std::runtime_error("parquet: truncated double"); p += 8; return;
            case CT_BINARY: skip_binary(); return;
            case CT_LIST: case CT_SET: {
                int et; uint32_t n;
                list_header(et, n);
                for (uint32_t i = 0; i < n; i++) skip_elem(et);
                return;
            }
            case CT_MAP: {
                uint32_t n = (uint32_t)varint();
                if (n == 0) return;
                uint8_t kv = byte();
                for (uint32_t i = 0; i < n; i++) { skip_elem(kv >> 4); skip_elem(kv & 0x0f); }
                return;
            }
            case CT_STRUCT: {
                int16_t id = 0;
                int t;
                while (field(id, t)) skip(t);
                return;
            }
            default: throw std::runtime_error("parquet: unknown thrift type");
        }
    }
    void skip_elem(int type) {
        if (type == CT_TRUE || type == CT_FALSE) { byte(); return; }   // bools in containers take one byte
        skip(type);
    }
};

SchemaElement read_schema_element(Reader &r) {
    SchemaElement e;
    int16_t id = 0;
    int t;
    while (r.field(id, t)) {
        switch (id) {
            case 1: e.type = (int32_t)r.zigzag(); break;
            case 2: e.type_length = (int32_t)r.zigzag(); break;
            case 3: e.repetition = (int32_t)r.zigzag(); break;
            case 4: e.name = r.binary(); break;
            case 5: e.num_children = (int32_t)r.zigzag(); break;
            case 6: e.converted_type = (int32_t)r.zigzag(); break;
            default: r.skip(t);
        }
    }
    return e;
}

ColumnChunk read_column_meta(Reader &r) {
    ColumnChunk c;
    int16_t id = 0;
    int t;
    while (r.field(id, t)) {
        switch (id) {
            case 1: c.type = (int32_t)r.zigzag(); break;
            case 2: {
                int et; uint32_t n;
                r.list_header(et, n);
                c.encodings.reserve(std::min<uint32_t>(n, 16));
                for (uint32_t i = 0; i < n; i++) c.encodings.push_back((int32_t)r.zigzag());
                break;
            }
            case 3: {
                int et; uint32_t n;
                r.list_header(et, n);
                c.path.reserve(std::min<uint32_t>(n, 16));
                for (uint32_t i = 0; i < n; i++) c.path.push_back(r.binary());
                break;
            }
            case 4: c.codec = (int32_t)r.zigzag(); break;
            case 5: c.num_values = r.zigzag(); break;
            case 6: c.total_uncompressed_size = r.zigzag(); break;
            case 7: c.total_compressed_size = r.zigzag(); break;
            case 9: c.data_page_offset = r.zigzag(); break;
            case 11: c.dictionary_page_offset = r.zigzag(); break;
            default: r.skip(t);
        }
    }
    return c;
}

ColumnChunk read_column_chunk(Reader &r) {
    ColumnChunk c;
    int16_t id = 0;
    int t;
    bool have = false;
    while (r.field(id, t)) {
        if (id == 3 && t == CT_STRUCT) { c = read_column_meta(r); have = true; }
        else r.skip(t);
    }
    if (!have) throw std::runtime_error("parquet: column chunk without meta_data");
    return c;
}

RowGroup read_row_group(Reader &r) {
    RowGroup g;
    int16_t id = 0;
    int t;
    while (r.field(id, t)) {
        switch (id) {
            case 1: {
                int et; uint32_t n;
                r.list_header(et, n);
                g.columns.reserve(std::min<uint32_t>(n, 4096));
                for (uint32_t i = 0; i < n; i++) g.columns.push_back(read_column_chunk(r));
                break;
            }
            case 2: g.total_byte_size = r.zigzag(); break;
            case 3: g.num_rows = r.zigzag(); break;
            default: r.skip(t);
        }
    }
    return g;
}

FileMetaData parse_footer_thrift(const uint8_t *footer, int64_t flen) {
    Reader r(footer, flen);
    FileMetaData m;
    int16_t id = 0;
    int t;
    while (r.field(id, t)) {
        switch (id) {
            case 1: m.version = (int32_t)r.zigzag(); break;
            case 2: {
                int et; uint32_t n;
                r.list_header(et, n);
                m.schema.reserve(std::min<uint32_t>(n, 4096));
                for (uint32_t i = 0; i < n; i++) m.schema.push_back(read_schema_element(r));
                break;
            }
            case 3: m.num_rows = r.zigzag(); break;
            case 4: {
                int et; uint32_t n;
                r.list_header(et, n);
                m.row_groups.reserve(std::min<uint32_t>(n, 4096));
                for (uint32_t i = 0; i < n; i++) m.row_groups.push_back(read_row_group(r));
                break;
            }
            case 6: m.created_by = r.binary(); break;
            default: r.skip(t);
        }
    }
    return m;
}

int64_t footer_length(const uint8_t *tail8) {
    if (tail8[4] != 'P' || tail8[5] != 'A' || tail8[6] != 'R' || tail8[7] != '1')
        throw std::runtime_error("parquet: missing PAR1 magic (encrypted or not a Parquet file)");
    return (int64_t)((uint32_t)tail8[0] | ((uint32_t)tail8[1] << 8) | ((uint32_t)tail8[2] << 16) | ((uint32_t)tail8[3] << 24));
}

}  // namespace

FileMetaData parse_footer(const uint8_t *file, int64_t size) {
    if (size < 12 || file[0] != 'P' || file[1] != 'A' || file[2] != 'R' || file[3] != '1')
        throw std::runtime_error("parquet: missing PAR1 magic (encrypted or not a Parquet file)");
    const int64_t flen = footer_length(file + size - 8);
    if (flen + 12 > size) throw std::runtime_error("parquet: bad footer length");
    return parse_footer_thrift(file + size - 8 - flen, flen);
}

std::vector<FileMetaData> read_footers(RangeReader &rd, const std::vector<uint64_t> &sizes) {
    const size_t nf = sizes.size();
    std::vector<uint8_t> tails(8 * nf);
    for (size_t f = 0; f < nf; f++) {
        if (sizes[f] < 12) throw std::runtime_error("parquet: missing PAR1 magic (encrypted or not a Parquet file)");
        rd.read((int)f, sizes[f] - 8, 8, &tails[8 * f]);
    }
    rd.flush();
    std::vector<std::vector<uint8_t>> footers(nf);
    for (size_t f = 0; f < nf; f++) {
        const int64_t flen = footer_length(&tails[8 * f]);
        if ((uint64_t)flen + 12 > sizes[f]) throw std::runtime_error("parquet: bad footer length");
        footers[f].resize((size_t)flen);
        rd.read((int)f, sizes[f] - 8 - (uint64_t)flen, (uint64_t)flen, footers[f].data());
    }
    rd.flush();
    std::vector<FooterBytes> spans(nf);
    for (size_t f = 0; f < nf; f++) spans[f] = FooterBytes{footers[f].data(), (int64_t)footers[f].size()};
    return parse_footers(spans);
}

std::vector<FileMetaData> parse_footers(const std::vector<FooterBytes> &footers) {
    // (on the calling thread: parsing the bench's 16 footers on 8 threads measured about 2 ms slower per section on
    // a shared host, DESIGN.md §5)
    std::vector<FileMetaData> m(footers.size());
    for (size_t f = 0; f < footers.size(); f++) m[f] = parse_footer_thrift(footers[f].bytes, footers[f].size);
    return m;
}

}  // namespace pq
