// parquet_meta.h — host-side Parquet metadata: Thrift compact-protocol reader and writer, footer (FileMetaData).
// Replaces what the reference takes from parquet-mr 1.16.0
// (org.apache.parquet.format.* via PQ3P/hadoop/ParquetFileReader.java:277-334 footer read, and the page headers and
// footer its writer serializes).  The algorithm restated here is the public Parquet format
// specification (parquet-format: "Thrift Compact Protocol" + parquet.thrift field ids), which is what
// parquet-mr implements; the dependency itself is not vendored in /root/reference.
#pragma once

#include <stdint.h>

#include <string>
#include <vector>

#include "range_reader.h"

namespace pq {

using pg::RangeReader;     // (range_reader.h: shared with the ORC tail reader)

enum PhysType { T_BOOLEAN = 0, T_INT32 = 1, T_INT64 = 2, T_INT96 = 3, T_FLOAT = 4, T_DOUBLE = 5, T_BYTE_ARRAY = 6,
                T_FIXED_LEN_BYTE_ARRAY = 7 };
enum Encoding { E_PLAIN = 0, E_PLAIN_DICTIONARY = 2, E_RLE = 3, E_BIT_PACKED = 4, E_DELTA_BINARY_PACKED = 5,
                E_DELTA_LENGTH_BYTE_ARRAY = 6, E_DELTA_BYTE_ARRAY = 7, E_RLE_DICTIONARY = 8, E_BYTE_STREAM_SPLIT = 9 };
enum Codec { C_UNCOMPRESSED = 0, C_SNAPPY = 1, C_GZIP = 2, C_LZO = 3, C_BROTLI = 4, C_LZ4 = 5, C_ZSTD = 6, C_LZ4_RAW = 7 };
enum PageType { P_DATA = 0, P_INDEX = 1, P_DICTIONARY = 2, P_DATA_V2 = 3 };
enum Repetition { R_REQUIRED = 0, R_OPTIONAL = 1, R_REPEATED = 2 };
// Thrift compact protocol wire types
enum TType { CT_STOP = 0, CT_TRUE = 1, CT_FALSE = 2, CT_BYTE = 3, CT_I16 = 4, CT_I32 = 5, CT_I64 = 6, CT_DOUBLE = 7,
             CT_BINARY = 8, CT_LIST = 9, CT_SET = 10, CT_MAP = 11, CT_STRUCT = 12 };

struct SchemaElement {
    int32_t type = -1;            // PhysType; -1 for groups
    int32_t type_length = 0;
    int32_t repetition = 0;
    std::string name;
    int32_t num_children = 0;
    int32_t converted_type = -1;
};

struct ColumnChunk {
    int32_t type = -1;
    int32_t codec = 0;
    int64_t num_values = 0;
    int64_t total_uncompressed_size = 0;
    int64_t total_compressed_size = 0;
    int64_t data_page_offset = 0;
    int64_t dictionary_page_offset = 0;   // 0 = none
    std::vector<int32_t> encodings;
    std::vector<std::string> path;
    int64_t start() const {
        return (dictionary_page_offset > 0 && dictionary_page_offset < data_page_offset) ? dictionary_page_offset
                                                                                        : data_page_offset;
    }
};

struct RowGroup {
    int64_t num_rows = 0;
    int64_t total_byte_size = 0;
    std::vector<ColumnChunk> columns;
};

struct FileMetaData {
    int32_t version = 0;
    int64_t num_rows = 0;
    std::vector<SchemaElement> schema;   // flattened, root first
    std::vector<RowGroup> row_groups;
    std::string created_by;
};

// Both throw std::runtime_error on malformed input.
// A file in host memory, whole.
FileMetaData parse_footer(const uint8_t *file, int64_t size);
// The footers of files of sizes[f] bytes whose bytes are elsewhere (device memory), read through rd in two rounds:
// the last 8 bytes of every file ([footer length:4 LE]["PAR1"]), then every footer.  No range is queued before it is
// checked against its file.  Unlike parse_footer, the leading "PAR1" is not read.
std::vector<FileMetaData> read_footers(RangeReader &rd, const std::vector<uint64_t> &sizes);
// The Thrift footers (without length and magic) of several files, in order.  Throws the error of the first malformed
// footer in the order given.
struct FooterBytes {
    const uint8_t *bytes;
    int64_t size;
};
std::vector<FileMetaData> parse_footers(const std::vector<FooterBytes> &footers);

inline void put_varint(std::vector<uint8_t> &b, uint64_t v) {
    while (v >= 0x80) { b.push_back((uint8_t)(v | 0x80)); v >>= 7; }
    b.push_back((uint8_t)v);
}

// Thrift compact protocol writer: the page headers and the footer of the files the device encoder writes
struct ThriftWriter {
    std::vector<uint8_t> b;
    std::vector<int> last{0};                           // per open struct: the id of its last field
    void varint(uint64_t v) { put_varint(b, v); }
    void zigzag(int64_t v) { varint(((uint64_t)v << 1) ^ (uint64_t)(v >> 63)); }
    void field(int id, int type) {
        int d = id - last.back();
        if (d > 0 && d <= 15) b.push_back((uint8_t)((d << 4) | type));
        else { b.push_back((uint8_t)type); zigzag(id); }
        last.back() = id;
    }
    void i32(int id, int32_t v) { field(id, CT_I32); zigzag(v); }
    void i64(int id, int64_t v) { field(id, CT_I64); zigzag(v); }
    void binary(const void *p, size_t n) { varint(n); b.insert(b.end(), (const uint8_t *)p, (const uint8_t *)p + n); }
    void bin(int id, const void *p, size_t n) { field(id, CT_BINARY); binary(p, n); }
    void str(int id, const std::string &s) { bin(id, s.data(), s.size()); }
    void list(int id, int elem_type, size_t n) {
        field(id, CT_LIST);
        if (n < 15) b.push_back((uint8_t)((n << 4) | elem_type));
        else { b.push_back((uint8_t)(0xF0 | elem_type)); varint(n); }
    }
    void struct_field(int id) { field(id, CT_STRUCT); last.push_back(0); }
    void struct_elem() { last.push_back(0); }           // list element
    void end() { b.push_back(CT_STOP); last.pop_back(); }
};

}  // namespace pq
