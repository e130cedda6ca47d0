// orc_meta.h — host-side ORC metadata: Protocol Buffers wire reader, PostScript, Footer, stripe footers.
// Replaces what the reference takes from orc-core 1.9.2 (org.apache.orc.impl.ReaderImpl / RecordReaderImpl behind
// paimon-format/src/main/java/org/apache/paimon/format/orc/OrcReaderFactory.java:98-163, createRecordReader :280-330);
// the dependency is not under /root/reference.  The layout restated here is the public ORC specification (file tail:
// footer, postscript, 1-byte postscript length; orc_proto.proto field numbers) and the protobuf wire format.
#pragma once

#include <stdint.h>

#include <string>
#include <vector>

#include "range_reader.h"

namespace orc {

using pg::RangeReader;     // (range_reader.h: shared with the Parquet footer reader)

enum Compression { C_NONE = 0, C_ZLIB = 1, C_SNAPPY = 2, C_LZO = 3, C_LZ4 = 4, C_ZSTD = 5 };
enum TypeKind { K_BOOLEAN = 0, K_BYTE = 1, K_SHORT = 2, K_INT = 3, K_LONG = 4, K_FLOAT = 5, K_DOUBLE = 6, K_STRING = 7,
                K_BINARY = 8, K_TIMESTAMP = 9, K_LIST = 10, K_MAP = 11, K_STRUCT = 12, K_UNION = 13, K_DECIMAL = 14,
                K_DATE = 15, K_VARCHAR = 16, K_CHAR = 17, K_TIMESTAMP_INSTANT = 18 };
enum StreamKind { S_PRESENT = 0, S_DATA = 1, S_LENGTH = 2, S_DICTIONARY_DATA = 3, S_DICTIONARY_COUNT = 4, S_SECONDARY = 5,
                  S_ROW_INDEX = 6, S_BLOOM_FILTER = 7, S_BLOOM_FILTER_UTF8 = 8 };
enum EncodingKind { E_DIRECT = 0, E_DICTIONARY = 1, E_DIRECT_V2 = 2, E_DICTIONARY_V2 = 3 };

struct Type {
    int kind = -1;
    std::vector<uint32_t> subtypes;
    std::vector<std::string> field_names;
    uint32_t precision = 0, scale = 0;
};
struct StripeInfo {
    uint64_t offset = 0, index_length = 0, data_length = 0, footer_length = 0, rows = 0;
};
struct StreamInfo {
    int kind = 0;
    uint32_t column = 0;
    uint64_t length = 0;
    uint64_t offset = 0;          // absolute file offset (derived)
};
struct ColumnEncoding {
    int kind = 0;
    uint32_t dictionary_size = 0;
};
struct StripeFooter {
    std::vector<StreamInfo> streams;
    std::vector<ColumnEncoding> columns;
};
struct FileTail {
    int compression = C_NONE;
    uint64_t block_size = 262144;
    std::vector<uint32_t> version;
    uint64_t rows = 0;
    std::vector<Type> types;
    std::vector<StripeInfo> stripes;
    std::vector<StripeFooter> stripe_footers;
};

// ---- the file tail.  Every parse below throws std::runtime_error on malformed / unsupported input (NONE, ZLIB, LZ4 and
// ZSTD metadata is inflated).  A file in host memory is parsed whole by parse_file; the files of a section in device
// memory come to the host a few byte ranges at a time through read_tails.  Both go through the same steps:
// parse_tail, then stripe_footer_offset + parse_stripe_footer per stripe.

// The PostScript and Footer of a file of `size` bytes from its last n bytes (tail = the file's bytes [size - n, size),
// n >= min(size, 256) so that the PostScript is inside): 0 when both are parsed into t (which is reset first), else the
// number of last bytes the Footer needs (> n).  The PostScript and Footer lengths are checked against the file.
uint64_t parse_tail(const uint8_t *tail, uint64_t n, uint64_t size, FileTail &t);
// where stripe i's footer starts; offset + index + data + footer length are checked against the file
uint64_t stripe_footer_offset(const FileTail &t, size_t i, uint64_t size);
// stripe i's footer from its stored bytes (t.stripes[i].footer_length of them): stored as t.stripe_footers[i], with
// the absolute offsets of its streams
void parse_stripe_footer(FileTail &t, size_t i, const uint8_t *stored);

FileTail parse_file(const uint8_t *file, int64_t size);

constexpr uint64_t kTailRead = 16384;
// The tails of files of sizes[f] bytes read through rd in at most three rounds, however many files there are: the
// last min(size, 16 KiB) bytes and the magic of every file; the rest of the Footers that did not fit; the stripe
// footers of every file.  No range is queued before it is checked against its file.
std::vector<FileTail> read_tails(RangeReader &rd, const std::vector<uint64_t> &sizes);

// ---- decode plan of one file: which streams to inflate, and one task per (stripe, wanted column)
struct PlanStream {
    uint64_t offset = 0, length = 0;     // in the file
    uint64_t out_bound = 0;              // host layout only: upper bound of the inflated bytes
    uint64_t out_off = 0;                // host layout only: position in the file's stream scratch (64-byte aligned)
};
struct PlanTask {
    int stripe = 0;
    int col = 0;                         // caller's column index
    int type_id = 0;                     // ORC type id (flat schema: file column + 1)
    int kind = 0, enc = 0, scale = 0;
    uint32_t dict_size = 0;
    uint64_t dict_off_base = 0;          // position in the dictionary-offset scratch (entries)
    int64_t row0 = 0, rows = 0;          // file-relative
    int s_present = -1, s_data = -1, s_length = -1, s_dict = -1, s_secondary = -1;   // indexes into Plan::streams
};
struct Plan {
    std::vector<PlanStream> streams;
    std::vector<PlanTask> tasks;
    uint64_t scratch_bytes = 0;          // host layout only: inflated streams
    uint64_t dict_entries = 0;           // dictionary-offset scratch entries
};
// file_col_of[c] = the file's column (0-based child of the root struct) for caller column c, or < 0 = skip.  The
// streams are checked against the file's size; their compression chunks are not read (the device decoder walks them
// with k_orc_walk and lays out its scratch with k_orc_scan).
Plan plan_file(const FileTail &t, int64_t size, const std::vector<int> &file_col_of);
// The same plan with the stream scratch laid out on the host, from the file's bytes in host memory: each stream's
// out_bound from its chunk headers (orcdev::chunk_bound, the function k_orc_walk calls), out_off, scratch_bytes.  For
// host builds of the decode path.
Plan plan_file(const FileTail &t, const uint8_t *file, int64_t size, const std::vector<int> &file_col_of);

// ---- writer side: the stripe footers, the row index sections and the file tail (Metadata, Footer, PostScript,
// PostScript length) of a flat file, written DIRECT / DIRECT_V2
struct PbWriter {
    std::vector<uint8_t> b;
    void varint(uint64_t v);
    void key(uint32_t field, int wire) { varint((uint64_t)field << 3 | (uint64_t)wire); }
    void u64(uint32_t field, uint64_t v) { key(field, 0); varint(v); }
    void s64(uint32_t field, int64_t v) { key(field, 0); varint(((uint64_t)v << 1) ^ (uint64_t)(v >> 63)); }
    void f64(uint32_t field, double v);
    void bytes(uint32_t field, const void *p, size_t n);
    void str(uint32_t field, const std::string &s) { bytes(field, s.data(), s.size()); }
    void msg(uint32_t field, const PbWriter &m) { bytes(field, m.b.data(), m.b.size()); }
};

struct OutType {
    int kind = 0;
    uint32_t precision = 0, scale = 0, max_length = 0;   // DECIMAL; VARCHAR
};
// one column of one stripe or of the file; the typed message written follows the column's kind
struct ColumnStats {
    uint64_t values = 0;          // non-null values
    bool has_null = false;
    bool has_minmax = false;      // integers, DATE, DECIMAL (unscaled), FLOAT / DOUBLE
    int64_t imin = 0, imax = 0;
    double dmin = 0, dmax = 0;
    bool has_sum = false;         // integers: the exact sum fits int64; DECIMAL: always
    __int128 sum = 0;
    int64_t bytes = 0;            // STRING / VARCHAR / BINARY: total bytes of the values
    uint64_t trues = 0;           // BOOLEAN
};
struct OutStream {
    int kind = 0;
    uint32_t column = 0;
    uint64_t length = 0;
};
struct OutStripe {
    uint64_t offset = 0, index_length = 0, data_length = 0, footer_length = 0, rows = 0;
    std::vector<ColumnStats> stats;   // [0] = the root struct
};

// an unscaled decimal as the text orc_proto's DecimalStatistics carries ("-123.45")
std::string decimal_string(__int128 unscaled, int scale);
// the serialized ColumnStatistics of a column of type t
std::vector<uint8_t> column_statistics(const OutType &t, const ColumnStats &s);
// a StripeFooter: the streams in file order, one encoding per column (root first)
std::vector<uint8_t> stripe_footer(const std::vector<OutStream> &streams, const std::vector<int> &encodings);
// a section stored under the file's compression: NONE = the bytes; ZSTD = chunks of at most block_size bytes, each one
// zstd frame behind a 3-byte header, or the original bytes when the frame is not smaller
std::vector<uint8_t> compress_section(const std::vector<uint8_t> &raw, int codec, uint64_t block_size);
// a RowIndex: per row group an entry with its positions (none: the field is left out) and its statistics
std::vector<uint8_t> row_index(const OutType &t, const std::vector<std::vector<uint64_t>> &positions,
                               const std::vector<ColumnStats> &stats);
// a BloomFilterIndex of n_filters BLOOM_FILTER_UTF8 filters of k hash functions, filter f the 64-bit little-endian
// words [f * n_words, (f + 1) * n_words)
std::vector<uint8_t> bloom_filter_index(int k, const uint64_t *words, size_t n_words, size_t n_filters);
// Metadata, Footer, PostScript and its length byte.  types / names: the columns (the root struct is added);
// file_stats[0] = the root; content_length: the bytes in front of the Metadata ("ORC" and the stripes);
// row_index_stride: 0 = no row index
std::vector<uint8_t> file_tail(const std::vector<OutType> &types, const std::vector<std::string> &names,
                               const std::vector<OutStripe> &stripes, const std::vector<ColumnStats> &file_stats,
                               uint64_t rows, uint64_t content_length, int codec, uint64_t block_size,
                               uint64_t row_index_stride = 0);

}  // namespace orc
