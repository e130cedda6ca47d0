// The Parquet footer (pq::FileMetaData) as text, for the host harnesses that compare two parses.
#pragma once

#include <string>

#include "parquet_meta.h"

// every field the decoder uses, as text: two parses are equal when their dumps are
inline std::string dump(const pq::FileMetaData &m) {
    std::string o = "v" + std::to_string(m.version) + " r" + std::to_string(m.num_rows) + " " + m.created_by;
    for (const pq::SchemaElement &e : m.schema)
        o += "\nE" + e.name + " t" + std::to_string(e.type) + " l" + std::to_string(e.type_length) + " r" +
             std::to_string(e.repetition) + " n" + std::to_string(e.num_children) + " c" + std::to_string(e.converted_type);
    for (const pq::RowGroup &g : m.row_groups) {
        o += "\nG" + std::to_string(g.num_rows) + " " + std::to_string(g.total_byte_size) + ":";
        for (const pq::ColumnChunk &c : g.columns) {
            o += " (" + std::to_string(c.type) + "," + std::to_string(c.codec) + "," + std::to_string(c.num_values) + "," +
                 std::to_string(c.total_uncompressed_size) + "," + std::to_string(c.total_compressed_size) + "," +
                 std::to_string(c.data_page_offset) + "," + std::to_string(c.dictionary_page_offset) + " e";
            for (int32_t e : c.encodings) o += std::to_string(e) + ".";
            for (const std::string &p : c.path) o += "/" + p;
            o += ")";
        }
    }
    return o;
}
