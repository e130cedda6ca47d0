// The ORC file tail (orc::FileTail) as text, for the host harnesses that compare two parses.
#pragma once

#include <string>

#include "orc_meta.h"

// every field the decoder uses, as text: two parses are equal when their dumps are
inline std::string dump(const orc::FileTail &t) {
    std::string o = "c" + std::to_string(t.compression) + " b" + std::to_string(t.block_size) + " r" + std::to_string(t.rows) + " v";
    for (uint32_t v : t.version) o += std::to_string(v) + ".";
    for (const orc::Type &ty : t.types) {
        o += "\nT" + std::to_string(ty.kind) + " p" + std::to_string(ty.precision) + " s" + std::to_string(ty.scale) + " [";
        for (uint32_t s : ty.subtypes) o += std::to_string(s) + ",";
        o += "] [";
        for (const std::string &n : ty.field_names) o += n + ",";
        o += "]";
    }
    for (size_t i = 0; i < t.stripes.size(); i++) {
        const orc::StripeInfo &si = t.stripes[i];
        o += "\nS" + std::to_string(si.offset) + " " + std::to_string(si.index_length) + " " + std::to_string(si.data_length) +
             " " + std::to_string(si.footer_length) + " " + std::to_string(si.rows) + ":";
        for (const orc::StreamInfo &st : t.stripe_footers[i].streams)
            o += " (" + std::to_string(st.kind) + "," + std::to_string(st.column) + "," + std::to_string(st.length) + "@" +
                 std::to_string(st.offset) + ")";
        o += " |";
        for (const orc::ColumnEncoding &e : t.stripe_footers[i].columns)
            o += " " + std::to_string(e.kind) + "/" + std::to_string(e.dictionary_size);
    }
    return o;
}
