// arrow_export.cu — hand a merged batch (or a decoded run) to the JVM through the Arrow C Data Interface.
//
// SURVEY.md §8(b): the Java side imports the batch with org.apache.arrow.c.Data.importVectorSchemaRoot and wraps it
// with paimon-arrow's ArrowBatchReader (paimon-arrow/src/main/java/org/apache/paimon/arrow/reader/ArrowBatchReader.java:
// 74-115), which maps columns BY FIELD NAME — so the exported schema carries the Paimon file field names
// (_KEY_*, _SEQUENCE_NUMBER, _VALUE_KIND, value fields; KeyValue.java:130-138, SpecialFields.java:76-83).
// The struct layouts below restate the public Arrow C Data Interface specification (ArrowSchema / ArrowArray with
// release callbacks); the buffers are page-locked host memory owned by the exported array and freed by its release
// callback, which is what RecordReader.RecordIterator.releaseBatch() calls on the Java side
// (paimon-common/.../reader/RecordReader.java:42-72).
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "pg_internal.h"

namespace pg {
namespace {

struct SchemaPriv {
    std::vector<std::string> names, formats;
    std::vector<ArrowSchema> children;
    std::vector<ArrowSchema *> child_ptrs;
};
void release_child_schema(ArrowSchema *s) { s->release = nullptr; }
void release_schema(ArrowSchema *s) {
    if (!s || !s->release) return;
    auto *p = (SchemaPriv *)s->private_data;
    for (auto &c : p->children) if (c.release) c.release(&c);
    delete p;
    s->release = nullptr;
}

struct ArrayPriv {
    void *pinned = nullptr;                            // one page-locked allocation behind every buffer
    std::vector<ArrowArray> children;
    std::vector<ArrowArray *> child_ptrs;
    std::vector<std::vector<const void *>> buffers;    // per child
    const void *top_buffers[1] = {nullptr};
};
void release_child_array(ArrowArray *a) { a->release = nullptr; }
void release_array(ArrowArray *a) {
    if (!a || !a->release) return;
    auto *p = (ArrayPriv *)a->private_data;
    for (auto &c : p->children) if (c.release) c.release(&c);
    if (p->pinned) cudaFreeHost(p->pinned);
    delete p;
    a->release = nullptr;
}

const char *arrow_format(int t) {
    switch (t) {
        case PG_INT8: return "c";
        case PG_INT16: return "s";
        case PG_INT32: return "i";
        case PG_INT64: return "l";
        case PG_FLOAT: return "f";
        case PG_DOUBLE: return "g";
        case PG_BOOL: return "b";
        case PG_STRING: return "u";
        default: return "z";
    }
}

}  // namespace

static pg_status export_arrow(uint64_t source, const char *const *names, int64_t row0, int64_t n_rows,
                              ArrowArray *out, ArrowSchema *out_schema) {
    BatchColumns batch;                                 // held until the copies below are done
    pg_status st = batch_columns(source, &batch);
    if (st) return st;
    const Schema *s = batch.schema.get();
    std::vector<DevColumn> &cols = batch.cols;
    if (n_rows < 0) n_rows = batch.n_rows - row0;
    if (row0 < 0 || n_rows < 0 || row0 + n_rows > batch.n_rows) return fail(PG_ERR_INVALID, "arrow export: row range outside the batch");
    // columns a read-type projection left out of the batch are not exported
    std::vector<int> present;
    for (int c = 0; c < s->n_cols(); c++)
        if (cols[c].data || cols[c].offsets || batch.n_rows == 0) present.push_back(c);
    {
        std::vector<DevColumn> pc;
        for (int c : present) pc.push_back(cols[c]);
        cols.swap(pc);
    }
    const int nc = (int)present.size();
    auto field_of = [&](int i) { return s->field(present[i]); };
    // validity bitmaps are byte-granular; an empty range starts at row0 itself: an importer sizes a var-len child's
    // payload from offsets[offset + length] but slices it from offsets[offset], so no rows must mean no offset either
    const int64_t lo = n_rows > 0 ? row0 & ~(int64_t)7 : row0;
    const int64_t delta = row0 - lo, m = n_rows + delta; // rows copied per column; children carry offset = delta
    auto pad = [](size_t b) { return (b + 63) & ~(size_t)63; };

    // ---- sizes: var-len payload ranges need the boundary offsets
    std::vector<int32_t> off_lo(nc, 0), off_hi(nc, 0);
    for (int c = 0; c < nc; c++) {
        if (!is_varlen(field_of(c).type) || m == 0) continue;
        PG_CUDA(cudaMemcpy(&off_lo[c], cols[c].offsets + lo, 4, cudaMemcpyDeviceToHost));
        PG_CUDA(cudaMemcpy(&off_hi[c], cols[c].offsets + lo + m, 4, cudaMemcpyDeviceToHost));
    }
    std::vector<size_t> o_val(nc), o_main(nc), o_data(nc);
    size_t bytes = 64;
    for (int c = 0; c < nc; c++) {
        const pg_field f = field_of(c);
        o_val[c] = bytes;
        if (cols[c].validity) bytes += pad((size_t)((m + 7) / 8) + 8);
        o_main[c] = bytes;
        if (is_varlen(f.type)) {
            bytes += pad(4 * (size_t)(m + 1));
            o_data[c] = bytes;
            bytes += pad((size_t)(off_hi[c] - off_lo[c]) + 8);
        } else if (f.type == PG_BOOL) {
            bytes += pad((size_t)m + 8);                // one byte per value from the device ...
            o_data[c] = bytes;
            bytes += pad((size_t)((m + 7) / 8) + 8);    // ... bit-packed for Arrow
        } else {
            bytes += pad((size_t)m * type_width(f.type) + 8);
        }
    }
    auto priv = std::make_unique<ArrayPriv>();
    PG_CUDA(cudaMallocHost(&priv->pinned, bytes));
    unsigned char *h = (unsigned char *)priv->pinned;
    // ---- device -> host
    for (int c = 0; c < nc && m > 0; c++) {
        const pg_field f = field_of(c);
        const DevColumn &dc = cols[c];
        if (dc.validity) PG_CUDA(cudaMemcpyAsync(h + o_val[c], dc.validity + lo / 8, (size_t)((m + 7) / 8), cudaMemcpyDeviceToHost, 0));
        if (is_varlen(f.type)) {
            PG_CUDA(cudaMemcpyAsync(h + o_main[c], dc.offsets + lo, 4 * (size_t)(m + 1), cudaMemcpyDeviceToHost, 0));
            if (off_hi[c] > off_lo[c])
                PG_CUDA(cudaMemcpyAsync(h + o_data[c], (const unsigned char *)dc.data + off_lo[c], (size_t)(off_hi[c] - off_lo[c]),
                                        cudaMemcpyDeviceToHost, 0));
        } else {
            const int w = type_width(f.type);
            PG_CUDA(cudaMemcpyAsync(h + o_main[c], (const unsigned char *)dc.data + lo * w, (size_t)m * w, cudaMemcpyDeviceToHost, 0));
        }
    }
    PG_CUDA(cudaStreamSynchronize(0));

    // ---- arrays
    priv->children.resize(nc);
    priv->child_ptrs.resize(nc);
    priv->buffers.resize(nc);
    for (int c = 0; c < nc; c++) {
        const pg_field f = field_of(c);
        ArrowArray &a = priv->children[c];
        memset(&a, 0, sizeof(a));
        a.length = n_rows;
        a.offset = delta;
        a.null_count = cols[c].validity ? -1 : 0;
        const void *val = cols[c].validity ? (const void *)(h + o_val[c]) : nullptr;
        if (is_varlen(f.type)) {
            int32_t *o = (int32_t *)(h + o_main[c]);
            const int32_t base = m > 0 ? o[0] : 0;
            for (int64_t i = 0; i <= m && m > 0; i++) o[i] -= base;
            if (m == 0) o[0] = 0;
            priv->buffers[c] = {val, o, h + o_data[c]};
        } else if (f.type == PG_BOOL) {
            const uint8_t *bytes8 = h + o_main[c];
            uint8_t *bits = h + o_data[c];
            memset(bits, 0, (size_t)((m + 7) / 8));
            for (int64_t i = 0; i < m; i++) if (bytes8[i]) bits[i >> 3] |= (uint8_t)(1u << (i & 7));
            priv->buffers[c] = {val, bits};
        } else {
            priv->buffers[c] = {val, h + o_main[c]};
        }
        a.n_buffers = (int64_t)priv->buffers[c].size();
        a.buffers = priv->buffers[c].data();
        a.release = release_child_array;
        priv->child_ptrs[c] = &a;
    }
    memset(out, 0, sizeof(*out));
    out->length = n_rows;
    out->null_count = 0;
    out->n_buffers = 1;
    out->buffers = priv->top_buffers;
    out->n_children = nc;
    out->children = priv->child_ptrs.data();
    out->release = release_array;
    out->private_data = priv.release();

    // ---- schema: a struct of the file fields, by name
    if (out_schema) {
        auto sp = std::make_unique<SchemaPriv>();
        sp->names.resize(nc);
        sp->children.resize(nc);
        sp->child_ptrs.resize(nc);
        for (int c = 0; c < nc; c++) {
            sp->names[c] = names && names[present[c]] ? names[present[c]] : ("c" + std::to_string(present[c]));
            ArrowSchema &cs = sp->children[c];
            memset(&cs, 0, sizeof(cs));
            cs.format = arrow_format(field_of(c).type);
            cs.name = sp->names[c].c_str();
            cs.flags = (field_of(c).nullable || cols[c].validity) ? 2 : 0;      // ARROW_FLAG_NULLABLE
            cs.release = release_child_schema;
            sp->child_ptrs[c] = &cs;
        }
        memset(out_schema, 0, sizeof(*out_schema));
        out_schema->format = "+s";
        out_schema->name = "";
        out_schema->n_children = nc;
        out_schema->children = sp->child_ptrs.data();
        out_schema->release = release_schema;
        out_schema->private_data = sp.release();
    }
    return PG_OK;
}

}  // namespace pg

using namespace pg;

extern "C" pg_status pg_export_arrow(uint64_t source, const char *const *column_names, int64_t row0, int64_t n_rows,
                                     struct ArrowArray *out, struct ArrowSchema *out_schema) {
    if (!out) return fail(PG_ERR_INVALID, "null argument");
    pg_status st = ensure_device();
    if (st) return st;
    return export_arrow(source, column_names, row0, n_rows, out, out_schema);
}
