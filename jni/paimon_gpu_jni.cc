// paimon_gpu_jni.cc — thin JNI shim over the C ABI of libpaimon_gpu.so (include/paimon_gpu.h).
//
// One Java native method per C function; handles are jlong, buffers are direct ByteBuffers
// (GetDirectBufferAddress), errors become java.lang.RuntimeException / UnsupportedOperationException /
// IllegalArgumentException with the message of pg_last_error() — the convention of the reference's only
// in-tree native code (paimon-tantivy/paimon-tantivy-jni/rust/src/lib.rs:32-35, 72-155).
//
// Every function include/paimon_gpu.h exports has a binding here (tests/test_abi_cpu.py checks the list).
// The build image has no JDK (no jni.h), so the real shim is built only where JAVA_HOME is set:
//   g++ -std=c++17 -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude
//       jni/paimon_gpu_jni.cc -Lpaimon_b200 -lpaimon_gpu -o libpaimon_gpu_jni.so
// Here it is syntax-checked against jni/stub/jni.h (the JNI specification's signatures):
//   g++ -std=c++17 -fsyntax-only -Ijni/stub -Iinclude jni/paimon_gpu_jni.cc          (`make jni-check`)
// The Java side (org.apache.paimon.gpu.NativeMerge) is listed in INTEGRATION.md.
#if __has_include(<jni.h>)
#include <jni.h>

#include <string>
#include <vector>

#include "paimon_gpu.h"

namespace {

void throw_for(JNIEnv *env, pg_status st) {
    const char *cls = "java/lang/RuntimeException";
    if (st == PG_ERR_UNSUPPORTED) cls = "java/lang/UnsupportedOperationException";
    if (st == PG_ERR_INVALID || st == PG_ERR_MERGE_FUNCTION) cls = "java/lang/IllegalArgumentException";
    env->ThrowNew(env->FindClass(cls), pg_last_error());
}

#define PG_CHECK(expr)                        \
    do {                                      \
        pg_status _st = (expr);               \
        if (_st != PG_OK) {                   \
            throw_for(env, _st);              \
            return 0;                         \
        }                                     \
    } while (0)

// names[] (String[]) -> C strings kept alive by `keep`
std::vector<const char *> utf_names(JNIEnv *env, jobjectArray names, std::vector<std::string> &keep) {
    const jsize nc = names ? env->GetArrayLength(names) : 0;
    keep.resize(nc);
    std::vector<const char *> ptrs(nc);
    for (jsize c = 0; c < nc; c++) {
        jstring js = (jstring)env->GetObjectArrayElement(names, c);
        const char *u = env->GetStringUTFChars(js, nullptr);
        keep[c] = u;
        env->ReleaseStringUTFChars(js, u);
        ptrs[c] = keep[c].c_str();
    }
    return ptrs;
}

}  // namespace

extern "C" {

JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_abiVersion(JNIEnv *, jclass) { return pg_abi_version(); }

JNIEXPORT jstring JNICALL Java_org_apache_paimon_gpu_NativeMerge_lastError(JNIEnv *env, jclass) {
    return env->NewStringUTF(pg_last_error());
}

JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_init(JNIEnv *env, jclass, jint device) {
    PG_CHECK(pg_init(device));
    return 0;
}

JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_shutdown(JNIEnv *env, jclass) {
    PG_CHECK(pg_shutdown());
    return 0;
}

// give cached device buffers back to the driver (e.g. from a memory-pressure hook)
JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_trim(JNIEnv *env, jclass) {
    PG_CHECK(pg_trim());
    return 0;
}

// int[] keyTypes, int[] valTypes, boolean[] valNullable -> schema handle
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_schemaCreate(JNIEnv *env, jclass, jintArray keyTypes,
                                                                             jintArray valTypes,
                                                                             jbooleanArray valNullable) {
    jsize nk = env->GetArrayLength(keyTypes), nv = env->GetArrayLength(valTypes);
    std::vector<jint> kt(nk), vt(nv);
    std::vector<jboolean> vn(nv);
    env->GetIntArrayRegion(keyTypes, 0, nk, kt.data());
    env->GetIntArrayRegion(valTypes, 0, nv, vt.data());
    env->GetBooleanArrayRegion(valNullable, 0, nv, vn.data());
    std::vector<pg_field> kf(nk), vf(nv);
    for (jsize i = 0; i < nk; i++) kf[i] = pg_field{kt[i], 0};
    for (jsize i = 0; i < nv; i++) vf[i] = pg_field{vt[i], vn[i] ? 1 : 0};
    pg_schema_desc d{nk, nv, kf.data(), vf.data()};
    uint64_t h = 0;
    PG_CHECK(pg_schema_create(&d, &h));
    return (jlong)h;
}

JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_schemaFree(JNIEnv *env, jclass, jlong h) {
    PG_CHECK(pg_schema_free((uint64_t)h));
    return 0;
}

// the declarative MergeFunction (what MergeFunctionFactory.create(readType) would have built)
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeSpecCreate(
    JNIEnv *env, jclass, jlong schema, jint engine, jboolean ignoreDelete, jboolean removeRecordOnDelete,
    jboolean dropDelete, jintArray seqFields, jboolean seqAscending, jintArray agg, jbooleanArray ignoreRetract,
    jintArray groupSeqStart, jintArray groupSeqFields, jintArray fieldGroup, jbooleanArray groupPartialDelete,
    jbooleanArray readFields, jintArray decimal) {
    // every per-field array has one entry per VALUE field of the schema (pg_merge_spec_create reads n_val entries)
    int32_t n_key = 0, n_val = 0;
    PG_CHECK(pg_schema_info((uint64_t)schema, &n_key, &n_val));
    const jsize nv = n_val;
    auto bad_len = [&](jarray a) { return a != nullptr && env->GetArrayLength(a) != nv; };
    if (bad_len(agg) || bad_len(ignoreRetract) || bad_len(fieldGroup) || bad_len(groupPartialDelete) || bad_len(readFields) ||
        bad_len(decimal)) {
        env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"),
                      "per-field arrays must have one entry per value field of the schema");
        return 0;
    }
    jsize ns = seqFields ? env->GetArrayLength(seqFields) : 0;
    std::vector<jint> sf(ns), ag(nv, 0);
    std::vector<jboolean> ir(nv, 0);
    if (ns) env->GetIntArrayRegion(seqFields, 0, ns, sf.data());
    if (nv && agg) env->GetIntArrayRegion(agg, 0, nv, ag.data());
    if (nv && ignoreRetract) env->GetBooleanArrayRegion(ignoreRetract, 0, nv, ir.data());
    std::vector<uint8_t> ir8(ir.begin(), ir.end());
    pg_merge_spec sp{};
    sp.engine = engine;
    sp.ignore_delete = ignoreDelete;
    sp.remove_record_on_delete = removeRecordOnDelete;
    sp.drop_delete = dropDelete;
    sp.n_seq_fields = ns;
    sp.seq_fields = ns ? sf.data() : nullptr;
    sp.seq_ascending = seqAscending;
    sp.agg = nv && agg ? ag.data() : nullptr;
    sp.ignore_retract = nv && ignoreRetract ? ir8.data() : nullptr;
    // partial-update sequence groups (PartialUpdateMergeFunction.Factory: fields.<seq>.sequence-group)
    std::vector<jint> gs, gf, fg;
    std::vector<uint8_t> gpd8;
    if (groupSeqStart && env->GetArrayLength(groupSeqStart) > 1 && groupSeqFields && fieldGroup) {
        gs.resize(env->GetArrayLength(groupSeqStart));
        gf.resize(env->GetArrayLength(groupSeqFields));
        fg.resize(nv);
        env->GetIntArrayRegion(groupSeqStart, 0, (jsize)gs.size(), gs.data());
        env->GetIntArrayRegion(groupSeqFields, 0, (jsize)gf.size(), gf.data());
        env->GetIntArrayRegion(fieldGroup, 0, nv, fg.data());
        if (groupPartialDelete) {
            std::vector<jboolean> gpd(nv);
            env->GetBooleanArrayRegion(groupPartialDelete, 0, nv, gpd.data());
            gpd8.assign(gpd.begin(), gpd.end());
        }
        sp.n_sequence_groups = (int32_t)gs.size() - 1;
        sp.group_seq_start = gs.data();
        sp.group_seq_fields = gf.data();
        sp.field_group = fg.data();
        sp.group_partial_delete = gpd8.empty() ? nullptr : gpd8.data();
    }
    // read-type projection (MergeFunctionFactory.create(readType)): null = every field
    std::vector<uint8_t> rf8;
    if (readFields) {
        std::vector<jboolean> rf(nv);
        if (nv) env->GetBooleanArrayRegion(readFields, 0, nv, rf.data());
        rf8.assign(rf.begin(), rf.end());
        sp.read_fields = rf8.data();
    }
    // DECIMAL value fields: precision << 8 | scale, 0 for other types; null = no DECIMAL field
    std::vector<jint> dec;
    if (decimal && nv) {
        dec.resize(nv);
        env->GetIntArrayRegion(decimal, 0, nv, dec.data());
        sp.decimal = dec.data();
    }
    uint64_t h = 0;
    PG_CHECK(pg_merge_spec_create((uint64_t)schema, &sp, &h));
    return (jlong)h;
}

JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeSpecFree(JNIEnv *env, jclass, jlong h) {
    PG_CHECK(pg_merge_spec_free((uint64_t)h));
    return 0;
}

// One sorted run from direct ByteBuffers: per column {data, offsets|null, validity|null}
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_runOpen(JNIEnv *env, jclass, jlong schema,
                                                                        jlong nRows, jobjectArray data,
                                                                        jobjectArray offsets, jobjectArray validity) {
    int32_t n_key = 0, n_val = 0;
    PG_CHECK(pg_schema_info((uint64_t)schema, &n_key, &n_val));
    jsize nc = env->GetArrayLength(data);
    if (nc != n_key + 2 + n_val || env->GetArrayLength(offsets) != nc || env->GetArrayLength(validity) != nc) {
        env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"),
                      "a run needs one {data, offsets, validity} entry per file column (n_key + 2 + n_val)");
        return 0;
    }
    std::vector<pg_column> cols(nc);
    for (jsize c = 0; c < nc; c++) {
        jobject d = env->GetObjectArrayElement(data, c);
        jobject o = env->GetObjectArrayElement(offsets, c);
        jobject v = env->GetObjectArrayElement(validity, c);
        cols[c].data = d ? env->GetDirectBufferAddress(d) : nullptr;
        cols[c].offsets = o ? (const int32_t *)env->GetDirectBufferAddress(o) : nullptr;
        cols[c].validity = v ? (const uint8_t *)env->GetDirectBufferAddress(v) : nullptr;
    }
    pg_run_desc rd{nRows, cols.data()};
    uint64_t h = 0;
    PG_CHECK(pg_run_open((uint64_t)schema, &rd, PG_MEM_HOST, &h));
    return (jlong)h;
}

JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_runFree(JNIEnv *env, jclass, jlong h) {
    PG_CHECK(pg_run_free((uint64_t)h));
    return 0;
}

JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeOpen(JNIEnv *env, jclass, jlong spec,
                                                                          jlongArray runs) {
    jsize k = env->GetArrayLength(runs);
    std::vector<jlong> r(k);
    env->GetLongArrayRegion(runs, 0, k, r.data());
    std::vector<uint64_t> ru(r.begin(), r.end());
    uint64_t h = 0;
    PG_CHECK(pg_merge_open((uint64_t)spec, ru.data(), k, &h));
    return (jlong)h;
}

// Re-use the merge handle for other runs of the same schema (the key-range streaming reader)
JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeRebind(JNIEnv *env, jclass, jlong merge,
                                                                          jlongArray runs, jlongArray startRows) {
    jsize k = env->GetArrayLength(runs);
    std::vector<jlong> r(k), sr(k, 0);
    env->GetLongArrayRegion(runs, 0, k, r.data());
    if (startRows) env->GetLongArrayRegion(startRows, 0, k, sr.data());
    std::vector<uint64_t> ru(r.begin(), r.end());
    std::vector<int64_t> st(sr.begin(), sr.end());
    PG_CHECK(pg_merge_rebind((uint64_t)merge, ru.data(), k, st.data()));
    return 0;
}

// Format seam: one Parquet data file (bytes read by the Java FileIO into a direct buffer) -> device-resident run
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_parquetOpen(JNIEnv *env, jclass, jlong schema,
                                                                           jobject fileBytes, jlong size) {
    uint64_t h = 0;
    PG_CHECK(pg_parquet_open((uint64_t)schema, (const uint8_t *)env->GetDirectBufferAddress(fileBytes), (int64_t)size, &h));
    return (jlong)h;
}
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_parquetReadRun(JNIEnv *env, jclass, jlong file) {
    uint64_t run = 0;
    PG_CHECK(pg_parquet_read_run((uint64_t)file, &run));
    return (jlong)run;
}
// ApplyDeletionVectorReader: the run minus the rows whose file position is set in the (expanded) deletion vector
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_applyDeletionVector(JNIEnv *env, jclass, jlong run,
                                                                                   jobject bitmap, jlong nBits) {
    uint64_t out = 0;
    PG_CHECK(pg_run_apply_deletion_vector((uint64_t)run, (const uint8_t *)env->GetDirectBufferAddress(bitmap), nBits, &out));
    return (jlong)out;
}
JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_parquetFree(JNIEnv *env, jclass, jlong file) {
    PG_CHECK(pg_parquet_free((uint64_t)file));
    return 0;
}

// Compaction output encode: rows [row0, row0 + nRows) of a merge batch / run -> one Parquet file on the device;
// pageIndex writes the ColumnIndex / OffsetIndex of every column chunk (pg_parquet_write_options.page_index)
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_parquetEncode(JNIEnv *env, jclass, jlong source,
                                                                             jobjectArray names, jlong row0,
                                                                             jlong nRows, jlong rowGroupRows,
                                                                             jlong pageRows, jboolean pageIndex) {
    std::vector<std::string> keep;
    std::vector<const char *> ptrs = utf_names(env, names, keep);
    pg_parquet_write_options opt{rowGroupRows, pageRows, pageIndex ? 1 : 0};
    uint64_t h = 0;
    PG_CHECK(pg_parquet_encode((uint64_t)source, ptrs.data(), row0, nRows, &opt, &h));
    return (jlong)h;
}
// The same with the page bodies compressed: codec = Parquet CompressionCodec (0 UNCOMPRESSED, 6 ZSTD), level =
// file.compression.zstd-level
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_parquetEncodeCompressed(JNIEnv *env, jclass, jlong source,
                                                                                       jobjectArray names, jlong row0,
                                                                                       jlong nRows, jlong rowGroupRows,
                                                                                       jlong pageRows, jboolean pageIndex,
                                                                                       jint codec, jint level) {
    std::vector<std::string> keep;
    std::vector<const char *> ptrs = utf_names(env, names, keep);
    pg_parquet_write_options opt{rowGroupRows, pageRows, pageIndex ? 1 : 0};
    uint64_t h = 0;
    PG_CHECK(pg_parquet_encode_compressed((uint64_t)source, ptrs.data(), row0, nRows, &opt, codec, level, &h));
    return (jlong)h;
}
// parquetEncodeCompressed with Parquet bloom filters: per i, file column bloomColumns[i] with ndv[i]
// (parquet.bloom.filter.expected.ndv#col, 0 = unset) and fpp[i] (parquet.bloom.filter.fpp#col); null = none:
// pg_parquet_encode_bloom.
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_parquetEncodeBloom(
        JNIEnv *env, jclass, jlong source, jobjectArray names, jlong row0, jlong nRows, jlong rowGroupRows,
        jlong pageRows, jboolean pageIndex, jint codec, jint level, jintArray bloomColumns, jlongArray ndv,
        jdoubleArray fpp) {
    std::vector<std::string> keep;
    std::vector<const char *> ptrs = utf_names(env, names, keep);
    pg_parquet_write_options opt{rowGroupRows, pageRows, pageIndex ? 1 : 0};
    const jsize n = bloomColumns ? env->GetArrayLength(bloomColumns) : 0;
    if ((n && (!ndv || !fpp)) || (ndv && env->GetArrayLength(ndv) != n) || (fpp && env->GetArrayLength(fpp) != n)) {
        env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"),
                      "parquetEncodeBloom: bloomColumns, ndv and fpp differ in length");
        return 0;
    }
    std::vector<jint> c(n);
    std::vector<jlong> d(n);
    std::vector<jdouble> f(n);
    if (n) {
        env->GetIntArrayRegion(bloomColumns, 0, n, c.data());
        env->GetLongArrayRegion(ndv, 0, n, d.data());
        env->GetDoubleArrayRegion(fpp, 0, n, f.data());
    }
    std::vector<pg_parquet_bloom_column> cols;
    for (jsize i = 0; i < n; i++) cols.push_back(pg_parquet_bloom_column{c[i], d[i], f[i]});
    pg_parquet_bloom_options bloom{(int32_t)n, cols.data()};
    uint64_t h = 0;
    PG_CHECK(pg_parquet_encode_bloom((uint64_t)source, ptrs.data(), row0, nRows, &opt, codec, level, &bloom, &h));
    return (jlong)h;
}
// types = 4 ints per column (kind, precision, scale, max length; pg_orc_column_type), or null for the kinds of the
// physical types
static std::vector<pg_orc_column_type> orc_types(JNIEnv *env, jintArray types) {
    std::vector<pg_orc_column_type> cols;
    if (types) {
        const jsize n = env->GetArrayLength(types);
        std::vector<jint> v((size_t)n);
        env->GetIntArrayRegion(types, 0, n, v.data());
        for (jsize i = 0; i + 3 < n; i += 4) cols.push_back(pg_orc_column_type{v[i], v[i + 1], v[i + 2], v[i + 3]});
    }
    return cols;
}
// The same rows as one ORC file: compression = ORC CompressionKind (0 NONE, 5 ZSTD), blockSize = orc.compress.size
// (0 = 256 KiB); types as orc_types reads them.  The result is a file handle for fileMeta / fileFetch / fileFree like
// Parquet's.
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_orcEncode(JNIEnv *env, jclass, jlong source,
                                                                         jobjectArray names, jlong row0, jlong nRows,
                                                                         jlong stripeRows, jint compression, jint level,
                                                                         jlong blockSize, jintArray types) {
    std::vector<std::string> keep;
    std::vector<const char *> ptrs = utf_names(env, names, keep);
    std::vector<pg_orc_column_type> cols = orc_types(env, types);
    pg_orc_write_options opt{stripeRows, compression, level, blockSize, types ? cols.data() : nullptr};
    uint64_t h = 0;
    PG_CHECK(pg_orc_encode((uint64_t)source, ptrs.data(), row0, nRows, &opt, &h));
    return (jlong)h;
}
// orcEncode with a row index of rowIndexStride rows per row group (orc.row.index.stride; 0 = none) and bloom filters
// of the file columns bloomColumns (orc.bloom.filter.columns, resolved to indexes; null = none) at bloomFpp
// (orc.bloom.filter.fpp): pg_orc_encode_indexed.
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_orcEncodeIndexed(
        JNIEnv *env, jclass, jlong source, jobjectArray names, jlong row0, jlong nRows, jlong stripeRows,
        jint compression, jint level, jlong blockSize, jintArray types, jlong rowIndexStride, jintArray bloomColumns,
        jdouble bloomFpp) {
    std::vector<std::string> keep;
    std::vector<const char *> ptrs = utf_names(env, names, keep);
    std::vector<pg_orc_column_type> cols = orc_types(env, types);
    pg_orc_write_options opt{stripeRows, compression, level, blockSize, types ? cols.data() : nullptr};
    std::vector<jint> bloom;
    if (bloomColumns) {
        bloom.resize((size_t)env->GetArrayLength(bloomColumns));
        env->GetIntArrayRegion(bloomColumns, 0, (jsize)bloom.size(), bloom.data());
    }
    std::vector<int32_t> bloom32(bloom.begin(), bloom.end());
    pg_orc_index_options index{rowIndexStride, (int32_t)bloom32.size(), bloom32.data(), bloomFpp};
    uint64_t h = 0;
    PG_CHECK(pg_orc_encode_indexed((uint64_t)source, ptrs.data(), row0, nRows, &opt, &index, &h));
    return (jlong)h;
}
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_fileMeta(JNIEnv *env, jclass, jlong file) {
    pg_file_meta m{};
    pg_status fst = pg_parquet_file_meta((uint64_t)file, &m);
    if (fst != PG_OK) { throw_for(env, fst); return nullptr; }
    jlong v[7] = {m.n_rows, m.file_bytes, m.min_sequence_number, m.max_sequence_number, m.delete_row_count,
                  m.n_row_groups, m.n_pages};
    jlongArray out = env->NewLongArray(7);
    env->SetLongArrayRegion(out, 0, 7, v);
    return out;
}
JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_fileFetch(JNIEnv *env, jclass, jlong file, jobject dst) {
    PG_CHECK(pg_parquet_file_fetch((uint64_t)file, env->GetDirectBufferAddress(dst), env->GetDirectBufferCapacity(dst)));
    return 0;
}
JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_fileFree(JNIEnv *env, jclass, jlong file) {
    PG_CHECK(pg_parquet_file_free((uint64_t)file));
    return 0;
}

// readBatch(): runs the merge; returns the row count.  Column sizes follow via batchColumnBytes().
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeExecute(JNIEnv *env, jclass, jlong merge) {
    PG_CHECK(pg_merge_execute((uint64_t)merge));
    pg_batch b{};
    PG_CHECK(pg_merge_device_batch((uint64_t)merge, &b));
    return (jlong)b.n_rows;
}

// long[3*nCols]: {dataBytes, hasOffsets, hasValidity} per column, so Java can size its direct buffers
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_batchLayout(JNIEnv *env, jclass, jlong merge) {
    pg_batch b{};
    pg_status st = pg_merge_device_batch((uint64_t)merge, &b);
    if (st != PG_OK) { throw_for(env, st); return nullptr; }
    std::vector<jlong> out(3 * (size_t)b.n_cols);
    for (int c = 0; c < b.n_cols; c++) {
        out[3 * c] = b.cols[c].data_bytes;
        out[3 * c + 1] = b.cols[c].offsets != nullptr;
        out[3 * c + 2] = b.cols[c].validity != nullptr;
    }
    jlongArray arr = env->NewLongArray((jsize)out.size());
    env->SetLongArrayRegion(arr, 0, (jsize)out.size(), out.data());
    return arr;
}

// copy the merged batch into caller-owned direct buffers (what ArrowBatchReader then wraps)
JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeFetch(JNIEnv *env, jclass, jlong merge,
                                                                          jobjectArray data, jobjectArray offsets,
                                                                          jobjectArray validity) {
    jsize nc = env->GetArrayLength(data);
    std::vector<pg_out_column> cols(nc);
    for (jsize c = 0; c < nc; c++) {
        jobject d = env->GetObjectArrayElement(data, c);
        jobject o = env->GetObjectArrayElement(offsets, c);
        jobject v = env->GetObjectArrayElement(validity, c);
        cols[c].data = d ? env->GetDirectBufferAddress(d) : nullptr;
        cols[c].offsets = o ? (int32_t *)env->GetDirectBufferAddress(o) : nullptr;
        cols[c].validity = v ? (uint8_t *)env->GetDirectBufferAddress(v) : nullptr;
        cols[c].data_bytes = d ? env->GetDirectBufferCapacity(d) : 0;
    }
    {
        // the library checks the data capacities; offsets / validity capacities are checked here
        pg_batch b{};
        PG_CHECK(pg_merge_device_batch((uint64_t)merge, &b));
        for (jsize c = 0; c < nc && c < b.n_cols; c++) {
            jobject o = env->GetObjectArrayElement(offsets, c);
            jobject v = env->GetObjectArrayElement(validity, c);
            const bool small = (o && b.cols[c].offsets && env->GetDirectBufferCapacity(o) < 4 * (b.n_rows + 1)) ||
                               (v && b.cols[c].validity && env->GetDirectBufferCapacity(v) < (b.n_rows + 7) / 8);
            if (small) {
                env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"), "offsets / validity buffer too small for the batch");
                return 0;
            }
        }
    }
    PG_CHECK(pg_merge_fetch((uint64_t)merge, cols.data(), nc));
    return 0;
}

JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeRelease(JNIEnv *env, jclass, jlong merge) {
    PG_CHECK(pg_merge_release((uint64_t)merge));
    return 0;
}

JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeFree(JNIEnv *env, jclass, jlong merge) {
    PG_CHECK(pg_merge_free((uint64_t)merge));
    return 0;
}

// ---- statistics, metadata, views, sections, Arrow ------------------------------------------------------------

// long[10]: rows_in, rows_out, bytes_h2d, bytes_d2h, bytes_out, n_tiles, n_levels, launches, then
// double[5] via mergeStatsMs: partition, plan, alloc, emit, total  (CompactionMetrics.Reporter feeds on these)
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeStats(JNIEnv *env, jclass, jlong merge) {
    pg_stats st{};
    pg_status rc = pg_merge_stats((uint64_t)merge, &st);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    jlong v[8] = {st.rows_in, st.rows_out, st.bytes_h2d, st.bytes_d2h, st.bytes_out, st.n_tiles, st.n_levels, st.launches};
    jlongArray out = env->NewLongArray(8);
    env->SetLongArrayRegion(out, 0, 8, v);
    return out;
}
JNIEXPORT jdoubleArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeStatsMs(JNIEnv *env, jclass, jlong merge) {
    pg_stats st{};
    pg_status rc = pg_merge_stats((uint64_t)merge, &st);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    jdouble v[5] = {st.ms_partition, st.ms_plan, st.ms_alloc, st.ms_emit, st.ms_total};
    jdoubleArray out = env->NewDoubleArray(5);
    env->SetDoubleArrayRegion(out, 0, 5, v);
    return out;
}

// the CUDA stream of a merge handle / of the calling thread's format readers (for interop with other CUDA users)
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_mergeStream(JNIEnv *env, jclass, jlong merge) {
    void *s = nullptr;
    PG_CHECK(pg_merge_stream((uint64_t)merge, &s));
    return (jlong)(uintptr_t)s;
}
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_threadStream(JNIEnv *env, jclass) {
    void *s = nullptr;
    PG_CHECK(pg_thread_stream(&s));
    return (jlong)(uintptr_t)s;
}

// asynchronous upload of the next section's files (direct ByteBuffers): begin -> handle; wait -> long[2 * n]
// {devicePointer, size} per file, to be passed to readSectionDevice; free
JNIEXPORT jlong JNICALL Java_org_apache_paimon_gpu_NativeMerge_uploadBegin(JNIEnv *env, jclass, jobjectArray fileBuffers,
                                                                           jlongArray sizes) {
    const jsize nf = env->GetArrayLength(fileBuffers);
    std::vector<jlong> sz(nf);
    env->GetLongArrayRegion(sizes, 0, nf, sz.data());
    std::vector<pg_file_desc> files(nf);
    for (jsize i = 0; i < nf; i++) {
        jobject b = env->GetObjectArrayElement(fileBuffers, i);
        if (!b || env->GetDirectBufferCapacity(b) < sz[i]) {
            env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"), "file buffer smaller than its size");
            return 0;
        }
        files[i] = pg_file_desc{(const uint8_t *)env->GetDirectBufferAddress(b), sz[i], PG_MEM_HOST, 0};
    }
    uint64_t up = 0;
    PG_CHECK(pg_files_upload_begin(files.data(), (int32_t)nf, &up));
    return (jlong)up;
}
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_uploadWait(JNIEnv *env, jclass, jlong upload, jint nFiles) {
    std::vector<pg_file_desc> d(nFiles > 0 ? nFiles : 1);
    pg_status rc = pg_files_upload_wait((uint64_t)upload, d.data(), nFiles);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    std::vector<jlong> out(2 * (size_t)nFiles);
    for (jint i = 0; i < nFiles; i++) { out[2 * i] = (jlong)(uintptr_t)d[i].bytes; out[2 * i + 1] = d[i].size; }
    jlongArray a = env->NewLongArray(2 * nFiles);
    env->SetLongArrayRegion(a, 0, 2 * nFiles, out.data());
    return a;
}
JNIEXPORT void JNICALL Java_org_apache_paimon_gpu_NativeMerge_uploadFree(JNIEnv *env, jclass, jlong upload) {
    pg_status rc = pg_files_upload_free((uint64_t)upload);
    if (rc != PG_OK) throw_for(env, rc);
}

// long[2 + 2 * nCols]: {nRows, nCols, then per column dataBytes, hasValidity}
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_runLayout(JNIEnv *env, jclass, jlong run, jint nCols) {
    std::vector<int64_t> bytes(nCols);
    std::vector<int32_t> hasv(nCols);
    int64_t n = 0;
    pg_status rc = pg_run_layout((uint64_t)run, &n, bytes.data(), hasv.data(), nCols);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    std::vector<jlong> out(2 + 2 * (size_t)nCols);
    out[0] = n; out[1] = nCols;
    for (int c = 0; c < nCols; c++) { out[2 + 2 * c] = bytes[c]; out[3 + 2 * c] = hasv[c]; }
    jlongArray arr = env->NewLongArray((jsize)out.size());
    env->SetLongArrayRegion(arr, 0, (jsize)out.size(), out.data());
    return arr;
}

// device-resident run -> caller-owned direct buffers (sizes from runLayout)
JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_runFetch(JNIEnv *env, jclass, jlong run, jobjectArray data,
                                                                        jobjectArray offsets, jobjectArray validity) {
    jsize nc = env->GetArrayLength(data);
    std::vector<pg_out_column> cols(nc);
    for (jsize c = 0; c < nc; c++) {
        jobject d = env->GetObjectArrayElement(data, c);
        jobject o = env->GetObjectArrayElement(offsets, c);
        jobject v = env->GetObjectArrayElement(validity, c);
        cols[c].data = d ? env->GetDirectBufferAddress(d) : nullptr;
        cols[c].offsets = o ? (int32_t *)env->GetDirectBufferAddress(o) : nullptr;
        cols[c].validity = v ? (uint8_t *)env->GetDirectBufferAddress(v) : nullptr;
        cols[c].data_bytes = d ? env->GetDirectBufferCapacity(d) : 0;
    }
    PG_CHECK(pg_run_fetch((uint64_t)run, cols.data(), nc));
    return 0;
}

// long[2]: {view run handle, start row inside the view}
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_runSlice(JNIEnv *env, jclass, jlong source, jlong rowLo,
                                                                             jlong rowHi) {
    uint64_t h = 0;
    int64_t start = 0;
    pg_status rc = pg_run_slice((uint64_t)source, rowLo, rowHi, &h, &start);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    jlong v[2] = {(jlong)h, start};
    jlongArray out = env->NewLongArray(2);
    env->SetLongArrayRegion(out, 0, 2, v);
    return out;
}

// long[7]: rows, row groups, columns, data pages, dictionary pages, launches, decode microseconds
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_parquetDescribe(JNIEnv *env, jclass, jlong reader) {
    pg_parquet_info pi{};
    pg_status rc = pg_parquet_describe((uint64_t)reader, &pi);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    jlong v[7] = {pi.n_rows, pi.n_row_groups, pi.n_columns, pi.n_data_pages, pi.n_dictionary_pages, pi.launches,
                  (jlong)(pi.ms_decode * 1000.0f)};
    jlongArray out = env->NewLongArray(7);
    env->SetLongArrayRegion(out, 0, 7, v);
    return out;
}

// MergeTreeReaders.readerForSection: every file of a section (direct ByteBuffers filled by the Java FileIO) in one
// batch of device launches; runOf[i] = sorted run of file i; returns one run handle per sorted run
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_readSection(
    JNIEnv *env, jclass, jint format, jlong schema, jobjectArray fileBuffers, jlongArray sizes, jintArray runOf, jint nRuns,
    jobjectArray columnNames, jbooleanArray readColumns) {
    const jsize nf = env->GetArrayLength(fileBuffers);
    if (env->GetArrayLength(sizes) != nf || env->GetArrayLength(runOf) != nf) {
        env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"), "one size and one run index per file");
        return nullptr;
    }
    std::vector<jlong> sz(nf);
    std::vector<jint> ro(nf);
    env->GetLongArrayRegion(sizes, 0, nf, sz.data());
    env->GetIntArrayRegion(runOf, 0, nf, ro.data());
    std::vector<pg_file_desc> files(nf);
    for (jsize i = 0; i < nf; i++) {
        jobject b = env->GetObjectArrayElement(fileBuffers, i);
        if (!b || env->GetDirectBufferCapacity(b) < sz[i]) {
            env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"), "file buffer smaller than its size");
            return nullptr;
        }
        files[i] = pg_file_desc{(const uint8_t *)env->GetDirectBufferAddress(b), sz[i], PG_MEM_HOST, ro[i]};
    }
    std::vector<std::string> keep;
    std::vector<const char *> names = utf_names(env, columnNames, keep);
    std::vector<uint64_t> runs(nRuns > 0 ? nRuns : 1);
    // read-type projection pushed into the decoder: one flag per file column, null = all
    std::vector<uint8_t> rc8;
    if (readColumns) {
        int32_t n_key = 0, n_val = 0;
        pg_status rs = pg_schema_info((uint64_t)schema, &n_key, &n_val);
        if (rs != PG_OK) { throw_for(env, rs); return nullptr; }
        const jsize ncol = env->GetArrayLength(readColumns);
        if (ncol != n_key + 2 + n_val) {
            env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"), "one read flag per file column");
            return nullptr;
        }
        std::vector<jboolean> rcb(ncol);
        env->GetBooleanArrayRegion(readColumns, 0, ncol, rcb.data());
        rc8.assign(rcb.begin(), rcb.end());
    }
    pg_section_info info{};
    // 'file.format': 0 = parquet, 1 = orc (FileFormat.fromIdentifier picks the reader by the data file's suffix)
    pg_status rc = format == 1
        ? pg_orc_read_section((uint64_t)schema, files.data(), nf, nRuns, columnNames ? names.data() : nullptr,
                              readColumns ? rc8.data() : nullptr, runs.data(), &info)
        : pg_parquet_read_section((uint64_t)schema, files.data(), nf, nRuns, columnNames ? names.data() : nullptr,
                                  readColumns ? rc8.data() : nullptr, runs.data(), &info);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    std::vector<jlong> out(runs.begin(), runs.begin() + (nRuns > 0 ? nRuns : 0));
    jlongArray arr = env->NewLongArray((jsize)out.size());
    env->SetLongArrayRegion(arr, 0, (jsize)out.size(), out.data());
    return arr;
}

// long[2]: {device address, size} of the encoded file's image (compaction output handed to the next read in HBM)
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_fileDeviceImage(JNIEnv *env, jclass, jlong file) {
    const uint8_t *p = nullptr;
    int64_t size = 0;
    pg_status rc = pg_parquet_file_device_image((uint64_t)file, &p, &size);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    jlong v[2] = {(jlong)(uintptr_t)p, size};
    jlongArray out = env->NewLongArray(2);
    env->SetLongArrayRegion(out, 0, 2, v);
    return out;
}

// long[4]: {nullCount, hasMinMax, min bits, max bits} (integers / BOOLEAN as long, FLOAT / DOUBLE as double bits):
// SimpleColStats of the DataFileMeta (KeyValueDataFileWriter.java:150-184)
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_fileColumnStats(JNIEnv *env, jclass, jlong file, jint column) {
    int64_t nulls = 0, mn = 0, mx = 0;
    int32_t has = 0;
    pg_status rc = pg_parquet_file_column_stats((uint64_t)file, column, &nulls, &has, &mn, &mx);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    jlong v[4] = {nulls, has, mn, mx};
    jlongArray out = env->NewLongArray(4);
    env->SetLongArrayRegion(out, 0, 4, v);
    return out;
}

// BloomFilter64(items, fpp) sizing: long[2] = {serialized bytes, hash function count}; the Java side allocates a
// direct ByteBuffer of that many bytes per indexed column for bloomFilterBuild
JNIEXPORT jlongArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_bloomFilterSize(JNIEnv *env, jclass, jint items,
                                                                                    jdouble fpp) {
    int64_t bytes = 0;
    int32_t k = 0;
    pg_status rc = pg_bloom_filter_size(items, fpp, &bytes, &k);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    jlong v[2] = {bytes, k};
    jlongArray out = env->NewLongArray(2);
    env->SetLongArrayRegion(out, 0, 2, v);
    return out;
}

// the serialized bloom filter of each (column, items, fpp) over rows [row0, row0 + nRows) of a merge or run handle,
// into out[i] (direct ByteBuffers): the per-column bytes DataFileIndexWriter hands to FileIndexFormat.Writer
JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_bloomFilterBuild(JNIEnv *env, jclass, jlong source,
                                                                              jlong row0, jlong nRows, jintArray columns,
                                                                              jintArray items, jdoubleArray fpp,
                                                                              jobjectArray out) {
    const jsize n = env->GetArrayLength(columns);
    if (env->GetArrayLength(items) != n || env->GetArrayLength(fpp) != n || env->GetArrayLength(out) != n) {
        env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"), "bloomFilterBuild: array lengths differ");
        return 0;
    }
    std::vector<jint> c((size_t)n), it((size_t)n);
    std::vector<jdouble> f((size_t)n);
    env->GetIntArrayRegion(columns, 0, n, c.data());
    env->GetIntArrayRegion(items, 0, n, it.data());
    env->GetDoubleArrayRegion(fpp, 0, n, f.data());
    std::vector<pg_bloom_filter_spec> specs((size_t)n);
    std::vector<uint8_t *> dst((size_t)n);
    std::vector<int64_t> cap((size_t)n);
    for (jsize i = 0; i < n; i++) {
        specs[i] = pg_bloom_filter_spec{c[i], it[i], f[i]};
        jobject buf = env->GetObjectArrayElement(out, i);
        dst[i] = (uint8_t *)env->GetDirectBufferAddress(buf);
        cap[i] = env->GetDirectBufferCapacity(buf);
    }
    PG_CHECK(pg_bloom_filter_build((uint64_t)source, row0, nRows, n, specs.data(), dst.data(), cap.data()));
    return 0;
}

// IntervalPartition.partition over (min, max) key bounds: int[2 * n + 1] = {sections, section of file i, run of file i}
JNIEXPORT jintArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_intervalPartition(JNIEnv *env, jclass, jlongArray minKey,
                                                                                     jlongArray maxKey) {
    const jsize n = env->GetArrayLength(minKey);
    if (env->GetArrayLength(maxKey) != n) {
        env->ThrowNew(env->FindClass("java/lang/IllegalArgumentException"), "one max key per min key");
        return nullptr;
    }
    std::vector<jlong> mn(n), mx(n);
    env->GetLongArrayRegion(minKey, 0, n, mn.data());
    env->GetLongArrayRegion(maxKey, 0, n, mx.data());
    std::vector<int64_t> a(mn.begin(), mn.end()), b(mx.begin(), mx.end());
    std::vector<int32_t> sec(n ? n : 1), run(n ? n : 1);
    int32_t ns = 0;
    pg_status rc = pg_interval_partition(n, a.data(), b.data(), sec.data(), run.data(), &ns);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    std::vector<jint> out(2 * (size_t)n + 1);
    out[0] = ns;
    for (jsize i = 0; i < n; i++) { out[1 + i] = sec[i]; out[1 + n + i] = run[i]; }
    jintArray arr = env->NewIntArray((jsize)out.size());
    env->SetIntArrayRegion(arr, 0, (jsize)out.size(), out.data());
    return arr;
}

// Arrow C Data Interface export: arrayAddr / schemaAddr are the addresses of an org.apache.arrow.c.ArrowArray /
// ArrowSchema allocated by the Java side (ArrowArray.allocateNew(allocator).memoryAddress()); afterwards
// Data.importVectorSchemaRoot(allocator, array, schema, null) yields the VectorSchemaRoot ArrowBatchReader wraps.
JNIEXPORT jint JNICALL Java_org_apache_paimon_gpu_NativeMerge_exportArrow(JNIEnv *env, jclass, jlong source,
                                                                          jobjectArray columnNames, jlong row0, jlong nRows,
                                                                          jlong arrayAddr, jlong schemaAddr) {
    std::vector<std::string> keep;
    std::vector<const char *> names = utf_names(env, columnNames, keep);
    PG_CHECK(pg_export_arrow((uint64_t)source, columnNames ? names.data() : nullptr, row0, nRows,
                             (struct ArrowArray *)(uintptr_t)arrayAddr, (struct ArrowSchema *)(uintptr_t)schemaAddr));
    return 0;
}

// int[2]: {n_key, n_val} of a schema handle
JNIEXPORT jintArray JNICALL Java_org_apache_paimon_gpu_NativeMerge_schemaInfo(JNIEnv *env, jclass, jlong schema) {
    int32_t v[2] = {0, 0};
    pg_status rc = pg_schema_info((uint64_t)schema, &v[0], &v[1]);
    if (rc != PG_OK) { throw_for(env, rc); return nullptr; }
    jintArray out = env->NewIntArray(2);
    env->SetIntArrayRegion(out, 0, 2, v);
    return out;
}

}  // extern "C"
#endif  // __has_include(<jni.h>)
