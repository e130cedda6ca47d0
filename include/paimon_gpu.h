/*
 * paimon_gpu.h — C ABI of libpaimon_gpu.so, the H100 (sm_90a) implementation of Apache
 * Paimon's merge-on-read / compaction hot path:
 *
 *     sorted-run columnar batches -> k-way merge by (key, sequence) -> per-key MergeFunction
 *
 * This is the drop-in boundary (SURVEY.md §8b).  Plain C, plain pointers and sizes, opaque
 * uint64 handles, every call returns a status (0 = OK) and leaves a message for
 * pg_last_error() otherwise; no C++/torch types cross it.  A JNI shim (jni/paimon_gpu_jni.cc)
 * binds one Java native method per function; see INTEGRATION.md.
 *
 * Reference interfaces each entry point replaces (paths under /root/reference/):
 *   pg_merge_spec_create  <- MergeFunctionFactory.create(readType)
 *                            paimon-core/.../mergetree/compact/MergeFunctionFactory.java:29-41 and the
 *                            option parsing in PartialUpdateMergeFunction.java:389-489,
 *                            aggregate/AggregateMergeFunction.java:146-204
 *   pg_run_open           <- one sorted run's RecordReader<KeyValue>:
 *                            paimon-core/.../mergetree/MergeTreeReaders.java:94-101 (readerForRun)
 *   pg_merge_open         <- SortMergeReader.createSortMergeReader(readers, keyComparator,
 *                            userDefinedSeqComparator, mergeFunctionWrapper, sortEngine)
 *                            paimon-core/.../mergetree/compact/SortMergeReader.java:41-57
 *                            (+ DropDeleteReader, paimon-core/.../mergetree/DropDeleteReader.java:50-68)
 *   pg_merge_execute/next <- RecordReader.readBatch()  paimon-common/.../reader/RecordReader.java:40-72;
 *                            like SortMergeReaderWithLoserTree.java:67-73 the merge yields ONE batch
 *   pg_merge_release      <- RecordIterator.releaseBatch()
 *   pg_*_free             <- RecordReader.close()
 *   pg_interval_partition <- IntervalPartition.partition()
 *                            paimon-core/.../mergetree/compact/IntervalPartition.java:67-125
 *   pg_parquet_*          <- FormatReaderFactory.createReader / FileRecordReader.readBatch
 *                            paimon-common/.../format/FormatReaderFactory.java:33-57,
 *                            paimon-format/.../parquet/ParquetReaderFactory.java:113-148
 *
 * Threading: the library is re-entrant across handles; one merge handle (one CUDA stream) per
 * Java reader thread, like the reference's thread-confined readers.
 */
#ifndef PAIMON_GPU_H
#define PAIMON_GPU_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PG_ABI_VERSION 2
#define PG_MAX_RUNS 32          /* runs merged by one call; more => merge in rounds on the host */
#define PG_MAX_SEQ_GROUPS 16
#define PG_MAX_KEY_FIELDS 4

typedef int32_t pg_status;
enum {
    PG_OK = 0,
    PG_ERR_INVALID = 1,         /* bad argument / handle */
    PG_ERR_UNSUPPORTED = 2,     /* spec refused at plan time (no CPU fallback) */
    PG_ERR_CUDA = 3,
    PG_ERR_MERGE_FUNCTION = 4,  /* the Java MergeFunction would have thrown; message says which */
    PG_ERR_INTERNAL = 5,
    PG_ERR_FORMAT = 6           /* malformed / unsupported file bytes */
};

/* physical column types; Paimon DATE/TIME -> INT32, TIMESTAMP(p<=6)/DECIMAL(p<=18) -> INT64,
 * CHAR/VARCHAR -> STRING, BINARY/VARBINARY -> BINARY, BOOLEAN -> one byte per value */
typedef enum {
    PG_INT8 = 1, PG_INT16 = 2, PG_INT32 = 3, PG_INT64 = 4,
    PG_FLOAT = 5, PG_DOUBLE = 6, PG_BOOL = 7, PG_STRING = 8, PG_BINARY = 9
} pg_type;

/* RowKind.toByteValue, paimon-api/.../types/RowKind.java:35-56 */
enum { PG_INSERT = 0, PG_UPDATE_BEFORE = 1, PG_UPDATE_AFTER = 2, PG_DELETE = 3 };

/* CoreOptions.MergeEngine */
enum { PG_ENGINE_DEDUPLICATE = 0, PG_ENGINE_PARTIAL_UPDATE = 1, PG_ENGINE_AGGREGATE = 2,
       PG_ENGINE_FIRST_ROW = 3 };

/* fields.<f>.aggregate-function */
enum {
    PG_AGG_NONE = 0, PG_AGG_SUM = 1, PG_AGG_PRODUCT = 2, PG_AGG_MAX = 3, PG_AGG_MIN = 4,
    PG_AGG_BOOL_AND = 5, PG_AGG_BOOL_OR = 6, PG_AGG_LAST_VALUE = 7, PG_AGG_LAST_NON_NULL_VALUE = 8,
    PG_AGG_FIRST_VALUE = 9, PG_AGG_FIRST_NON_NULL_VALUE = 10, PG_AGG_PRIMARY_KEY = 11
};

enum { PG_MEM_HOST = 0, PG_MEM_DEVICE = 1 };

typedef struct {
    int32_t type;       /* pg_type */
    int32_t nullable;
} pg_field;

/* file schema [_KEY_*..., _SEQUENCE_NUMBER BIGINT, _VALUE_KIND TINYINT, value...]
 * (paimon-core/.../KeyValue.java:130-138) */
typedef struct {
    int32_t n_key;
    int32_t n_val;
    const pg_field *key_fields;
    const pg_field *val_fields;
} pg_schema_desc;

/* declarative MergeFunction: what the reference factories derive from table options */
typedef struct {
    int32_t engine;
    int32_t ignore_delete;              /* 'ignore-delete' */
    int32_t remove_record_on_delete;    /* partial-update.* / aggregation.remove-record-on-delete */
    int32_t drop_delete;                /* wrap the merge in DropDeleteReader */
    int32_t n_seq_fields;               /* 'sequence.field' (value-field indexes), 0 = none */
    const int32_t *seq_fields;
    int32_t seq_ascending;              /* 'sequence.field.sort-order' */
    const int32_t *agg;                 /* [n_val] PG_AGG_*; NULL = all NONE */
    const uint8_t *ignore_retract;      /* [n_val]; NULL = all false */
    /* partial-update sequence groups ('fields.<seq,...>.sequence-group' = 'a,b'; PartialUpdateMergeFunction.java:
     * 190-342, option parsing :389-489): a group's fields only move when the row's group sequence is >= the
     * accumulated one */
    int32_t n_sequence_groups;          /* 0 = none; at most PG_MAX_SEQ_GROUPS */
    const int32_t *group_seq_start;     /* [n_sequence_groups + 1] CSR into group_seq_fields */
    const int32_t *group_seq_fields;    /* value-field indexes of each group's sequence fields (<= 4 per group) */
    const int32_t *field_group;         /* [n_val] group protecting the field (its sequence fields included), -1 */
    const uint8_t *group_partial_delete;/* [n_val] sequence field listed in
                                           'partial-update.remove-record-on-sequence-group'; NULL = none */
    /* read-type projection (MergeFunctionFactory.create(readType), MergeFileSplitRead.withReadType :133-163): value
     * fields with 0 are not part of the merged batch (no output buffers, no emit work); the runs may come without
     * buffers for them (pg_parquet_read_section's read_columns), except for fields the merge itself compares
     * ('sequence.field', sequence-group fields: PartialUpdateMergeFunction.adjustReadType :576-606 keeps those) */
    const uint8_t *read_fields;         /* [n_val]; NULL = every field */
    /* DECIMAL value fields (unscaled INT64 columns): sum / product follow the reference's DECIMAL rules (FieldSumAgg /
     * FieldProductAgg on DecimalType: NULL on int64 overflow or when a product / quotient has more than p digits,
     * HALF_UP rescaling, exact division on retract) instead of wrapping int64 arithmetic.  precision 1..18. */
    const int32_t *decimal;             /* [n_val] precision << 8 | scale, 0 = not DECIMAL; NULL = none */
} pg_merge_spec;

/* one column, Arrow buffer layout */
typedef struct {
    const void *data;          /* fixed width: values[n_rows]; var-len: bytes */
    const int32_t *offsets;    /* var-len: int32[n_rows + 1], else NULL */
    const uint8_t *validity;   /* bitmap LSB-first, or NULL when the column has no nulls */
} pg_column;

typedef struct {
    int64_t n_rows;
    const pg_column *cols;     /* n_key + 2 + n_val columns in file order */
} pg_run_desc;

typedef struct {
    void *data;
    int32_t *offsets;
    uint8_t *validity;         /* NULL for NOT NULL columns */
    int64_t data_bytes;        /* bytes in data (var-len: payload bytes) */
} pg_out_column;

typedef struct {
    int64_t n_rows;
    int32_t n_cols;
    const pg_out_column *cols; /* owned by the merge handle, valid until pg_merge_release/free */
} pg_batch;

typedef struct {
    int64_t rows_in;
    int64_t rows_out;
    int64_t bytes_h2d;
    int64_t bytes_d2h;
    int64_t bytes_out;             /* device bytes of the output batch */
    int32_t n_tiles;
    int32_t n_levels;              /* sampled partition levels above level 0 */
    float ms_partition;            /* CUDA-event times of the last execute, on the handle's stream */
    float ms_plan;                 /* plan kernel + row-count scan */
    float ms_alloc;                /* size read-back + output allocation (host-paced gap on the stream) */
    float ms_emit;                 /* emit kernel only */
    float ms_total;
    int32_t launches;              /* kernels launched by the last execute */
} pg_stats;

const char *pg_last_error(void);
int32_t pg_abi_version(void);

/* bind the library to a device; idempotent for the same ordinal.  One process drives ONE GPU (one process per GPU,
 * like bucket_scheduler / torchrun): a second ordinal is refused — handles, streams and the recycled device buffers
 * all belong to the first one. */
pg_status pg_init(int32_t device_ordinal);
pg_status pg_shutdown(void);
/* give the cached device buffers of freed host-opened runs back to the driver */
pg_status pg_trim(void);

pg_status pg_schema_create(const pg_schema_desc *desc, uint64_t *out_schema);
pg_status pg_schema_free(uint64_t schema);
pg_status pg_schema_info(uint64_t schema, int32_t *n_key, int32_t *n_val);

pg_status pg_merge_spec_create(uint64_t schema, const pg_merge_spec *spec, uint64_t *out_spec);
pg_status pg_merge_spec_free(uint64_t spec);

/* Register one sorted run.  PG_MEM_HOST: the buffers are copied to the device now (they may be
 * freed after the call).  PG_MEM_DEVICE: the pointers are device pointers that the caller keeps
 * alive until pg_run_free; every buffer must be 16-byte aligned and readable up to the next multiple
 * of 16 bytes (true for any cudaMalloc'ed / framework-allocated buffer): the kernels stage column
 * segments with 16-byte bulk async copies. */
pg_status pg_run_open(uint64_t schema, const pg_run_desc *run, int32_t mem, uint64_t *out_run);
pg_status pg_run_free(uint64_t run);

/* k-way merge of `k` runs (all of `schema`) with the merge function of `spec`. */
pg_status pg_merge_open(uint64_t spec, const uint64_t *runs, int32_t k, uint64_t *out_merge);
/* run the kernels; asynchronous on the handle's stream except for one size read-back */
/* Re-use a merge handle (its stream, descriptors and arenas) for another set of runs of the same schema, and
 * start each run at start_rows[i] (NULL = 0): rows before it do not take part.  This is what a reader uses that
 * streams a bucket through the device in key ranges: range j of run i is copied from the 8-row boundary below
 * its first row (validity bitmaps are byte-granular), and start_rows skips the rows that belong to range j-1. */
pg_status pg_merge_rebind(uint64_t merge, const uint64_t *runs, int32_t k, const int64_t *start_rows);
pg_status pg_merge_execute(uint64_t merge);
/* the single output batch, device-resident (pointers are device pointers) */
pg_status pg_merge_device_batch(uint64_t merge, pg_batch *out);
/* copy the output batch into caller-allocated host buffers (sizes from pg_merge_device_batch); host_cols[c].data_bytes
 * is the CAPACITY of host_cols[c].data and is checked (offsets need 4 * (n_rows + 1) bytes, validity (n_rows + 7) / 8) */
pg_status pg_merge_fetch(uint64_t merge, const pg_out_column *host_cols, int32_t n_cols);
pg_status pg_merge_release(uint64_t merge);      /* releaseBatch(): drop the output buffers */
pg_status pg_merge_stats(uint64_t merge, pg_stats *out);
pg_status pg_merge_stream(uint64_t merge, void **out_cuda_stream);
pg_status pg_merge_free(uint64_t merge);

/* A registered run's shape, and a device->host copy of its columns (sizes from pg_run_layout). */
pg_status pg_run_layout(uint64_t run, int64_t *n_rows, int64_t *data_bytes, int32_t *has_validity, int32_t n_cols);
pg_status pg_run_fetch(uint64_t run, const pg_out_column *host_cols, int32_t n_cols);

/* ---- Arrow C Data Interface export (SURVEY §8b): the batch the JVM imports ------------------------------------
 * The struct definitions restate the public Arrow C Data Interface (https://arrow.apache.org/docs/format/
 * CDataInterface.html); they are guarded with the specification's own macro so that including Arrow's abi.h first
 * is fine. */
#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE
struct ArrowSchema {
    const char *format;
    const char *name;
    const char *metadata;
    int64_t flags;
    int64_t n_children;
    struct ArrowSchema **children;
    struct ArrowSchema *dictionary;
    void (*release)(struct ArrowSchema *);
    void *private_data;
};
struct ArrowArray {
    int64_t length;
    int64_t null_count;
    int64_t offset;
    int64_t n_buffers;
    int64_t n_children;
    const void **buffers;
    struct ArrowArray **children;
    struct ArrowArray *dictionary;
    void (*release)(struct ArrowArray *);
    void *private_data;
};
#endif
/* Rows [row0, row0 + n_rows) (n_rows < 0 = to the end) of a merge handle's current batch, or of a run handle, as
 * one Arrow struct array whose children are the file columns, named `column_names[i]` (the Paimon field names
 * _KEY_*, _SEQUENCE_NUMBER, _VALUE_KIND, value fields: paimon-arrow's ArrowBatchReader.java:74-115 maps columns by
 * name).  The buffers are page-locked host memory owned by `out` and freed by out->release (what the Java reader's
 * releaseBatch() / close() call after Data.importVectorSchemaRoot); BOOLEAN columns are bit-packed as Arrow wants
 * them.  A reader hands a large batch out piece by piece by calling this with consecutive row ranges
 * (RecordReader.readBatch(), paimon-common/.../reader/RecordReader.java:42-72). */
pg_status pg_export_arrow(uint64_t source, const char *const *column_names, int64_t row0, int64_t n_rows,
                          struct ArrowArray *out, struct ArrowSchema *out_schema);

/* A VIEW (no copy) of rows [row_lo, row_hi) of a run handle, or of the current batch of a merge handle: a new run
 * handle whose columns point into the source's device buffers (the source must outlive it; pg_run_free drops the
 * view only).  The view starts at the 128-row boundary at or below row_lo (every buffer stays 16-byte aligned);
 * *start_row receives row_lo's position inside the view — pass it as start_rows[i] to pg_merge_rebind, or skip that
 * many rows after pg_run_fetch.  Used to re-merge / read back a key range of a bucket (parity samples at full size,
 * readers that hand out a large batch piece by piece). */
pg_status pg_run_slice(uint64_t source, int64_t row_lo, int64_t row_hi, uint64_t *out_run, int64_t *start_row);

/* the CUDA stream the calling thread's format readers (pg_parquet_*) launch on, for event timing */
pg_status pg_thread_stream(void **out_cuda_stream);

/* ---- format seam: Parquet data file -> device-resident sorted run -------------------------------------
 * Replaces FormatReaderFactory.createReader(context) + FileRecordReader.readBatch()
 * (paimon-common/.../format/FormatReaderFactory.java:33-57, paimon-format/.../parquet/ParquetReaderFactory.java:
 * 113-148, reader/VectorizedParquetRecordReader.java:178-241) for KeyValue data files: the file bytes (read by the
 * Java FileIO) are parsed on the host for footer + page headers and decoded on the device straight into the
 * columnar run the merge consumes.  Decoded: flat schemas, BOOLEAN/INT32/INT64/FLOAT/DOUBLE/BYTE_ARRAY, PLAIN and
 * dictionary encodings, RLE booleans, DELTA_BINARY_PACKED integers, data pages V1/V2, uncompressed, Snappy-, zstd- and
 * gzip-compressed pages (decompressed on the device); anything else (lz4, brotli, byte-array DELTA encodings,
 * INT96 / FIXED_LEN_BYTE_ARRAY, nested columns) returns PG_ERR_UNSUPPORTED.  pg_parquet_open walks the page headers
 * on the host once so that such files are refused before any device work. */
typedef struct {
    int64_t n_rows;
    int32_t n_row_groups;
    int32_t n_columns;
    int32_t n_data_pages;
    int32_t n_dictionary_pages;
    float ms_decode;               /* CUDA-event time of the last pg_parquet_read_run */
    int32_t launches;
} pg_parquet_info;

pg_status pg_parquet_open(uint64_t schema, const uint8_t *file_bytes, int64_t size, uint64_t *out_reader);
pg_status pg_parquet_describe(uint64_t reader, pg_parquet_info *out);
/* decode the whole file into a run handle (free it with pg_run_free); usable directly in pg_merge_open */
pg_status pg_parquet_read_run(uint64_t reader, uint64_t *out_run);
pg_status pg_parquet_free(uint64_t reader);

/* ---- a whole SECTION in one batch of launches ------------------------------------------------------------
 * Replaces MergeTreeReaders.readerForSection's reader construction (paimon-core/.../mergetree/MergeTreeReaders.java:
 * 67-101): every data file of every sorted run of a section is decoded by one set of kernel launches, and the files
 * of one run (key-disjoint, ascending: SortedRun.java:59-61) are CONCATENATED into one device run, exactly as
 * readerForRun's ConcatRecordReader does — the k-way merge then sees k = number of runs inputs, not number of files.
 * `files[i].run` names the output run of file i; files of a run must be listed in key order.  `bytes` is host memory
 * (copied to the device by the call) or device memory (PG_MEM_DEVICE: the bytes already sit in HBM, e.g. read by
 * GPUDirect storage or produced by pg_parquet_encode; must stay valid during the call only).  Only the footers are
 * parsed on the host; page headers are parsed on the device.
 * `column_names` (n_key + 2 + n_val entries, or NULL = positional) are the names the read schema's fields have in the
 * files: columns are resolved BY NAME like the reference does (ParquetReaderFactory.java:113-148 clipParquetSchema):
 * a nullable read field the file does not have decodes as all-NULL (file written before ADD COLUMN), file columns
 * the read schema does not name are ignored (DROP COLUMN), and a file column that is narrower than the read field is
 * widened on the fly (INT-family -> BIGINT, FLOAT -> DOUBLE: the casts of DataFileRecordReader.java:55-57 that need
 * no rewrite).  Anything else (renames without the old name, other casts) is refused with PG_ERR_UNSUPPORTED.
 * `read_columns` ([n_key + 2 + n_val] bytes, or NULL = all) is the read-type projection pushed into the decoder
 * (MergeFileSplitRead.withReadType, operation/MergeFileSplitRead.java:133-163): columns with 0 are not decoded and the
 * runs carry no buffers for them; key, sequence-number and kind columns are always read (keys are never projected
 * before a merge, :276-277).  out_runs[n_runs] receives run handles (pg_run_free each). */
typedef struct {
    const uint8_t *bytes;
    int64_t size;
    int32_t mem;                   /* PG_MEM_HOST / PG_MEM_DEVICE */
    int32_t run;                   /* output run of this file, 0 <= run < n_runs */
} pg_file_desc;

typedef struct {
    int64_t n_rows;
    int64_t file_bytes;            /* sum of the file sizes */
    int64_t page_bytes;            /* uncompressed page bodies: the encoded bytes the decode kernels read */
    int64_t decoded_bytes;         /* bytes of the decoded columns (values, offsets, payload, validity) */
    int32_t n_files, n_runs, n_chunks, n_data_pages, n_dictionary_pages;
    int32_t launches;
    float ms_decode;               /* CUDA-event time from the first copy / kernel to the last kernel */
} pg_section_info;

pg_status pg_parquet_read_section(uint64_t schema, const pg_file_desc *files, int32_t n_files, int32_t n_runs,
                                  const char *const *column_names, const uint8_t *read_columns, uint64_t *out_runs,
                                  pg_section_info *info);

/* The same for ORC data files ('file.format' = 'orc'; OrcReaderFactory.createReader, paimon-format/.../orc/
 * OrcReaderFactory.java:98-163): every stripe of every file of a section, the files of a run concatenated.  Decoded:
 * flat schemas, BOOLEAN / TINYINT / SMALLINT / INT / BIGINT / FLOAT / DOUBLE / DATE / DECIMAL(p <= 18) / STRING-family /
 * BINARY, integer RLE v1 and v2, DIRECT and DICTIONARY string encodings, PRESENT streams, compression NONE / ZLIB /
 * ZSTD; columns are resolved by field name (missing nullable fields -> NULL, integer / float widening).  Timestamps,
 * DECIMAL(p > 18), nested types and the other codecs return PG_ERR_UNSUPPORTED.  The file bytes must be host memory
 * (footers and compression-chunk headers are walked on the host); pg_section_info.n_chunks counts (stripe, column)
 * tasks and n_data_pages counts streams. */
pg_status pg_orc_read_section(uint64_t schema, const pg_file_desc *files, int32_t n_files, int32_t n_runs,
                              const char *const *column_names, const uint8_t *read_columns, uint64_t *out_runs,
                              pg_section_info *info);

/* Asynchronous host -> device copy of a section's data files, so that the NEXT section's bytes move while the current
 * one decodes and merges (the copy of the encoded files is the longest leg of an end-to-end step).
 *   pg_files_upload_begin: starts the copies on the library's upload stream and returns at once (host buffers should be
 *     page-locked; descriptors that are already PG_MEM_DEVICE pass through untouched);
 *   pg_files_upload_wait:  blocks until the bytes are resident and fills out_files[n_files] with PG_MEM_DEVICE
 *     descriptors (same order, same run indexes) for pg_parquet_read_section;
 *   pg_files_upload_free:  releases the device copies; call it from the thread that decoded them, after
 *     pg_parquet_read_section returned (it waits for that thread's decode launches).
 * Replaces: the blocking file read in front of FormatReaderFactory.createReader
 * (paimon-core/.../io/KeyValueFileReaderFactory.java:104-140) for the device path. */
pg_status pg_files_upload_begin(const pg_file_desc *files, int32_t n_files, uint64_t *out_upload);
pg_status pg_files_upload_wait(uint64_t upload, pg_file_desc *out_files, int32_t n_files);
pg_status pg_files_upload_free(uint64_t upload);


/* ApplyDeletionVectorReader (paimon-core/.../deletionvectors/ApplyDeletionVectorReader.java:31-54): a new run holding
 * the rows of `run` whose file position is NOT set in the deletion vector.  `deleted_bitmap` is host memory, LSB
 * first, bit i = row i of the file is deleted (the Java side expands its RoaringBitmap32; DeletionVector.java);
 * positions >= n_bits are kept.  The input run stays valid. */
pg_status pg_run_apply_deletion_vector(uint64_t run, const uint8_t *deleted_bitmap, int64_t n_bits, uint64_t *out_run);

/* ---- compaction output encode: device batch -> Parquet data file ------------------------------------------
 * Replaces KeyValueDataFileWriter.write()/result() (paimon-core/.../io/KeyValueDataFileWriter.java:108-184: row
 * count, min/max key, min/max sequence number, delete row count, per-column stats -> DataFileMeta) and the
 * Parquet writer behind it (paimon-format/.../parquet/writer/ParquetRowDataWriter.java,
 * RowDataParquetBuilder.java:58-119; type mapping ParquetSchemaConverter.java:76-160) on the rewrite side of
 * MergeTreeCompactRewriter.rewriteCompaction (:78-116).  `source` is a merge handle holding a batch or a run
 * handle; rows [row0, row0 + n_rows) are encoded (row0 a multiple of 8, n_rows < 0 = to the end), so a rolling
 * writer (RollingFileWriterImpl.java:64-105) cuts one batch into several files.  Written: data pages V1, PLAIN,
 * uncompressed, definition levels for nullable columns, per-chunk statistics. */
typedef struct {
    int64_t row_group_rows;        /* 0 = 1 Mi rows */
    int64_t page_rows;             /* 0 = 32 Ki rows; rounded up to a multiple of 8 */
} pg_parquet_write_options;

typedef struct {
    int64_t n_rows;
    int64_t file_bytes;
    int64_t min_sequence_number;
    int64_t max_sequence_number;
    int64_t delete_row_count;      /* rows whose _VALUE_KIND is a retract (UPDATE_BEFORE / DELETE) */
    int32_t n_row_groups;
    int32_t n_pages;
    float ms_encode;               /* CUDA-event time of the encode */
    int32_t launches;
} pg_file_meta;

pg_status pg_parquet_encode(uint64_t source, const char *const *column_names, int64_t row0, int64_t n_rows,
                            const pg_parquet_write_options *options, uint64_t *out_file);
pg_status pg_parquet_file_meta(uint64_t file, pg_file_meta *out);
/* whole-file statistics of one column: null count; min / max for fixed-width columns (integers and BOOLEAN as
 * int64, FLOAT / DOUBLE as double; absent when every value is NULL or a NaN was seen) */
pg_status pg_parquet_file_column_stats(uint64_t file, int32_t column, int64_t *null_count, int32_t *has_min_max,
                                       void *min8, void *max8);
pg_status pg_parquet_file_fetch(uint64_t file, void *host_buffer, int64_t capacity);
/* the complete file image in device memory (page headers and footer patched in on first use); valid until
 * pg_parquet_file_free.  Lets a compaction hand its output to the next read without leaving HBM, and is how the
 * benchmark builds 100 M-row Parquet inputs. */
pg_status pg_parquet_file_device_image(uint64_t file, const uint8_t **device_bytes, int64_t *size);
pg_status pg_parquet_file_free(uint64_t file);

/* IntervalPartition over int64 (min,max) key bounds of data files: section and run id per file */
pg_status pg_interval_partition(int32_t n_files, const int64_t *min_key, const int64_t *max_key,
                                int32_t *section_of, int32_t *run_of, int32_t *n_sections);

#ifdef __cplusplus
}
#endif
#endif
