/*
 * paimon_oracle.h — TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement (plain C) of Apache Paimon's merge-on-read hot path, used as
 * the parity oracle for the CUDA implementation in paimon_b200/.  Only tests/,
 * __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference) may
 * load this library.  The product path (libpaimon_gpu.so) never links or calls
 * it, and has no CPU fallback.
 *
 * Reference files restated (all under /root/reference/paimon-core/src/main/java/
 * org/apache/paimon/):
 *   mergetree/compact/LoserTree.java:45-356
 *   mergetree/compact/SortMergeReaderWithLoserTree.java:39-118
 *   mergetree/compact/SortMergeReaderWithMinHeap.java:54-70,135-179
 *   mergetree/compact/ReducerMergeFunctionWrapper.java:45-73
 *   mergetree/compact/DeduplicateMergeFunction.java:42-60
 *   mergetree/compact/FirstRowMergeFunction.java:32-73
 *   mergetree/compact/PartialUpdateMergeFunction.java:111-362
 *   mergetree/compact/aggregate/AggregateMergeFunction.java:72-125
 *   mergetree/compact/aggregate/Field{Sum,Product,Max,Min,BoolAnd,BoolOr,LastValue,
 *       LastNonNullValue,FirstValue,FirstNonNullValue,PrimaryKey,IgnoreRetract}Agg.java
 *   mergetree/DropDeleteReader.java:50-68
 *   mergetree/compact/IntervalPartition.java:38-125
 * Comparator rules: paimon-codegen/.../GenerateUtils.scala:113-173,
 *   paimon-common/.../data/BinaryString.java:109-126, utils/InternalRowUtils.java:387-444.
 *
 * Parity pinning: the restatement is checked (tests/test_oracle_golden.py) against the
 * reference's own fixed vectors and expected-result calculators transcribed from
 * paimon-core/src/test/java/org/apache/paimon/mergetree/compact/{SortMergeReaderTestBase,
 * CombiningRecordReaderTestBase,MergeFunctionTestUtils,PartialUpdateMergeFunctionTest,
 * aggregate/FieldAggregatorTest,aggregate/AggregateMergeFunctionTest,IntervalPartitionTest}.java.
 * The Java reference itself cannot run here (no JVM in the image).
 */
#ifndef PAIMON_ORACLE_H
#define PAIMON_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* physical column types (Paimon logical -> physical: DATE/TIME -> INT32, TIMESTAMP(<=6) and
 * DECIMAL(p<=18) -> INT64, CHAR/VARCHAR -> STRING, BINARY/VARBINARY -> BINARY, BOOLEAN -> 1 byte) */
enum {
    PO_INT8 = 1, PO_INT16 = 2, PO_INT32 = 3, PO_INT64 = 4,
    PO_FLOAT = 5, PO_DOUBLE = 6, PO_BOOL = 7, PO_STRING = 8, PO_BINARY = 9
};

/* RowKind byte values, paimon-api/.../types/RowKind.java:35-56 */
enum { PO_INSERT = 0, PO_UPDATE_BEFORE = 1, PO_UPDATE_AFTER = 2, PO_DELETE = 3 };

enum { PO_ENGINE_DEDUPLICATE = 0, PO_ENGINE_PARTIAL_UPDATE = 1, PO_ENGINE_AGGREGATE = 2,
       PO_ENGINE_FIRST_ROW = 3 };

/* CoreOptions.SortEngine + a brute-force checker (sort all rows by key,[seq fields],seq; fold) */
enum { PO_SORT_LOSER_TREE = 0, PO_SORT_MIN_HEAP = 1, PO_SORT_BRUTE_FORCE = 2 };

enum {
    PO_AGG_NONE = 0,            /* partial-update column without aggregator */
    PO_AGG_SUM = 1, PO_AGG_PRODUCT = 2, PO_AGG_MAX = 3, PO_AGG_MIN = 4,
    PO_AGG_BOOL_AND = 5, PO_AGG_BOOL_OR = 6,
    PO_AGG_LAST_VALUE = 7, PO_AGG_LAST_NON_NULL_VALUE = 8,
    PO_AGG_FIRST_VALUE = 9, PO_AGG_FIRST_NON_NULL_VALUE = 10,
    PO_AGG_PRIMARY_KEY = 11
};

/* one column of one run, Arrow layout */
typedef struct {
    const void *data;        /* fixed width: values; var-len: bytes */
    const int32_t *offsets;  /* var-len only: n_rows+1 offsets */
    const uint8_t *valid;    /* Arrow validity bitmap (LSB first) or NULL = no nulls */
} po_col;

/* file-order columns: [key_0..key_{nk-1}, _SEQUENCE_NUMBER i64, _VALUE_KIND i8, val_0..val_{nv-1}]
 * (paimon-core/.../KeyValue.java:130-138) */
typedef struct {
    int64_t n_rows;
    const po_col *cols;      /* n_key + 2 + n_val entries */
} po_run;

typedef struct {
    int32_t n_key;
    int32_t n_val;
    const int32_t *key_types;      /* [n_key] */
    const int32_t *val_types;      /* [n_val] */
    const uint8_t *val_nullable;   /* [n_val] 1 = nullable */
} po_schema;

typedef struct {
    int32_t engine;
    int32_t sort_engine;
    int32_t ignore_delete;             /* 'ignore-delete' */
    int32_t remove_record_on_delete;   /* partial-update.* / aggregation.remove-record-on-delete */
    int32_t drop_delete;               /* wrap in DropDeleteReader */
    /* 'sequence.field': user defined sequence comparator over value fields */
    int32_t n_seq_fields;
    const int32_t *seq_fields;         /* value-field indexes */
    int32_t seq_ascending;
    /* per value field */
    const int32_t *agg;                /* [n_val] PO_AGG_* */
    const uint8_t *ignore_retract;     /* [n_val] */
    /* partial-update sequence groups (fields.<a,b>.sequence-group = c,d) */
    int32_t n_groups;
    const int32_t *group_seq_start;    /* [n_groups+1] CSR into group_seq_fields */
    const int32_t *group_seq_fields;   /* value-field indexes of each group's sequence fields */
    const int32_t *field_group;        /* [n_val] group id protecting this field (incl. the sequence
                                          fields themselves), -1 = none */
    const uint8_t *group_partial_delete; /* [n_val] field is in sequenceGroupPartialDelete */
    /* test hook: call MergeFunction.add for every record, without ReducerMergeFunctionWrapper's
     * single-record passthrough — this is how the reference's MergeFunction unit tests
     * (PartialUpdateMergeFunctionTest, AggregateMergeFunctionTest) drive the function */
    int32_t bypass_wrapper;
    /* [n_val] precision << 8 | scale of a DECIMAL(p <= 18) field (unscaled INT64), 0 = not DECIMAL; NULL = none.
     * sum / product on such a field follow FieldSumAgg / FieldProductAgg's DECIMAL branch (DecimalUtils.add /
     * subtract, BigDecimal multiply / divide, Decimal.fromBigDecimal), not int64 arithmetic. */
    const int32_t *decimal;
} po_spec;

typedef struct {
    void *data;
    int32_t *offsets;
    uint8_t *valid;       /* bitmap, always allocated */
    int64_t data_bytes;   /* var-len: bytes used */
} po_out_col;

typedef struct {
    int64_t n_rows;
    int32_t n_cols;
    po_out_col *cols;
} po_result;

/* Merge k sorted runs.  Returns 0, or <0 on a Java-exception-equivalent (message via
 * po_last_error()).  *out must be freed with po_result_free. */
int po_merge(const po_schema *schema, const po_spec *spec, int32_t k, const po_run *runs,
             po_result **out);
void po_result_free(po_result *r);
const char *po_last_error(void);

/* the (run,row) pop order of the bare LoserTree / MinHeap (LoserTreeTest.java:51-68) */
int po_merge_order(const po_schema *schema, const po_spec *spec, int32_t k, const po_run *runs,
                   int32_t *out_run, int64_t *out_row, int64_t *out_n);

/* IntervalPartition.java:67-125 over int64 (min,max) file key bounds.
 * Writes, per file (input order), its section id and run id within the section. */
int po_interval_partition(int32_t n_files, const int64_t *min_key, const int64_t *max_key,
                          int32_t *section_of, int32_t *run_of, int32_t *n_sections);

#ifdef __cplusplus
}
#endif
#endif
