/*
 * paimon_oracle.c — TEST INFRASTRUCTURE ONLY (see paimon_oracle.h).
 *
 * Row-at-a-time CPU restatement of the reference's SortMergeReader / LoserTree /
 * MergeFunction stack over Arrow-layout columnar runs.  Deliberately written the way
 * the Java code is structured (state machine, wrapper, per-record add) so that each
 * function can be read next to the reference lines it cites.  Not optimised.
 */
#include "paimon_oracle.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define REF_BASE "paimon-core/src/main/java/org/apache/paimon/mergetree/compact/"

static __thread char g_err[512];
const char *po_last_error(void) { return g_err; }
static int fail(const char *msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg);
    return -1;
}

/* ------------------------------------------------------------------ values */

typedef struct {
    uint8_t is_null;
    union { int64_t i; double d; float f; } v;
    const uint8_t *p;   /* var-len payload */
    int32_t len;
} po_val;

typedef struct { int32_t run; int64_t row; } kvref;   /* a KeyValue = (run,row); run<0 = null */

typedef struct {
    const po_schema *s;
    const po_spec *spec;
    int32_t k;
    const po_run *runs;
} ctx_t;

static int is_varlen(int t) { return t == PO_STRING || t == PO_BINARY; }
static int type_width(int t) {
    switch (t) {
        case PO_INT8: case PO_BOOL: return 1;
        case PO_INT16: return 2;
        case PO_INT32: case PO_FLOAT: return 4;
        case PO_INT64: case PO_DOUBLE: return 8;
        default: return 0;
    }
}

static po_val read_val(int type, const po_col *c, int64_t row) {
    po_val v;
    memset(&v, 0, sizeof(v));
    if (c->valid && !((c->valid[row >> 3] >> (row & 7)) & 1)) { v.is_null = 1; return v; }
    switch (type) {
        case PO_INT8:  v.v.i = ((const int8_t *)c->data)[row]; break;
        case PO_BOOL:  v.v.i = ((const uint8_t *)c->data)[row] ? 1 : 0; break;
        case PO_INT16: v.v.i = ((const int16_t *)c->data)[row]; break;
        case PO_INT32: v.v.i = ((const int32_t *)c->data)[row]; break;
        case PO_INT64: v.v.i = ((const int64_t *)c->data)[row]; break;
        case PO_FLOAT: v.v.f = ((const float *)c->data)[row]; break;
        case PO_DOUBLE: v.v.d = ((const double *)c->data)[row]; break;
        case PO_STRING: case PO_BINARY:
            v.p = (const uint8_t *)c->data + c->offsets[row];
            v.len = c->offsets[row + 1] - c->offsets[row];
            break;
    }
    return v;
}

/* KeyValue accessors — KeyValueSerializer.fromRow (paimon-core/.../KeyValueSerializer.java:77-84) */
static const po_col *key_col(const ctx_t *c, kvref kv, int f) { return &c->runs[kv.run].cols[f]; }
static int64_t kv_seq(const ctx_t *c, kvref kv) {
    return ((const int64_t *)c->runs[kv.run].cols[c->s->n_key].data)[kv.row];
}
static int8_t kv_kind(const ctx_t *c, kvref kv) {
    return ((const int8_t *)c->runs[kv.run].cols[c->s->n_key + 1].data)[kv.row];
}
static po_val kv_value(const ctx_t *c, kvref kv, int f) {
    return read_val(c->s->val_types[f], &c->runs[kv.run].cols[c->s->n_key + 2 + f], kv.row);
}
/* RowKind.isRetract / isAdd, paimon-api/.../types/RowKind.java:101-108 */
static int is_retract(int8_t kind) { return kind == PO_UPDATE_BEFORE || kind == PO_DELETE; }

/* ------------------------------------------------------------- comparators */

static int cmp_bytes(const uint8_t *a, int32_t la, const uint8_t *b, int32_t lb) {
    /* BinaryString.compareTo :109-126 and SortUtil.compareBinary :212-241 — both reduce to
     * unsigned bytewise comparison, then length */
    int32_t n = la < lb ? la : lb;
    for (int32_t i = 0; i < n; i++) {
        int d = (int)a[i] - (int)b[i];
        if (d != 0) return d;
    }
    return la - lb;
}

/* generated comparator body for one non-null field, GenerateUtils.scala:113-126:
 * numeric: (a > b ? 1 : a < b ? -1 : 0)  — NaN compares equal to everything */
static int cmp_codegen(int type, const po_val *a, const po_val *b) {
    switch (type) {
        case PO_INT8: case PO_INT16: case PO_INT32: case PO_INT64:
            return a->v.i > b->v.i ? 1 : a->v.i < b->v.i ? -1 : 0;
        case PO_BOOL:
            return a->v.i == b->v.i ? 0 : (a->v.i ? 1 : -1);
        case PO_FLOAT:
            return a->v.f > b->v.f ? 1 : a->v.f < b->v.f ? -1 : 0;
        case PO_DOUBLE:
            return a->v.d > b->v.d ? 1 : a->v.d < b->v.d ? -1 : 0;
        default: {
            int d = cmp_bytes(a->p, a->len, b->p, b->len);
            return d > 0 ? 1 : d < 0 ? -1 : 0;
        }
    }
}

/* userKeyComparator.compare(a.key(), b.key()); PK fields are NOT NULL */
static int cmp_key(const ctx_t *c, kvref a, kvref b) {
    for (int f = 0; f < c->s->n_key; f++) {
        po_val va = read_val(c->s->key_types[f], key_col(c, a, f), a.row);
        po_val vb = read_val(c->s->key_types[f], key_col(c, b, f), b.row);
        int d = cmp_codegen(c->s->key_types[f], &va, &vb);
        if (d != 0) return d;
    }
    return 0;
}

/* generateRowCompare with nullIsLast=false (GenerateUtils.scala:305-345): both null -> next
 * field; one null -> that side is smaller, returned BEFORE the descending sign flip */
static int cmp_fields_vals(const po_schema *s, const int32_t *fields, int n, int ascending,
                           const po_val *a, const po_val *b) {
    for (int j = 0; j < n; j++) {
        int f = fields[j];
        if (a[f].is_null && b[f].is_null) continue;
        if (a[f].is_null) return -1;
        if (b[f].is_null) return 1;
        int d = cmp_codegen(s->val_types[f], &a[f], &b[f]);
        if (d != 0) return ascending ? d : -d;
    }
    return 0;
}

/* userDefinedSeqComparator.compare(a.value(), b.value()) on two stored rows */
static int cmp_udseq(const ctx_t *c, kvref a, kvref b) {
    const po_spec *sp = c->spec;
    for (int j = 0; j < sp->n_seq_fields; j++) {
        int f = sp->seq_fields[j];
        po_val va = kv_value(c, a, f), vb = kv_value(c, b, f);
        if (va.is_null && vb.is_null) continue;
        if (va.is_null) return -1;
        if (vb.is_null) return 1;
        int d = cmp_codegen(c->s->val_types[f], &va, &vb);
        if (d != 0) return sp->seq_ascending ? d : -d;
    }
    return 0;
}

static int cmp_i64(int64_t a, int64_t b) { return a < b ? -1 : a > b ? 1 : 0; }

/* total order used by the min-heap (SortMergeReaderWithMinHeap.java:56-70) and by the
 * brute-force checker: key, [user sequence fields], sequence number */
static int cmp_full(const ctx_t *c, kvref a, kvref b) {
    int d = cmp_key(c, a, b);
    if (d != 0) return d;
    if (c->spec->n_seq_fields > 0) {
        d = cmp_udseq(c, a, b);
        if (d != 0) return d;
    }
    return cmp_i64(kv_seq(c, a), kv_seq(c, b));
}

/* ------------------------------------------------------------- LoserTree */

/* LoserTree.java:338-355 */
enum { LOSER_WITH_NEW_KEY, LOSER_WITH_SAME_KEY, LOSER_POPPED,
       WINNER_WITH_NEW_KEY, WINNER_WITH_SAME_KEY, WINNER_POPPED };
static int state_is_winner(int st) { return st >= WINNER_WITH_NEW_KEY; }

typedef struct {
    int32_t run;
    int64_t next;       /* next row to hand out (iterator position) */
    kvref kv;           /* current minimum kv; run = -1 => null */
    int end_of_input;
    int first_same_key_index;
    int state;
} leaf_t;

typedef struct {
    const ctx_t *c;
    int *tree;
    int size;
    leaf_t *leaves;
    int initialized;
    int bug;            /* set when a "This is a bug" branch is reached */
} loser_tree;

/* LoserTree.java:66-73 + SortMergeReaderWithLoserTree.java:48 — first comparator: nulls lose,
 * user key comparator REVERSED so that the smallest key "wins" */
static int lt_first_cmp(const loser_tree *t, kvref e1, kvref e2) {
    if (e1.run < 0) return -1;
    if (e2.run < 0) return 1;
    return cmp_key(t->c, e2, e1);
}
/* SortMergeReaderWithLoserTree.java:52-65 */
static int lt_second_cmp(const loser_tree *t, kvref e1, kvref e2) {
    if (e1.run < 0) return -1;
    if (e2.run < 0) return 1;
    if (t->c->spec->n_seq_fields > 0) {
        int r = cmp_udseq(t->c, e2, e1);
        if (r != 0) return r;
    }
    return cmp_i64(kv_seq(t->c, e2), kv_seq(t->c, e1));
}

static void leaf_set_first_same_key_index(leaf_t *l, int index) {      /* :288-292 */
    if (l->first_same_key_index == -1) l->first_same_key_index = index;
}

/* LeafIterator.advanceIfAvailable :295-316 — each run is a single batch */
static void leaf_advance_if_available(const loser_tree *t, leaf_t *l) {
    l->first_same_key_index = -1;
    l->state = WINNER_WITH_NEW_KEY;
    if (!l->end_of_input && l->next < t->c->runs[l->run].n_rows) {
        l->kv.run = l->run;
        l->kv.row = l->next++;
    } else {
        l->end_of_input = 1;
        l->kv.run = -1;
    }
}

/* :173-197 */
static void lt_adjust_with_same_winner_key(loser_tree *t, int index, leaf_t *parent, leaf_t *winner) {
    switch (parent->state) {
        case LOSER_WITH_SAME_KEY: {
            int second = lt_second_cmp(t, parent->kv, winner->kv);
            if (second > 0) {
                parent->state = WINNER_WITH_SAME_KEY;
                winner->state = LOSER_WITH_SAME_KEY;
                leaf_set_first_same_key_index(parent, index);
            } else {
                leaf_set_first_same_key_index(winner, index);
            }
            return;
        }
        case LOSER_WITH_NEW_KEY:
        case LOSER_POPPED:
            return;
        default:
            t->bug = 1;
    }
}

/* :203-245 */
static void lt_adjust_with_new_winner_key(loser_tree *t, int index, leaf_t *parent, leaf_t *winner) {
    switch (parent->state) {
        case LOSER_WITH_NEW_KEY: {
            int first = lt_first_cmp(t, parent->kv, winner->kv);
            if (first == 0) {
                int second = lt_second_cmp(t, parent->kv, winner->kv);
                if (second < 0) {
                    parent->state = LOSER_WITH_SAME_KEY;
                    leaf_set_first_same_key_index(winner, index);
                } else {
                    winner->state = LOSER_WITH_SAME_KEY;
                    parent->state = WINNER_WITH_NEW_KEY;
                    leaf_set_first_same_key_index(parent, index);
                }
            } else if (first > 0) {
                parent->state = WINNER_WITH_NEW_KEY;
                winner->state = LOSER_WITH_NEW_KEY;
            }
            return;
        }
        case LOSER_WITH_SAME_KEY:
            t->bug = 1;
            return;
        case LOSER_POPPED:
            parent->state = WINNER_POPPED;
            parent->first_same_key_index = -1;
            winner->state = LOSER_WITH_NEW_KEY;
            return;
        default:
            t->bug = 1;
    }
}

/* :126-170 */
static void lt_adjust(loser_tree *t, int winner) {
    int parent;
    for (parent = (winner + t->size) / 2; parent > 0 && winner >= 0; parent /= 2) {
        leaf_t *winner_node = &t->leaves[winner];
        leaf_t *parent_node;
        if (t->tree[parent] == -1) {
            winner_node->state = LOSER_WITH_NEW_KEY;
        } else {
            parent_node = &t->leaves[t->tree[parent]];
            switch (winner_node->state) {
                case WINNER_WITH_NEW_KEY:
                    lt_adjust_with_new_winner_key(t, parent, parent_node, winner_node);
                    break;
                case WINNER_WITH_SAME_KEY:
                    lt_adjust_with_same_winner_key(t, parent, parent_node, winner_node);
                    break;
                case WINNER_POPPED:
                    if (winner_node->first_same_key_index < 0) {
                        parent = -1;
                    } else {
                        parent = winner_node->first_same_key_index;
                        parent_node = &t->leaves[t->tree[parent]];
                        winner_node->state = LOSER_POPPED;
                        parent_node->state = WINNER_WITH_SAME_KEY;
                    }
                    break;
                default:
                    t->bug = 1;
            }
        }
        if (parent < 0) break;   /* Java: parent = -1 then "parent /= 2" leaves the loop (-1/2 == 0) */
        if (!state_is_winner(winner_node->state)) {
            int tmp = winner;
            winner = t->tree[parent];
            t->tree[parent] = tmp;
        }
    }
    t->tree[0] = winner;
}

/* :83-92 */
static void lt_initialize_if_needed(loser_tree *t) {
    if (!t->initialized) {
        for (int i = 0; i < t->size; i++) t->tree[i] = -1;
        for (int i = t->size - 1; i >= 0; i--) {
            leaf_advance_if_available(t, &t->leaves[i]);
            lt_adjust(t, i);
        }
        t->initialized = 1;
    }
}
/* :95-102 */
static void lt_adjust_for_next_loop(loser_tree *t) {
    leaf_t *winner = &t->leaves[t->tree[0]];
    while (winner->state == WINNER_POPPED) {
        leaf_advance_if_available(t, winner);
        lt_adjust(t, t->tree[0]);
        winner = &t->leaves[t->tree[0]];
    }
}
/* :105-115 */
static kvref lt_pop_winner(loser_tree *t) {
    kvref null_kv = { -1, 0 };
    leaf_t *winner = &t->leaves[t->tree[0]];
    if (winner->state == WINNER_POPPED) return null_kv;
    winner->state = WINNER_POPPED;          /* LeafIterator.pop :283-286 */
    kvref result = winner->kv;
    lt_adjust(t, t->tree[0]);
    return result;
}
/* :118-120 */
static kvref lt_peek_winner(loser_tree *t) {
    kvref null_kv = { -1, 0 };
    leaf_t *w = &t->leaves[t->tree[0]];
    return w->state != WINNER_POPPED ? w->kv : null_kv;
}

static loser_tree *lt_new(const ctx_t *c) {
    loser_tree *t = (loser_tree *)calloc(1, sizeof(*t));
    t->c = c;
    t->size = c->k;
    t->tree = (int *)calloc(c->k > 0 ? c->k : 1, sizeof(int));
    t->leaves = (leaf_t *)calloc(c->k > 0 ? c->k : 1, sizeof(leaf_t));
    for (int i = 0; i < c->k; i++) {
        t->leaves[i].run = i;
        t->leaves[i].kv.run = -1;
        t->leaves[i].first_same_key_index = -1;
        t->leaves[i].state = WINNER_WITH_NEW_KEY;
    }
    return t;
}
static void lt_free(loser_tree *t) { free(t->tree); free(t->leaves); free(t); }

/* ---------------------------------------------------------- merge functions */

typedef struct {
    const ctx_t *c;
    /* DeduplicateMergeFunction / FirstRowMergeFunction */
    kvref latest;
    /* PartialUpdate / Aggregate accumulators */
    po_val *row;              /* GenericRow(getters.length) */
    uint8_t *agg_initialized; /* FieldFirst*Agg.initialized */
    kvref current_key;        /* the kv whose key() is currentKey / latestKv */
    int64_t latest_seq;
    int current_delete_row;
    int not_null_column_filled;
    int meet_insert;
    /* scratch */
    po_val *in;
    uint8_t *empty_group;
    uint8_t *updated_seq_fields;
} mf_t;

/* result of getResult(): */
enum { RES_NULL = 0, RES_REF = 1, RES_ROW = 2 };
typedef struct {
    int kind;
    kvref ref;        /* RES_REF: the source kv; RES_ROW: kv supplying the key */
    int64_t seq;
    int8_t value_kind;
    const po_val *row;
} result_t;

static void row_clear(const ctx_t *c, po_val *row) {
    for (int i = 0; i < c->s->n_val; i++) { memset(&row[i], 0, sizeof(po_val)); row[i].is_null = 1; }
}

static void mf_reset(mf_t *m) {
    const ctx_t *c = m->c;
    switch (c->spec->engine) {
        case PO_ENGINE_DEDUPLICATE:          /* DeduplicateMergeFunction.java:42-45 */
        case PO_ENGINE_FIRST_ROW:            /* FirstRowMergeFunction.java:44-48 */
            m->latest.run = -1;
            break;
        case PO_ENGINE_PARTIAL_UPDATE:       /* PartialUpdateMergeFunction.java:111-119 */
            m->current_key.run = -1;
            m->meet_insert = 0;
            m->not_null_column_filled = 0;
            row_clear(c, m->row);
            m->latest_seq = 0;
            memset(m->agg_initialized, 0, c->s->n_val);
            break;
        case PO_ENGINE_AGGREGATE:            /* AggregateMergeFunction.java:72-78 */
            m->current_key.run = -1;
            row_clear(c, m->row);
            memset(m->agg_initialized, 0, c->s->n_val);
            m->current_delete_row = 0;
            break;
    }
}

/* Float.compare / Double.compare total order used by FieldMax/MinAgg through
 * InternalRowUtils.compare (paimon-common/.../utils/InternalRowUtils.java:409-414) */
static int java_double_compare(double a, double b) {
    if (a < b) return -1;
    if (a > b) return 1;
    int64_t x, y;
    memcpy(&x, &a, 8); memcpy(&y, &b, 8);
    /* doubleToLongBits canonicalises NaN */
    if (a != a) x = 0x7ff8000000000000LL;
    if (b != b) y = 0x7ff8000000000000LL;
    return x == y ? 0 : (x < y ? -1 : 1);
}
static int java_float_compare(float a, float b) {
    if (a < b) return -1;
    if (a > b) return 1;
    int32_t x, y;
    memcpy(&x, &a, 4); memcpy(&y, &b, 4);
    if (a != a) x = 0x7fc00000;
    if (b != b) y = 0x7fc00000;
    return x == y ? 0 : (x < y ? -1 : 1);
}
static int cmp_internal_row_utils(int type, const po_val *a, const po_val *b, int *err) {
    switch (type) {
        case PO_INT8: case PO_INT16: case PO_INT32: case PO_INT64:
            return cmp_i64(a->v.i, b->v.i);
        case PO_FLOAT: return java_float_compare(a->v.f, b->v.f);
        case PO_DOUBLE: return java_double_compare(a->v.d, b->v.d);
        case PO_STRING: case PO_BINARY: return cmp_bytes(a->p, a->len, b->p, b->len);
        default: *err = 1; return 0;   /* "Incomparable type" */
    }
}

/* ---- DECIMAL(p, s) sum / product on unscaled int64 values (p <= 18)
 * sum / subtract: DecimalUtils.add / subtract (paimon-common/.../utils/DecimalUtils.java:52-87): exact int64; on
 *   overflow the BigDecimal result has more than 18 digits and Decimal.fromBigDecimal returns NULL; a result over p
 *   digits that fits int64 is kept (fromUnscaledLong does not check the precision).
 * product: round_half_up(a * b / 10^s), NULL over p digits (FieldProductAgg.java:47-58, Decimal.java:182-193).
 * product retract: BigDecimal.divide is exact: it throws on a zero divisor and when the quotient does not terminate;
 *   otherwise round_half_up(a * 10^s / b), NULL over p digits (FieldProductAgg.java:95-106).
 * sum retract into a NULL accumulator: negative() = fromBigDecimal(-a), NULL over p digits (FieldSumAgg.java:140-143).
 * |a|, |b| <= 2^63 and 10^s <= 10^18, so a * b and a * 10^s fit __int128. */
static int field_decimal(const mf_t *m, int f) {
    return m->c->spec->decimal ? m->c->spec->decimal[f] : 0;
}
static unsigned __int128 dec_pow10(int e) {
    unsigned __int128 r = 1;
    while (e-- > 0) r *= 10u;
    return r;
}
static unsigned __int128 dec_abs(__int128 v) { return v < 0 ? (unsigned __int128)0 - (unsigned __int128)v : (unsigned __int128)v; }
static __int128 dec_div_half_up(__int128 n, unsigned __int128 d) {       /* d > 0; RoundingMode.HALF_UP */
    unsigned __int128 m = dec_abs(n), q = m / d, r = m - q * d;
    if (r >= d - r) q += 1;
    return n < 0 ? -(__int128)q : (__int128)q;
}
/* out := the DECIMAL r, or NULL when it has more than p digits */
static void dec_set(po_val *out, __int128 r, int precision) {
    if (dec_abs(r) >= dec_pow10(precision)) { memset(out, 0, sizeof(*out)); out->is_null = 1; }
    else { out->is_null = 0; out->v.i = (int64_t)r; }
}
/* fn: 0 add, 1 subtract, 2 multiply, 3 divide, 4 negate a.  Returns -1 when BigDecimal would have thrown. */
static int dec_arith(int decimal, int fn, int64_t a, int64_t b, po_val *out) {
    const int precision = decimal >> 8, scale = decimal & 0xff;
    if (fn == 0 || fn == 1) {
        int64_t r;
        int overflow = fn == 0 ? __builtin_add_overflow(a, b, &r) : __builtin_sub_overflow(a, b, &r);
        if (overflow) { memset(out, 0, sizeof(*out)); out->is_null = 1; }
        else { out->is_null = 0; out->v.i = r; }
        return 0;
    }
    if (fn == 4) { dec_set(out, -(__int128)a, precision); return 0; }
    if (fn == 2) { dec_set(out, dec_div_half_up((__int128)a * b, dec_pow10(scale)), precision); return 0; }
    if (b == 0) return fail(a == 0 ? "ArithmeticException: Division undefined" : "ArithmeticException: Division by zero");
    /* a / b terminates iff b / gcd(a, b) has no prime factor other than 2 and 5 */
    uint64_t x = (uint64_t)dec_abs(a), y = (uint64_t)dec_abs(b);
    while (x != 0) { uint64_t t = y % x; y = x; x = t; }
    uint64_t den = (uint64_t)dec_abs(b) / y;
    while (den % 2 == 0) den /= 2;
    while (den % 5 == 0) den /= 5;
    if (den != 1)
        return fail("ArithmeticException: Non-terminating decimal expansion; no exact representable decimal result.");
    __int128 n = (__int128)a * (__int128)dec_pow10(scale);
    dec_set(out, dec_div_half_up(b < 0 ? -n : n, dec_abs(b)), precision);
    return 0;
}

/* FieldAggregator.agg for the fixed-width aggregators (files listed in the header) */
static int agg_apply(mf_t *m, int f, int agg, const po_val *acc, const po_val *in, po_val *out) {
    int type = m->c->s->val_types[f];
    int err = 0;
    switch (agg) {
        case PO_AGG_SUM: case PO_AGG_PRODUCT:       /* FieldSumAgg.java:41-84, FieldProductAgg */
            if (acc->is_null || in->is_null) { *out = acc->is_null ? *in : *acc; return 0; }
            *out = *acc;
            if (field_decimal(m, f)) return dec_arith(field_decimal(m, f), agg == PO_AGG_PRODUCT ? 2 : 0, acc->v.i, in->v.i, out);
            {
                int mul = agg == PO_AGG_PRODUCT;
                switch (type) {
                    case PO_INT8:  out->v.i = (int8_t)(mul ? (int8_t)acc->v.i * (int8_t)in->v.i
                                                           : (int8_t)acc->v.i + (int8_t)in->v.i); break;
                    case PO_INT16: out->v.i = (int16_t)(mul ? (int16_t)acc->v.i * (int16_t)in->v.i
                                                            : (int16_t)acc->v.i + (int16_t)in->v.i); break;
                    case PO_INT32: out->v.i = (int32_t)(mul ? (uint32_t)acc->v.i * (uint32_t)in->v.i
                                                            : (uint32_t)acc->v.i + (uint32_t)in->v.i); break;
                    case PO_INT64: out->v.i = (int64_t)(mul ? (uint64_t)acc->v.i * (uint64_t)in->v.i
                                                            : (uint64_t)acc->v.i + (uint64_t)in->v.i); break;
                    case PO_FLOAT: out->v.f = mul ? acc->v.f * in->v.f : acc->v.f + in->v.f; break;
                    case PO_DOUBLE: out->v.d = mul ? acc->v.d * in->v.d : acc->v.d + in->v.d; break;
                    default: return fail("type not support in FieldSumAgg/FieldProductAgg");
                }
            }
            return 0;
        case PO_AGG_MAX: case PO_AGG_MIN: {          /* FieldMaxAgg.java:35-43, FieldMinAgg */
            if (acc->is_null || in->is_null) { *out = acc->is_null ? *in : *acc; return 0; }
            int d = cmp_internal_row_utils(type, acc, in, &err);
            if (err) return fail("Incomparable type");
            if (agg == PO_AGG_MAX) *out = d < 0 ? *in : *acc;
            else *out = d < 0 ? *acc : *in;
            return 0;
        }
        case PO_AGG_BOOL_AND: case PO_AGG_BOOL_OR:
            if (acc->is_null || in->is_null) { *out = acc->is_null ? *in : *acc; return 0; }
            *out = *acc;
            out->v.i = agg == PO_AGG_BOOL_AND ? (acc->v.i && in->v.i) : (acc->v.i || in->v.i);
            return 0;
        case PO_AGG_LAST_VALUE: case PO_AGG_PRIMARY_KEY:   /* FieldLastValueAgg.java:33-36 */
            *out = *in;
            return 0;
        case PO_AGG_LAST_NON_NULL_VALUE:                   /* FieldLastNonNullValueAgg.java:33-36 */
            *out = in->is_null ? *acc : *in;
            return 0;
        case PO_AGG_FIRST_VALUE:                           /* FieldFirstValueAgg.java:37-44 */
            if (!m->agg_initialized[f]) { m->agg_initialized[f] = 1; *out = *in; }
            else *out = *acc;
            return 0;
        case PO_AGG_FIRST_NON_NULL_VALUE:                  /* FieldFirstNonNullValueAgg.java:37-44 */
            if (!m->agg_initialized[f] && !in->is_null) { m->agg_initialized[f] = 1; *out = *in; }
            else *out = *acc;
            return 0;
    }
    return fail("unknown aggregator");
}

/* aggReversed = agg(inputField, accumulator), FieldAggregator.java:40-42 */
static int agg_apply_reversed(mf_t *m, int f, int agg, const po_val *acc, const po_val *in, po_val *out) {
    return agg_apply(m, f, agg, in, acc, out);
}

static int agg_retract(mf_t *m, int f, int agg, const po_val *acc, const po_val *in, po_val *out) {
    int type = m->c->s->val_types[f];
    if (m->c->spec->ignore_retract && m->c->spec->ignore_retract[f]) {   /* FieldIgnoreRetractAgg :43-45 */
        *out = *acc;
        return 0;
    }
    switch (agg) {
        case PO_AGG_SUM:                                   /* FieldSumAgg.java:87-131, negative :133-163 */
            if (acc->is_null || in->is_null) {
                if (!acc->is_null) { *out = *acc; return 0; }
                *out = *in;                                  /* negative(inputField) */
                if (in->is_null) return 0;
                if (field_decimal(m, f)) return dec_arith(field_decimal(m, f), 4, in->v.i, 0, out);
                switch (type) {
                    case PO_INT8:  out->v.i = (int8_t)(-(int8_t)in->v.i); break;
                    case PO_INT16: out->v.i = (int16_t)(-(int16_t)in->v.i); break;
                    case PO_INT32: out->v.i = (int32_t)(0u - (uint32_t)in->v.i); break;
                    case PO_INT64: out->v.i = (int64_t)(0ull - (uint64_t)in->v.i); break;
                    case PO_FLOAT: out->v.f = -in->v.f; break;
                    case PO_DOUBLE: out->v.d = -in->v.d; break;
                    default: return fail("type not support in FieldSumAgg");
                }
                return 0;
            }
            *out = *acc;
            if (field_decimal(m, f)) return dec_arith(field_decimal(m, f), 1, acc->v.i, in->v.i, out);
            switch (type) {
                case PO_INT8:  out->v.i = (int8_t)((int8_t)acc->v.i - (int8_t)in->v.i); break;
                case PO_INT16: out->v.i = (int16_t)((int16_t)acc->v.i - (int16_t)in->v.i); break;
                case PO_INT32: out->v.i = (int32_t)((uint32_t)acc->v.i - (uint32_t)in->v.i); break;
                case PO_INT64: out->v.i = (int64_t)((uint64_t)acc->v.i - (uint64_t)in->v.i); break;
                case PO_FLOAT: out->v.f = acc->v.f - in->v.f; break;
                case PO_DOUBLE: out->v.d = acc->v.d - in->v.d; break;
                default: return fail("type not support in FieldSumAgg");
            }
            return 0;
        case PO_AGG_PRODUCT:                               /* FieldProductAgg retract: divide */
            if (acc->is_null || in->is_null) { *out = *acc; return 0; }
            *out = *acc;
            if (field_decimal(m, f)) return dec_arith(field_decimal(m, f), 3, acc->v.i, in->v.i, out);
            switch (type) {
                case PO_INT8: case PO_INT16: case PO_INT32: case PO_INT64:
                    if (in->v.i == 0) return fail("ArithmeticException: / by zero");
                    /* Java integer division truncates toward zero; MIN/-1 wraps */
                    if (in->v.i == -1) out->v.i = (int64_t)(0ull - (uint64_t)acc->v.i);
                    else out->v.i = acc->v.i / in->v.i;
                    if (type == PO_INT8) out->v.i = (int8_t)out->v.i;
                    if (type == PO_INT16) out->v.i = (int16_t)out->v.i;
                    if (type == PO_INT32) out->v.i = (int32_t)out->v.i;
                    break;
                case PO_FLOAT: out->v.f = acc->v.f / in->v.f; break;
                case PO_DOUBLE: out->v.d = acc->v.d / in->v.d; break;
                default: return fail("type not support in FieldProductAgg");
            }
            return 0;
        case PO_AGG_LAST_VALUE:                            /* FieldLastValueAgg.java:38-40 */
            memset(out, 0, sizeof(*out)); out->is_null = 1;
            return 0;
        case PO_AGG_LAST_NON_NULL_VALUE:                   /* FieldLastNonNullValueAgg.java:38-40 */
            if (!in->is_null) { memset(out, 0, sizeof(*out)); out->is_null = 1; }
            else *out = *acc;
            return 0;
        case PO_AGG_PRIMARY_KEY:                           /* FieldPrimaryKeyAgg.java:38-40 */
            *out = *in;
            return 0;
        default:                                           /* FieldAggregator.java:47-54 */
            return fail("Aggregate function does not support retraction, If you allow this function "
                        "to ignore retraction messages, you can configure "
                        "'fields.${field_name}.ignore-retract'='true'.");
    }
}

/* initRow, PartialUpdateMergeFunction.java:344-352 / AggregateMergeFunction.java:104-112 */
static int init_row(mf_t *m, po_val *row, const po_val *value) {
    for (int i = 0; i < m->c->s->n_val; i++) {
        if (!m->c->s->val_nullable[i] && value[i].is_null) return fail("Field can not be null");
        row[i] = value[i];
    }
    return 0;
}

static void load_value_row(mf_t *m, kvref kv) {
    for (int i = 0; i < m->c->s->n_val; i++) m->in[i] = kv_value(m->c, kv, i);
}

/* isEmptySequenceGroup :249-269 */
static int pu_is_empty_group(mf_t *m, int g) {
    const po_spec *sp = m->c->spec;
    const int32_t *fields = sp->group_seq_fields + sp->group_seq_start[g];
    int n = sp->group_seq_start[g + 1] - sp->group_seq_start[g];
    if (m->empty_group[fields[0]]) return 1;
    for (int j = 0; j < n; j++) if (!m->in[fields[j]].is_null) return 0;
    for (int j = 0; j < n; j++) m->empty_group[fields[j]] = 1;
    return 1;
}
static int pu_group_has_field(const po_spec *sp, int g, int f) {
    for (int j = sp->group_seq_start[g]; j < sp->group_seq_start[g + 1]; j++)
        if (sp->group_seq_fields[j] == f) return 1;
    return 0;
}
static int pu_cmp_group(mf_t *m, int g) {      /* seqComparator.compare(kv.value(), row) */
    const po_spec *sp = m->c->spec;
    return cmp_fields_vals(m->c->s, sp->group_seq_fields + sp->group_seq_start[g],
                           sp->group_seq_start[g + 1] - sp->group_seq_start[g], 1, m->in, m->row);
}

/* updateWithSequenceGroup :190-247 */
static int pu_update_with_sequence_group(mf_t *m) {
    const po_spec *sp = m->c->spec;
    int n = m->c->s->n_val;
    memset(m->empty_group, 0, n);
    for (int i = 0; i < n; i++) {
        int g = sp->field_group ? sp->field_group[i] : -1;
        int agg = sp->agg ? sp->agg[i] : PO_AGG_NONE;
        po_val accumulator = m->row[i];
        if (g < 0) {
            po_val field = m->in[i];
            if (agg != PO_AGG_NONE) {
                po_val out;
                if (agg_apply(m, i, agg, &accumulator, &field, &out)) return -1;
                m->row[i] = out;
            } else if (!field.is_null) {
                m->row[i] = field;
            }
        } else {
            if (pu_is_empty_group(m, g)) continue;
            po_val field = m->in[i];
            if (pu_cmp_group(m, g) >= 0) {
                if (pu_group_has_field(sp, g, i)) {
                    for (int j = sp->group_seq_start[g]; j < sp->group_seq_start[g + 1]; j++)
                        m->row[sp->group_seq_fields[j]] = m->in[sp->group_seq_fields[j]];
                    continue;
                }
                if (agg == PO_AGG_NONE) m->row[i] = field;
                else {
                    po_val out;
                    if (agg_apply(m, i, agg, &accumulator, &field, &out)) return -1;
                    m->row[i] = out;
                }
            } else if (agg != PO_AGG_NONE) {
                po_val out;
                if (agg_apply_reversed(m, i, agg, &accumulator, &field, &out)) return -1;
                m->row[i] = out;
            }
        }
    }
    return 0;
}

/* retractWithSequenceGroup :271-342; returns 1 if it performed the early "return" */
static int pu_retract_with_sequence_group(mf_t *m, kvref kv) {
    const po_spec *sp = m->c->spec;
    int n = m->c->s->n_val;
    memset(m->empty_group, 0, n);
    memset(m->updated_seq_fields, 0, n);
    for (int i = 0; i < n; i++) {
        int g = sp->field_group ? sp->field_group[i] : -1;
        int agg = sp->agg ? sp->agg[i] : PO_AGG_NONE;
        if (g < 0) continue;
        if (pu_is_empty_group(m, g)) continue;
        if (pu_cmp_group(m, g) >= 0) {
            if (pu_group_has_field(sp, g, i)) {
                for (int j = sp->group_seq_start[g]; j < sp->group_seq_start[g + 1]; j++) {
                    int field = sp->group_seq_fields[j];
                    if (!m->updated_seq_fields[field]) {
                        if (kv_kind(m->c, kv) == PO_DELETE && sp->group_partial_delete &&
                            sp->group_partial_delete[field]) {
                            m->current_delete_row = 1;
                            row_clear(m->c, m->row);
                            if (init_row(m, m->row, m->in)) return -1;
                            return 1;
                        } else {
                            m->row[field] = m->in[field];
                            m->updated_seq_fields[field] = 1;
                        }
                    }
                }
            } else {
                if (agg == PO_AGG_NONE) { memset(&m->row[i], 0, sizeof(po_val)); m->row[i].is_null = 1; }
                else {
                    po_val out, acc = m->row[i];
                    if (agg_retract(m, i, agg, &acc, &m->in[i], &out)) return -1;
                    m->row[i] = out;
                }
            }
        } else if (agg != PO_AGG_NONE) {
            po_val out, acc = m->row[i];
            if (agg_retract(m, i, agg, &acc, &m->in[i], &out)) return -1;
            m->row[i] = out;
        }
    }
    return 0;
}

static int mf_add(mf_t *m, kvref kv) {
    const ctx_t *c = m->c;
    const po_spec *sp = c->spec;
    int8_t kind = kv_kind(c, kv);
    switch (sp->engine) {
        case PO_ENGINE_DEDUPLICATE:                       /* DeduplicateMergeFunction.java:47-55 */
            if (sp->ignore_delete && is_retract(kind)) return 0;
            m->latest = kv;
            return 0;
        case PO_ENGINE_FIRST_ROW:                         /* FirstRowMergeFunction.java:50-69 */
            if (is_retract(kind)) {
                if (sp->ignore_delete) return 0;
                return fail("By default, First row merge engine can not accept DELETE/UPDATE_BEFORE records.\n"
                            "You can config 'ignore-delete' to ignore the DELETE/UPDATE_BEFORE records.");
            }
            if (m->latest.run < 0) m->latest = kv;
            return 0;
        case PO_ENGINE_PARTIAL_UPDATE: {                  /* PartialUpdateMergeFunction.java:121-175 */
            m->current_key = kv;
            m->current_delete_row = 0;
            load_value_row(m, kv);
            if (is_retract(kind)) {
                if (!m->not_null_column_filled) {
                    if (init_row(m, m->row, m->in)) return -1;
                    m->not_null_column_filled = 1;
                }
                if (sp->ignore_delete) return 0;
                m->latest_seq = kv_seq(c, kv);
                if (sp->n_groups > 0) {                   /* fieldSequenceEnabled */
                    int r = pu_retract_with_sequence_group(m, kv);
                    return r < 0 ? -1 : 0;
                }
                if (sp->remove_record_on_delete) {
                    if (kind == PO_DELETE) {
                        m->current_delete_row = 1;
                        row_clear(c, m->row);
                        if (init_row(m, m->row, m->in)) return -1;
                    }
                    return 0;
                }
                return fail("By default, Partial update can not accept delete records, you can choose one of "
                            "the following solutions:\n1. Configure 'ignore-delete' to ignore delete records.\n"
                            "2. Configure 'partial-update.remove-record-on-delete' to remove the whole row when "
                            "receiving delete records.\n3. Configure 'sequence-group's to retract partial columns. "
                            "Also configure 'partial-update.remove-record-on-sequence-group' to remove the whole "
                            "row when receiving deleted records of `specified sequence group`.");
            }
            m->latest_seq = kv_seq(c, kv);
            if (sp->n_groups == 0) {                      /* updateNonNullFields :177-188 */
                for (int i = 0; i < c->s->n_val; i++) {
                    if (!m->in[i].is_null) m->row[i] = m->in[i];
                    else if (!c->s->val_nullable[i]) return fail("Field can not be null");
                }
            } else {
                if (pu_update_with_sequence_group(m)) return -1;
            }
            m->meet_insert = 1;
            m->not_null_column_filled = 1;
            return 0;
        }
        case PO_ENGINE_AGGREGATE: {                       /* AggregateMergeFunction.java:80-102 */
            m->current_key = kv;                           /* latestKv */
            load_value_row(m, kv);
            m->current_delete_row = sp->remove_record_on_delete && kind == PO_DELETE;
            if (m->current_delete_row) {
                row_clear(c, m->row);
                return init_row(m, m->row, m->in);
            }
            int retract = is_retract(kind);
            for (int i = 0; i < c->s->n_val; i++) {
                po_val acc = m->row[i], out;
                int r = retract ? agg_retract(m, i, sp->agg[i], &acc, &m->in[i], &out)
                                : agg_apply(m, i, sp->agg[i], &acc, &m->in[i], &out);
                if (r) return -1;
                m->row[i] = out;
            }
            return 0;
        }
    }
    return fail("unknown engine");
}

static void mf_get_result(mf_t *m, result_t *r) {
    const po_spec *sp = m->c->spec;
    memset(r, 0, sizeof(*r));
    switch (sp->engine) {
        case PO_ENGINE_DEDUPLICATE:
        case PO_ENGINE_FIRST_ROW:
            if (m->latest.run < 0) { r->kind = RES_NULL; return; }
            r->kind = RES_REF; r->ref = m->latest;
            return;
        case PO_ENGINE_PARTIAL_UPDATE:                    /* :354-362 */
            r->kind = RES_ROW; r->ref = m->current_key; r->seq = m->latest_seq;
            r->value_kind = (m->current_delete_row || !m->meet_insert) ? PO_DELETE : PO_INSERT;
            r->row = m->row;
            return;
        case PO_ENGINE_AGGREGATE:                         /* :114-125 */
            r->kind = RES_ROW; r->ref = m->current_key; r->seq = kv_seq(m->c, m->current_key);
            r->value_kind = m->current_delete_row ? PO_DELETE : PO_INSERT;
            r->row = m->row;
            return;
    }
}

/* ReducerMergeFunctionWrapper.java:45-73 */
typedef struct {
    mf_t *mf;
    kvref initial_kv;
    int is_initialized;
    int bypass;         /* test hook, see po_spec.bypass_wrapper */
} wrapper_t;

static void wr_reset(wrapper_t *w) {
    w->initial_kv.run = -1;
    mf_reset(w->mf);
    w->is_initialized = 0;
}
static int wr_add(wrapper_t *w, kvref kv) {
    if (w->bypass) {
        w->initial_kv = kv;
        w->is_initialized = 1;
        return mf_add(w->mf, kv);
    }
    if (w->initial_kv.run < 0) {
        w->initial_kv = kv;
    } else {
        if (!w->is_initialized) {
            if (mf_add(w->mf, w->initial_kv)) return -1;
            w->is_initialized = 1;
        }
        if (mf_add(w->mf, kv)) return -1;
    }
    return 0;
}
static void wr_get_result(wrapper_t *w, result_t *r) {
    if (w->is_initialized) { mf_get_result(w->mf, r); return; }
    memset(r, 0, sizeof(*r));
    r->kind = RES_REF; r->ref = w->initial_kv;
}

/* ------------------------------------------------------------- output */

typedef struct { uint8_t *p; int64_t len, cap; } buf_t;
static void buf_reserve(buf_t *b, int64_t extra) {
    if (b->len + extra > b->cap) {
        int64_t nc = b->cap ? b->cap * 2 : 4096;
        while (nc < b->len + extra) nc *= 2;
        if (b->p == NULL) {
            b->p = (uint8_t *)calloc(1, (size_t)nc);          /* lazily zeroed pages */
        } else {
            b->p = (uint8_t *)realloc(b->p, (size_t)nc);
            memset(b->p + b->cap, 0, (size_t)(nc - b->cap));
        }
        b->cap = nc;
    }
}
static void buf_append(buf_t *b, const void *src, int64_t n) {
    buf_reserve(b, n);
    if (n) memcpy(b->p + b->len, src, (size_t)n);
    b->len += n;
}

typedef struct {
    const ctx_t *c;
    int ncols;
    int64_t n_rows;
    buf_t *data, *offsets, *valid;
} writer_t;

static int col_type(const ctx_t *c, int col) {
    if (col < c->s->n_key) return c->s->key_types[col];
    if (col == c->s->n_key) return PO_INT64;
    if (col == c->s->n_key + 1) return PO_INT8;
    return c->s->val_types[col - c->s->n_key - 2];
}

static writer_t *wr_new(const ctx_t *c) {
    writer_t *w = (writer_t *)calloc(1, sizeof(*w));
    w->c = c;
    w->ncols = c->s->n_key + 2 + c->s->n_val;
    w->data = (buf_t *)calloc(w->ncols, sizeof(buf_t));
    w->offsets = (buf_t *)calloc(w->ncols, sizeof(buf_t));
    w->valid = (buf_t *)calloc(w->ncols, sizeof(buf_t));
    /* size every output buffer for the worst case (all input rows survive) up front: a growing realloc
     * per column makes many-thread runs serialise in the kernel's mmap path, which would understate the
     * CPU baseline */
    int64_t n_in = 0;
    for (int r = 0; r < c->k; r++) n_in += c->runs[r].n_rows;
    for (int i = 0; i < w->ncols; i++) {
        int t = col_type(c, i);
        if (is_varlen(t)) {
            int64_t bytes = 0;
            for (int r = 0; r < c->k; r++)
                if (c->runs[r].n_rows > 0) bytes += c->runs[r].cols[i].offsets[c->runs[r].n_rows];
            buf_reserve(&w->data[i], bytes + 16);
            buf_reserve(&w->offsets[i], 4 * (n_in + 1) + 16);
        } else {
            buf_reserve(&w->data[i], n_in * type_width(t) + 16);
        }
        buf_reserve(&w->valid[i], n_in / 8 + 16);
    }
    int32_t zero = 0;
    for (int i = 0; i < w->ncols; i++)
        if (is_varlen(col_type(c, i))) buf_append(&w->offsets[i], &zero, 4);
    return w;
}

static void wr_put(writer_t *w, int col, const po_val *v) {
    int t = col_type(w->c, col);
    int64_t r = w->n_rows;
    buf_t *vb = &w->valid[col];
    if ((r >> 3) >= vb->len) { uint8_t z = 0; buf_append(vb, &z, 1); }
    if (!v->is_null) vb->p[r >> 3] |= (uint8_t)(1u << (r & 7));
    if (is_varlen(t)) {
        if (!v->is_null) buf_append(&w->data[col], v->p, v->len);
        int32_t off = (int32_t)w->data[col].len;
        buf_append(&w->offsets[col], &off, 4);
    } else {
        int wd = type_width(t);
        uint8_t tmp[8] = {0};
        if (!v->is_null) {
            switch (t) {
                case PO_INT8: case PO_BOOL: { int8_t x = (int8_t)v->v.i; memcpy(tmp, &x, 1); break; }
                case PO_INT16: { int16_t x = (int16_t)v->v.i; memcpy(tmp, &x, 2); break; }
                case PO_INT32: { int32_t x = (int32_t)v->v.i; memcpy(tmp, &x, 4); break; }
                case PO_INT64: memcpy(tmp, &v->v.i, 8); break;
                case PO_FLOAT: memcpy(tmp, &v->v.f, 4); break;
                case PO_DOUBLE: memcpy(tmp, &v->v.d, 8); break;
            }
        }
        buf_append(&w->data[col], tmp, wd);
    }
}

static void wr_emit(writer_t *w, const result_t *r) {
    const ctx_t *c = w->c;
    int nk = c->s->n_key;
    for (int f = 0; f < nk; f++) {
        po_val v = read_val(c->s->key_types[f], key_col(c, r->ref, f), r->ref.row);
        wr_put(w, f, &v);
    }
    po_val seq, kind;
    memset(&seq, 0, sizeof(seq)); memset(&kind, 0, sizeof(kind));
    if (r->kind == RES_REF) { seq.v.i = kv_seq(c, r->ref); kind.v.i = kv_kind(c, r->ref); }
    else { seq.v.i = r->seq; kind.v.i = r->value_kind; }
    wr_put(w, nk, &seq);
    wr_put(w, nk + 1, &kind);
    for (int f = 0; f < c->s->n_val; f++) {
        po_val v = r->kind == RES_REF ? kv_value(c, r->ref, f) : r->row[f];
        wr_put(w, nk + 2 + f, &v);
    }
    w->n_rows++;
}

static po_result *wr_finish(writer_t *w) {
    po_result *res = (po_result *)calloc(1, sizeof(*res));
    res->n_rows = w->n_rows;
    res->n_cols = w->ncols;
    res->cols = (po_out_col *)calloc(w->ncols, sizeof(po_out_col));
    for (int i = 0; i < w->ncols; i++) {
        buf_reserve(&w->data[i], 8);
        buf_reserve(&w->valid[i], 8);
        res->cols[i].data = w->data[i].p;
        res->cols[i].data_bytes = w->data[i].len;
        res->cols[i].offsets = (int32_t *)w->offsets[i].p;
        res->cols[i].valid = w->valid[i].p;
    }
    free(w->data); free(w->offsets); free(w->valid); free(w);
    return res;
}
static void wr_abort(writer_t *w) {
    for (int i = 0; i < w->ncols; i++) { free(w->data[i].p); free(w->offsets[i].p); free(w->valid[i].p); }
    free(w->data); free(w->offsets); free(w->valid); free(w);
}

void po_result_free(po_result *r) {
    if (!r) return;
    for (int i = 0; i < r->n_cols; i++) { free(r->cols[i].data); free(r->cols[i].offsets); free(r->cols[i].valid); }
    free(r->cols);
    free(r);
}

/* result filter: SortMergeReaderWithLoserTree.java:97-100 (null result => key emits nothing)
 * followed by DropDeleteReader.java:50-68 */
static void emit_filtered(writer_t *w, const result_t *r) {
    if (r->kind == RES_NULL) return;
    if (w->c->spec->drop_delete) {
        int8_t kind = r->kind == RES_REF ? kv_kind(w->c, r->ref) : r->value_kind;
        if (is_retract(kind)) return;      /* !kv.isAdd() */
    }
    wr_emit(w, r);
}

/* ------------------------------------------------------------- drivers */

static mf_t *mf_new(const ctx_t *c) {
    mf_t *m = (mf_t *)calloc(1, sizeof(*m));
    int n = c->s->n_val > 0 ? c->s->n_val : 1;
    m->c = c;
    m->row = (po_val *)calloc(n, sizeof(po_val));
    m->in = (po_val *)calloc(n, sizeof(po_val));
    m->agg_initialized = (uint8_t *)calloc(n, 1);
    m->empty_group = (uint8_t *)calloc(n, 1);
    m->updated_seq_fields = (uint8_t *)calloc(n, 1);
    return m;
}
static void mf_free(mf_t *m) {
    free(m->row); free(m->in); free(m->agg_initialized); free(m->empty_group);
    free(m->updated_seq_fields); free(m);
}

/* SortMergeReaderWithLoserTree.SortMergeIterator.next / merge :87-112 */
static int run_loser_tree(const ctx_t *c, writer_t *w, wrapper_t *wrap) {
    loser_tree *t = lt_new(c);
    int rc = 0;
    lt_initialize_if_needed(t);
    if (c->k > 0) {
        while (1) {
            lt_adjust_for_next_loop(t);
            kvref winner = lt_pop_winner(t);
            if (winner.run < 0) break;
            wr_reset(wrap);
            if (wr_add(wrap, winner)) { rc = -1; break; }
            while (lt_peek_winner(t).run >= 0) {
                if (wr_add(wrap, lt_pop_winner(t))) { rc = -1; break; }
            }
            if (rc) break;
            result_t r;
            wr_get_result(wrap, &r);
            emit_filtered(w, &r);
        }
    }
    if (t->bug && !rc) rc = fail("LoserTree reached a 'This is a bug' branch");
    lt_free(t);
    return rc;
}

/* binary min-heap of (run,row) on cmp_full, then by run index to make ties deterministic */
typedef struct { const ctx_t *c; kvref *a; int n; } heap_t;
static int heap_less(const heap_t *h, kvref x, kvref y) {
    int d = cmp_full(h->c, x, y);
    if (d != 0) return d < 0;
    return x.run < y.run;
}
static void heap_push(heap_t *h, kvref x) {
    int i = h->n++;
    h->a[i] = x;
    while (i > 0) {
        int p = (i - 1) / 2;
        if (!heap_less(h, h->a[i], h->a[p])) break;
        kvref t = h->a[i]; h->a[i] = h->a[p]; h->a[p] = t;
        i = p;
    }
}
static kvref heap_pop(heap_t *h) {
    kvref top = h->a[0];
    h->a[0] = h->a[--h->n];
    int i = 0;
    while (1) {
        int l = 2 * i + 1, r = l + 1, m = i;
        if (l < h->n && heap_less(h, h->a[l], h->a[m])) m = l;
        if (r < h->n && heap_less(h, h->a[r], h->a[m])) m = r;
        if (m == i) break;
        kvref t = h->a[i]; h->a[i] = h->a[m]; h->a[m] = t;
        i = m;
    }
    return top;
}

/* SortMergeReaderWithMinHeap.SortMergeIterator.nextImpl :135-179 (single batch per run) */
static int run_min_heap(const ctx_t *c, writer_t *w, wrapper_t *wrap) {
    heap_t h;
    h.c = c; h.n = 0;
    h.a = (kvref *)calloc(c->k > 0 ? c->k : 1, sizeof(kvref));
    kvref *polled = (kvref *)calloc(c->k > 0 ? c->k : 1, sizeof(kvref));
    int n_polled = 0, rc = 0;
    for (int r = 0; r < c->k; r++)
        if (c->runs[r].n_rows > 0) { kvref kv = { r, 0 }; heap_push(&h, kv); }
    while (1) {
        for (int i = 0; i < n_polled; i++) {          /* add polled elements back */
            kvref kv = polled[i];
            if (kv.row + 1 < c->runs[kv.run].n_rows) { kv.row++; heap_push(&h, kv); }
        }
        n_polled = 0;
        if (h.n == 0) break;
        wr_reset(wrap);
        kvref key = h.a[0];
        while (h.n > 0) {
            kvref e = h.a[0];
            if (cmp_key(c, key, e) != 0) break;
            heap_pop(&h);
            if (wr_add(wrap, e)) { rc = -1; break; }
            polled[n_polled++] = e;
        }
        if (rc) break;
        result_t r;
        wr_get_result(wrap, &r);
        emit_filtered(w, &r);
    }
    free(h.a); free(polled);
    return rc;
}

/* brute force: concatenate, sort by (key,[seq fields],seq), fold per key —
 * legitimised by MergeFunctionTestUtils.java:35-150 and LoserTreeTest.java:51-68 */
static __thread const ctx_t *g_sort_ctx;
static int qsort_cmp(const void *a, const void *b) {
    kvref x = *(const kvref *)a, y = *(const kvref *)b;
    int d = cmp_full(g_sort_ctx, x, y);
    if (d != 0) return d;
    return x.run < y.run ? -1 : x.run > y.run ? 1 : 0;
}
static int run_brute_force(const ctx_t *c, writer_t *w, wrapper_t *wrap) {
    int64_t n = 0;
    for (int r = 0; r < c->k; r++) n += c->runs[r].n_rows;
    kvref *all = (kvref *)malloc((size_t)(n > 0 ? n : 1) * sizeof(kvref));
    int64_t p = 0;
    for (int r = 0; r < c->k; r++)
        for (int64_t i = 0; i < c->runs[r].n_rows; i++) { all[p].run = r; all[p].row = i; p++; }
    g_sort_ctx = c;
    qsort(all, (size_t)n, sizeof(kvref), qsort_cmp);
    int rc = 0;
    int64_t i = 0;
    while (i < n && !rc) {
        int64_t j = i;
        wr_reset(wrap);
        while (j < n && cmp_key(c, all[i], all[j]) == 0) {
            if (wr_add(wrap, all[j])) { rc = -1; break; }
            j++;
        }
        if (rc) break;
        result_t r;
        wr_get_result(wrap, &r);
        emit_filtered(w, &r);
        i = j;
    }
    free(all);
    return rc;
}

int po_merge(const po_schema *schema, const po_spec *spec, int32_t k, const po_run *runs,
             po_result **out) {
    ctx_t c = { schema, spec, k, runs };
    g_err[0] = 0;
    *out = NULL;
    writer_t *w = wr_new(&c);
    mf_t *mf = mf_new(&c);
    wrapper_t wrap = { mf, { -1, 0 }, 0, spec->bypass_wrapper };
    int rc;
    switch (spec->sort_engine) {
        case PO_SORT_LOSER_TREE: rc = run_loser_tree(&c, w, &wrap); break;
        case PO_SORT_MIN_HEAP: rc = run_min_heap(&c, w, &wrap); break;
        case PO_SORT_BRUTE_FORCE: rc = run_brute_force(&c, w, &wrap); break;
        default: rc = fail("unknown sort engine");
    }
    mf_free(mf);
    if (rc) { wr_abort(w); return rc; }
    *out = wr_finish(w);
    return 0;
}

int po_merge_order(const po_schema *schema, const po_spec *spec, int32_t k, const po_run *runs,
                   int32_t *out_run, int64_t *out_row, int64_t *out_n) {
    ctx_t c = { schema, spec, k, runs };
    int64_t n = 0;
    g_err[0] = 0;
    if (spec->sort_engine == PO_SORT_LOSER_TREE) {
        /* LoserTreeTest.java:95-110: adjustForNextLoop; pop until null */
        loser_tree *t = lt_new(&c);
        lt_initialize_if_needed(t);
        while (k > 0) {
            lt_adjust_for_next_loop(t);
            kvref wkv = lt_pop_winner(t);
            if (wkv.run < 0) break;
            out_run[n] = wkv.run; out_row[n] = wkv.row; n++;
            while (lt_peek_winner(t).run >= 0) {
                wkv = lt_pop_winner(t);
                out_run[n] = wkv.run; out_row[n] = wkv.row; n++;
            }
        }
        int bug = t->bug;
        lt_free(t);
        if (bug) return fail("LoserTree reached a 'This is a bug' branch");
    } else {
        heap_t h;
        h.c = &c; h.n = 0;
        h.a = (kvref *)calloc(k > 0 ? k : 1, sizeof(kvref));
        for (int r = 0; r < k; r++)
            if (runs[r].n_rows > 0) { kvref kv = { r, 0 }; heap_push(&h, kv); }
        while (h.n > 0) {
            kvref e = heap_pop(&h);
            out_run[n] = e.run; out_row[n] = e.row; n++;
            if (e.row + 1 < runs[e.run].n_rows) { e.row++; heap_push(&h, e); }
        }
        free(h.a);
    }
    *out_n = n;
    return 0;
}

/* ------------------------------------------------------ IntervalPartition */

typedef struct { int64_t mn, mx; int32_t idx; } fmeta;
static int fmeta_cmp(const void *a, const void *b) {                 /* IntervalPartition.java:40-46 */
    const fmeta *x = (const fmeta *)a, *y = (const fmeta *)b;
    if (x->mn != y->mn) return x->mn < y->mn ? -1 : 1;
    if (x->mx != y->mx) return x->mx < y->mx ? -1 : 1;
    return x->idx < y->idx ? -1 : x->idx > y->idx ? 1 : 0;           /* List.sort is stable */
}

/* partition(List<DataFileMeta>) :95-124 — greedy: the run with the smallest last-maxKey takes the
 * file if it does not overlap, else a new run is opened */
static void partition_section(const fmeta *files, int n, int section, int32_t *section_of, int32_t *run_of) {
    int64_t *run_max = (int64_t *)malloc((size_t)n * sizeof(int64_t));
    int n_runs = 0;
    for (int i = 0; i < n; i++) {
        int best = -1;
        for (int r = 0; r < n_runs; r++)
            if (best < 0 || run_max[r] < run_max[best]) best = r;   /* queue.poll(): smallest max key */
        if (i > 0 && files[i].mn > run_max[best]) {
            run_max[best] = files[i].mx;
            run_of[files[i].idx] = best;
        } else {
            run_max[n_runs] = files[i].mx;
            run_of[files[i].idx] = n_runs++;
        }
        section_of[files[i].idx] = section;
    }
    free(run_max);
}

int po_interval_partition(int32_t n_files, const int64_t *min_key, const int64_t *max_key,
                          int32_t *section_of, int32_t *run_of, int32_t *n_sections) {
    fmeta *files = (fmeta *)malloc((size_t)(n_files > 0 ? n_files : 1) * sizeof(fmeta));
    for (int i = 0; i < n_files; i++) { files[i].mn = min_key[i]; files[i].mx = max_key[i]; files[i].idx = i; }
    qsort(files, (size_t)n_files, sizeof(fmeta), fmeta_cmp);
    int sections = 0, start = 0, have_bound = 0;
    int64_t bound = 0;
    for (int i = 0; i < n_files; i++) {                              /* partition() :67-93 */
        if (i > start && files[i].mn > bound) {
            partition_section(files + start, i - start, sections++, section_of, run_of);
            start = i;
            have_bound = 0;
        }
        if (!have_bound || files[i].mx > bound) { bound = files[i].mx; have_bound = 1; }
    }
    if (n_files > start) partition_section(files + start, n_files - start, sections++, section_of, run_of);
    *n_sections = sections;
    free(files);
    return 0;
}
