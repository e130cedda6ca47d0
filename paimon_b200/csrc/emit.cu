// emit.cu — the dominant kernel of the merge: per tile and column, stage the k run segments into
// shared memory with 1-D bulk async copies (TMA, cp.async.bulk + mbarrier), resolve every output row
// from its key group's members (select / fold per the plan's op codes), and store the result column
// coalesced.  All random access happens in shared memory; global memory only sees contiguous streams.
//
// Replaces, per output row and column, MergeFunction.add()/getResult() of the reference:
//   DeduplicateMergeFunction.java:47-60, PartialUpdateMergeFunction.java:177-188 (updateNonNullFields),
//   aggregate/AggregateMergeFunction.java:91-101 + FieldAggregator implementations.
//
// Pipeline per CTA (one tile): column c+1's segments are in flight (async proxy) while column c is being
// resolved from the other stage; validity words of column c+1 are prefetched into registers.
// Var-len columns get their output byte offsets from a decoupled look-back over tiles (tiles are taken
// in ticket order), so no second pass over the data is needed to size them.
//
// Round 2 measured four restructurings of this kernel against it on the same box (profiles/experiments/README.md):
// a size pass + copy pass per var-len column with full / empty mbarriers instead of block barriers, a ballot-based
// bitmap select, a single-winner path for deduplicate, deeper payload gathers and an L2 prefetch of the payload.  All
// lost on C3.  What did help: pointers to the staged data are computed from the shared-memory
// symbol at every use (picked out of a local array they became generic loads through L1TEX), global stores /
// loads are marked global, the tile prologue loads its run bounds with one lane per run, and the pass descriptors
// (column, ColDesc, output buffers) are staged in shared memory once per tile instead of being read from the device
// tables at the top of every pass (two dependent global round trips in front of all 16 warps).
#include <stdio.h>

#include "device_utils.cuh"

namespace pg {

constexpr int kStages = 2;
constexpr int kEmitThreads = 512;
constexpr int kEmitWarps = kEmitThreads / 32;
#define kFlagAgg (1ull << 62)
#define kFlagPrefix (2ull << 62)
#define kValMask ((1ull << 62) - 1)

// per merged position: staged row position (13 bits) | op (2 bits) | first-member-of-group (1 bit)
constexpr uint32_t kPmPosMask = 0x1FFF;
constexpr int kPmOpShift = 13;
constexpr uint32_t kPmHead = 0x8000;

struct EmitLayout {
    int rt;              // staged rows capacity per stage (multiple of 32)
    size_t stage_bytes;
    size_t total;
};
__host__ __device__ inline EmitLayout emit_layout(int k) {
    EmitLayout L;
    L.rt = kTileMax + 64 * k;
    L.stage_bytes = (((size_t)L.rt * 8 + (size_t)L.rt / 32 * 4) + 127) & ~(size_t)127;
    L.total = kStages * L.stage_bytes + (size_t)kTileMax * (2 + 2 + 1) + (PG_MAX_RUNS + 1) * 4 * 3 +
              PG_MAX_RUNS * 8 + kStages * PG_MAX_RUNS * 8 + kStages * 8 + 34 * 4 + 64;
    return L;
}

__device__ __forceinline__ bool staged_valid(const uint32_t *vw, int p) { return (vw[p >> 5] >> (p & 31)) & 1; }

template <int W> __device__ __forceinline__ uint64_t lds_fixed(const unsigned char *vals, int p);
template <> __device__ __forceinline__ uint64_t lds_fixed<1>(const unsigned char *v, int p) { return v[p]; }
template <> __device__ __forceinline__ uint64_t lds_fixed<2>(const unsigned char *v, int p) { return ((const uint16_t *)v)[p]; }
template <> __device__ __forceinline__ uint64_t lds_fixed<4>(const unsigned char *v, int p) { return ((const uint32_t *)v)[p]; }
template <> __device__ __forceinline__ uint64_t lds_fixed<8>(const unsigned char *v, int p) { return ((const uint64_t *)v)[p]; }
// output / run column pointers come out of device tables as generic pointers: tell the compiler they are global
// (STG / LDG instead of generic ST / LD).  Only for non-null pointers.
template <typename T> __device__ __forceinline__ T *as_global(T *p) { __builtin_assume(__isGlobal(p)); return p; }
template <int W> __device__ __forceinline__ void stg_fixed(void *d, int64_t row, uint64_t v);
template <> __device__ __forceinline__ void stg_fixed<1>(void *d, int64_t r, uint64_t v) { as_global((uint8_t *)d)[r] = (uint8_t)v; }
template <> __device__ __forceinline__ void stg_fixed<2>(void *d, int64_t r, uint64_t v) { as_global((uint16_t *)d)[r] = (uint16_t)v; }
template <> __device__ __forceinline__ void stg_fixed<4>(void *d, int64_t r, uint64_t v) { as_global((uint32_t *)d)[r] = (uint32_t)v; }
template <> __device__ __forceinline__ void stg_fixed<8>(void *d, int64_t r, uint64_t v) { as_global((uint64_t *)d)[r] = v; }

// ops-based select, newest member first: the newest UPD member with a non-null cell wins; a SET member
// ends the scan (its cell, null or not, is the result).  Returns the staged position or -1 (NULL).
template <bool GAGG>
__device__ __forceinline__ int select_pos(const uint16_t *pm, const uint32_t *vw, int last) {
    int j = last;
    while (true) {
        uint32_t e = pm[j];
        uint32_t op = (e >> kPmOpShift) & 3;
        // (only with aggregates inside sequence groups does the plan mark retracts on a partial-update merge) a
        // RETRACT member leaves select columns alone, unless it is the group's first record (initRow: verbatim)
        if (GAGG && op == OP_RETRACT) op = (e & kPmHead) ? OP_SET : OP_NOOP;
        if (op != OP_NOOP) {
            int pj = e & kPmPosMask;
            if (staged_valid(vw, pj)) return pj;
            if (op == OP_SET) return -1;
        }
        if (e & kPmHead) return -1;
        --j;
    }
}
// same, but returns the member's merged position (needed for its run id)
template <bool GAGG>
__device__ __forceinline__ int select_member_idx(const uint16_t *pm, const uint32_t *vw, int last) {
    int j = last;
    while (true) {
        uint32_t e = pm[j];
        uint32_t op = (e >> kPmOpShift) & 3;
        if (GAGG && op == OP_RETRACT) op = (e & kPmHead) ? OP_SET : OP_NOOP;
        if (op != OP_NOOP) {
            if (staged_valid(vw, e & kPmPosMask)) return j;
            if (op == OP_SET) return -1;
        }
        if (e & kPmHead) return -1;
        --j;
    }
}

// partial-update sequence group column: the member the plan kernel marked (merged position), or -1
__device__ __forceinline__ int select_marked_idx(const uint16_t *pm, const uint32_t *gplan, uint32_t bit, int last) {
    int j = last;
    while (true) {
        if (gplan[j] & bit) return j;
        if (pm[j] & kPmHead) return -1;
        --j;
    }
}

__device__ __forceinline__ int group_first(const uint16_t *pm, int last) {
    int j = last;
    while (!(pm[j] & kPmHead)) --j;
    return j;
}

// aggregate engine on a var-len column: fold with the member index as accumulator
__device__ int fold_member_idx(const ColDesc &cd, const uint16_t *pm, const uint8_t *mrun, const uint32_t *vw,
                               const int32_t *offs, const uint8_t *const *cdata, int last, int32_t *err) {
    int acc = -1;
    bool initialized = false;
    for (int j = group_first(pm, last); j <= last; j++) {
        uint32_t e = pm[j];
        int op = (e >> kPmOpShift) & 3;
        if (op == OP_NOOP) continue;
        bool v = staged_valid(vw, e & kPmPosMask);
        int in = v ? j : -1;
        if (op == OP_SET) { acc = in; continue; }
        if (op == OP_RETRACT) {
            if (cd.retract == RT_IGNORE) continue;
            switch (cd.agg) {
                case PG_AGG_LAST_VALUE: acc = -1; break;
                case PG_AGG_LAST_NON_NULL_VALUE: if (v) acc = -1; break;
                case PG_AGG_PRIMARY_KEY: acc = in; break;
                default: atomicCAS(err, KERR_NONE, KERR_AGG_RETRACT); break;
            }
            continue;
        }
        switch (cd.agg) {
            case PG_AGG_LAST_VALUE: case PG_AGG_PRIMARY_KEY: acc = in; break;
            case PG_AGG_LAST_NON_NULL_VALUE: if (v) acc = in; break;
            case PG_AGG_FIRST_VALUE: if (!initialized) { initialized = true; acc = in; } break;
            case PG_AGG_FIRST_NON_NULL_VALUE: if (!initialized && v) { initialized = true; acc = in; } break;
            case PG_AGG_MAX: case PG_AGG_MIN:
                if (acc < 0 || in < 0) { if (acc < 0) acc = in; break; }
                {
                    int pa = pm[acc] & kPmPosMask, pb = e & kPmPosMask;
                    int d = bytes_compare(cdata[mrun[acc]] + offs[pa], offs[pa + 1] - offs[pa],
                                          cdata[mrun[j]] + offs[pb], offs[pb + 1] - offs[pb]);
                    if (cd.agg == PG_AGG_MAX) { if (d < 0) acc = in; }
                    else { if (!(d < 0)) acc = in; }
                }
                break;
            default: break;
        }
    }
    return acc;
}

// SUM / PRODUCT step of a fixed-width fold (fn as in arith, 4 = negate a).  Integer and float results are never
// NULL; a DECIMAL one can be (decimal_arith).  DEC = true only inside emit_decimal_column.
template <bool DEC>
__device__ __forceinline__ uint64_t fold_arith(const ColDesc &cd, int fn, uint64_t a, uint64_t b, bool *valid,
                                               int32_t *err) {
    if (DEC) {
        const DecimalResult d = decimal_arith(cd.decimal, fn, a, b, err);
        *valid = d.valid;
        return d.value;
    }
    *valid = true;
    return fn == 4 ? negate_fixed(cd.type, cd.width, a) : arith(cd.type, cd.width, fn, a, b, err);
}

// strict left fold of a fixed-width column in sequence order (AggregateMergeFunction.java:91-101)
template <bool DEC>
__device__ void fold_fixed(const ColDesc &cd, const uint16_t *pm, const uint32_t *vw, const unsigned char *vals,
                           int last, uint64_t *out_val, bool *out_valid, int32_t *err) {
    const int w = cd.width;
    uint64_t val = 0;
    bool is_valid = false, initialized = false;
    for (int j = group_first(pm, last); j <= last; j++) {
        uint32_t e = pm[j];
        int op = (e >> kPmOpShift) & 3;
        if (op == OP_NOOP) continue;
        int pj = e & kPmPosMask;
        bool v = staged_valid(vw, pj);
        uint64_t in = v ? load_fixed(vals, w, pj) : 0;
        if (op == OP_SET) { val = in; is_valid = v; continue; }
        if (op == OP_RETRACT) {
            if (cd.retract == RT_IGNORE) continue;
            switch (cd.agg) {
                case PG_AGG_SUM:       // FieldSumAgg.retract :87-131, negative :133-163
                    if (!is_valid) { if (v) val = fold_arith<DEC>(cd, 4, in, 0, &is_valid, err); }
                    else if (v) val = fold_arith<DEC>(cd, 1, val, in, &is_valid, err);
                    break;
                case PG_AGG_PRODUCT:
                    if (is_valid && v) val = fold_arith<DEC>(cd, 3, val, in, &is_valid, err);
                    break;
                case PG_AGG_LAST_VALUE: is_valid = false; val = 0; break;
                case PG_AGG_LAST_NON_NULL_VALUE: if (v) { is_valid = false; val = 0; } break;
                case PG_AGG_PRIMARY_KEY: val = in; is_valid = v; break;
                default: atomicCAS(err, KERR_NONE, KERR_AGG_RETRACT); break;
            }
            continue;
        }
        switch (cd.agg) {
            case PG_AGG_SUM: case PG_AGG_PRODUCT:
                if (!is_valid || !v) { if (!is_valid) { val = in; is_valid = v; } }
                else val = fold_arith<DEC>(cd, cd.agg == PG_AGG_SUM ? 0 : 2, val, in, &is_valid, err);
                break;
            case PG_AGG_MAX: case PG_AGG_MIN:
                if (!is_valid || !v) { if (!is_valid) { val = in; is_valid = v; } }
                else {
                    int d = compare_fixed(cd.type, w, val, in);
                    if (cd.agg == PG_AGG_MAX) { if (d < 0) val = in; }
                    else { if (!(d < 0)) val = in; }
                }
                break;
            case PG_AGG_BOOL_AND: case PG_AGG_BOOL_OR:
                if (!is_valid || !v) { if (!is_valid) { val = in; is_valid = v; } }
                else val = cd.agg == PG_AGG_BOOL_AND ? ((val != 0) && (in != 0)) : ((val != 0) || (in != 0));
                break;
            case PG_AGG_LAST_VALUE: case PG_AGG_PRIMARY_KEY: val = in; is_valid = v; break;
            case PG_AGG_LAST_NON_NULL_VALUE: if (v) { val = in; is_valid = true; } break;
            case PG_AGG_FIRST_VALUE:
                if (!initialized) { initialized = true; val = in; is_valid = v; }
                break;
            case PG_AGG_FIRST_NON_NULL_VALUE:
                if (!initialized && v) { initialized = true; val = in; is_valid = true; }
                break;
            default: break;
        }
    }
    *out_val = val;
    *out_valid = is_valid;
}

// agg(accumulator = a, input = b) of a fixed-width aggregator as a function of both operands, so that
// aggReversed(acc, in) = agg(in, acc) (FieldAggregator.java:40-42) can be evaluated too
template <bool DEC>
__device__ void agg_pair(const ColDesc &cd, uint64_t a, bool av, uint64_t b, bool bv, bool *initialized,
                         uint64_t *out, bool *out_valid, int32_t *err) {
    const int w = cd.width;
    switch (cd.agg) {
        case PG_AGG_SUM: case PG_AGG_PRODUCT:
            if (!av || !bv) { *out = av ? a : b; *out_valid = av || bv; }
            else *out = fold_arith<DEC>(cd, cd.agg == PG_AGG_SUM ? 0 : 2, a, b, out_valid, err);
            return;
        case PG_AGG_MAX: case PG_AGG_MIN:
            if (!av || !bv) { *out = av ? a : b; *out_valid = av || bv; return; }
            {
                const int d = compare_fixed(cd.type, w, a, b);
                const bool take_b = cd.agg == PG_AGG_MAX ? d < 0 : !(d < 0);
                *out = take_b ? b : a; *out_valid = true;
            }
            return;
        case PG_AGG_BOOL_AND: case PG_AGG_BOOL_OR:
            if (!av || !bv) { *out = av ? a : b; *out_valid = av || bv; return; }
            *out = cd.agg == PG_AGG_BOOL_AND ? ((a != 0) && (b != 0)) : ((a != 0) || (b != 0));
            *out_valid = true;
            return;
        case PG_AGG_LAST_VALUE: case PG_AGG_PRIMARY_KEY: *out = b; *out_valid = bv; return;
        case PG_AGG_LAST_NON_NULL_VALUE: *out = bv ? b : a; *out_valid = bv ? true : av; return;
        case PG_AGG_FIRST_VALUE:
            if (!*initialized) { *initialized = true; *out = b; *out_valid = bv; }
            else { *out = a; *out_valid = av; }
            return;
        case PG_AGG_FIRST_NON_NULL_VALUE:
            if (!*initialized && bv) { *initialized = true; *out = b; *out_valid = true; }
            else { *out = a; *out_valid = av; }
            return;
        default: *out = a; *out_valid = av; return;
    }
}

// Field of a partial-update sequence group that has an aggregate function
// (PartialUpdateMergeFunction.updateWithSequenceGroup :228-244, retractWithSequenceGroup :323-339): every member
// whose group is not empty takes part — in order (agg) when its group sequence is >= the accumulated one, else
// reversed (aggReversed); retract members call retract(); the first record of a key initialises the row.
template <bool DEC>
__device__ void fold_group_agg(const ColDesc &cd, const uint16_t *pm, const uint32_t *gagg, const uint32_t *vw,
                               const unsigned char *vals, int last, uint64_t *out_val, bool *out_valid, int32_t *err) {
    const int w = cd.width, g = cd.group;
    uint64_t val = 0;
    bool is_valid = false, initialized = false;
    for (int j = group_first(pm, last); j <= last; j++) {
        const uint32_t e = pm[j];
        const int op = (e >> kPmOpShift) & 3;
        if (op == OP_NOOP) continue;
        const int pj = e & kPmPosMask;
        const bool v = staged_valid(vw, pj);
        const uint64_t in = v ? load_fixed(vals, w, pj) : 0;
        if (op == OP_SET) { val = in; is_valid = v; continue; }            // initRow / row restart: verbatim
        const uint32_t marks = gagg[j];
        if (op == OP_RETRACT) {
            if (e & kPmHead) { val = in; is_valid = v; }                    // initRow, then the retract itself
            if (!((marks >> g) & 1) || cd.retract == RT_IGNORE) continue;
            switch (cd.agg) {
                case PG_AGG_SUM:
                    if (!is_valid) { if (v) val = fold_arith<DEC>(cd, 4, in, 0, &is_valid, err); }
                    else if (v) val = fold_arith<DEC>(cd, 1, val, in, &is_valid, err);
                    break;
                case PG_AGG_PRODUCT:
                    if (is_valid && v) val = fold_arith<DEC>(cd, 3, val, in, &is_valid, err);
                    break;
                case PG_AGG_LAST_VALUE: is_valid = false; val = 0; break;
                case PG_AGG_LAST_NON_NULL_VALUE: if (v) { is_valid = false; val = 0; } break;
                case PG_AGG_PRIMARY_KEY: val = in; is_valid = v; break;
                default: atomicCAS(err, KERR_NONE, KERR_AGG_RETRACT); break;
            }
            continue;
        }
        uint64_t r;
        bool rv;
        if ((marks >> g) & 1) agg_pair<DEC>(cd, val, is_valid, in, v, &initialized, &r, &rv, err);
        else if ((marks >> (16 + g)) & 1) agg_pair<DEC>(cd, in, v, val, is_valid, &initialized, &r, &rv, err);
        else continue;                                                       // empty group in this record
        val = rv ? r : 0;
        is_valid = rv;
    }
    *out_val = val;
    *out_valid = is_valid;
}

struct TileView {
    const uint16_t *pm;
    const uint16_t *glast;
    int n_out;
    int o_shift;
    int64_t out_base;
    int64_t in_base;
    int n_out_a;                 // output rows of the first plan tile of the pair
    int seq_shift;               // tmp_seq / tmp_kind are laid out per plan tile: rows of the second one sit
                                 // (n_a - n_out_a) entries further
};
__device__ __forceinline__ int64_t result_index(const TileView &tv, int ob) {
    return tv.in_base + ob + (ob >= tv.n_out_a ? tv.seq_shift : 0);
}

// one output validity word per warp iteration: interior words are plain stores, tile-boundary words OR
__device__ __forceinline__ void put_validity_word(uint8_t *validity, int64_t out_base, int wb, int n_out,
                                                  bool bit) {
    unsigned mask = __ballot_sync(0xffffffffu, bit);
    if ((threadIdx.x & 31) == 0) {
        int64_t word = (out_base + wb) >> 5;
        bool full = wb >= 0 && wb + 32 <= n_out;
        uint32_t *bm = as_global((uint32_t *)validity);
        if (full) bm[word] = mask;
        else if (mask) atomicOr(&bm[word], mask);
    }
}

template <int W, bool GAGG>
__device__ __forceinline__ void emit_fixed_column(const EmitArgs &ea, const ColDesc &cd, const pg_out_column &oc,
                                                  const TileView &tv, const unsigned char *vals, const uint32_t *vw) {
    const int tid = threadIdx.x, lane = tid & 31;
    for (int wb = (tid & ~31) - tv.o_shift; wb < tv.n_out; wb += kEmitThreads) {   // warp-uniform trip count
        const int ob = wb + lane;
        const bool active = ob >= 0 && ob < tv.n_out;
        bool is_valid = false;
        if (active) {
            uint64_t val = 0;
            const int last = tv.glast[ob];
            if (cd.mode == CM_SELECT) {
                int pj = select_pos<GAGG>(tv.pm, vw, last);
                if (pj >= 0) { val = lds_fixed<W>(vals, pj); is_valid = true; }
            } else if (cd.mode == CM_GVAL || cd.mode == CM_GSEQ) {
                const uint32_t gbit = 1u << (cd.agg + (cd.mode == CM_GSEQ ? 16 : 0));
                const int j = select_marked_idx(tv.pm, ea.gplan + tv.in_base, gbit, last);
                if (j >= 0) {
                    const int pj = tv.pm[j] & kPmPosMask;
                    if (staged_valid(vw, pj)) { val = lds_fixed<W>(vals, pj); is_valid = true; }
                }
            } else if (GAGG && cd.mode == CM_GAGG) {
                fold_group_agg<false>(cd, tv.pm, ea.gagg + tv.in_base, vw, vals, last, &val, &is_valid, ea.err);
                if (!is_valid) val = 0;
            } else if (cd.mode == CM_KEY) {
                val = lds_fixed<W>(vals, tv.pm[last] & kPmPosMask); is_valid = true;
            } else if (cd.mode == CM_SEQ) {
                val = (uint64_t)ea.tmp_seq[result_index(tv, ob)]; is_valid = true;
            } else if (cd.mode == CM_KIND) {
                val = (uint8_t)ea.tmp_kind[result_index(tv, ob)]; is_valid = true;
            } else {
                fold_fixed<false>(cd, tv.pm, vw, vals, last, &val, &is_valid, ea.err);
                if (!is_valid) val = 0;
            }
            stg_fixed<W>(oc.data, tv.out_base + ob, val);
        }
        if (oc.validity != nullptr) put_validity_word(oc.validity, tv.out_base, wb, tv.n_out, is_valid);
    }
}

// A DECIMAL sum / product column (CM_FOLD or CM_GAGG, cd.decimal != 0): the same folds with the DECIMAL arithmetic.
// It is its own pass branch (chosen once per column and tile, like the width) so that the common folds carry no
// decimal test in their loops.  Out of line, the call costs the kernel a stack frame and spills in every pass; inlined,
// k_emit<false> keeps 64 registers and 8 bytes of stack (k_emit<true>: 16 -> 24 bytes of stack).
template <bool GAGG>
__device__ __forceinline__ void emit_decimal_column(const ColDesc &cd, const pg_out_column &oc, const TileView &tv,
                                                    const unsigned char *vals, const uint32_t *vw, const uint32_t *gagg,
                                                    int32_t *err) {
    const int tid = threadIdx.x, lane = tid & 31;
    for (int wb = (tid & ~31) - tv.o_shift; wb < tv.n_out; wb += kEmitThreads) {   // warp-uniform trip count
        const int ob = wb + lane;
        bool is_valid = false;
        if (ob >= 0 && ob < tv.n_out) {
            uint64_t val = 0;
            const int last = tv.glast[ob];
            if (GAGG && cd.mode == CM_GAGG) fold_group_agg<true>(cd, tv.pm, gagg, vw, vals, last, &val, &is_valid, err);
            else fold_fixed<true>(cd, tv.pm, vw, vals, last, &val, &is_valid, err);
            stg_fixed<8>(oc.data, tv.out_base + ob, is_valid ? val : 0);
        }
        if (oc.validity != nullptr) put_validity_word(oc.validity, tv.out_base, wb, tv.n_out, is_valid);
    }
}

#ifdef PG_EMIT_TIMING
__device__ long long g_emit_ts[64 * 256];
#define TS(slot) do { if (tid == 0 && ts_on) g_emit_ts[(ts_tile) * 256 + (slot)] = clock64(); } while (0)
#else
#define TS(slot) do { } while (0)
#endif

// GAGG: the merge has aggregate functions inside sequence groups (the fold for them is compiled into its own
// kernel variant: inlined into the common one it costs every workload registers and spills)
struct PassEnt { ColDesc cd; pg_out_column oc; int32_t c, pad; };
constexpr int kPassCache = 64;

template <bool GAGG>
__global__ void __launch_bounds__(kEmitThreads, 2)
k_emit(EmitArgs ea) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ PassEnt s_pass[kPassCache];
    const int k = ea.k, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const EmitLayout L = emit_layout(k);
    auto stage_vals = [&](int s) -> unsigned char * { return smem + (size_t)s * L.stage_bytes; };
    auto stage_vw = [&](int s) -> uint32_t * { return (uint32_t *)(smem + (size_t)s * L.stage_bytes + (size_t)L.rt * 8); };
    unsigned char *p = smem + kStages * L.stage_bytes;
    uint16_t *pm = (uint16_t *)p;              p += kTileMax * 2;
    uint16_t *glast = (uint16_t *)p;           p += kTileMax * 2;   // per output row: last member position
    uint8_t *mrun = (uint8_t *)p;              p += kTileMax;
    int64_t *rstart = (int64_t *)p;            p += PG_MAX_RUNS * 8;
    const uint8_t **cdata = (const uint8_t **)p; p += kStages * PG_MAX_RUNS * 8;   // payload base per run (var-len)
    uint64_t *mbar = (uint64_t *)p;            p += kStages * 8;
    int64_t *s_i64 = (int64_t *)p;             p += 16;
    int *seg = (int *)p;                       p += (PG_MAX_RUNS + 1) * 4;
    int *seg_a = (int *)p;                     p += (PG_MAX_RUNS + 1) * 4;        // first plan tile: slot base per run
    int *rr = (int *)p;                        p += (PG_MAX_RUNS + 1) * 4;         // staged row base per run
    int *ws = (int *)p;                        p += 34 * 4;
    int *s_i32 = (int *)p;                     p += 16;

    // ---- tile ticket (tiles are started in order => look-back never waits on an unscheduled tile)
    if (tid == 0) {
        s_i32[0] = atomicAdd(ea.tile_counter, 1);
        for (int s = 0; s < kStages; s++) mbar_init(&mbar[s], 1);
        mbar_fence_init();
    }
    __syncthreads();
    const int tile = s_i32[0];
    if (tid < ea.n_passes && tid < kPassCache) {
        const int c = ea.col_order[tid];
        s_pass[tid].c = c;
        s_pass[tid].cd = ea.cols[c];
        s_pass[tid].oc = ea.out_cols[c];
    }
#ifdef PG_EMIT_TIMING
    const bool ts_on = tile >= 2000 && tile < 2064;
    const int ts_tile = tile - 2000;
#endif
    TS(0);
    // an emit tile is two consecutive plan tiles (the last one may be single)
    const int plan_a = 2 * tile, plan_end = min(plan_a + 2, ea.n_plan_tiles);
    if (warp == 0) {
        // lane r = run r (its three bounds in flight together); slot / staged-row bases by warp scans
        int64_t b0 = 0, bm = 0, b1 = 0;
        if (lane < k) {
            b0 = ea.bounds[(int64_t)plan_a * k + lane];
            bm = ea.bounds[(int64_t)(plan_a + 1) * k + lane];
            b1 = ea.bounds[(int64_t)plan_end * k + lane];
        }
        const int len = (int)(b1 - b0), len_a = (int)(bm - b0);
        const int rlen = lane < k ? (((int)(b0 & 31) + len + 1) + 31) & ~31 : 0;
        const int i_len = warp_scan_incl(len), i_a = warp_scan_incl(len_a), i_r = warp_scan_incl(rlen);
        if (lane < k) {
            rstart[lane] = b0;
            seg[lane] = i_len - len;
            seg_a[lane] = i_a - len_a;
            rr[lane] = i_r - rlen;
        }
        if (lane == 31) { seg[k] = i_len; seg_a[k] = i_a; rr[k] = i_r; }
    }
    __syncthreads();
    const int n = seg[k];
    const int n_vw = rr[k] >> 5;                       // staged validity words
    int64_t in_base = 0;
    for (int r = 0; r < k; r++) in_base += rstart[r];

    // ---- plan -> (staged position | op | head), output rows
    constexpr int VT = kTileMax / kEmitThreads;
    const int p0 = tid * VT, p1 = min(p0 + VT, n);
    int my = 0;
    uint32_t emit_bits = 0;
    // slot -> (staged position, run) tables, built per run segment (no searches); they live in memory that
    // is not in use yet (glast, stage 1)
    uint16_t *spos = glast;
    uint8_t *srun = stage_vals(1);
    // plan slots are run-major inside their plan tile: table index = slot (first tile) or n_a + slot (second)
    const int n_a = seg_a[k];
    for (int r = 0; r < k; r++) {
        const int len_a = seg_a[r + 1] - seg_a[r], len = seg[r + 1] - seg[r];
        const int p0r = rr[r] + (int)(rstart[r] & 31);                  // staged position of the run's first row
        const int sb0 = n_a + (seg[r] - seg_a[r]);                      // second tile: slot base of run r
        for (int j = tid; j < len; j += kEmitThreads) {
            const int idx = j < len_a ? seg_a[r] + j : sb0 + (j - len_a);
            spos[idx] = (uint16_t)(p0r + j);
            srun[idx] = (uint8_t)r;
        }
    }
    __syncthreads();
    for (int i = p0; i < p1; i++) {
        uint16_t e = ea.plan[in_base + i];
        int slot = (e & kPlanSlotMask) + (i < n_a ? 0 : n_a);
        mrun[i] = srun[slot];
        uint32_t pos = spos[slot];
        uint32_t op = (e >> kPlanOpShift) & 3;
        pm[i] = (uint16_t)(pos | (op << kPmOpShift) | ((e & kPlanHead) ? kPmHead : 0));
        if ((e & kPlanHead) && (e & kPlanEmit)) { my++; emit_bits |= 1u << (i - p0); }
    }
    int n_out = 0;
    int o = block_scan_excl(my, ws, &n_out);          // (syncs: pm is complete afterwards)
    for (int i = p0; i < p1; i++) {
        if (emit_bits & (1u << (i - p0))) {
            int e = i + 1;
            while (e < n && !(pm[e] & kPmHead)) e++;
            glast[o++] = (uint16_t)(e - 1);
        }
    }
    // validity word owned by this thread: (run, global word index), fixed for the whole tile
    int vw_run = -1;
    int64_t vw_gword = 0;
    if (tid < n_vw) {
        int r = 0;
        while (r + 1 < k && (rr[r + 1] >> 5) <= tid) r++;
        vw_run = r;
        vw_gword = (rstart[r] >> 5) + (tid - (rr[r] >> 5));
        if (vw_gword > ((ea.run_rows[r] - 1) >> 5)) vw_run = -1;      // beyond the run's bitmap: never used
    }
    __syncthreads();

    TileView tv;
    tv.pm = pm;
    tv.glast = glast;
    tv.n_out = n_out;
    tv.out_base = ea.row_base[plan_a];
    tv.o_shift = (int)(tv.out_base & 31);
    tv.in_base = in_base;
    tv.n_out_a = ea.tile_rows[plan_a];
    tv.seq_shift = n_a - tv.n_out_a;
    const int ncols = ea.n_passes;
    uint32_t phase = 0;                                // bit s = parity to wait for on stage s

    auto col_staged = [&](const ColDesc &cd) { return cd.mode != CM_SEQ && cd.mode != CM_KIND; };
    // pass descriptors of the tile (column, ColDesc, output buffers) come into shared memory once: read from the device
    // tables at the top of every pass they are two dependent global round trips in front of all 16 warps
    auto pass_col = [&](int ci) -> int { return ci < kPassCache ? s_pass[ci].c : ea.col_order[ci]; };
    auto pass_desc = [&](int ci, int c) -> ColDesc { return ci < kPassCache ? s_pass[ci].cd : ea.cols[c]; };

    // issue the bulk copies of column c into stage s (warp 0; lane r = run r)
    auto issue = [&](int c, const ColDesc &cd, int s) {
        if (!col_staged(cd)) return;
        // the stage was last touched through the generic proxy (scratch + validity words)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        uint32_t bytes = 0;
        const unsigned char *src = nullptr;
        unsigned char *dst = nullptr;
        if (lane < k) {
            const int r = lane;
            const int len = seg[r + 1] - seg[r];
            const int64_t row0 = rstart[r] & ~(int64_t)31;
            const int head = (int)(rstart[r] & 31);
            if (cd.width > 0) {
                if (len > 0) {
                    bytes = (uint32_t)(((head + len) * cd.width + 15) & ~15);
                    src = (const unsigned char *)ea.ptrs.data[(int64_t)c * k + r] + row0 * cd.width;
                    dst = stage_vals(s) + (size_t)rr[r] * cd.width;
                }
            } else {
                if (len > 0) {
                    bytes = (uint32_t)(((head + len + 1) * 4 + 15) & ~15);
                    src = (const unsigned char *)(ea.ptrs.offsets[(int64_t)c * k + r] + row0);
                    dst = stage_vals(s) + (size_t)rr[r] * 4;
                }
                cdata[s * PG_MAX_RUNS + r] = (const uint8_t *)ea.ptrs.data[(int64_t)c * k + r];
            }
        }
        uint32_t total = bytes;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) total += __shfl_xor_sync(0xffffffffu, total, d);
        if (lane == 0) mbar_arrive_expect_tx(&mbar[s], total);
        __syncwarp();
        if (bytes) bulk_g2s(dst, src, bytes, &mbar[s]);
    };
    auto load_vw = [&](int c) -> uint32_t {
        if (vw_run < 0) return 0xffffffffu;
        const uint32_t *vp = ea.ptrs.validity[(int64_t)c * k + vw_run];
        return vp ? vp[vw_gword] : 0xffffffffu;
    };

    // ---- prologue: column 0
    // columns are walked in ea.col_order (var-len columns first: their look-back then happens while the
    // CTAs of a wave are still close together in time)
    if (warp == 0 && ncols > 0) issue(pass_col(0), pass_desc(0, pass_col(0)), 0);
    if (tid < n_vw && ncols > 0) stage_vw(0)[tid] = load_vw(pass_col(0));
    __syncthreads();

    TS(1);
    for (int ci = 0; ci < ncols; ci++) {
        const int s = ci & 1;
        const int c = pass_col(ci);
        const int cn = ci + 1 < ncols ? pass_col(ci + 1) : -1;
        const ColDesc cd = pass_desc(ci, c);
        const pg_out_column oc = ci < kPassCache ? s_pass[ci].oc : ea.out_cols[c];
        if (warp == 0 && cn >= 0) issue(cn, pass_desc(ci + 1, cn), s ^ 1);
        uint32_t next_vw = (cn >= 0 && tid < n_vw) ? load_vw(cn) : 0;
        if (col_staged(cd)) {
            mbar_wait(&mbar[s], (phase >> s) & 1);
            phase ^= 1u << s;
        }
        const unsigned char *vals = stage_vals(s);
        const uint32_t *vw = stage_vw(s);

        if (cd.decimal) emit_decimal_column<GAGG>(cd, oc, tv, vals, vw, GAGG ? ea.gagg + tv.in_base : nullptr, ea.err);
        else if (cd.width == 8) emit_fixed_column<8, GAGG>(ea, cd, oc, tv, vals, vw);
        else if (cd.width == 4) emit_fixed_column<4, GAGG>(ea, cd, oc, tv, vals, vw);
        else if (cd.width == 1) emit_fixed_column<1, GAGG>(ea, cd, oc, tv, vals, vw);
        else if (cd.width == 2) emit_fixed_column<2, GAGG>(ea, cd, oc, tv, vals, vw);
        else {
            // ---- var-len column: offsets staged as int32 at the staged row positions; the upper half of the
            // stage is free (offsets are 4 bytes per row) and holds the per-row source + per-warp scratch
            const int32_t *offs = (const int32_t *)vals;
            uint16_t *vsrc = (uint16_t *)(vals + (size_t)L.rt * 4);
            int *wpre = (int *)(vsrc + kTileMax);                                   // per warp: 33 ints
            const uint8_t **wsrc = (const uint8_t **)(wpre + ((kEmitWarps * 33 + 1) & ~1));   // 8-byte aligned
            int *wend = (int *)(wsrc + kEmitWarps * 32);                             // per warp: 32 ints
            int64_t *wtot = (int64_t *)(wend + kEmitWarps * 32);                     // per warp: its byte total
            static_assert(kTileMax * 2 + ((kEmitWarps * 33 + 1) & ~1) * 4 + kEmitWarps * 32 * (8 + 4) + kEmitWarps * 8 <=
                              (kTileMax + 64) * 4, "var-len scratch fits the upper half of a stage at k = 1");
            const uint8_t *const *cd_data = cdata + s * PG_MAX_RUNS;
            // Rows are dealt to warps in contiguous chunks of RW rows (RW a multiple of 32, aligned to the
            // output's 32-row validity words), so that offsets come from warp-level scans and the only
            // block-level steps are one 16-entry scan and the look-back.
            const int span = tv.o_shift + n_out;
            const int RW = (((span + kEmitWarps - 1) / kEmitWarps) + 31) & ~31;
            const int wbeg = -tv.o_shift + warp * RW;
            // pass 1: source member per output row, byte total of this warp's rows.  Every value is below 2 GiB,
            // but a warp's or a tile's rows together need not be: the totals are 64-bit.
            int64_t my_bytes = 0;
            for (int ob0 = wbeg; ob0 < wbeg + RW && ob0 < n_out; ob0 += 32) {
                const int ob = ob0 + lane;
                if (ob >= 0 && ob < n_out) {
                    const int last = glast[ob];
                    int src;
                    if (cd.mode == CM_KEY) src = last;
                    else if (cd.mode == CM_FOLD) src = fold_member_idx(cd, pm, mrun, vw, offs, cd_data, last, ea.err);
                    else if (cd.mode == CM_GVAL || cd.mode == CM_GSEQ) {
                        src = select_marked_idx(pm, ea.gplan + in_base,
                                                1u << (cd.agg + (cd.mode == CM_GSEQ ? 16 : 0)), last);
                        if (src >= 0 && !staged_valid(vw, pm[src] & kPmPosMask)) src = -1;
                    } else src = select_member_idx<GAGG>(pm, vw, last);
                    vsrc[ob] = src < 0 ? (uint16_t)0xFFFF : (uint16_t)src;
                    if (src >= 0) { int ps = pm[src] & kPmPosMask; my_bytes += offs[ps + 1] - offs[ps]; }
                }
            }
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) my_bytes += __shfl_xor_sync(0xffffffffu, my_bytes, d);
            if (lane == 0) wtot[warp] = my_bytes;
            __syncthreads();
            if (ci < 60) TS(8 + 4 * ci + 0);
            // warp 0: exclusive scan of the 16 warp totals + decoupled look-back over earlier tiles
            uint64_t *state = ea.vl_state + (int64_t)cd.varlen_index * ea.n_tiles;
            if (warp == 0) {
                const int64_t x = lane < kEmitWarps ? wtot[lane] : 0;
                int64_t xi = x;
#pragma unroll
                for (int d = 1; d < kEmitWarps; d <<= 1) {
                    const int64_t y = __shfl_up_sync(0xffffffffu, xi, d);
                    if (lane >= d) xi += y;
                }
                const uint64_t tile_bytes = (uint64_t)__shfl_sync(0xffffffffu, xi, kEmitWarps - 1);
                // (only read by pass 2, which runs only when the tile ends below 2 GiB: then these fit in int)
                if (lane < kEmitWarps) ws[lane] = (int)(xi - x);
                uint64_t excl = 0;
                if (lane == 0 && tile > 0) {
                    __threadfence();
                    atomicExch((unsigned long long *)&state[tile], kFlagAgg | (uint64_t)tile_bytes);
                }
                // The CTAs of a wave reach a column at about the same time, so the nearest tile that already knows
                // its prefix is usually a whole wave (~300 tiles) back: every lane looks at kLook consecutive
                // predecessors per step (all loads of a step are independent).
                constexpr int kLook = 8;
                int t = tile - 1;
                while (t >= 0) {
                    uint64_t sv[kLook];
#pragma unroll
                    for (int q = 0; q < kLook; q++) {
                        const int idx = t - (lane * kLook + q);
                        sv[q] = idx >= 0 ? *((volatile uint64_t *)&state[idx]) : kFlagPrefix;
                    }
                    // position p = lane * kLook + q (0 = nearest predecessor): first prefix, nothing unpublished in front
                    int lp = 32 * kLook;
#pragma unroll
                    for (int q = kLook - 1; q >= 0; q--) if ((unsigned)(sv[q] >> 62) == 2) lp = lane * kLook + q;
                    int first = lp;
#pragma unroll
                    for (int d = 16; d > 0; d >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, d));
                    bool inval = false;
                    uint64_t contrib = 0;
#pragma unroll
                    for (int q = 0; q < kLook; q++) {
                        if (lane * kLook + q <= first) {
                            if ((unsigned)(sv[q] >> 62) == 0) inval = true;
                            contrib += sv[q] & kValMask;
                        }
                    }
                    if (__any_sync(0xffffffffu, inval)) continue;      // a needed predecessor has not published yet
#pragma unroll
                    for (int d = 16; d > 0; d >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, d);
                    excl += contrib;
                    if (first < 32 * kLook) break;
                    t -= 32 * kLook;
                }
                if (lane == 0) {
                    __threadfence();
                    const uint64_t tot = excl + tile_bytes;
                    atomicExch((unsigned long long *)&state[tile], kFlagPrefix | tot);
                    // Offsets are int32: a tile that ends past 2 GiB refuses the batch and stores nothing (its
                    // payload could lie past the buffer, its in-tile offsets past int).  Its prefix is published
                    // all the same, so every later tile sees the overflow too.
                    const bool fits = tot <= 0x7fffffffull;
                    if (!fits) atomicCAS(ea.err, KERR_NONE, KERR_OFFSET_OVERFLOW);
                    s_i64[0] = fits ? (int64_t)excl : -1;
                    if (tile == ea.n_tiles - 1) {
                        ea.totals[1 + cd.varlen_index] = (int64_t)tot;
                        if (fits) oc.offsets[ea.totals[0]] = (int32_t)tot;
                    }
                }
            }
            __syncthreads();
            if (ci < 60) TS(8 + 4 * ci + 1);
            const int64_t byte_base = s_i64[0];
            uint8_t *dbase = (uint8_t *)oc.data + (byte_base < 0 ? 0 : byte_base);
            // pass 2: offsets, validity, payload copy — warp-local.  Byte positions inside the tile fit in int (the
            // tile ends below 2 GiB), but the 8-lane copy below steps up to 31 bytes past a row's end: its indexes
            // are 64-bit.
            int carry = ws[warp];
            int *my_pre = wpre + warp * 33;
            int *my_end = wend + warp * 32;
            const uint8_t **my_src = wsrc + warp * 32;
            const int ob_end = byte_base < 0 ? wbeg : min(wbeg + RW, n_out);      // a tile past 2 GiB stores nothing
            for (int ob0 = wbeg; ob0 < ob_end; ob0 += 32) {
                const int ob = ob0 + lane;
                const bool active = ob >= 0 && ob < n_out;
                int len = 0;
                const uint8_t *sp = nullptr;
                bool has = false;
                if (active) {
                    int src = vsrc[ob];
                    if (src != 0xFFFF) {
                        int ps = pm[src] & kPmPosMask;
                        int st = offs[ps];
                        len = offs[ps + 1] - st;
                        sp = cd_data[mrun[src]] + st;
                        has = true;
                    }
                }
                const int incl = warp_scan_incl(len);
                const int off = carry + incl - len;
                carry += __shfl_sync(0xffffffffu, incl, 31);
                if (active) oc.offsets[tv.out_base + ob] = (int32_t)(byte_base + off);
                if (oc.validity != nullptr) put_validity_word(oc.validity, tv.out_base, ob0, n_out, has);
                // warp-cooperative payload copy: the warp's 32 rows form one contiguous destination range;
                // rows without payload (NULL / empty) are squeezed out first, then 8 lanes serve one row (so
                // stores coalesce and short strings do not idle a whole warp), two row groups are in flight at
                // a time and all loads are issued before the stores
                const unsigned pay = __ballot_sync(0xffffffffu, len > 0);
                const int n_pay = __popc(pay);
                if (len > 0) {
                    const int ci = __popc(pay & ((1u << lane) - 1));
                    my_pre[ci] = off;
                    my_end[ci] = off + len;
                    my_src[ci] = sp;
                }
                __syncwarp();
                for (int rg = 0; rg < n_pay; rg += 8) {
                    const int ra = rg + (lane >> 3), rb = ra + 4;
                    int a0 = 0, a1 = 0, b0 = 0, b1 = 0;
                    const uint8_t *pa = nullptr, *pb = nullptr;
                    if (ra < n_pay) { a0 = my_pre[ra]; a1 = my_end[ra]; pa = my_src[ra] - a0; }
                    if (rb < n_pay) { b0 = my_pre[rb]; b1 = my_end[rb]; pb = my_src[rb] - b0; }
                    const int64_t ia = (int64_t)a0 + (lane & 7), ib = (int64_t)b0 + (lane & 7);
                    uint8_t xa0 = 0, xa1 = 0, xa2 = 0, xb0 = 0, xb1 = 0, xb2 = 0;
                    if (ia < a1) xa0 = pa[ia];
                    if (ia + 8 < a1) xa1 = pa[ia + 8];
                    if (ia + 16 < a1) xa2 = pa[ia + 16];
                    if (ib < b1) xb0 = pb[ib];
                    if (ib + 8 < b1) xb1 = pb[ib + 8];
                    if (ib + 16 < b1) xb2 = pb[ib + 16];
                    if (ia < a1) dbase[ia] = xa0;
                    if (ia + 8 < a1) dbase[ia + 8] = xa1;
                    if (ia + 16 < a1) dbase[ia + 16] = xa2;
                    if (ib < b1) dbase[ib] = xb0;
                    if (ib + 8 < b1) dbase[ib + 8] = xb1;
                    if (ib + 16 < b1) dbase[ib + 16] = xb2;
                    for (int64_t b = ia + 24; b < a1; b += 8) dbase[b] = pa[b];
                    for (int64_t b = ib + 24; b < b1; b += 8) dbase[b] = pb[b];
                }
                __syncwarp();
            }
        }
        if (cn >= 0 && tid < n_vw) stage_vw(s ^ 1)[tid] = next_vw;
        __syncthreads();
        if (ci < 60) TS(8 + 4 * ci + 3);
    }
}

#ifdef PG_EMIT_TIMING
void emit_timing_dump() {
    static long long h[64 * 256];
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(h, g_emit_ts, sizeof(h));
    double acc[256] = {0};
    int cntv[256] = {0};
    for (int t = 0; t < 64; t++)
        for (int sl = 1; sl < 256; sl++) {
            if (h[t * 256 + sl] == 0) continue;
            int pv = sl - 1;
            while (pv > 0 && h[t * 256 + pv] == 0) pv--;
            if (h[t * 256 + pv] == 0) continue;
            acc[sl] += (double)(h[t * 256 + sl] - h[t * 256 + pv]);
            cntv[sl]++;
        }
    fprintf(stderr, "[emit timing] cycles since previous slot (avg over tiles):");
    for (int sl = 1; sl < 256; sl++) if (cntv[sl]) fprintf(stderr, " %d:%.0f", sl, acc[sl] / cntv[sl]);
    fprintf(stderr, "\n");
    static long long z[64 * 256];
    cudaMemcpyToSymbol(g_emit_ts, z, sizeof(z));
}
#endif

static bool g_emit_attr = false;
void launch_emit(const EmitArgs &ea) {
    EmitLayout L = emit_layout(ea.k);
    if (!g_emit_attr) {
        cudaFuncSetAttribute(k_emit<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        cudaFuncSetAttribute(k_emit<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        g_emit_attr = true;
    }
    if (ea.gagg) k_emit<true><<<ea.n_tiles, kEmitThreads, L.total, ea.stream>>>(ea);
    else k_emit<false><<<ea.n_tiles, kEmitThreads, L.total, ea.stream>>>(ea);
#ifdef PG_EMIT_TIMING
    emit_timing_dump();
#endif
}

}  // namespace pg
