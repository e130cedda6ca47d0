// merge.cu — sm_90a kernels of the k-way merge + per-key-group reduce.
//
// Replaces the per-record loop of SortMergeReaderWithLoserTree.SortMergeIterator.next()
// (reference: paimon-core/.../mergetree/compact/SortMergeReaderWithLoserTree.java:87-112,
// LoserTree.java:95-170) with a data-parallel pipeline over columnar runs resident in HBM:
//
//   1. sampled partition   every S-th key of each run forms the next level; levels are merged
//                          top-down so that level 0 is cut into key-range tiles of <= kPlanTile rows
//                          (all rows of one key fall into one tile => the reduce is tile-local)
//   2. plan kernel         one CTA per tile: k sorted segments -> shared memory -> log2(k) rounds of
//                          merge-path pair merges -> key groups -> members ordered by sequence number
//                          -> per-member op (the MergeFunction's row-level semantics) -> uint16 plan
//   3. scan                tile row counts / var-len byte counts -> output offsets
//   4. emit kernel         per tile and column: select / fold the group's members, coalesced stores
//
// No tensor cores: the path is integer compare + gather (HBM bound).
#include <mutex>

#include "device_utils.cuh"

namespace pg {

// ------------------------------------------------------------------ helpers

__device__ __forceinline__ uint64_t norm_field(const void *base, int type, int64_t row) {
    // order-preserving unsigned image of a signed integer key field (GenerateUtils.scala:122-123:
    // integers compare with signed < / >)
    switch (type) {
        case PG_INT8:  return (uint64_t)(uint8_t)(((const int8_t *)base)[row] ^ (int8_t)0x80);
        case PG_BOOL:  return ((const uint8_t *)base)[row] ? 1u : 0u;
        case PG_INT16: return (uint64_t)(uint16_t)(((const int16_t *)base)[row] ^ (int16_t)0x8000);
        case PG_INT32: return (uint64_t)(uint32_t)(((const int32_t *)base)[row] ^ (int32_t)0x80000000);
        default:       return (uint64_t)(((const int64_t *)base)[row]) ^ 0x8000000000000000ull;
    }
}

// Order-preserving 64-bit window of a row's primary key.  The key is read as a byte stream: the key fields
// big-endian, most significant first; a var-len field contributes its bytes and ends the stream.  The window
// holds stream bytes [skip, skip + 8), zero padded.  With `skip` = a common prefix length of all keys that are
// compared with each other, window(a) < window(b) implies a < b; equal windows decide nothing unless the keys
// are known to end inside the window (kd.exact, or a tile whose keys all have the same covered length).
__device__ __forceinline__ uint64_t load_key(const KeySrc &ks, const KeyDesc &kd, int run, int64_t row, int skip = 0) {
    if (kd.n_fields == 1 && kd.width[0] == 8 && skip == 0) return norm_field(ks.data[run], kd.type[0], row);
    uint64_t k = 0;
    int pos = 0;                                         // stream offset of the current field
    const int end = skip + 8;
    for (int f = 0; f < kd.n_fields && pos < end; f++) {
        const void *base = ks.data[run * kd.n_fields + f];
        const int w = kd.width[f];
        if (w > 0) {
            if (pos + w > skip) {
                const uint64_t v = norm_field(base, kd.type[f], row);
                for (int j = max(0, skip - pos); j < w && pos + j < end; j++)
                    k |= ((v >> (8 * (w - 1 - j))) & 0xFF) << (8 * (7 - (pos + j - skip)));
            }
            pos += w;
        } else {
            const int32_t *offs = ks.offsets[run * kd.n_fields + f];
            const uint8_t *bytes = (const uint8_t *)base + offs[row];
            const int len = offs[row + 1] - offs[row];
            for (int j = max(0, skip - pos); j < len && pos + j < end; j++)
                k |= (uint64_t)bytes[j] << (8 * (7 - (pos + j - skip)));
            pos = end;
        }
    }
    return k;
}

// Length of the key's byte stream (see load_key); -1 when the stream does not cover the whole key (a var-len
// field that is not the last one)
__device__ __forceinline__ int key_stream_len(const KeySrc &ks, const KeyDesc &kd, int run, int64_t row) {
    int pos = 0;
    for (int f = 0; f < kd.n_fields; f++) {
        const int w = kd.width[f];
        if (w > 0) pos += w;
        else {
            if (f != kd.n_fields - 1) return -1;
            const int32_t *offs = ks.offsets[run * kd.n_fields + f];
            pos += offs[row + 1] - offs[row];
        }
    }
    return pos;
}

// Number of leading stream bytes two rows' keys have in common
__device__ int key_stream_lcp(const KeySrc &ks, const KeyDesc &kd, int ra, int64_t row_a, int rb, int64_t row_b) {
    int pos = 0;
    for (int f = 0; f < kd.n_fields; f++) {
        const void *da = ks.data[ra * kd.n_fields + f], *db = ks.data[rb * kd.n_fields + f];
        const int w = kd.width[f];
        if (w > 0) {
            const uint64_t x = norm_field(da, kd.type[f], row_a), y = norm_field(db, kd.type[f], row_b);
            if (x != y) return pos + (__clzll((long long)(x ^ y)) >> 3) - (8 - w);
            pos += w;
        } else {
            const int32_t *oa = ks.offsets[ra * kd.n_fields + f], *ob = ks.offsets[rb * kd.n_fields + f];
            const uint8_t *pa = (const uint8_t *)da + oa[row_a], *pb = (const uint8_t *)db + ob[row_b];
            const int la = oa[row_a + 1] - oa[row_a], lb = ob[row_b + 1] - ob[row_b];
            int j = 0;
            while (j < la && j < lb && pa[j] == pb[j]) j++;
            return pos + j;                              // a var-len field ends the stream
        }
    }
    return pos;
}

// Full comparison of two rows' keys, field by field, with the generated comparator's rules
// (GenerateUtils.scala:113-126): integers signed, BOOLEAN false < true, CHAR/VARCHAR/BINARY unsigned bytewise
// then length (BinaryString.java:109-126, SortUtil.java:212-241).
__device__ int full_key_compare(const KeySrc &ks, const KeyDesc &kd, int ra, int64_t row_a, int rb, int64_t row_b) {
    for (int f = 0; f < kd.n_fields; f++) {
        const void *da = ks.data[ra * kd.n_fields + f], *db = ks.data[rb * kd.n_fields + f];
        const int w = kd.width[f];
        if (w > 0) {
            uint64_t x = norm_field(da, kd.type[f], row_a), y = norm_field(db, kd.type[f], row_b);
            if (x != y) return x < y ? -1 : 1;
        } else {
            const int32_t *oa = ks.offsets[ra * kd.n_fields + f], *ob = ks.offsets[rb * kd.n_fields + f];
            int la = oa[row_a + 1] - oa[row_a], lb = ob[row_b + 1] - ob[row_b];
            int d = bytes_compare((const uint8_t *)da + oa[row_a], la, (const uint8_t *)db + ob[row_b], lb);
            if (d != 0) return d < 0 ? -1 : 1;
        }
    }
    return 0;
}

// ------------------------------------------------------------------ partition

__global__ void k_partition(int k, KeyDesc kd, KeySrc ks, LevelView lv, const uint64_t *__restrict__ sk,
                            const uint64_t *__restrict__ sref, int q, int n_tiles, int64_t *bounds,
                            const int *__restrict__ skip_p) {
    const int skip = skip_p ? *skip_p : 0;
    int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= (int64_t)(n_tiles + 1) * k) return;
    int t = (int)(idx / k), r = (int)(idx % k);
    int64_t res;
    if (t == 0) res = 0;
    else if (t == n_tiles) res = lv.count[r];
    else {
        const uint64_t x = sk[(int64_t)t * q];
        const uint64_t xr = kd.exact ? 0 : sref[(int64_t)t * q];      // splitter row: run << 40 | row
        const int s_run = (int)(xr >> 40);
        const int64_t s_row = (int64_t)(xr & ((1ull << 40) - 1));
        int64_t lo = 0, hi = lv.count[r];
        while (lo < hi) {                      // lower_bound: first j with key(j) >= splitter key
            int64_t mid = (lo + hi) >> 1;
            const int64_t row = lv.row0[r] + (mid + 1) * lv.stride - 1;
            uint64_t km = load_key(ks, kd, r, row, skip);
            bool less = km < x;
            if (!less && km == x && !kd.exact) less = full_key_compare(ks, kd, r, row, s_run, s_row) < 0;
            if (less) lo = mid + 1; else hi = mid;
        }
        res = lo;
    }
    // level 0 hands out absolute rows (plan / emit index the runs with them), upper levels level-local indexes
    bounds[idx] = lv.stride == 1 ? res + lv.row0[r] : res;
}

// ------------------------------------------------------------------ in-tile merge

// shared-memory index padding: one extra slot per 16 elements, so that the merge-path threads (which start
// 16 elements apart) fall into different banks instead of all hitting the same one
#define PADI(i) ((i) + ((i) >> 4))
constexpr int kTilePad = kPlanTile + kPlanTile / 16;

struct TileCtx {
    uint64_t *key[2];
    uint16_t *idx[2];
    int *lb[2];          // list boundaries, k+1 entries each
    int *seg;            // slot base per run, k+1 entries
    int64_t *rstart;     // first row (at this level) of every run's segment
    int n;               // rows in the tile
    int fin;             // which buffer holds the merged result
    bool exact;          // equal windows mean equal keys in this tile
};

// Loads the tile's k segments and merges them.  Returns false when the tile overflows.
template <bool EXACT>
__device__ bool merge_tile(TileCtx &tc, int k, const KeyDesc &kd, const KeySrc &ks,
                           const int64_t *bounds, int tile, int64_t stride, const int64_t *row0, int32_t *err,
                           int skip, bool refine) {
    const int tid = threadIdx.x;
    __shared__ int s_skip, s_len0;
    if (tid < 32) {
        // lane r = run r: both loads of every run in flight at once, slot bases by a warp scan
        int64_t b0 = 0, b1 = 0;
        if (tid < k) { b0 = bounds[(int64_t)tile * k + tid]; b1 = bounds[(int64_t)(tile + 1) * k + tid]; }
        const int64_t len = b1 - b0;
        const bool odd = len < 0 || len > kPlanTile;
        const int l = odd ? 0 : (int)len;
        const int incl = warp_scan_incl(l);
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        const bool over = __any_sync(0xffffffffu, odd) || total > kPlanTile;
        if (tid < k) {
            tc.rstart[tid] = b0;
            tc.seg[tid] = incl - l;
            tc.lb[0][tid] = incl - l;
        }
        if (tid == 0) {
            tc.seg[k] = over ? kPlanTile + 1 : total;
            tc.lb[0][k] = over ? kPlanTile + 1 : total;
        }
    }
    __syncthreads();
    tc.n = tc.seg[k];
    if (tc.n > kPlanTile) {
        if (tid == 0) atomicCAS(err, KERR_NONE, KERR_TILE_OVERFLOW);
        return false;
    }
    const int n = tc.n;
    tc.exact = EXACT;
    if (!EXACT && refine) {
        // the tile's keys share at least the prefix its 2k segment end points share with one of them: start the
        // 8-byte window behind it, so that keys with a long common prefix ("user_0000123") still sort by window
        if (tid == 0) { s_skip = 0x7fffffff; s_len0 = -2; }
        __syncthreads();
        int ref_r = 0;
        while (ref_r < k && tc.seg[ref_r + 1] == tc.seg[ref_r]) ref_r++;
        if (tid < 2 * k && ref_r < k) {
            const int r = tid >> 1;
            const int len = tc.seg[r + 1] - tc.seg[r];
            if (len > 0) {
                const int64_t row = ((tid & 1) ? tc.rstart[r] + len - 1 : tc.rstart[r]);
                atomicMin(&s_skip, key_stream_lcp(ks, kd, ref_r, tc.rstart[ref_r], r, row));
            }
        }
        __syncthreads();
        skip = s_skip == 0x7fffffff ? 0 : s_skip;
    }
    bool odd_len = false;                            // a key that does not end inside the window, or whose length
    int len0 = -2;                                   // differs from the tile's first key
    if (!EXACT && refine && n > 0) {
        int ref_r = 0;
        while (tc.seg[ref_r + 1] == tc.seg[ref_r]) ref_r++;
        len0 = key_stream_len(ks, kd, ref_r, tc.rstart[ref_r]);
        if (len0 < 0 || len0 > skip + 8) odd_len = true;
    }
    {
        // slots tid, tid + blockDim, ...: neighbours in a warp are neighbours in a run (coalesced), and all of a
        // thread's loads are in flight before the first one is stored (a loop over the runs with the store inside
        // serialises k memory latencies per tile)
        constexpr int VTL = kPlanTile / kThreads;
        uint64_t kv[VTL];
#pragma unroll
        for (int u = 0; u < VTL; u++) {
            const int i = tid + u * kThreads;
            kv[u] = 0;
            if (i < n) {
                const int r = run_of_slot(tc.seg, k, i);
                const int64_t rb = row0 ? row0[r] : 0;       // (level 0 bounds are absolute rows already)
                const int64_t row = rb + (tc.rstart[r] + (i - tc.seg[r]) + 1) * stride - 1;
                kv[u] = load_key(ks, kd, r, row, skip);
                if (!EXACT && refine && !odd_len && key_stream_len(ks, kd, r, row) != len0) odd_len = true;
            }
        }
#pragma unroll
        for (int u = 0; u < VTL; u++) {
            const int i = tid + u * kThreads;
            if (i < n) { tc.key[0][PADI(i)] = kv[u]; tc.idx[0][PADI(i)] = (uint16_t)i; }
        }
    }
    if (!EXACT && refine) tc.exact = !__syncthreads_or(odd_len);
    else __syncthreads();

    // a <= b on (prefix, slot) pairs; equal prefixes of a non-exact key fall back to the full comparison
    auto le = [&](uint64_t ka, int sa, uint64_t kb, int sb) -> bool {
        if (ka != kb) return ka < kb;
        if (EXACT || tc.exact) return true;
        const int ra = run_of_slot(tc.seg, k, sa), rb = run_of_slot(tc.seg, k, sb);
        const int64_t row_a = (row0 ? row0[ra] : 0) + (tc.rstart[ra] + (sa - tc.seg[ra]) + 1) * stride - 1;
        const int64_t row_b = (row0 ? row0[rb] : 0) + (tc.rstart[rb] + (sb - tc.seg[rb]) + 1) * stride - 1;
        return full_key_compare(ks, kd, ra, row_a, rb, row_b) <= 0;
    };

    int L = k, cur = 0;
    constexpr int VT = kPlanTile / kThreads;
    while (L > 1) {
        const uint64_t *sk = tc.key[cur];
        const uint16_t *si = tc.idx[cur];
        uint64_t *dk = tc.key[cur ^ 1];
        uint16_t *di = tc.idx[cur ^ 1];
        const int *lb = tc.lb[cur];
        int pos = tid * VT, end = min(pos + VT, n);
        int p = 0;
        while (pos < end) {
            // pair p merges lists 2p and 2p+1
            while (lb[min(2 * p + 2, L)] <= pos) p++;
            int a0 = lb[2 * p], a1 = lb[min(2 * p + 1, L)], b1 = lb[min(2 * p + 2, L)];
            int na = a1 - a0, nb = b1 - a1;
            int d = pos - a0;
            int cnt = min(end, b1) - pos;
            int lo = max(0, d - nb), hi = min(d, na);
            while (lo < hi) {                    // merge path: #elements taken from A among the first d
                int mid = (lo + hi) >> 1;
                if (le(sk[PADI(a0 + mid)], si[PADI(a0 + mid)], sk[PADI(a1 + d - 1 - mid)], si[PADI(a1 + d - 1 - mid)]))
                    lo = mid + 1;
                else
                    hi = mid;
            }
            int ai = lo, bi = d - lo;
            uint64_t ka = ai < na ? sk[PADI(a0 + ai)] : 0, kb = bi < nb ? sk[PADI(a1 + bi)] : 0;
            uint16_t ia = ai < na ? si[PADI(a0 + ai)] : 0, ib = bi < nb ? si[PADI(a1 + bi)] : 0;
            for (int s = 0; s < cnt; s++) {
                bool take_a = (bi >= nb) || (ai < na && le(ka, ia, kb, ib));   // stable: lower run first on ties
                if (take_a) {
                    dk[PADI(pos + s)] = ka; di[PADI(pos + s)] = ia;
                    ai++;
                    if (ai < na) { ka = sk[PADI(a0 + ai)]; ia = si[PADI(a0 + ai)]; }
                } else {
                    dk[PADI(pos + s)] = kb; di[PADI(pos + s)] = ib;
                    bi++;
                    if (bi < nb) { kb = sk[PADI(a1 + bi)]; ib = si[PADI(a1 + bi)]; }
                }
            }
            pos += cnt;
        }
        int P = (L + 1) >> 1;
        if (tid <= P) tc.lb[cur ^ 1][tid] = lb[min(2 * tid, L)];
        __syncthreads();
        L = P;
        cur ^= 1;
    }
    tc.fin = cur;
    return true;
}

__device__ __forceinline__ void carve_tile(TileCtx &tc, unsigned char *smem, int k) {
    tc.key[0] = (uint64_t *)smem;
    tc.key[1] = tc.key[0] + kTilePad;
    tc.idx[0] = (uint16_t *)(tc.key[1] + kTilePad);
    tc.idx[1] = tc.idx[0] + kTilePad;
    tc.rstart = (int64_t *)(tc.idx[1] + kTilePad);
    tc.lb[0] = (int *)(tc.rstart + PG_MAX_RUNS);
    tc.lb[1] = tc.lb[0] + PG_MAX_RUNS + 1;
    tc.seg = tc.lb[1] + PG_MAX_RUNS + 1;
}
constexpr size_t kTileSmem = (size_t)kTilePad * (8 + 8 + 2 + 2) + PG_MAX_RUNS * 8 + 3 * (PG_MAX_RUNS + 1) * 4;

template <bool EXACT>
__global__ void __launch_bounds__(kThreads)
k_merge_keys(int k, KeyDesc kd, KeySrc ks, LevelView lv, const int64_t *bounds, uint64_t *sorted_keys,
             uint64_t *sorted_refs, int32_t *err, const int *__restrict__ skip_p) {
    extern __shared__ __align__(16) unsigned char smem[];
    TileCtx tc;
    carve_tile(tc, smem, k);
    int tile = blockIdx.x;
    if (!merge_tile<EXACT>(tc, k, kd, ks, bounds, tile, lv.stride, lv.row0, err, skip_p ? *skip_p : 0, false)) return;
    int64_t base = 0;
    for (int r = 0; r < k; r++) base += tc.rstart[r];
    const uint64_t *fk = tc.key[tc.fin];
    const uint16_t *fi = tc.idx[tc.fin];
    for (int i = threadIdx.x; i < tc.n; i += blockDim.x) {
        sorted_keys[base + i] = fk[PADI(i)];
        if (!EXACT) {                          // the sample's row, for full comparisons against it
            const int slot = fi[PADI(i)];
            const int r = run_of_slot(tc.seg, k, slot);
            const int64_t row = lv.row0[r] + (tc.rstart[r] + (slot - tc.seg[r]) + 1) * lv.stride - 1;
            sorted_refs[base + i] = ((uint64_t)r << 40) | (uint64_t)row;
        }
    }
}

// ------------------------------------------------------------------ 'sequence.field' comparator

// userDefinedSeqComparator.compare(a.value(), b.value()) for two members given by their tile slots.
// Generated-comparator rules (paimon-codegen GenerateUtils.scala:113-126, 305-345; nullIsLast = false):
// both null -> next field; one null -> that side is smaller, decided BEFORE the descending sign flip;
// numbers compare with > / < (NaN is "equal" to everything); BOOLEAN false < true.
__device__ int compare_seq_fields(const SeqFields &sf, const ColPtrs &ptrs, int k, const int *seg,
                                  const int64_t *rstart, int slot_a, int slot_b) {
    const int ra = run_of_slot(seg, k, slot_a), rb = run_of_slot(seg, k, slot_b);
    const int64_t row_a = rstart[ra] + (slot_a - seg[ra]), row_b = rstart[rb] + (slot_b - seg[rb]);
    for (int f = 0; f < sf.n; f++) {
        const int col = sf.col[f];
        const uint8_t *va = (const uint8_t *)ptrs.validity[(int64_t)col * k + ra];
        const uint8_t *vb = (const uint8_t *)ptrs.validity[(int64_t)col * k + rb];
        const bool na = !valid_bit(va, row_a), nb = !valid_bit(vb, row_b);
        if (na && nb) continue;
        if (na) return -1;
        if (nb) return 1;
        const void *da = ptrs.data[(int64_t)col * k + ra], *db = ptrs.data[(int64_t)col * k + rb];
        int d;
        switch (sf.type[f]) {
            case PG_FLOAT: {
                float x = ((const float *)da)[row_a], y = ((const float *)db)[row_b];
                d = x > y ? 1 : x < y ? -1 : 0;
                break;
            }
            case PG_DOUBLE: {
                double x = ((const double *)da)[row_a], y = ((const double *)db)[row_b];
                d = x > y ? 1 : x < y ? -1 : 0;
                break;
            }
            default: {
                const int w = sf.width[f];
                int64_t x = sext(load_fixed(da, w, row_a), w), y = sext(load_fixed(db, w, row_b), w);
                if (sf.type[f] == PG_BOOL) { x = x != 0; y = y != 0; }
                d = x > y ? 1 : x < y ? -1 : 0;
            }
        }
        if (d != 0) return sf.ascending ? d : -d;
    }
    return 0;
}

// ---- partial-update sequence groups (PartialUpdateMergeFunction.java:190-342)

// one value cell of a member given by its tile slot
struct CellRef { const void *data; const uint8_t *validity; int64_t row; };
__device__ __forceinline__ CellRef cell_of(const ColPtrs &ptrs, int k, const int *seg, const int64_t *rstart, int col,
                                           int slot) {
    const int r = run_of_slot(seg, k, slot);
    CellRef c;
    c.data = ptrs.data[(int64_t)col * k + r];
    c.validity = (const uint8_t *)ptrs.validity[(int64_t)col * k + r];
    c.row = rstart[r] + (slot - seg[r]);
    return c;
}

// isEmptySequenceGroup (:249-269): every sequence field of the group is NULL in this member
__device__ bool group_is_empty(const SeqGroups &sg, int g, const ColPtrs &ptrs, int k, const int *seg,
                               const int64_t *rstart, int slot) {
    for (int f = sg.start[g]; f < sg.start[g + 1]; f++) {
        CellRef c = cell_of(ptrs, k, seg, rstart, sg.col[f], slot);
        if (valid_bit(c.validity, c.row)) return false;
    }
    return true;
}

// seqComparator.compare(kv.value(), row) for group g: member `slot_a` against the accumulated sequence fields,
// which are those of member `slot_b` (slot_b < 0: all NULL).  Ascending, NULL first (a5).
__device__ int compare_group_seq(const SeqGroups &sg, int g, const ColPtrs &ptrs, int k, const int *seg,
                                 const int64_t *rstart, int slot_a, int slot_b) {
    for (int f = sg.start[g]; f < sg.start[g + 1]; f++) {
        CellRef a = cell_of(ptrs, k, seg, rstart, sg.col[f], slot_a);
        const bool na = !valid_bit(a.validity, a.row);
        bool nb = true;
        CellRef b{};
        if (slot_b >= 0) {
            b = cell_of(ptrs, k, seg, rstart, sg.col[f], slot_b);
            nb = !valid_bit(b.validity, b.row);
        }
        if (na && nb) continue;
        if (na) return -1;
        if (nb) return 1;
        int d;
        switch (sg.type[f]) {
            case PG_FLOAT: {
                float x = ((const float *)a.data)[a.row], y = ((const float *)b.data)[b.row];
                d = x > y ? 1 : x < y ? -1 : 0;
                break;
            }
            case PG_DOUBLE: {
                double x = ((const double *)a.data)[a.row], y = ((const double *)b.data)[b.row];
                d = x > y ? 1 : x < y ? -1 : 0;
                break;
            }
            default: {
                const int w = sg.width[f];
                int64_t x = sext(load_fixed(a.data, w, a.row), w), y = sext(load_fixed(b.data, w, b.row), w);
                if (sg.type[f] == PG_BOOL) { x = x != 0; y = y != 0; }
                d = x > y ? 1 : x < y ? -1 : 0;
            }
        }
        if (d != 0) return d;
    }
    return 0;
}

// ------------------------------------------------------------------ plan kernel

struct PlanSmemExtra {
    uint16_t *res_slot;   // per head position: slot whose sequence number is the result's (0xFFFF = 0)
    uint8_t *res_kind;    // per head position: result RowKind
    int *ws;              // 33 ints scan scratch
};
constexpr size_t kPlanSmem = kTileSmem + (size_t)kPlanTile * 3 + 34 * 4 + kPlanTile / 8 + 16;

template <bool EXACT>
__global__ void __launch_bounds__(kThreads, 4)
k_plan(int k, KeyDesc kd, KeySrc ks, PlanArgs pa, int32_t *err) {
    extern __shared__ __align__(16) unsigned char smem[];
    TileCtx tc;
    carve_tile(tc, smem, k);
    PlanSmemExtra px;
    px.res_slot = (uint16_t *)(smem + ((kTileSmem + 15) & ~(size_t)15));
    px.res_kind = (uint8_t *)(px.res_slot + kPlanTile);
    px.ws = (int *)(px.res_kind + kPlanTile);
    uint8_t *head_bits = (uint8_t *)(px.ws + 34);            // bit i: merged position i starts a key group

    const int tile = blockIdx.x, tid = threadIdx.x;
    if (!merge_tile<EXACT>(tc, k, kd, ks, pa.bounds, tile, 1, nullptr, err, 0, true)) {
        if (tid == 0) pa.tile_rows[tile] = 0;
        return;
    }
    const int n = tc.n;
    const uint64_t *fk = tc.key[tc.fin];
    uint16_t *fi = tc.idx[tc.fin];
    int64_t *seq_s = (int64_t *)tc.key[tc.fin ^ 1];          // staged by slot
    uint8_t *kind_s = (uint8_t *)tc.idx[tc.fin ^ 1];          // first 4 KiB: kinds by slot
    uint8_t *ops = kind_s + kPlanTile;                         // second 4 KiB: op per merged position

    int64_t in_base = 0;
    for (int r = 0; r < k; r++) in_base += tc.rstart[r];

    // do the merged positions a and b hold the same key?  (equal prefixes decide only for exact keys)
    auto same_key = [&](int a, int b) -> bool {
        if (fk[PADI(a)] != fk[PADI(b)]) return false;
        if (EXACT || tc.exact) return true;
        const int sa = fi[PADI(a)], sb = fi[PADI(b)];
        const int ra = run_of_slot(tc.seg, k, sa), rb = run_of_slot(tc.seg, k, sb);
        return full_key_compare(ks, kd, ra, tc.rstart[ra] + (sa - tc.seg[ra]), rb, tc.rstart[rb] + (sb - tc.seg[rb])) == 0;
    };

    // stage sequence numbers and kinds (slot order: coalesced inside a run; all loads before the stores)
    {
        constexpr int VTL = kPlanTile / kThreads;
        int64_t sq[VTL];
        uint8_t kn[VTL];
#pragma unroll
        for (int u = 0; u < VTL; u++) {
            const int sl = tid + u * kThreads;
            sq[u] = 0; kn[u] = 0;
            if (sl < n) {
                const int r = run_of_slot(tc.seg, k, sl);
                const int64_t row = tc.rstart[r] + (sl - tc.seg[r]);
                sq[u] = pa.seq_ptrs[r][row];
                kn[u] = (uint8_t)pa.kind_ptrs[r][row];
            }
        }
#pragma unroll
        for (int u = 0; u < VTL; u++) {
            const int sl = tid + u * kThreads;
            if (sl < n) { seq_s[sl] = sq[u]; kind_s[sl] = kn[u]; }
        }
    }
    __syncthreads();

    constexpr int VT = kPlanTile / kThreads;
    const int p0 = tid * VT, p1 = min(p0 + VT, n);
    const MergeFlags fl = pa.flags;
    int my_emit = 0;

    // group heads first, for every position, BEFORE any group is re-ordered: same_key() of a non-exact key reads
    // the slots of both positions, and the position in front of a head belongs to another thread's group
    static_assert(kPlanTile / kThreads == 8, "one byte of head bits per thread");
    {
        uint32_t hb = 0;
        for (int i = p0; i < p1; i++)
            if (i == 0 || !same_key(i - 1, i)) hb |= 1u << (i - p0);
        head_bits[tid] = (uint8_t)hb;
    }
    __syncthreads();
    auto is_head = [&](int i) -> bool { return (head_bits[i >> 3] >> (i & 7)) & 1; };

    for (int i = p0; i < p1; i++) {
        if (!is_head(i)) continue;
        int e = i + 1;
        while (e < n && !is_head(e)) e++;
        const int g = e - i;
        // members in ascending sequence order (SortMergeReaderWithLoserTree.java:52-65); ties (which the
        // reference leaves unspecified) resolve by run order = slot order
        for (int a = i + 1; a < e; a++) {
            uint16_t sa = fi[PADI(a)];
            int64_t qa = seq_s[sa];
            int b = a - 1;
            while (b >= i) {
                uint16_t sb = fi[PADI(b)];
                int64_t qb = seq_s[sb];
                // 'sequence.field': the user defined sequence fields order the members first
                // (SortMergeReaderWithLoserTree.java:58-64), then the sequence number
                int ud = pa.seq.n ? compare_seq_fields(pa.seq, pa.ptrs, k, tc.seg, tc.rstart, sb, sa) : 0;
                if (ud < 0 || (ud == 0 && (qb < qa || (qb == qa && sb < sa)))) break;
                fi[PADI(b + 1)] = sb;
                b--;
            }
            fi[PADI(b + 1)] = sa;
        }
        // row-level semantics of the merge function
        bool emit = true;
        int res_kind = PG_INSERT;
        uint16_t res_slot = 0xFFFF;
        if (g == 1) {
            // ReducerMergeFunctionWrapper.java:53-73: a lone record is returned untouched
            ops[i] = OP_SET;
            res_slot = fi[PADI(i)];
            res_kind = kind_s[fi[PADI(i)]];
            if (pa.groups) pa.gplan[in_base + i] = 0xFFFFFFFFu;      // every group field from this record
            if (pa.gagg) pa.gagg[in_base + i] = 0;
        } else if (fl.engine == PG_ENGINE_DEDUPLICATE) {
            // DeduplicateMergeFunction.java:47-60
            int win = -1;
            for (int j = e - 1; j >= i; j--) {
                if (fl.ignore_delete && kind_is_retract(kind_s[fi[PADI(j)]])) continue;
                win = j;
                break;
            }
            for (int j = i; j < e; j++) ops[j] = (j == win) ? OP_SET : OP_NOOP;
            if (win < 0) emit = false;
            else { res_slot = fi[PADI(win)]; res_kind = kind_s[fi[PADI(win)]]; }
        } else if (fl.engine == PG_ENGINE_FIRST_ROW) {
            // FirstRowMergeFunction.java:50-73
            int win = -1;
            for (int j = i; j < e; j++) {
                ops[j] = OP_NOOP;
                if (kind_is_retract(kind_s[fi[PADI(j)]])) {
                    if (!fl.ignore_delete) atomicCAS(err, KERR_NONE, KERR_FIRST_ROW_RETRACT);
                    continue;
                }
                if (win < 0) win = j;
            }
            if (win < 0) emit = false;
            else { ops[win] = OP_SET; res_slot = fi[PADI(win)]; res_kind = kind_s[fi[PADI(win)]]; }
        } else if (fl.engine == PG_ENGINE_PARTIAL_UPDATE) {
            // PartialUpdateMergeFunction.java:121-175 (no sequence groups), getResult :354-362
            bool filled = false, meet = false, cur_del = false;
            // sequence groups: which member currently provides group g's sequence fields / its other fields
            // (-1: NULL).  Groups only see inserts whose group sequence is >= the accumulated one (:190-247);
            // a retract with a >= sequence takes the sequence fields and NULLs the group's fields (:271-342)
            int8_t seq_src[PG_MAX_SEQ_GROUPS], val_src[PG_MAX_SEQ_GROUPS];
            const SeqGroups *sg = pa.groups;
            const int ng = sg ? sg->n : 0;
            for (int g = 0; g < ng; g++) { seq_src[g] = -1; val_src[g] = -1; }
            for (int j = i; j < e; j++) {
                int kind = kind_s[fi[PADI(j)]];
                int op = OP_NOOP;
                cur_del = false;
                if (ng > 0) {
                    const int slot = fi[PADI(j)];
                    const int mj = j - i;
                    uint32_t am = 0;                                             // aggregation marks of this member
                    if (kind_is_retract(kind)) {
                        if (!filled) {                                           // initRow: every field verbatim
                            op = OP_SET; filled = true;
                            for (int g = 0; g < ng; g++) { seq_src[g] = (int8_t)mj; val_src[g] = (int8_t)mj; }
                        }
                        if (!fl.ignore_delete) {
                            // (a retract that is also the first record: op RETRACT on the head = initRow, then
                            // the retract; the select / fold code treats a RETRACT head like SET first)
                            if (pa.gagg) op = OP_RETRACT;           // only the aggregate-in-group fold needs to see it
                            res_slot = (uint16_t)slot;
                            for (int g = 0; g < ng; g++) {
                                if (group_is_empty(*sg, g, pa.ptrs, k, tc.seg, tc.rstart, slot)) continue;
                                am |= 1u << g;                                   // aggregated fields retract either way
                                const int sb = seq_src[g] < 0 ? -1 : fi[PADI(i + seq_src[g])];
                                if (compare_group_seq(*sg, g, pa.ptrs, k, tc.seg, tc.rstart, slot, sb) < 0) continue;
                                if (kind == PG_DELETE && sg->partial_delete[g]) {
                                    // remove-record-on-sequence-group: the row restarts from this record
                                    cur_del = true; op = OP_SET; am = 0;
                                    for (int h = 0; h < ng; h++) { seq_src[h] = (int8_t)mj; val_src[h] = (int8_t)mj; }
                                    break;
                                }
                                seq_src[g] = (int8_t)mj;
                                val_src[g] = -1;
                            }
                        }
                    } else {
                        res_slot = (uint16_t)slot;
                        op = OP_UPD; meet = true; filled = true;
                        for (int g = 0; g < ng; g++) {
                            if (group_is_empty(*sg, g, pa.ptrs, k, tc.seg, tc.rstart, slot)) continue;
                            const int sb = seq_src[g] < 0 ? -1 : fi[PADI(i + seq_src[g])];
                            if (compare_group_seq(*sg, g, pa.ptrs, k, tc.seg, tc.rstart, slot, sb) >= 0) {
                                seq_src[g] = (int8_t)mj; val_src[g] = (int8_t)mj;
                                am |= 1u << g;
                            } else {
                                am |= 1u << (16 + g);                            // aggReversed
                            }
                        }
                    }
                    if (pa.gagg) pa.gagg[in_base + j] = am;
                    ops[j] = (uint8_t)op;
                    continue;
                }
                if (kind_is_retract(kind)) {
                    if (!filled) { op = OP_SET; filled = true; }          // initRow
                    if (!fl.ignore_delete) {
                        res_slot = fi[PADI(j)];                                  // latestSequenceNumber
                        if (fl.remove_record_on_delete) {
                            if (kind == PG_DELETE) { cur_del = true; op = OP_SET; }
                        } else {
                            atomicCAS(err, KERR_NONE, KERR_PU_DELETE);
                        }
                    }
                } else {
                    res_slot = fi[PADI(j)];
                    op = OP_UPD;
                    meet = true;
                    filled = true;
                }
                ops[j] = (uint8_t)op;
            }
            res_kind = (cur_del || !meet) ? PG_DELETE : PG_INSERT;
            if (ng > 0) {
                for (int j = i; j < e; j++) {
                    uint32_t mk = 0;
                    for (int g = 0; g < ng; g++) {
                        if (val_src[g] == j - i) mk |= 1u << g;
                        if (seq_src[g] == j - i) mk |= 1u << (16 + g);
                    }
                    pa.gplan[in_base + j] = mk;
                }
            }
        } else {
            // AggregateMergeFunction.java:80-125
            bool cur_del = false;
            for (int j = i; j < e; j++) {
                int kind = kind_s[fi[PADI(j)]];
                cur_del = fl.remove_record_on_delete && kind == PG_DELETE;
                ops[j] = cur_del ? OP_SET : (kind_is_retract(kind) ? OP_RETRACT : OP_UPD);
            }
            res_slot = fi[PADI(e - 1)];
            res_kind = cur_del ? PG_DELETE : PG_INSERT;
        }
        // DropDeleteReader.java:58: only kv.isAdd() survives
        if (emit && fl.drop_delete && kind_is_retract(res_kind)) emit = false;
        px.res_slot[i] = res_slot;
        px.res_kind[i] = (uint8_t)(res_kind | (emit ? 0x80 : 0));
        if (emit) my_emit++;
    }
    __syncthreads();

    // plan entries + per-output sequence number / kind
    int total = 0;
    int o = block_scan_excl(my_emit, px.ws, &total);
    for (int i = p0; i < p1; i++) {
        const bool head = is_head(i);
        uint16_t entry = (uint16_t)(fi[PADI(i)] | (ops[i] << kPlanOpShift));
        if (head) {
            entry |= kPlanHead;
            if (px.res_kind[i] & 0x80) {
                entry |= kPlanEmit;
                uint16_t rs = px.res_slot[i];
                pa.tmp_seq[in_base + o] = rs == 0xFFFF ? 0 : seq_s[rs];
                pa.tmp_kind[in_base + o] = (int8_t)(px.res_kind[i] & 0x7f);
                o++;
            }
        }
        pa.plan[in_base + i] = entry;
    }
    if (tid == 0) pa.tile_rows[tile] = total;
}

// ------------------------------------------------------------------ common key prefix of a whole merge

// *skip = number of leading key-stream bytes all rows of all runs share (from the runs' first and last rows)
__global__ void k_key_lcp(int k, KeyDesc kd, KeySrc ks, LevelView lv, int *skip) {
    __shared__ int s;
    if (threadIdx.x == 0) s = 0x7fffffff;
    __syncthreads();
    int ref = 0;
    while (ref < k && lv.count[ref] == 0) ref++;
    if ((int)threadIdx.x < 2 * k && ref < k) {
        const int r = threadIdx.x >> 1;
        if (lv.count[r] > 0) {
            const int64_t row = (threadIdx.x & 1) ? lv.row0[r] + lv.count[r] - 1 : lv.row0[r];
            atomicMin(&s, key_stream_lcp(ks, kd, ref, lv.row0[ref], r, row));
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) *skip = s == 0x7fffffff ? 0 : s;
}

// ------------------------------------------------------------------ scan of tile row counts

__global__ void k_scan(const int32_t *tile_rows, int n_tiles, int64_t *row_base, int64_t *totals) {
    __shared__ int64_t part[1024];
    int per = (n_tiles + blockDim.x - 1) / blockDim.x;
    int b = threadIdx.x * per, e = min(b + per, n_tiles);
    int64_t s = 0;
    for (int i = b; i < e; i++) s += tile_rows[i];
    part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t acc = 0;
        for (int i = 0; i < (int)blockDim.x; i++) { int64_t t = part[i]; part[i] = acc; acc += t; }
        totals[0] = acc;
    }
    __syncthreads();
    int64_t acc = part[threadIdx.x];
    for (int i = b; i < e; i++) { row_base[i] = acc; acc += tile_rows[i]; }
}

// ------------------------------------------------------------------ launchers

// once per process, whichever thread launches first: the other threads wait until the attributes are set
static std::once_flag g_attr_once;
static void set_attrs() {
    std::call_once(g_attr_once, [] {
        cudaFuncSetAttribute(k_merge_keys<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTileSmem);
        cudaFuncSetAttribute(k_merge_keys<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTileSmem);
        cudaFuncSetAttribute(k_plan<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPlanSmem);
        cudaFuncSetAttribute(k_plan<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPlanSmem);
    });
}

void launch_partition(const MergeLaunch &ml, const LevelView &lv, const uint64_t *splitter_keys,
                      const uint64_t *splitter_refs, int q, int n_tiles, int64_t *bounds) {
    int64_t total = (int64_t)(n_tiles + 1) * ml.k;
    int blocks = (int)((total + 127) / 128);
    k_partition<<<blocks, 128, 0, ml.stream>>>(ml.k, ml.key, ml.ks, lv, splitter_keys, splitter_refs, q, n_tiles,
                                                 bounds, ml.skip);
}

void launch_merge_keys(const MergeLaunch &ml, const LevelView &lv, const int64_t *bounds, int n_tiles,
                       uint64_t *sorted_keys, uint64_t *sorted_refs) {
    set_attrs();
    if (ml.key.exact)
        k_merge_keys<true><<<n_tiles, kThreads, kTileSmem, ml.stream>>>(ml.k, ml.key, ml.ks, lv, bounds, sorted_keys,
                                                                          sorted_refs, ml.err, nullptr);
    else
        k_merge_keys<false><<<n_tiles, kThreads, kTileSmem, ml.stream>>>(ml.k, ml.key, ml.ks, lv, bounds,
                                                                           sorted_keys, sorted_refs, ml.err, ml.skip);
}

void launch_key_lcp(const MergeLaunch &ml, const LevelView &lv0, int *skip) {
    k_key_lcp<<<1, 64, 0, ml.stream>>>(ml.k, ml.key, ml.ks, lv0, skip);
}

void launch_plan(const MergeLaunch &ml, const PlanArgs &pa) {
    set_attrs();
    if (ml.key.exact) k_plan<true><<<pa.n_tiles, kThreads, kPlanSmem, ml.stream>>>(ml.k, ml.key, ml.ks, pa, ml.err);
    else k_plan<false><<<pa.n_tiles, kThreads, kPlanSmem, ml.stream>>>(ml.k, ml.key, ml.ks, pa, ml.err);
}

void launch_scan(cudaStream_t stream, const int32_t *tile_rows, int n_tiles, int64_t *row_base, int64_t *totals) {
    k_scan<<<1, 1024, 0, stream>>>(tile_rows, n_tiles, row_base, totals);
}

}  // namespace pg
