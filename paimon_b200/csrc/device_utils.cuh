// Device-side helpers shared by merge.cu and emit.cu.
#pragma once

#include "pg_internal.h"

namespace pg {

__device__ __forceinline__ int warp_scan_incl(int v) {
    int lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int n = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += n;
    }
    return v;
}

// exclusive scan over the block; *total receives the block sum.  `ws` = 33 ints of shared memory.
__device__ __forceinline__ int block_scan_excl(int v, int *ws, int *total) {
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int incl = warp_scan_incl(v);
    if (lane == 31) ws[w] = incl;
    __syncthreads();
    if (w == 0) {
        int x = lane < nw ? ws[lane] : 0;
        int xi = warp_scan_incl(x);
        ws[lane] = xi - x;
        if (lane == 31) ws[32] = xi;
    }
    __syncthreads();
    int res = ws[w] + incl - v;
    *total = ws[32];
    __syncthreads();
    return res;
}

__device__ __forceinline__ bool valid_bit(const uint8_t *bm, int64_t row) {
    return bm == nullptr || ((bm[row >> 3] >> (row & 7)) & 1);
}

__device__ __forceinline__ bool kind_is_retract(int kind) {   // RowKind.java:101-103
    return kind == PG_UPDATE_BEFORE || kind == PG_DELETE;
}

__device__ __forceinline__ int run_of_slot(const int *seg, int k, int slot) {
    int r = 0;
    while (r + 1 < k && seg[r + 1] <= slot) r++;
    return r;
}

__device__ __forceinline__ uint64_t load_fixed(const void *data, int width, int64_t row) {
    switch (width) {
        case 1: return ((const uint8_t *)data)[row];
        case 2: return ((const uint16_t *)data)[row];
        case 4: return ((const uint32_t *)data)[row];
        default: return ((const uint64_t *)data)[row];
    }
}
__device__ __forceinline__ void store_fixed(void *data, int width, int64_t row, uint64_t v) {
    switch (width) {
        case 1: ((uint8_t *)data)[row] = (uint8_t)v; break;
        case 2: ((uint16_t *)data)[row] = (uint16_t)v; break;
        case 4: ((uint32_t *)data)[row] = (uint32_t)v; break;
        default: ((uint64_t *)data)[row] = v; break;
    }
}

// Float.compare / Double.compare total order (InternalRowUtils.java:409-414)
__device__ __forceinline__ int java_double_compare(double a, double b) {
    if (a < b) return -1;
    if (a > b) return 1;
    long long x = __double_as_longlong(a), y = __double_as_longlong(b);
    if (a != a) x = 0x7ff8000000000000LL;
    if (b != b) y = 0x7ff8000000000000LL;
    return x == y ? 0 : (x < y ? -1 : 1);
}
__device__ __forceinline__ int java_float_compare(float a, float b) {
    if (a < b) return -1;
    if (a > b) return 1;
    int x = __float_as_int(a), y = __float_as_int(b);
    if (a != a) x = 0x7fc00000;
    if (b != b) y = 0x7fc00000;
    return x == y ? 0 : (x < y ? -1 : 1);
}

__device__ __forceinline__ int64_t sext(uint64_t v, int width) {
    switch (width) {
        case 1: return (int8_t)v;
        case 2: return (int16_t)v;
        case 4: return (int32_t)v;
        default: return (int64_t)v;
    }
}

// a (fn) b for SUM / PRODUCT and their retractions; integer results wrap exactly like the Java casts
// (FieldSumAgg.java:57-74, FieldProductAgg.java); fp uses the IEEE round-to-nearest single operation
// (no FMA contraction) so that a left fold is bit-identical to the JVM's
__device__ __forceinline__ uint64_t arith(int type, int width, int fn, uint64_t a, uint64_t b, int32_t *err) {
    // fn: 0 add, 1 sub, 2 mul, 3 div
    if (type == PG_DOUBLE) {
        double x = __longlong_as_double((long long)a), y = __longlong_as_double((long long)b), r;
        r = fn == 0 ? __dadd_rn(x, y) : fn == 1 ? __dsub_rn(x, y) : fn == 2 ? __dmul_rn(x, y) : __ddiv_rn(x, y);
        return (uint64_t)__double_as_longlong(r);
    }
    if (type == PG_FLOAT) {
        float x = __int_as_float((int)a), y = __int_as_float((int)b), r;
        r = fn == 0 ? __fadd_rn(x, y) : fn == 1 ? __fsub_rn(x, y) : fn == 2 ? __fmul_rn(x, y) : __fdiv_rn(x, y);
        return (uint32_t)__float_as_int(r);
    }
    int64_t x = sext(a, width), y = sext(b, width);
    uint64_t r;
    if (fn == 0) r = (uint64_t)x + (uint64_t)y;
    else if (fn == 1) r = (uint64_t)x - (uint64_t)y;
    else if (fn == 2) r = (uint64_t)x * (uint64_t)y;
    else {
        if (y == 0) { atomicCAS(err, KERR_NONE, KERR_DIV_ZERO); r = 0; }
        else if (y == -1) r = 0ull - (uint64_t)x;
        else r = (uint64_t)(x / y);
    }
    return r;        // store_fixed truncates to the column width == Java's narrowing cast
}

// ---- DECIMAL(p, s) sum / product on unscaled int64 values (FieldSumAgg / FieldProductAgg on DecimalType)
// sum, subtract: DecimalUtils.add / subtract (DecimalUtils.java:52-87): exact int64; on overflow the BigDecimal result
//   has more than 18 digits and Decimal.fromBigDecimal gives NULL.  A result over p digits that fits int64 is kept
//   (fromUnscaledLong does not check the precision).
// product: round_half_up(a * b / 10^s), NULL over p digits (FieldProductAgg.java:47-58, Decimal.java:182-193).
// retract of a product: BigDecimal.divide is exact (throws when the quotient does not terminate, or on a zero
//   divisor); the result is round_half_up(a * 10^s / b), NULL over p digits (FieldProductAgg.java:95-106).
// negate (retract of a sum into a NULL accumulator): fromBigDecimal(-a), NULL over p digits (FieldSumAgg.java:140-143).
// |a|, |b| <= 2^63 and 10^s <= 10^18, so a * b and a * 10^s fit __int128.
__device__ __forceinline__ unsigned __int128 dec_pow10(int e) {
    unsigned __int128 r = 1;
    for (int i = 0; i < e; i++) r *= 10u;
    return r;
}
// round_half_up(n / d) for d > 0: ties away from zero (RoundingMode.HALF_UP)
__device__ __forceinline__ __int128 dec_div_half_up(__int128 n, unsigned __int128 d) {
    const bool neg = n < 0;
    const unsigned __int128 m = neg ? (unsigned __int128)0 - (unsigned __int128)n : (unsigned __int128)n;
    unsigned __int128 q = m / d;
    const unsigned __int128 r = m - q * d;
    if (r >= d - r) q += 1;
    return neg ? -(__int128)q : (__int128)q;
}
__device__ __forceinline__ bool dec_fits(__int128 v, int precision) {     // BigDecimal.precision() <= p
    const unsigned __int128 m = v < 0 ? (unsigned __int128)0 - (unsigned __int128)v : (unsigned __int128)v;
    return m < dec_pow10(precision);
}
// fn: 0 add, 1 sub, 2 mul, 3 div, 4 negate a
struct DecimalResult {
    uint64_t value;      // unscaled
    bool valid;          // false = NULL
};
__device__ __forceinline__ DecimalResult decimal_arith(int decimal, int fn, uint64_t ua, uint64_t ub, int32_t *err) {
    const int precision = decimal >> 8, scale = decimal & 0xff;
    const int64_t a = (int64_t)ua, b = (int64_t)ub;
    __int128 r;
    if (fn == 0 || fn == 1) {
        const uint64_t u = fn == 0 ? ua + ub : ua - ub;
        const int64_t x = (int64_t)u;
        const bool overflow = fn == 0 ? ((a ^ x) & (b ^ x)) < 0 : ((a ^ b) & (a ^ x)) < 0;
        return DecimalResult{overflow ? 0 : u, !overflow};
    }
    if (fn == 4) {
        r = -(__int128)a;
    } else if (fn == 2) {
        r = dec_div_half_up((__int128)a * (__int128)b, dec_pow10(scale));
    } else {
        if (b == 0) {
            atomicCAS(err, KERR_NONE, a == 0 ? KERR_DEC_DIV_UNDEFINED : KERR_DEC_DIV_ZERO);
            return DecimalResult{0, false};
        }
        // a / b terminates iff b / gcd(a, b) has no prime factor other than 2 and 5
        const uint64_t mb = b < 0 ? 0ull - ub : ub;
        uint64_t x = a < 0 ? 0ull - ua : ua, y = mb;
        while (x != 0) { const uint64_t t = y % x; y = x; x = t; }
        uint64_t den = mb / y;
        while (den % 2 == 0) den /= 2;
        while (den % 5 == 0) den /= 5;
        if (den != 1) {
            atomicCAS(err, KERR_NONE, KERR_DEC_NON_TERMINATING);
            return DecimalResult{0, false};
        }
        const __int128 n = (__int128)a * (__int128)dec_pow10(scale);
        r = dec_div_half_up(b < 0 ? -n : n, (unsigned __int128)mb);
    }
    const bool fits = dec_fits(r, precision);
    return DecimalResult{fits ? (uint64_t)(int64_t)r : 0, fits};
}

__device__ __forceinline__ uint64_t negate_fixed(int type, int width, uint64_t a) {
    if (type == PG_DOUBLE) return a ^ 0x8000000000000000ull;
    if (type == PG_FLOAT) return (uint32_t)a ^ 0x80000000u;
    return 0ull - (uint64_t)sext(a, width);
}

__device__ __forceinline__ int compare_fixed(int type, int width, uint64_t a, uint64_t b) {
    if (type == PG_DOUBLE)
        return java_double_compare(__longlong_as_double((long long)a), __longlong_as_double((long long)b));
    if (type == PG_FLOAT) return java_float_compare(__int_as_float((int)a), __int_as_float((int)b));
    int64_t x = sext(a, width), y = sext(b, width);
    return x < y ? -1 : x > y ? 1 : 0;
}

__device__ __forceinline__ int bytes_compare(const uint8_t *a, int la, const uint8_t *b, int lb) {
    int n = min(la, lb);
    for (int i = 0; i < n; i++) {
        int d = (int)a[i] - (int)b[i];
        if (d) return d;
    }
    return la - lb;
}

// ---- mbarrier + bulk async copy (TMA 1-D) ----

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}
// global -> shared bulk copy; dst/src 16-byte aligned, bytes a multiple of 16
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

}  // namespace pg
