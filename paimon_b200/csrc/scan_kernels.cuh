// scan_kernels.cuh — device-wide inclusive scan of an int32 array in place (lengths -> offsets), three small kernels.
// Included by the Parquet and the ORC decoder (static: one copy per translation unit).
#pragma once

#include "device_utils.cuh"

namespace pg {

// ---- device-wide inclusive scan of int32 (three small kernels; used by the deletion-vector filter)
static __global__ void k_scan_block_sums(const int32_t *data, int64_t n, int64_t *block_sums) {
    __shared__ int64_t sh[256];
    int64_t b0 = (int64_t)blockIdx.x * 4096;
    int64_t s = 0;
    for (int i = threadIdx.x; i < 4096 && b0 + i < n; i += blockDim.x) s += data[b0 + i];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int d = 128; d > 0; d >>= 1) { if (threadIdx.x < d) sh[threadIdx.x] += sh[threadIdx.x + d]; __syncthreads(); }
    if (threadIdx.x == 0) block_sums[blockIdx.x] = sh[0];
}
static __global__ void __launch_bounds__(1024) k_scan_block_prefix(int64_t *block_sums, int64_t n_blocks, int32_t *err) {
    // exclusive scan of the block sums by one CTA: every thread owns a contiguous slice
    __shared__ int64_t part[1024];
    const int64_t per = (n_blocks + blockDim.x - 1) / blockDim.x;
    const int64_t b = threadIdx.x * per, e = min(b + per, n_blocks);
    int64_t s = 0;
    for (int64_t i = b; i < e; i++) s += block_sums[i];
    part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t acc = 0;
        for (int i = 0; i < (int)blockDim.x; i++) { const int64_t t = part[i]; part[i] = acc; acc += t; }
        if (acc > 0x7fffffffLL) atomicCAS(err, KERR_NONE, KERR_OFFSET_OVERFLOW);
    }
    __syncthreads();
    int64_t acc = part[threadIdx.x];
    for (int64_t i = b; i < e; i++) { const int64_t t = block_sums[i]; block_sums[i] = acc; acc += t; }
}
static __global__ void __launch_bounds__(256) k_scan_apply(int32_t *data, int64_t n, const int64_t *block_sums) {
    __shared__ int ws[34];
    int64_t b0 = (int64_t)blockIdx.x * 4096;
    int carry = (int)block_sums[blockIdx.x];
    for (int base = 0; base < 4096; base += 256) {
        int64_t i = b0 + base + threadIdx.x;
        int v = i < n ? data[i] : 0;
        int tot = 0;
        int ex = block_scan_excl(v, ws, &tot);
        if (i < n) data[i] = carry + ex + v;
        carry += tot;
    }
}


// data[0..n) -> its inclusive scan, in place.  `sums` = scratch of n / 4096 + 2 int64.
static inline void launch_inclusive_scan(int32_t *data, int64_t n, int64_t *sums, int32_t *err, cudaStream_t st) {
    if (n <= 0) return;
    const int64_t nb = (n + 4095) / 4096;
    k_scan_block_sums<<<(unsigned)nb, 256, 0, st>>>(data, n, sums);
    k_scan_block_prefix<<<1, 1024, 0, st>>>(sums, nb, err);
    k_scan_apply<<<(unsigned)nb, 256, 0, st>>>(data, n, sums);
}

// offsets[1..n] hold lengths, offsets[0] = 0: turn them into Arrow offsets
static inline void launch_offsets_scan(int32_t *offsets, int64_t n, int64_t *sums, int32_t *err, cudaStream_t st) {
    launch_inclusive_scan(offsets + 1, n, sums, err, st);
}

}  // namespace pg
