// stage_bw.cu — how fast can one SM stage scattered run segments into shared memory?
//
// Mimics the load pattern of k_emit without any compute: every CTA walks `ncols` columns of its tile; per column it
// copies k segments of `seg_bytes` bytes (one per run, from k far-apart arrays) into a shared-memory stage and waits
// for them, with `depth` columns in flight.  Variants:
//   mode 0: 1-D bulk async copies (cp.async.bulk + mbarrier), one per segment          (what k_emit does)
//   mode 1: cp.async 16-byte copies issued by all threads (Ampere-style LDGSTS)
//   mode 2: plain LDG.128 -> STS.128 by all threads
// Prints achieved GB/s (bytes staged / time).  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o stage_bw stage_bw.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

template <int MODE>
__global__ void __launch_bounds__(512) k_stage(const uint8_t *base, size_t col_stride, size_t run_stride, int k, int seg_bytes,
                                               int ncols, int depth, unsigned long long *sink) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t stage_bytes = (size_t)k * seg_bytes;
    uint64_t *mbar = (uint64_t *)(smem + (size_t)depth * stage_bytes);
    if (MODE == 0 && tid == 0) {
        for (int s = 0; s < depth; s++) mbar_init(&mbar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const size_t tile_off = (size_t)blockIdx.x * seg_bytes;                 // this tile's segment inside every run
    unsigned long long acc = 0;
    auto issue = [&](int c) {
        unsigned char *dst = smem + (size_t)(c % depth) * stage_bytes;
        const uint8_t *src = base + (size_t)c * col_stride + tile_off;
        if (MODE == 0) {
            if (warp == 0) {
                if (lane == 0) mbar_expect(&mbar[c % depth], (uint32_t)stage_bytes);
                __syncwarp();
                if (lane < k) bulk_g2s(dst + (size_t)lane * seg_bytes, src + (size_t)lane * run_stride, seg_bytes, &mbar[c % depth]);
            }
        } else if (MODE == 1) {
            for (int i = tid * 16; i < (int)stage_bytes; i += 512 * 16) {
                const int r = i / seg_bytes, o = i % seg_bytes;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst + i)), "l"(src + (size_t)r * run_stride + o) : "memory");
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        } else {
            for (int i = tid * 16; i < (int)stage_bytes; i += 512 * 16) {
                const int r = i / seg_bytes, o = i % seg_bytes;
                *(uint4 *)(dst + i) = *(const uint4 *)(src + (size_t)r * run_stride + o);
            }
        }
    };
    for (int c = 0; c < depth - 1 && c < ncols; c++) issue(c);
    for (int c = 0; c < ncols; c++) {
        if (c + depth - 1 < ncols) issue(c + depth - 1);
        else if (MODE == 1) asm volatile("cp.async.commit_group;" ::: "memory");
        if (MODE == 0) mbar_wait(&mbar[c % depth], (c / depth) & 1);
        else if (MODE == 1) {
            if (depth == 2) asm volatile("cp.async.wait_group 1;" ::: "memory");
            else if (depth == 3) asm volatile("cp.async.wait_group 2;" ::: "memory");
            else asm volatile("cp.async.wait_group 3;" ::: "memory");
            __syncthreads();
        } else __syncthreads();
        // touch the stage so that the copies cannot be dropped
        acc += *(const unsigned long long *)(smem + (size_t)(c % depth) * stage_bytes + (tid * 8) % stage_bytes);
        __syncthreads();
    }
    if (acc == 0x1234567) *sink = acc;
}

int main(int argc, char **argv) {
    const int k = argc > 1 ? atoi(argv[1]) : 16, seg_bytes = argc > 2 ? atoi(argv[2]) : 2048;
    const int ncols = argc > 3 ? atoi(argv[3]) : 52, depth = argc > 4 ? atoi(argv[4]) : 2, ctas_per_sm = argc > 5 ? atoi(argv[5]) : 2;
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int tiles = sms * ctas_per_sm * 24;
    const size_t run_stride = (size_t)tiles * seg_bytes + 4096, col_stride = run_stride * k;
    const size_t total = col_stride * ncols;
    uint8_t *d = nullptr;
    unsigned long long *sink = nullptr;
    if (cudaMalloc(&d, total) != cudaSuccess) { printf("alloc of %zu bytes failed\n", total); return 1; }
    cudaMalloc(&sink, 8);
    cudaMemset(d, 1, total);
    const size_t smem = (size_t)depth * k * seg_bytes + 64;
    for (int mode = 0; mode < 3; mode++) {
        auto kern = mode == 0 ? k_stage<0> : mode == 1 ? k_stage<1> : k_stage<2>;
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int it = 0; it < 2; it++) {
            cudaEventRecord(e0);
            kern<<<tiles, 512, smem>>>(d, col_stride, run_stride, k, seg_bytes, ncols, depth, sink);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
        }
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        cudaError_t e = cudaGetLastError();
        const double gb = (double)tiles * ncols * k * seg_bytes / 1e9;
        printf("k=%d seg=%dB cols=%d depth=%d ctas/SM=%d smem=%zuKB mode=%d (%s): %.3f ms  %.0f GB/s  %s\n", k, seg_bytes, ncols, depth,
               ctas_per_sm, smem >> 10, mode, mode == 0 ? "cp.async.bulk" : mode == 1 ? "cp.async 16B" : "LDG.128+STS", ms, gb / (ms * 1e-3),
               e == cudaSuccess ? "" : cudaGetErrorString(e));
    }
    return 0;
}
