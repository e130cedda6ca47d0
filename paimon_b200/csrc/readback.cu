// readback.cu — small device -> host reads that do not wait behind large DMA copies.
//
// A decode + merge step has a handful of tiny read-backs (page counts, exact payload sizes, the output row count,
// error words, Parquet footers of device-resident files).  Issued as cudaMemcpyAsync they go through the
// device -> host copy engine, which serves its queue in order: when another thread is reading a multi-GB merged batch
// back (the end-to-end pipeline of bench.py, or any reader that fetches bucket i while bucket i + 1 merges), every one
// of them waits for hundreds of milliseconds.  Here a few threads of a kernel store the bytes into page-locked,
// device-mapped host memory instead; the host reads them after synchronising the stream.
#include <algorithm>
#include <cstring>
#include <stdexcept>
#include <utility>
#include <vector>

#include "pg_internal.h"

namespace pg {

namespace {

struct Staging {
    uint8_t *h = nullptr, *d = nullptr;
    size_t cap = 0;
    ~Staging() { if (h) cudaFreeHost(h); }
};
thread_local Staging g_stage;
constexpr size_t kStageBytes = 4u << 20;

__global__ void k_small_read(const uint8_t *src, uint8_t *dst, size_t n) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
    if ((((uintptr_t)src | (uintptr_t)dst) & 3) == 0) {
        const size_t n4 = n >> 2;
        for (size_t i = t; i < n4; i += step) ((uint32_t *)dst)[i] = ((const uint32_t *)src)[i];
        for (size_t i = (n4 << 2) + t; i < n; i += step) dst[i] = src[i];
    } else {
        for (size_t i = t; i < n; i += step) dst[i] = src[i];
    }
}

}  // namespace

// host -> device: the same idea in the other direction.  Job tables and descriptors (pageable host vectors) are
// copied into a device-mapped page-locked ring and a kernel moves them to their device buffer, so that they do not
// queue behind an asynchronous upload of the next section's files on the host -> device copy engine.
namespace {
struct Ring {
    uint8_t *h = nullptr, *d = nullptr;
    size_t cap = 0, off = 0;
    ~Ring() { if (h) cudaFreeHost(h); }
};
constexpr size_t kRingBytes = 8u << 20;
}  // namespace

pg_status small_h2d(void *dev_dst, const void *host_src, size_t n, cudaStream_t stream) {
    if (n == 0) return PG_OK;
    thread_local std::vector<std::pair<cudaStream_t, Ring *>> rings;       // one ring per (thread, stream)
    Ring *r = nullptr;
    for (auto &p : rings) if (p.first == stream) r = p.second;
    if (!r) {
        r = new Ring();
        if (cudaHostAlloc((void **)&r->h, kRingBytes, cudaHostAllocMapped) == cudaSuccess &&
            cudaHostGetDevicePointer((void **)&r->d, r->h, 0) == cudaSuccess)
            r->cap = kRingBytes;
        else
            cudaGetLastError();
        rings.push_back({stream, r});
    }
    if (n > r->cap) {
        PG_CUDA(cudaMemcpyAsync(dev_dst, host_src, n, cudaMemcpyHostToDevice, stream));
        return PG_OK;
    }
    size_t off = (r->off + 15) & ~(size_t)15;
    if (off + n > r->cap) {
        PG_CUDA(cudaStreamSynchronize(stream));        // every kernel that read the ring so far is done
        off = 0;
    }
    memcpy(r->h + off, host_src, n);
    const int blocks = (int)std::min<size_t>(128, (n + 4095) / 4096);
    k_small_read<<<blocks, 256, 0, stream>>>(r->d + off, (uint8_t *)dev_dst, n);
    r->off = off + n;
    return PG_OK;
}

pg_status SmallReads::add(void *host_dst, const void *dev_src, size_t n) {
    if (n == 0) return PG_OK;
    if (!g_stage.h) {
        if (cudaHostAlloc((void **)&g_stage.h, kStageBytes, cudaHostAllocMapped) == cudaSuccess &&
            cudaHostGetDevicePointer((void **)&g_stage.d, g_stage.h, 0) == cudaSuccess)
            g_stage.cap = kStageBytes;
        else
            cudaGetLastError();                        // (no mapped memory: plain copies below)
    }
    const size_t off = (used_ + 15) & ~(size_t)15;
    if (off + n > g_stage.cap) {
        PG_CUDA(cudaMemcpyAsync(host_dst, dev_src, n, cudaMemcpyDeviceToHost, stream_));
        return PG_OK;
    }
    const int blocks = (int)std::min<size_t>(64, (n + 4095) / 4096);
    k_small_read<<<blocks, 256, 0, stream_>>>((const uint8_t *)dev_src, g_stage.d + off, n);
    items_.push_back(Item{host_dst, off, n});
    used_ = off + n;
    return PG_OK;
}

pg_status SmallReads::finish(cudaEvent_t after) {
    if (after) PG_CUDA(cudaEventSynchronize(after));
    else PG_CUDA(cudaStreamSynchronize(stream_));
    for (const Item &it : items_) memcpy(it.dst, g_stage.h + it.off, it.n);
    items_.clear();
    used_ = 0;
    return PG_OK;
}

DeviceRanges::DeviceRanges(cudaStream_t s, const pg_file_desc *section, int n_files) : section(section), rb(s) {
    for (int f = 0; f < n_files; f++)
        if (section[f].mem == PG_MEM_DEVICE) { files.push_back(f); sizes.push_back((uint64_t)section[f].size); }
}

void DeviceRanges::read(int file, uint64_t off, uint64_t n, uint8_t *dst) {
    if (st == PG_OK) st = rb.add(dst, section[files[file]].bytes + off, (size_t)n);
}

void DeviceRanges::flush() {
    if (st == PG_OK) st = rb.finish();
    if (st != PG_OK) throw std::runtime_error("a read-back of the file metadata failed");
}

}  // namespace pg
