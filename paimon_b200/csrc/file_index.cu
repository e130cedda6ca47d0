// file_index.cu — the bloom-filter file index of a data file (pg_bloom_filter_build): one BloomFilter64 per indexed
// column over rows [row0, row0 + n_rows) of a merge or run handle, built in device memory and serialized the way
// BloomFilterFileIndex.Writer.serializedBytes does (the hash function count as a big-endian int32, then the bit set).
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "device_utils.cuh"
#include "encoded_file.h"
#include "xxhash64_device.cuh"

namespace pg {

struct BloomJob {
    const void *data;
    const int32_t *offsets;      // var-len columns
    const uint8_t *validity;     // NULL = no nulls
    uint32_t *bits;              // the bit set as little-endian words: bit p is bit p & 31 of word p >> 5
    uint32_t num_bits;
    int32_t k;
    int32_t type;                // pg_type (BOOLEAN is refused before the launch)
    int32_t width;               // bytes, 0 = var-len
};

// one thread per value: skip NULLs, hash by the physical type (FastHash), set the k bits (BloomFilter64.addHash).
// blockIdx.y = the job (column), the rows are strided over blockIdx.x.
__global__ void __launch_bounds__(256) k_bloom_build(const BloomJob *jobs, int64_t row0, int64_t n_rows) {
    const BloomJob j = jobs[blockIdx.y];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rows; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = row0 + i;
        if (!valid_bit(j.validity, row)) continue;
        int64_t h;
        if (j.width == 0) {
            const int32_t a = j.offsets[row], b = j.offsets[row + 1];
            h = (int64_t)fi::xxh64((const uint8_t *)j.data + a, b - a);
        } else {
            const uint64_t v = load_fixed(j.data, j.width, row);
            h = fi::wang64(j.type == PG_FLOAT    ? fi::float_key((uint32_t)v)
                           : j.type == PG_DOUBLE ? fi::double_key(v)
                                                 : sext(v, j.width));
        }
        for (int t = 1; t <= j.k; t++) {
            const uint32_t p = fi::bloom_bit(h, t, j.num_bits);
            atomicOr(j.bits + (p >> 5), 1u << (p & 31));
        }
    }
}

}  // namespace pg

using namespace pg;

extern "C" {

pg_status pg_bloom_filter_size(int32_t items, double fpp, int64_t *bytes, int32_t *num_hash_functions) {
    if (items <= 0 || !(fpp > 0 && fpp < 1))
        return fail(PG_ERR_INVALID, "bloom filter: items must be > 0 and fpp inside (0, 1), got items " +
                                        std::to_string(items) + ", fpp " + std::to_string(fpp));
    int32_t num_bits = 0, k = 0;
    if (!fi::bloom_sizing(items, fpp, &num_bits, &k))
        return fail(PG_ERR_INVALID, "bloom filter: items " + std::to_string(items) + " at fpp " + std::to_string(fpp) +
                                        " need a bit set of 2^31 bits or more");
    if (bytes) *bytes = 4 + (int64_t)num_bits / 8;
    if (num_hash_functions) *num_hash_functions = k;
    return PG_OK;
}

pg_status pg_bloom_filter_build(uint64_t source, int64_t row0, int64_t n_rows, int32_t n,
                                const pg_bloom_filter_spec *specs, uint8_t *const *host_out, const int64_t *capacity) {
    static const char *who = "bloom filter";
    if (n < 0 || (n > 0 && (!specs || !host_out || !capacity))) return fail(PG_ERR_INVALID, "bloom filter: bad arguments");
    std::vector<int32_t> num_bits(n), k(n);
    for (int i = 0; i < n; i++) {
        int64_t bytes = 0;
        pg_status st = pg_bloom_filter_size(specs[i].items, specs[i].fpp, &bytes, &k[i]);
        if (st) return st;
        num_bits[i] = (int32_t)((bytes - 4) * 8);
        if (!host_out[i] || capacity[i] < bytes)
            return fail(PG_ERR_INVALID, "bloom filter: the output of spec " + std::to_string(i) + " holds " +
                                            std::to_string(capacity[i]) + " bytes, the filter needs " + std::to_string(bytes));
    }
    BatchColumns batch;
    pg_status st = encode_source(source, who, row0, &n_rows, &batch);
    if (st) return st;
    const Schema &s = *batch.schema;
    std::vector<BloomJob> jobs(n);
    std::vector<size_t> at(n);
    size_t total = 0;
    for (int i = 0; i < n; i++) {
        const int c = specs[i].column;
        if (c < 0 || c >= s.n_cols()) return fail(PG_ERR_INVALID, "bloom filter: column " + std::to_string(c) + " out of range");
        const int t = s.field(c).type;
        if (t == PG_BOOL) return fail(PG_ERR_UNSUPPORTED, "bloom filter: column " + std::to_string(c) + " is BOOLEAN");
        const DevColumn &dc = batch.cols[c];
        jobs[i] = BloomJob{dc.data, dc.offsets, dc.validity, nullptr, (uint32_t)num_bits[i], k[i], t, type_width(t)};
        at[i] = total;
        total += align256(((size_t)num_bits[i] + 31) / 32 * 4);
    }
    if (n == 0) return PG_OK;
    Scratch scratch(0);
    uint8_t *d_bits = (uint8_t *)scratch.take(total);
    BloomJob *d_jobs = (BloomJob *)scratch.take(sizeof(BloomJob) * n);
    if (!d_bits || !d_jobs) return oom(who, "the bit sets", total);
    for (int i = 0; i < n; i++) jobs[i].bits = (uint32_t *)(d_bits + at[i]);
    PG_CUDA(cudaMemsetAsync(d_bits, 0, total, 0));
    PG_CUDA(cudaMemcpy(d_jobs, jobs.data(), sizeof(BloomJob) * n, cudaMemcpyHostToDevice));
    if (n_rows > 0) {
        const int64_t blocks = std::min<int64_t>((n_rows + 255) / 256, 4096);
        k_bloom_build<<<dim3((unsigned)blocks, (unsigned)n), 256>>>(d_jobs, row0, n_rows);
        PG_CUDA(cudaGetLastError());
    }
    for (int i = 0; i < n; i++) {
        const uint32_t kk = (uint32_t)k[i];
        const uint8_t be[4] = {(uint8_t)(kk >> 24), (uint8_t)(kk >> 16), (uint8_t)(kk >> 8), (uint8_t)kk};
        memcpy(host_out[i], be, 4);
        PG_CUDA(cudaMemcpy(host_out[i] + 4, d_bits + at[i], (size_t)num_bits[i] / 8, cudaMemcpyDeviceToHost));
    }
    return PG_OK;
}

}  // extern "C"
