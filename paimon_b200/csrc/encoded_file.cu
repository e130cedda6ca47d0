// encoded_file.cu — the back end the compaction output encoders (parquet_encode.cu, orc_encode.cu) share; what it
// holds is listed in encoded_file.h.
#include <algorithm>
#include <memory>
#include <string>

#include "device_utils.cuh"
#include "encoded_file.h"
#include "zstd_encode_device.cuh"

namespace pg {

// per job (one CTA): min / max of the non-null values of a fixed-width numeric column, as int64 / double bit patterns
// (FLOAT / DOUBLE: of the non-NaN values, whichever zero comes first; FileStats applies the zero rule), whether a
// non-null value is NaN; also used for the sequence number range and the delete count (kind column)
__global__ void k_pw_stats(const EncColumn *cols, const StatJob *jobs, int64_t *out /* [job][kStatWords] */) {
    const StatJob j = jobs[blockIdx.x];
    const EncColumn c = cols[j.col];
    const bool fp = c.type == PG_FLOAT || c.type == PG_DOUBLE;
    int64_t imin = INT64_MAX, imax = INT64_MIN;
    double dmin = INFINITY, dmax = -INFINITY;
    long long nn = 0, retr = 0;
    bool nan_seen = false;
    for (int64_t i = threadIdx.x; i < j.n_rows; i += blockDim.x) {
        const int64_t row = j.row0 + i;
        if (c.validity && !valid_bit(c.validity, row)) continue;
        nn++;
        if (c.width == 0) continue;
        if (fp) {
            double x = c.type == PG_FLOAT ? (double)((const float *)c.data)[row] : ((const double *)c.data)[row];
            if (x != x) { nan_seen = true; continue; }
            dmin = fmin(dmin, x); dmax = fmax(dmax, x);
        } else {
            int64_t x = sext(load_fixed(c.data, c.width, row), c.width);
            if (c.type == PG_BOOL) x = x != 0;
            imin = min(imin, x); imax = max(imax, x);
            if (c.type == PG_INT8 && (x == 1 || x == 3)) retr++;        // RowKind retracts, used for _VALUE_KIND
        }
    }
    __shared__ long long s_i[2], s_n[2];
    __shared__ double s_d[2];
    __shared__ int s_nan;
    if (threadIdx.x == 0) { s_i[0] = INT64_MAX; s_i[1] = INT64_MIN; s_d[0] = INFINITY; s_d[1] = -INFINITY; s_n[0] = s_n[1] = 0; s_nan = 0; }
    __syncthreads();
    if (fp) {
        // doubles: order-preserving via atomicMin/Max on the transformed bit pattern is overkill here: serialise
        // per warp leader through a CAS loop on the shared doubles
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            dmin = fmin(dmin, __shfl_xor_sync(0xffffffffu, dmin, d));
            dmax = fmax(dmax, __shfl_xor_sync(0xffffffffu, dmax, d));
        }
        if ((threadIdx.x & 31) == 0) {
            unsigned long long *pmin = (unsigned long long *)&s_d[0], *pmax = (unsigned long long *)&s_d[1];
            unsigned long long old = *pmin;
            while (dmin < __longlong_as_double((long long)old)) {
                unsigned long long prev = atomicCAS(pmin, old, (unsigned long long)__double_as_longlong(dmin));
                if (prev == old) break;
                old = prev;
            }
            old = *pmax;
            while (dmax > __longlong_as_double((long long)old)) {
                unsigned long long prev = atomicCAS(pmax, old, (unsigned long long)__double_as_longlong(dmax));
                if (prev == old) break;
                old = prev;
            }
        }
        if (nan_seen) s_nan = 1;
    } else {
        atomicMin(&s_i[0], (long long)imin);
        atomicMax(&s_i[1], (long long)imax);
    }
    atomicAdd((unsigned long long *)&s_n[0], (unsigned long long)nn);
    atomicAdd((unsigned long long *)&s_n[1], (unsigned long long)retr);
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t *o = out + kStatWords * (int64_t)blockIdx.x;
        if (fp) { o[0] = __double_as_longlong(s_d[0]); o[1] = __double_as_longlong(s_d[1]); }
        else { o[0] = s_i[0]; o[1] = s_i[1]; }
        o[2] = s_n[0];
        o[3] = s_n[1];
        o[4] = s_nan;
    }
}

// host-built pieces of the file (headers, level prefixes, footers) -> their places in the device image
struct PatchJob { int64_t dst; int32_t src, len; };
__global__ void k_pw_patch(const PatchJob *jobs, int n, const uint8_t *bytes, uint8_t *file) {
    const int j = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (j >= n) return;
    const PatchJob pj = jobs[j];
    for (int i = lane; i < pj.len; i += 32) file[pj.dst + i] = bytes[pj.src + i];
}

// ------------------------------------------------------------------ zstd framing (ZstdFrames)

struct ZsBlockJob {
    int64_t src;                  // offset of the block in the image
    int64_t out;                  // offset of its payload slot (n bytes)
    int64_t seq;                  // first sequence slot (n / 4 + 1 of them)
    int32_t n;                    // input bytes (<= 128 KiB)
    int32_t body;                 // its body
};
struct ZsBody {
    int64_t src, bytes;           // offset in the image, bytes
    int32_t first_block, n_blocks;
};

constexpr size_t kZsSmem = (sizeof(int32_t) << zs::kHashLog) + sizeof(zs::EncWork);

__global__ void __launch_bounds__(32)
k_zs_block(const ZsBlockJob *jobs, const uint8_t *img, uint8_t *out, zs::Seq *seqs, uint8_t *lits, int2 *res) {
    extern __shared__ __align__(16) uint8_t zs_smem[];
    int32_t *htab = (int32_t *)zs_smem;
    zs::EncWork &W = *(zs::EncWork *)(zs_smem + (sizeof(int32_t) << zs::kHashLog));
    const ZsBlockJob j = jobs[blockIdx.x];
    const zs::BlockOut r = zs::compress_block(img + j.src, j.n, out + j.out, htab, seqs + j.seq, lits + j.src, W);
    if (threadIdx.x == 0) res[blockIdx.x] = make_int2(r.type, r.size);
}

// per body: where each block's header goes inside the frame, and the frame size
__global__ void k_zs_frame_sizes(const ZsBody *bodies, int n_bodies, const int2 *res, int32_t *boff, int64_t *frame_bytes) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_bodies) return;
    const ZsBody b = bodies[p];
    int64_t off = zs::frame_header_size((uint64_t)b.bytes);
    for (int k = 0; k < b.n_blocks; k++) {
        boff[b.first_block + k] = (int32_t)off;
        off += 3 + res[b.first_block + k].y;
    }
    frame_bytes[p] = off;
}

// one CTA per block, at its body's file offset: the frame header (first block of a body), the block header and the
// payload; or, for a body stored raw (raw != NULL and raw[body] set), the block's input bytes as they are
__global__ void k_zs_gather(const ZsBlockJob *jobs, const ZsBody *bodies, const int2 *res, const int32_t *boff,
                            const int64_t *dst_off, const uint8_t *raw, const uint8_t *img, const uint8_t *out,
                            uint8_t *file) {
    const ZsBlockJob j = jobs[blockIdx.x];
    const ZsBody b = bodies[j.body];
    uint8_t *frame = file + dst_off[j.body];
    if (raw && raw[j.body]) {
        uint8_t *dst = frame + (j.src - b.src);
        for (int i = threadIdx.x; i < j.n; i += blockDim.x) dst[i] = img[j.src + i];
        return;
    }
    const int2 r = res[blockIdx.x];
    uint8_t *dst = frame + boff[blockIdx.x];
    if (threadIdx.x == 0) {
        if ((int)blockIdx.x == b.first_block) zs::write_frame_header(frame, (uint64_t)b.bytes);
        zs::write_block_header(dst, (int)blockIdx.x == b.first_block + b.n_blocks - 1, r.x,
                               r.x == 2 ? (uint32_t)r.y : (uint32_t)j.n);
    }
    const uint8_t *pay = r.x == 0 ? img + j.src : out + j.out;
    for (int i = threadIdx.x; i < r.y; i += blockDim.x) dst[3 + i] = pay[i];
}

// ------------------------------------------------------------------ host side

static Table<EncodedFile> g_enc(6);

void launch_pw_stats(const EncColumn *cols, const StatJob *jobs, int n_jobs, int64_t *out) {
    if (n_jobs) k_pw_stats<<<(unsigned)n_jobs, 256>>>(cols, jobs, out);
}

pg_status patch(Scratch &scratch, const std::vector<Part> &parts, uint8_t *dst, const char *what) {
    if (parts.empty()) return PG_OK;
    std::vector<PatchJob> jobs;
    std::vector<uint8_t> bytes;
    for (const Part &p : parts) {
        if (bytes.size() + p.second.size() > 0x7fffffffull) return fail(PG_ERR_UNSUPPORTED, "parquet encode: too many header bytes");
        jobs.push_back(PatchJob{p.first, (int32_t)bytes.size(), (int32_t)p.second.size()});
        bytes.insert(bytes.end(), p.second.begin(), p.second.end());
    }
    PatchJob *d_jobs = (PatchJob *)scratch.take(sizeof(PatchJob) * jobs.size() + 16);
    uint8_t *d_bytes = (uint8_t *)scratch.take(bytes.size() + 16);
    if (!d_jobs || !d_bytes) return fail(PG_ERR_CUDA, std::string("parquet encode: out of device memory for ") + what);
    PG_CUDA(cudaMemcpy(d_jobs, jobs.data(), sizeof(PatchJob) * jobs.size(), cudaMemcpyHostToDevice));
    PG_CUDA(cudaMemcpy(d_bytes, bytes.data(), bytes.size(), cudaMemcpyHostToDevice));
    k_pw_patch<<<(unsigned)((jobs.size() * 32 + 127) / 128), 128>>>(d_jobs, (int)jobs.size(), d_bytes, dst);
    return PG_OK;
}

pg_status encode_source(uint64_t source, const char *who, int64_t row0, int64_t *n_rows, BatchColumns *out) {
    pg_status st = ensure_device();
    if (st) return st;
    if ((st = batch_columns(source, out))) return st;
    for (int c = 0; c < out->schema->n_cols() && out->n_rows > 0; c++)
        if (!out->cols[c].data && !out->cols[c].offsets)
            return fail(PG_ERR_INVALID, std::string(who) + ": the batch was produced under a read-type projection and has "
                                        "no column " + std::to_string(c) + "; a data file needs every column");
    if (*n_rows < 0) *n_rows = out->n_rows - row0;
    if (row0 < 0 || (row0 & 7) || row0 + *n_rows > out->n_rows)
        return fail(PG_ERR_INVALID, std::string(who) + ": row range outside the batch or not starting at a multiple of 8");
    return PG_OK;
}

pg_status start_encode(SectionTimer &tm) {
    PG_CUDA(cudaEventCreate(&tm.e0));
    PG_CUDA(cudaEventCreate(&tm.e1));
    PG_CUDA(cudaEventRecord(tm.e0, 0));
    return PG_OK;
}

pg_status finish_encode(SectionTimer &tm, std::unique_ptr<EncodedFile> ef, int launches, const char *who,
                        uint64_t *out_file) {
    PG_CUDA(cudaEventRecord(tm.e1, 0));
    PG_CUDA(cudaEventSynchronize(tm.e1));
    cudaError_t le = cudaGetLastError();
    if (le != cudaSuccess) return fail(PG_ERR_CUDA, std::string(who) + ": " + cudaGetErrorString(le));
    ef->meta.file_bytes = ef->file_bytes;
    ef->meta.ms_encode = tm.ms();
    ef->meta.launches = launches;
    *out_file = g_enc.put(std::move(ef));
    return PG_OK;
}

FileStats::FileStats(const Schema &s)
    : n_key_(s.n_key), cols_(s.n_cols(), ColStats{INT64_MAX, INT64_MIN, 0, 0}), nan_(s.n_cols(), 0) {}

ColStats piece_stats(const EncColumn &ec, const int64_t *sw, int64_t rows) {
    ColStats p;
    p.null_count = rows - sw[2];
    p.has_minmax = ec.width > 0 && sw[2] > 0 && !sw[4];
    p.min = sw[0];
    p.max = sw[1];
    if ((ec.type == PG_FLOAT || ec.type == PG_DOUBLE) && p.has_minmax) {
        p.min = zero_as(p.min, -0.0);
        p.max = zero_as(p.max, 0.0);
    }
    return p;
}

ColStats FileStats::add(int col, const EncColumn &ec, const int64_t *sw, int64_t rows) {
    const bool fp = ec.type == PG_FLOAT || ec.type == PG_DOUBLE;
    const ColStats p = piece_stats(ec, sw, rows);
    nan_[col] |= sw[4] != 0;
    if (col == n_key_ + 1) deletes_ += sw[3];
    // the merge keeps the zero rule: the zero min it can take is -0.0, the zero max +0.0
    ColStats &f = cols_[col];
    f.null_count += p.null_count;
    if (p.has_minmax) {
        if (!f.has_minmax) { f.min = p.min; f.max = p.max; f.has_minmax = 1; }
        else if (fp) {
            double a, b, x, y;
            memcpy(&a, &f.min, 8); memcpy(&b, &f.max, 8); memcpy(&x, &p.min, 8); memcpy(&y, &p.max, 8);
            a = std::min(a, x); b = std::max(b, y);
            memcpy(&f.min, &a, 8); memcpy(&f.max, &b, 8);
        } else { f.min = std::min(f.min, p.min); f.max = std::max(f.max, p.max); }
    }
    return p;
}

void FileStats::finish(EncodedFile &ef) {
    for (size_t c = 0; c < cols_.size(); c++)
        if (nan_[c]) cols_[c] = ColStats{INT64_MAX, INT64_MIN, cols_[c].null_count, 0};
    ef.meta.delete_row_count = deletes_;
    const ColStats &sq = cols_[n_key_];
    ef.meta.min_sequence_number = sq.has_minmax ? sq.min : 0;
    ef.meta.max_sequence_number = sq.has_minmax ? sq.max : 0;
    ef.stats = std::move(cols_);
}

pg_status ZstdFrames::compress(Scratch &scratch, const uint8_t *img, const std::vector<Body> &bodies,
                               std::vector<int64_t> *frame_bytes, int *launches) {
    frame_bytes->assign(bodies.size(), 0);
    if (bodies.empty()) return PG_OK;
    std::vector<ZsBlockJob> jobs;
    std::vector<ZsBody> zb;
    int64_t img_end = 0, out = 0, seq = 0;
    for (const Body &b : bodies) {
        ZsBody z{b.off, b.bytes, (int32_t)jobs.size(), 0};
        for (int64_t b0 = 0; b0 == 0 || b0 < b.bytes; b0 += zs::kMaxBlock) {   // an empty body: one empty block
            const int32_t n = (int32_t)std::min<int64_t>(zs::kMaxBlock, b.bytes - b0);
            jobs.push_back(ZsBlockJob{b.off + b0, out, seq, n, (int32_t)zb.size()});
            out += n;
            seq += n / 4 + 1;
            z.n_blocks++;
        }
        zb.push_back(z);
        img_end = std::max(img_end, b.off + b.bytes);
    }
    img_ = img;
    n_blocks_ = jobs.size();
    n_bodies_ = zb.size();
    out_ = (uint8_t *)scratch.take((size_t)out + 64);
    uint8_t *lits = (uint8_t *)scratch.take((size_t)img_end + 64);
    zs::Seq *seqs = (zs::Seq *)scratch.take(sizeof(zs::Seq) * (size_t)seq);
    raw_ = (uint8_t *)scratch.take(n_bodies_);
    jobs_ = (ZsBlockJob *)scratch.take(sizeof(ZsBlockJob) * n_blocks_);
    bodies_ = (ZsBody *)scratch.take(sizeof(ZsBody) * n_bodies_);
    res_ = (int2 *)scratch.take(sizeof(int2) * n_blocks_);
    boff_ = (int32_t *)scratch.take(sizeof(int32_t) * n_blocks_);
    frame_ = (int64_t *)scratch.take(sizeof(int64_t) * n_bodies_);
    if (!out_ || !lits || !seqs || !raw_ || !jobs_ || !bodies_ || !res_ || !boff_ || !frame_)
        return fail(PG_ERR_CUDA, std::string(who_) + ": out of device memory for the zstd frames");
    PG_CUDA(cudaMemcpy(jobs_, jobs.data(), sizeof(ZsBlockJob) * n_blocks_, cudaMemcpyHostToDevice));
    PG_CUDA(cudaMemcpy(bodies_, zb.data(), sizeof(ZsBody) * n_bodies_, cudaMemcpyHostToDevice));
    k_zs_block<<<(unsigned)n_blocks_, 32, kZsSmem>>>(jobs_, img, out_, seqs, lits, res_);
    k_zs_frame_sizes<<<(unsigned)((n_bodies_ + 127) / 128), 128>>>(bodies_, (int)n_bodies_, res_, boff_, frame_);
    *launches += 2;
    SmallReads rd(0);
    pg_status st = rd.add(frame_bytes->data(), frame_, sizeof(int64_t) * n_bodies_);
    if (st) return st;
    ++*launches;
    return rd.finish();
}

pg_status ZstdFrames::gather(const std::vector<int64_t> &dst_off, const std::vector<uint8_t> &raw, uint8_t *file,
                             int *launches) {
    if (!n_blocks_) return PG_OK;
    // (the frame sizes have been read: their buffer takes the destination offsets)
    PG_CUDA(cudaMemcpy(frame_, dst_off.data(), sizeof(int64_t) * n_bodies_, cudaMemcpyHostToDevice));
    if (!raw.empty()) PG_CUDA(cudaMemcpy(raw_, raw.data(), n_bodies_, cudaMemcpyHostToDevice));
    k_zs_gather<<<(unsigned)n_blocks_, 256>>>(jobs_, bodies_, res_, boff_, frame_, raw.empty() ? nullptr : raw_, img_,
                                              out_, file);
    ++*launches;
    return PG_OK;
}

}  // namespace pg

using namespace pg;

extern "C" {

pg_status pg_parquet_file_meta(uint64_t file, pg_file_meta *out) {
    std::shared_ptr<EncodedFile> ef = g_enc.get(file);
    if (!ef || !out) return fail(PG_ERR_INVALID, "unknown encoded file handle");
    *out = ef->meta;
    return PG_OK;
}

pg_status pg_parquet_file_column_stats(uint64_t file, int32_t column, int64_t *null_count, int32_t *has_min_max,
                                       void *min8, void *max8) {
    std::shared_ptr<EncodedFile> ef = g_enc.get(file);
    if (!ef) return fail(PG_ERR_INVALID, "unknown encoded file handle");
    if (column < 0 || column >= (int32_t)ef->stats.size()) return fail(PG_ERR_INVALID, "column out of range");
    const ColStats &cs = ef->stats[column];
    if (null_count) *null_count = cs.null_count;
    if (has_min_max) *has_min_max = cs.has_minmax;
    if (min8) memcpy(min8, &cs.min, 8);
    if (max8) memcpy(max8, &cs.max, 8);
    return PG_OK;
}

pg_status pg_parquet_file_fetch(uint64_t file, void *host_buffer, int64_t capacity) {
    std::shared_ptr<EncodedFile> ef = g_enc.get(file);
    if (!ef || !host_buffer) return fail(PG_ERR_INVALID, "unknown encoded file handle");
    if (capacity < ef->file_bytes) return fail(PG_ERR_INVALID, "buffer smaller than the file");
    pg_status st = ensure_device();
    if (st) return st;
    PG_CUDA(cudaMemcpy(host_buffer, ef->d_file, (size_t)ef->data_end, cudaMemcpyDeviceToHost));
    for (const auto &p : ef->host_parts) memcpy((uint8_t *)host_buffer + p.first, p.second.data(), p.second.size());
    return PG_OK;
}

pg_status pg_parquet_file_device_image(uint64_t file, const uint8_t **device_bytes, int64_t *size) {
    std::shared_ptr<EncodedFile> ef = g_enc.get(file);
    if (!ef || !device_bytes || !size) return fail(PG_ERR_INVALID, "unknown encoded file handle");
    pg_status st = ensure_device();
    if (st) return st;
    if (!ef->image_complete) {
        Scratch scratch(0);
        if ((st = patch(scratch, ef->host_parts, ef->d_file, "the header patch"))) return st;
        cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) return fail(PG_ERR_CUDA, std::string("parquet encode: ") + cudaGetErrorString(e));
        ef->image_complete = true;
    }
    *device_bytes = ef->d_file;
    *size = ef->file_bytes;
    return PG_OK;
}

pg_status pg_parquet_file_free(uint64_t file) {
    return g_enc.take(file) ? PG_OK : fail(PG_ERR_INVALID, "unknown encoded file handle");
}

}  // extern "C"
