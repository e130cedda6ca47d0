// upload.cu — start moving the data files of the NEXT section to the device while the current one merges.
//
// The Java read path fetches a bucket's data files through FileIO and hands them to the format readers
// (KeyValueFileReaderFactory.java:104-140); a compaction / scan task walks many sections and buckets one after the
// other (MergeTreeCompactRewriter.java:77-106 per section).  On the device path the host -> device copy of a section's
// file bytes (the encoded pages: ~0.3 of the decoded bytes) is the longest leg of a step, so it runs on its own copy
// stream: pg_files_upload_begin returns at once, pg_files_upload_wait blocks until the bytes are resident and hands
// back device descriptors for pg_parquet_read_section.  Host buffers should be page-locked (a pageable source makes
// the copy synchronous and staged by the driver).
#include <memory>
#include <mutex>
#include <vector>

#include "pg_internal.h"

namespace pg {
namespace {

struct Upload {
    std::vector<DeviceBuffer> bufs;
    std::vector<pg_file_desc> files;
    cudaEvent_t done = nullptr;
    ~Upload() { if (done) cudaEventDestroy(done); }
};

Table<Upload> g_up(7);
std::mutex g_up_mu;                                    // creation of the upload stream
cudaStream_t g_up_stream = nullptr;

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" pg_status pg_files_upload_begin(const pg_file_desc *files, int32_t n_files, uint64_t *out_upload) {
    if (!out_upload || n_files < 0 || (n_files > 0 && !files)) return fail(PG_ERR_INVALID, "null argument");
    for (int i = 0; i < n_files; i++) {
        pg_status st = check_file_desc(files[i]);
        if (st) return st;
    }
    pg_status st = ensure_device();
    if (st) return st;
    auto up = std::make_unique<Upload>();
    {
        std::lock_guard<std::mutex> lk(g_up_mu);
        if (!g_up_stream) PG_CUDA(cudaStreamCreateWithFlags(&g_up_stream, cudaStreamNonBlocking));
    }
    PG_CUDA(cudaEventCreateWithFlags(&up->done, cudaEventDisableTiming));
    Scratch scratch(g_up_stream);                      // the buffers until the upload is registered
    for (int i = 0; i < n_files; i++) {
        pg_file_desc d = files[i];
        if (d.mem == PG_MEM_HOST) {
            st = file_image(scratch, d.bytes, d.size, "upload", &d.bytes);
            if (st) return st;
            d.mem = PG_MEM_DEVICE;
        }
        up->files.push_back(d);
    }
    PG_CUDA(cudaEventRecord(up->done, g_up_stream));
    up->bufs.swap(scratch.bufs);
    *out_upload = g_up.put(std::move(up));
    return PG_OK;
}

extern "C" pg_status pg_files_upload_wait(uint64_t upload, pg_file_desc *out_files, int32_t n_files) {
    std::shared_ptr<Upload> up = g_up.get(upload);
    if (!up) return fail(PG_ERR_INVALID, "unknown upload handle");
    if (n_files != (int32_t)up->files.size() || (n_files > 0 && !out_files)) return fail(PG_ERR_INVALID, "upload: one descriptor per file");
    PG_CUDA(cudaEventSynchronize(up->done));
    for (int i = 0; i < n_files; i++) out_files[i] = up->files[i];
    return PG_OK;
}

extern "C" pg_status pg_files_upload_free(uint64_t upload) {
    std::shared_ptr<Upload> up = g_up.take(upload);
    if (!up) return fail(PG_ERR_INVALID, "unknown upload handle");
    // the copy itself, and the decode launches of the calling thread that read the bytes, must be done before the
    // buffers go back to the cache
    cudaEventSynchronize(up->done);
    cudaStreamSynchronize(copy_stream());
    return PG_OK;
}
