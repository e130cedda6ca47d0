// Host build of paimon_b200/csrc/zstd_encode_device.cuh (the same source the device kernels compile): C entry points for
// tests/test_zstd_encode_cpu.py, which decompresses every frame with libzstd (through pyarrow) and with the project's
// own decoder, without a GPU.
#include <stdlib.h>

#include "zstd_encode_device.cuh"

// one zstd frame of src[0, n) into dst (cap bytes); returns the frame size or -1
extern "C" long long zse_host_compress(const unsigned char *src, long long n, unsigned char *dst, long long cap) {
    int32_t *htab = (int32_t *)malloc(sizeof(int32_t) << zs::kHashLog);
    zs::Seq *seqs = (zs::Seq *)malloc(sizeof(zs::Seq) * (zs::kMaxBlock / 4 + 1));
    unsigned char *lits = (unsigned char *)malloc(zs::kMaxBlock);
    unsigned char *blk = (unsigned char *)malloc(zs::kMaxBlock);
    zs::EncWork *W = (zs::EncWork *)calloc(1, sizeof(zs::EncWork));
    const long long r = zs::compress_frame(src, n, dst, cap, htab, seqs, lits, blk, *W);
    free(W);
    free(blk);
    free(lits);
    free(seqs);
    free(htab);
    return r;
}

extern "C" long long zse_host_bound(long long n) { return zs::frame_bound(n); }

extern "C" long long zse_host_decode(const unsigned char *src, long long n, unsigned char *dst, long long cap) {
    zs::Tables *T = (zs::Tables *)calloc(1, sizeof(zs::Tables));
    unsigned char *lit = (unsigned char *)malloc(zs::kMaxBlock + 64);
    const long long r = zs::decode(src, n, dst, cap, lit, *T);
    free(lit);
    free(T);
    return r;
}

// the value -> code maps of the encoder against the decoder's code tables: 0 when every value lands in its code's range
extern "C" int zse_host_check_codes() {
    for (uint32_t v = 0; v < (1u << 17); v++) {
        uint32_t base;
        int bits;
        zs::ll_code_info(zs::ll_code(v), base, bits);
        if (v < base || v - base >= (1u << bits)) return 1;
        zs::ml_code_info(zs::ml_code(v + 3), base, bits);
        if (v + 3 < base || v + 3 - base >= (1u << bits)) return 2;
    }
    return 0;
}
