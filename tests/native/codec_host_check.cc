// Host build of the page decompressors snappy_device.cuh, zstd_device.cuh, inflate_device.cuh and lz4_device.cuh (the
// same sources the device kernels compile) as a filter program, so that the tests (through tests/codec_filter.py) can
// run them under AddressSanitizer / UBSan without preloading the sanitizer runtime into Python.  Input on stdin, records
// of [u8 mode: 0 Snappy, 1 zstd, 2 raw DEFLATE, 3 gzip, 4 zlib, 5 raw LZ4 block, 6 Hadoop-framed LZ4][i64 cap][i64 n]
// [n bytes]; output on stdout, per record [i64 result][result bytes when result > 0].  Every input and output buffer,
// the decoder tables and the zstd literals buffer are heap-allocated at their exact sizes, so a read or write one byte
// outside is reported.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "inflate_device.cuh"
#include "lz4_device.cuh"
#include "snappy_device.cuh"
#include "zstd_device.cuh"

static bool read_all(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

int main() {
    uint8_t mode;
    int64_t cap, n;
    while (read_all(&mode, 1)) {
        if (!read_all(&cap, 8) || !read_all(&n, 8) || cap < 0 || n < 0 || mode > 6) return 2;
        uint8_t *src = (uint8_t *)malloc(n ? (size_t)n : 1);
        uint8_t *dst = (uint8_t *)malloc(cap ? (size_t)cap : 1);
        if (!src || !dst || !read_all(src, (size_t)n)) return 2;
        int64_t r;
        if (mode == 0) {
            r = snappy::decode(src, n, dst, cap);
        } else if (mode == 1) {
            zs::Tables *T = (zs::Tables *)calloc(1, sizeof(zs::Tables));
            uint8_t *lit = (uint8_t *)malloc(zs::kMaxBlock);
            r = zs::decode(src, n, dst, cap, lit, *T);
            free(lit);
            free(T);
        } else if (mode >= 5) {
            r = mode == 5 ? lz4::decode_block(src, n, dst, cap) : lz4::decode_hadoop(src, n, dst, cap);
        } else {
            inflate::Tables *T = (inflate::Tables *)calloc(1, sizeof(inflate::Tables));
            r = mode == 2 ? inflate::inflate_raw(src, n, dst, cap, *T, nullptr)
                : mode == 3 ? inflate::inflate_gzip(src, n, dst, cap, *T) : inflate::inflate_zlib(src, n, dst, cap, *T);
            free(T);
        }
        fwrite(&r, 8, 1, stdout);
        if (r > 0) fwrite(dst, 1, (size_t)r, stdout);
        free(src);
        free(dst);
    }
    return 0;
}
