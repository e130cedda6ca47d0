// Host build of paimon_b200/csrc/lz4_device.cuh (the same source the device kernels compile) as a filter program, so
// that tests/test_lz4_cpu.py can run it under AddressSanitizer / UBSan without preloading the sanitizer runtime into
// Python.  Input on stdin, records of [u8 mode: 0 raw block, 1 Hadoop framing][i64 cap][i64 n][n bytes]; output on
// stdout, per record [i64 result][result bytes when result > 0].  Every input and output buffer is heap-allocated at
// its exact size, so a read or write one byte outside is reported.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "lz4_device.cuh"

static bool read_all(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

int main() {
    uint8_t mode;
    int64_t cap, n;
    while (read_all(&mode, 1)) {
        if (!read_all(&cap, 8) || !read_all(&n, 8) || cap < 0 || n < 0) return 2;
        uint8_t *src = (uint8_t *)malloc(n ? (size_t)n : 1);
        uint8_t *dst = (uint8_t *)malloc(cap ? (size_t)cap : 1);
        if (!src || !dst || !read_all(src, (size_t)n)) return 2;
        const int64_t r = mode == 0 ? lz4::decode_block(src, n, dst, cap) : lz4::decode_hadoop(src, n, dst, cap);
        fwrite(&r, 8, 1, stdout);
        if (r > 0) fwrite(dst, 1, (size_t)r, stdout);
        free(src);
        free(dst);
    }
    return 0;
}
