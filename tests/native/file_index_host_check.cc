// Host build of xxhash64_device.cuh (the same source k_bloom_build compiles) as a filter program, so that the tests
// (test_file_index_cpu.py) run it under AddressSanitizer / UBSan against the Python model in file_index_reference.py.
// One command per input line, one answer line each:
//   x <align> <hex bytes>     XXH64 (seed 0) of the bytes, placed at offset <align> of a buffer that ends with them
//   w <int64>                 Thomas Wang's hash of the value
//   f <uint32 bits>           the hash of a FLOAT with these bits (NaN folded)
//   d <uint64 bits>           the hash of a DOUBLE with these bits (NaN folded)
//   s <items> <fpp>           BloomFilter64 sizing: "<num_bits> <k>", or "refused"
//   b <hash> <k> <num_bits>   the k bit positions of a hash
#include <inttypes.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "xxhash64_device.cuh"

int main() {
    static char line[1 << 16];
    while (fgets(line, sizeof line, stdin)) {
        char *p = line + 2;
        if (line[0] == 'x') {
            const int align = (int)strtol(p, &p, 10);
            while (*p == ' ') p++;
            size_t n = 0;
            while (p[2 * n] && p[2 * n] != '\n') n++;
            uint8_t *buf = (uint8_t *)malloc(align + n ? align + n : 1);   // exact: a read past the end is reported
            for (size_t i = 0; i < n; i++) {
                unsigned v;
                sscanf(p + 2 * i, "%2x", &v);
                buf[align + i] = (uint8_t)v;
            }
            printf("%" PRIu64 "\n", fi::xxh64(buf + align, (int64_t)n));
            free(buf);
        } else if (line[0] == 'w') {
            printf("%" PRId64 "\n", fi::wang64(strtoll(p, nullptr, 10)));
        } else if (line[0] == 'f') {
            printf("%" PRId64 "\n", fi::wang64(fi::float_key((uint32_t)strtoull(p, nullptr, 10))));
        } else if (line[0] == 'd') {
            printf("%" PRId64 "\n", fi::wang64(fi::double_key(strtoull(p, nullptr, 10))));
        } else if (line[0] == 's') {
            const int32_t items = (int32_t)strtol(p, &p, 10);
            const double fpp = strtod(p, nullptr);
            int32_t bits = 0, k = 0;
            if (fi::bloom_sizing(items, fpp, &bits, &k)) printf("%d %d\n", bits, k);
            else printf("refused\n");
        } else if (line[0] == 'b') {
            const int64_t h = strtoll(p, &p, 10);
            const int k = (int)strtol(p, &p, 10);
            const uint32_t bits = (uint32_t)strtoul(p, nullptr, 10);
            for (int i = 1; i <= k; i++) printf(i < k ? "%u " : "%u\n", fi::bloom_bit(h, i, bits));
        } else {
            return 2;
        }
    }
    return 0;
}
