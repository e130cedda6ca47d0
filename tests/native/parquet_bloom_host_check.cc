// Host build of sbbf_device.cuh (the same source k_pw_sbbf compiles) as a filter program, so that the tests
// (test_parquet_bloom_cpu.py) run it under AddressSanitizer / UBSan against the Python model in
// parquet_bloom_reference.py.  One command per input line, one answer line each:
//   s <ndv> <fpp>                        the bitset bytes of a filter for ndv values at fpp
//   4 <uint32>                           the hash of 4 little-endian bytes (hash4), then fi::xxh64 of the same bytes
//   8 <uint64>                           the same for 8 bytes (hash8)
//   f <bytes> <hex value> <hex value>…   a filter of <bytes> over the values ("-" = the empty value), as hex
#include <inttypes.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "sbbf_device.cuh"

static std::vector<uint8_t> unhex(const char *p, size_t n) {
    std::vector<uint8_t> b(n / 2);
    for (size_t i = 0; i < b.size(); i++) {
        unsigned v;
        sscanf(p + 2 * i, "%2x", &v);
        b[i] = (uint8_t)v;
    }
    return b;
}

int main() {
    static char line[1 << 20];
    while (fgets(line, sizeof line, stdin)) {
        char *p = line + 2;
        if (line[0] == 's') {
            const int64_t ndv = strtoll(p, &p, 10);
            printf("%" PRId64 "\n", sbbf::num_bytes(ndv, strtod(p, nullptr)));
        } else if (line[0] == '4') {
            const uint32_t v = (uint32_t)strtoull(p, nullptr, 10);
            const uint8_t b[4] = {(uint8_t)v, (uint8_t)(v >> 8), (uint8_t)(v >> 16), (uint8_t)(v >> 24)};
            printf("%" PRIu64 " %" PRIu64 "\n", sbbf::hash4(v), fi::xxh64(b, 4));
        } else if (line[0] == '8') {
            const uint64_t v = strtoull(p, nullptr, 10);
            uint8_t b[8];
            for (int i = 0; i < 8; i++) b[i] = (uint8_t)(v >> (8 * i));
            printf("%" PRIu64 " %" PRIu64 "\n", sbbf::hash8(v), fi::xxh64(b, 8));
        } else if (line[0] == 'f') {
            const int64_t bytes = strtoll(p, &p, 10);
            std::vector<uint32_t> words((size_t)bytes / 4);
            const uint32_t n_blocks = (uint32_t)(bytes / 32);
            for (;;) {
                while (*p == ' ') p++;
                if (!*p || *p == '\n') break;
                size_t n = 0;
                while (p[n] && p[n] != ' ' && p[n] != '\n') n++;
                // an exact-size buffer: a read past the value is reported
                std::vector<uint8_t> v = *p == '-' ? std::vector<uint8_t>() : unhex(p, n);
                uint8_t *buf = (uint8_t *)malloc(v.size() ? v.size() : 1);
                if (!v.empty()) memcpy(buf, v.data(), v.size());
                const uint64_t h = fi::xxh64(buf, (int64_t)v.size());
                free(buf);
                const uint32_t blk = sbbf::block_of(h, n_blocks);
                for (int i = 0; i < 8; i++) words[8 * (size_t)blk + i] |= sbbf::mask_word(h, i);
                p += n;
            }
            for (uint32_t w : words)
                printf("%02x%02x%02x%02x", w & 0xFF, (w >> 8) & 0xFF, (w >> 16) & 0xFF, w >> 24);
            printf("\n");
        } else {
            return 2;
        }
    }
    return 0;
}
