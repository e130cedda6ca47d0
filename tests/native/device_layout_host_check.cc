// Host build of the device-memory carver (device_layout.h) for tests/test_device_layout_cpu.py: a list of regions,
// each n values of one element size, carved once with a null base (the sizing pass) and once on a real block.
#include <stdint.h>
#include <stdlib.h>

#include "device_layout.h"

using pg::Carver;

namespace {

template <size_t N>
struct Blob {
    unsigned char b[N];
};

void *take(Carver &cv, int elem, size_t n) {
    switch (elem) {
        case 1: return cv.take<uint8_t>(n);
        case 2: return cv.take<uint16_t>(n);
        case 3: return cv.take<Blob<3>>(n);
        case 4: return cv.take<int32_t>(n);
        case 8: return cv.take<int64_t>(n);
        case 24: return cv.take<Blob<24>>(n);
        case 32: return cv.take<Blob<32>>(n);
        default: abort();
    }
}

}  // namespace

// elem[i], count[i]: region i.  offsets[i] <- its byte offset in the carved block, bytes[0] <- the sizing pass's
// bytes(), bytes[1] <- the carving pass's.  Returns 0, or -1 when the sizing pass returned a non-null pointer.
extern "C" int layout_check(int n, const int *elem, const long long *count, long long *offsets, long long *bytes) {
    Carver size(nullptr);
    for (int i = 0; i < n; i++)
        if (take(size, elem[i], (size_t)count[i])) return -1;
    bytes[0] = (long long)size.bytes();
    const size_t cap = (size.bytes() + 255) & ~(size_t)255;
    unsigned char *base = (unsigned char *)aligned_alloc(256, cap ? cap : 256);
    Carver at(base);
    for (int i = 0; i < n; i++) offsets[i] = (long long)((unsigned char *)take(at, elem[i], (size_t)count[i]) - base);
    bytes[1] = (long long)at.bytes();
    free(base);
    return 0;
}
