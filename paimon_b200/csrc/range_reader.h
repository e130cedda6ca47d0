// range_reader.h — byte ranges of the files of a section whose bytes are not in host memory, for the metadata readers
// (orc::read_tails, pq::read_footers).  Host-only: builds with or without CUDA.
#pragma once

#include <stdint.h>

namespace pg {

// read() queues the copy of [off, off + n) of file `file` into dst, flush() delivers every queued range (one round
// trip) and throws std::runtime_error when it cannot.
struct RangeReader {
    virtual ~RangeReader() = default;
    virtual void read(int file, uint64_t off, uint64_t n, uint8_t *dst) = 0;
    virtual void flush() = 0;
};

}  // namespace pg
