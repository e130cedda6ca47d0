// device_layout.h — how one block of device memory is split into regions.  Host-only: builds with or without CUDA.
#pragma once

#include <stddef.h>

namespace pg {

// bytes a kernel may read past the end of a column buffer or a scratch region: the readers load whole words and look
// past a page's or a column's last byte without a bounds test
constexpr size_t kReadPast = 64;

// A bump carver.  A block's regions are written once, as code that takes them in order from a Carver; it runs with a
// null base to size the block (bytes()), then on the block's memory to place them, so size and layout cannot disagree.
// Every region starts on a 256-byte boundary.
class Carver {
 public:
    explicit Carver(void *base) : base_((unsigned char *)base) {}
    template <typename T>
    T *take(size_t n) {                  // n values of T; NULL when the base is
        const size_t at = (size_ + 255) & ~(size_t)255;
        size_ = at + n * sizeof(T);
        return base_ ? (T *)(base_ + at) : nullptr;
    }
    size_t bytes() const { return size_; }

 private:
    unsigned char *base_;
    size_t size_ = 0;
};

}  // namespace pg
