// Layout of one call's staging buffer: consecutive regions, each starting 256-byte aligned.  CUDA-free, so that the
// host-only build of the CRAM record code (tests/hostsim) lays out its std::vector image exactly as the device path
// lays out ctx->d_stage.
#pragma once
#include <stddef.h>
#include <stdint.h>

struct StageLayout {
    struct Seg { size_t off, bytes; };
    size_t total = 0;                  // bytes the buffer must have
    size_t slack = 0;                  // extra bytes behind every region
    uint8_t *base = nullptr;           // the buffer, once bound (hgpu_stage_ensure, or a host image)

    StageLayout() = default;
    explicit StageLayout(size_t per_seg_slack) : slack(per_seg_slack) {}

    // A region of `bytes` bytes (plus `slack`).  Regions never overlap: each one starts where the previous one ended,
    // rounded up to 256.
    Seg seg(size_t bytes)
    {
        const Seg s{total, bytes};
        total += align(bytes + slack);
        return s;
    }
    static size_t align(size_t x) { return (x + 255) & ~(size_t)255; }
    template <class T = uint8_t> T *at(const Seg &s) const { return reinterpret_cast<T *>(base + s.off); }
};
