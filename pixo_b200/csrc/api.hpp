// api.hpp — what the C ABI's area files (api_jpeg.cu, api_png.cu, api_decode.cu) share from api.cu.  Private to the
// library: its functions are hidden, so the library exports the same symbols however its sources are split.
#pragma once

#include <array>
#include <functional>

#include "common.cuh"

#define PIXO_HIDDEN __attribute__((visibility("hidden")))

namespace pixo {

PIXO_HIDDEN bool is_page_locked(const void *p);

// Host -> device copy of any host memory, queued on `st` (see api.cu).
PIXO_HIDDEN int h2d_copy(pixo_b200_ctx *ctx, void *dst, const void *src, size_t bytes, cudaStream_t st);

// Device -> host copy into any host memory on `st`; returns when `dst` holds the bytes.
PIXO_HIDDEN int d2h_copy_sync(pixo_b200_ctx *ctx, void *dst, const void *src, size_t bytes, cudaStream_t st);

// Synchronises every stream of the context when an entry point leaves early, so that no queued
// copy still reads the caller's pixels or writes the caller's output after the error return.
struct DrainOnError {
    pixo_b200_ctx *ctx;
    bool armed = true;
    explicit DrainOnError(pixo_b200_ctx *c) : ctx(c) {}
    ~DrainOnError();
};

// One result a host-buffer entry point copies back: `bytes` at device `src` to the caller's `dst` (none: nothing is
// copied).  With `out_len`, the length is stored there first and a result longer than `cap` is refused.
struct HostResult {
    void *dst = nullptr;
    const void *src = nullptr;
    size_t bytes = 0;
    size_t *out_len = nullptr;
    size_t cap = 0;
};
using HostResults = std::array<HostResult, 4>;

// The device side of every host-buffer entry point, once its checks have passed: sets the device, stages the
// caller's `in_bytes` at `in` in d_in, binds `outputs` in d_out, then `queue(d_in, back)` queues the `_dev` twin on
// them and names the results, which are copied back in order.  Every stream is drained on an error return.
PIXO_HIDDEN int stage_host_call(pixo_b200_ctx *ctx, const void *in, size_t in_bytes,
                                const std::function<void(Layout &)> &outputs,
                                const std::function<int(const uint8_t *d_in, HostResults &back)> &queue);

}  // namespace pixo
