// decode_host.hpp — what the JPEG and PNG decoders share: the status of a decoded file and, for the .cu files, the
// prefix search their kernels use to find an item's file and the pass driver that cuts, packs and uploads a batch.
#pragma once

#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

#include "../../include/pixo_b200.h"

namespace pixo {

// What pixo's decoder returns for one file: code is 0 or the PIXO_B200_ERR_* of its error, msg the error's Display
// text ("Decode error: ...", "Unsupported: ...", "Invalid image dimensions: ...", "Image ... exceeds ...")
struct DecodeStatus {
    int code = 0;
    std::string msg;
};

// pixo's Error::InvalidDecode and Error::UnsupportedDecode, the codes of most decode errors
constexpr int kInvalidDecode = PIXO_B200_ERR_INVALID_DECODE, kUnsupportedDecode = PIXO_B200_ERR_UNSUPPORTED_DECODE;

// Sets s to an error: code, and the formatted message behind the Display prefix of InvalidDecode and
// UnsupportedDecode (the other codes' messages carry their own).  Returns false, for parsers that stop there.
inline bool decode_fail(DecodeStatus &s, int code, const char *fmt, ...) __attribute__((format(printf, 3, 4)));
inline bool decode_fail(DecodeStatus &s, int code, const char *fmt, ...)
{
    char buf[256];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    s.code = code;
    s.msg = code == kInvalidDecode ? std::string("Decode error: ") + buf
          : code == kUnsupportedDecode ? std::string("Unsupported: ") + buf : std::string(buf);
    return false;
}

}  // namespace pixo

#ifdef __CUDACC__
#include <algorithm>
#include <numeric>
#include <vector>

#include "common.cuh"

namespace pixo {

// The item of a pass's prefix sums (prefix[0] = 0, prefix[n] = total) that holds g
__device__ inline uint32_t item_of(const uint64_t *__restrict__ prefix, uint32_t n, uint64_t g)
{
    uint32_t lo = 0, hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) / 2;
        if (__ldg(prefix + mid) <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// A decode pass: files go in while their scratch, as `charge` counts it, stays within kDecodePassBytes and their
// count within kDecodePassFiles; a file larger than kDecodePassBytes goes alone.
constexpr uint64_t kDecodePassBytes = (uint64_t)1 << 30;
constexpr uint32_t kDecodePassFiles = 1u << 16;

// The end of the pass that starts at file p0 of n
template <class Parsed, class Charge>
uint32_t pass_end(const Parsed *const *files, uint32_t p0, uint32_t n, Charge charge)
{
    uint32_t p1 = p0;
    uint64_t need = 0;
    while (p1 < n && p1 - p0 < kDecodePassFiles && (p1 == p0 || need + charge(*files[p1]) <= kDecodePassBytes))
        need += charge(*files[p1++]);
    return p1;
}

// A pass's uploaded part (its first `up` bytes), built on the host in the device's layout: H's pointers are bound
// to the returned image by the pass's describe_pass
template <class Pass, class Sizes>
std::vector<uint8_t> host_image(const Sizes &s, Pass &H)
{
    Layout count;
    describe_pass(count, s, H);
    std::vector<uint8_t> image(H.up);
    Layout L(image.data());
    describe_pass(L, s, H);
    return image;
}

// Orders the pass's s.n files longest stream first (H.order, by H.files[i].src_len), binds the device scratch D in
// buf and queues the upload of the filled image on the context's stream
template <class Pass, class Sizes>
int upload_pass(pixo_b200_ctx *ctx, DevBuf &buf, const Sizes &s, Pass &H, const std::vector<uint8_t> &image, Pass &D)
{
    std::iota(H.order, H.order + s.n, 0u);
    std::stable_sort(H.order, H.order + s.n,
                     [&](uint32_t a, uint32_t b) { return H.files[a].src_len > H.files[b].src_len; });
    PIXO_TRY(bind(ctx, buf, [&](Layout &L) { describe_pass(L, s, D); }));
    PIXO_CUDA(ctx, cudaMemcpyAsync(D.files, image.data(), H.up, cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

}  // namespace pixo
#endif
