// api_decode.cu — the JPEG and PNG decode entry points of the C ABI.
#include <vector>

#include "api.hpp"
#include "jpeg_decode_host.hpp"
#include "png_decode_host.hpp"

using namespace pixo;

// One set of entry points for both decoders, over the parsed file (JdecParsed, PdecParsed); parse and launch_decode
// are overloaded on it.

static int decode_error(pixo_b200_ctx *ctx, const DecodeStatus &s)
{
    return set_error(ctx, s.code, "%s", s.msg.c_str());
}

template <class Parsed>
static void decode_geometry(const Parsed &p, uint32_t *width, uint32_t *height, uint32_t *color_type)
{
    if (width) *width = p.width;
    if (height) *height = p.height;
    if (color_type) *color_type = p.out_ct;
}

template <class Parsed>
static int decode_info(const uint8_t *data, size_t len, uint32_t *width, uint32_t *height, uint32_t *color_type,
                       int32_t *producible)
{
    if (!data && len) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "data is null");
    Parsed p;
    parse(data, len, p);
    if (p.status.code) return decode_error(nullptr, p.status);
    decode_geometry(p, width, height, color_type);
    if (producible) *producible = p.producible();
    return 0;
}

template <class Parsed>
static int decode_one(pixo_b200_ctx *ctx, const uint8_t *data, size_t len, uint8_t *pixels, size_t pixels_cap,
                      uint32_t *width, uint32_t *height, uint32_t *color_type)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    if (!data && len) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "data is null");
    Parsed p;
    parse(data, len, p);
    if (p.status.code) return decode_error(ctx, p.status);
    decode_geometry(p, width, height, color_type);
    // a file whose stream cannot produce its rows is decoded for its error only: no frame, no output capacity
    const bool producible = p.producible();
    const size_t bytes = p.out_bytes();
    if (producible && pixels_cap < bytes)
        return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu below %zu", pixels_cap, bytes);
    if (producible && bytes == 0) return 0;   // a JPEG frame 0 rows high: nothing to decode
    if (producible && !pixels) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "pixels is null");
    uint8_t *d_pixels = nullptr;
    auto outputs = [&](Layout &L) { if (producible) d_pixels = L.take(bytes); };
    // launch_decode uploads the file itself
    return stage_host_call(ctx, nullptr, 0, outputs, [&](const uint8_t *, HostResults &back) {
        const Parsed *files[1] = {&p};
        const uint64_t off[1] = {0};
        DecodeStatus res;
        PIXO_TRY(launch_decode(ctx, files, &data, 1, off, d_pixels, &res));
        if (res.code) return decode_error(ctx, res);
        if (!producible) return set_error(ctx, PIXO_B200_ERR_CUDA, "png decode: a stream produced more than its bound");
        back = {{{pixels, d_pixels, bytes}}};
        return 0;
    });
}

template <class Parsed>
static int decode_to_device(pixo_b200_ctx *ctx, const uint8_t *const *files, const size_t *lens, uint32_t n,
                            uint8_t *d_out, const size_t *out_offsets, int32_t *status)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    if (n == 0) return 0;
    if (!files || !lens || !out_offsets || !status || !d_out)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null array");
    std::vector<Parsed> parsed(n);
    std::vector<const Parsed *> ok;
    std::vector<const uint8_t *> data;
    std::vector<uint64_t> off;
    std::vector<uint32_t> idx;
    for (uint32_t i = 0; i < n; ++i) {
        if (!files[i] && lens[i]) {
            status[i] = PIXO_B200_ERR_INVALID_ARGUMENT;
            continue;
        }
        parse(files[i], lens[i], parsed[i]);
        status[i] = parsed[i].status.code;
        if (status[i]) continue;
        ok.push_back(&parsed[i]);
        data.push_back(files[i]);
        off.push_back(out_offsets[i]);
        idx.push_back(i);
    }
    if (ok.empty()) return 0;
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<DecodeStatus> res(ok.size());
    PIXO_TRY(launch_decode(ctx, ok.data(), data.data(), (uint32_t)ok.size(), off.data(), d_out, res.data()));
    for (size_t k = 0; k < ok.size(); ++k)
        if (res[k].code) status[idx[k]] = res[k].code;
    return 0;
}

extern "C" {

int pixo_b200_jpeg_decode_info(const uint8_t *data, size_t len, uint32_t *width, uint32_t *height,
                               uint32_t *color_type)
{
    return decode_info<JdecParsed>(data, len, width, height, color_type, nullptr);
}

int pixo_b200_jpeg_decode(pixo_b200_ctx *ctx, const uint8_t *data, size_t len, uint8_t *pixels, size_t pixels_cap,
                          uint32_t *width, uint32_t *height, uint32_t *color_type)
{
    return decode_one<JdecParsed>(ctx, data, len, pixels, pixels_cap, width, height, color_type);
}

int pixo_b200_jpeg_decode_to_device(pixo_b200_ctx *ctx, const uint8_t *const *files, const size_t *lens, uint32_t n,
                                    uint8_t *d_out, const size_t *out_offsets, int32_t *status)
{
    return decode_to_device<JdecParsed>(ctx, files, lens, n, d_out, out_offsets, status);
}

int pixo_b200_png_decode_info(const uint8_t *data, size_t len, uint32_t *width, uint32_t *height,
                              uint32_t *color_type, int32_t *producible)
{
    return decode_info<PdecParsed>(data, len, width, height, color_type, producible);
}

int pixo_b200_png_decode(pixo_b200_ctx *ctx, const uint8_t *data, size_t len, uint8_t *pixels, size_t pixels_cap,
                         uint32_t *width, uint32_t *height, uint32_t *color_type)
{
    return decode_one<PdecParsed>(ctx, data, len, pixels, pixels_cap, width, height, color_type);
}

int pixo_b200_png_decode_to_device(pixo_b200_ctx *ctx, const uint8_t *const *files, const size_t *lens, uint32_t n,
                                   uint8_t *d_out, const size_t *out_offsets, int32_t *status)
{
    return decode_to_device<PdecParsed>(ctx, files, lens, n, d_out, out_offsets, status);
}

}  // extern "C"
