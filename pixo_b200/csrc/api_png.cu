// api_png.cu — the PNG encode and resize entry points of the C ABI: filter, reduce, quantise, Adler-32, DEFLATE and
// resize, with their checks.
#include <string.h>

#include <algorithm>

#include "api.hpp"
#include "resize_host.hpp"

using namespace pixo;

extern "C" {

// Frames of a batch (n > 1) must not overlap: each frame's input is read whole while other frames'
// threads write their outputs.  out_name: the caller's name of the output stride.
static int check_batch_strides(pixo_b200_ctx *ctx, uint32_t n, size_t in_stride, size_t in_bytes,
                               const char *out_name, size_t out_stride, size_t out_bytes)
{
    if (n > 1 && in_stride < in_bytes)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DATA_LENGTH, "Invalid data length: expected %zu bytes, got %zu",
                         in_bytes, in_stride);
    if (n > 1 && out_stride < out_bytes)
        return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "%s %zu below %zu", out_name, out_stride, out_bytes);
    return 0;
}

// encode_into's dimension checks (src/png/mod.rs:442-467); empty_rows: rows of 0 bytes
static int check_png_dimensions(pixo_b200_ctx *ctx, uint32_t width, uint32_t height, bool empty_rows = false)
{
    if (width == 0 || height == 0 || empty_rows)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DIMENSIONS, "Invalid image dimensions: %ux%u", width, height);
    if (width > (1u << 24) || height > (1u << 24))  // src/png/mod.rs:21
        return set_error(ctx, PIXO_B200_ERR_IMAGE_TOO_LARGE, "Image dimensions %ux%u exceed maximum %u", width, height, 1u << 24);
    return 0;
}

static int validate_png(pixo_b200_ctx *ctx, uint32_t width, uint32_t height, size_t row_bytes,
                        uint32_t bpp, uint32_t strategy)
{
    PIXO_TRY(check_png_dimensions(ctx, width, height, row_bytes == 0));
    if (bpp < 1 || bpp > 4)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "bytes_per_pixel %u not in 1..4", bpp);
    if ((strategy & ~PIXO_B200_PNG_OPTIMIZE_ALPHA) > PIXO_B200_FILTER_BIGRAMS)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "unknown filter strategy %u", strategy);
    return 0;
}

int pixo_b200_png_filter_dev(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride,
                             uint32_t n_images, uint32_t width, uint32_t height,
                             size_t row_bytes, uint32_t bytes_per_pixel, uint32_t strategy,
                             uint8_t *d_out, size_t out_stride, uint32_t *d_adler)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_png(ctx, width, height, row_bytes, bytes_per_pixel, strategy));
    if (!d_data || !d_out) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    PIXO_TRY(check_batch_strides(ctx, n_images, in_stride, row_bytes * height, "out_stride", out_stride,
                                 (row_bytes + 1) * (size_t)height));
    if (n_images == 0) return 0;
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return launch_png_filter_rows(ctx, d_data, in_stride, n_images, width, height, row_bytes,
                                  bytes_per_pixel, strategy, d_out, out_stride, d_adler, nullptr, height);
}

int pixo_b200_png_filter(pixo_b200_ctx *ctx, const uint8_t *data, uint32_t width,
                         uint32_t height, size_t row_bytes, uint32_t bytes_per_pixel,
                         uint32_t strategy, uint8_t *out, uint32_t *adler32_out)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_png(ctx, width, height, row_bytes, bytes_per_pixel, strategy));
    if (!data || !out) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    const size_t in_bytes = row_bytes * height, out_bytes = (row_bytes + 1) * (size_t)height;
    uint8_t *d_out;
    uint32_t *d_adler;   // the Adler word after the filtered stream
    auto outputs = [&](Layout &L) { d_out = L.take(out_bytes + 16), d_adler = L.take<uint32_t>(1); };
    return stage_host_call(ctx, data, in_bytes, outputs, [&](const uint8_t *d_in, HostResults &back) {
        PIXO_TRY(pixo_b200_png_filter_dev(ctx, d_in, in_bytes, 1, width, height, row_bytes, bytes_per_pixel, strategy,
                                          d_out, out_bytes, adler32_out ? d_adler : nullptr));
        back = {{{out, d_out, out_bytes}, {adler32_out, d_adler, 4}}};
        return 0;
    });
}

int pixo_b200_png_filter_rows_dev(pixo_b200_ctx *ctx, const uint8_t *d_rows, const uint8_t *d_row_above,
                                  uint32_t width, uint32_t image_height, uint32_t band_rows,
                                  size_t row_bytes, uint32_t bytes_per_pixel, uint32_t strategy,
                                  uint8_t *d_out, uint32_t *d_adler)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_png(ctx, width, image_height, row_bytes, bytes_per_pixel, strategy));
    if (!d_rows || !d_out) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if (band_rows == 0 || band_rows > image_height)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "band_rows %u outside 1..%u", band_rows, image_height);
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return launch_png_filter_rows(ctx, d_rows, row_bytes * band_rows, 1, width, band_rows, row_bytes, bytes_per_pixel,
                                  strategy, d_out, (row_bytes + 1) * (size_t)band_rows, d_adler, d_row_above,
                                  image_height);
}

// encode_into's checks (src/png/mod.rs:442-467) plus the strategy word of the reduce entry points
static int validate_png_reduce(pixo_b200_ctx *ctx, uint32_t width, uint32_t height, uint32_t color_type,
                               uint32_t strategy_and_flags)
{
    PIXO_TRY(check_png_dimensions(ctx, width, height));
    if (color_type > PIXO_B200_RGBA)
        return set_error(ctx, PIXO_B200_ERR_UNSUPPORTED_COLOR, "Unsupported color type: %u", color_type);
    const uint32_t known = 0xFFu | PIXO_B200_PNG_OPTIMIZE_ALPHA | PIXO_B200_PNG_REDUCE_COLOR_TYPE | PIXO_B200_PNG_REDUCE_PALETTE;
    if ((strategy_and_flags & ~known) || (strategy_and_flags & 0xFFu) > PIXO_B200_FILTER_BIGRAMS)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "unknown filter strategy or flags %#x", strategy_and_flags);
    return 0;
}

int pixo_b200_png_reduce_filter_dev(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride,
                                    uint32_t n_images, uint32_t width, uint32_t height, uint32_t color_type,
                                    uint32_t strategy_and_flags, pixo_b200_png_reduced *info, uint8_t *d_out,
                                    size_t out_stride, uint32_t *d_adler)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_png_reduce(ctx, width, height, color_type, strategy_and_flags));
    if (!d_data || !d_out || !info) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    PIXO_TRY(check_batch_strides(ctx, n_images, in_stride, (size_t)width * height * (color_type + 1), "out_stride",
                                 out_stride, (size_t)height * ((size_t)width * (color_type + 1) + 1)));
    if (n_images == 0) return 0;
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return png_reduce_filter(ctx, d_data, in_stride, n_images, width, height, color_type, strategy_and_flags, info,
                             d_out, out_stride, d_adler);
}

int pixo_b200_png_reduce_filter(pixo_b200_ctx *ctx, const uint8_t *data, size_t data_len, uint32_t width,
                                uint32_t height, uint32_t color_type, uint32_t strategy_and_flags,
                                pixo_b200_png_reduced *info, uint8_t *out, size_t out_cap, size_t *out_len,
                                uint32_t *adler32_out)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_png_reduce(ctx, width, height, color_type, strategy_and_flags));
    if (!data || !out || !info || !out_len) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    const size_t in_bytes = (size_t)width * height * (color_type + 1);
    if (data_len != in_bytes)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DATA_LENGTH, "Invalid data length: expected %zu bytes, got %zu",
                         in_bytes, data_len);
    const size_t out_bytes = (size_t)height * ((size_t)width * (color_type + 1) + 1);
    uint8_t *d_out;
    uint32_t *d_adler;   // the Adler word after the filtered stream
    auto outputs = [&](Layout &L) { d_out = L.take(out_bytes + 16), d_adler = L.take<uint32_t>(1); };
    return stage_host_call(ctx, data, in_bytes, outputs, [&](const uint8_t *d_in, HostResults &back) {
        PIXO_TRY(pixo_b200_png_reduce_filter_dev(ctx, d_in, in_bytes, 1, width, height, color_type, strategy_and_flags,
                                                 info, d_out, out_bytes, d_adler));
        back = {{{out, d_out, (size_t)height * (info->row_bytes + 1), out_len, out_cap}, {adler32_out, d_adler, 4}}};
        return 0;
    });
}

// the reduce entry points' checks, the quantisation flags and QuantizationOptions::max_colors (a u16)
static int validate_png_quantize(pixo_b200_ctx *ctx, uint32_t width, uint32_t height, uint32_t color_type,
                                 uint32_t strategy_and_flags, uint32_t max_colors)
{
    const uint32_t qflags = PIXO_B200_PNG_QUANTIZE_AUTO | PIXO_B200_PNG_QUANTIZE_FORCE | PIXO_B200_PNG_DITHER;
    PIXO_TRY(validate_png_reduce(ctx, width, height, color_type, strategy_and_flags & ~qflags));
    if ((strategy_and_flags & PIXO_B200_PNG_QUANTIZE_AUTO) && (strategy_and_flags & PIXO_B200_PNG_QUANTIZE_FORCE))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "QUANTIZE_AUTO and QUANTIZE_FORCE are exclusive");
    if (max_colors > 65535)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "max_colors %u is not a u16", max_colors);
    return 0;
}

int pixo_b200_png_quantize_filter_dev(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride,
                                      uint32_t n_images, uint32_t width, uint32_t height, uint32_t color_type,
                                      uint32_t strategy_and_flags, uint32_t max_colors, const uint8_t *palettes,
                                      const uint32_t *palette_lens, pixo_b200_png_reduced *info, uint8_t *d_out,
                                      size_t out_stride, uint32_t *d_adler)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_png_quantize(ctx, width, height, color_type, strategy_and_flags, max_colors));
    if (!d_data || !d_out || !info) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if (palettes && !palette_lens) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "palettes without palette_lens");
    for (uint32_t i = 0; palettes && i < n_images; ++i)
        if (palette_lens[i] > 256)
            return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "palette_lens[%u] = %u not in 0..256", i, palette_lens[i]);
    PIXO_TRY(check_batch_strides(ctx, n_images, in_stride, (size_t)width * height * (color_type + 1), "out_stride",
                                 out_stride, (size_t)height * ((size_t)width * (color_type + 1) + 1)));
    if (n_images == 0) return 0;
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return png_quantize_filter(ctx, d_data, in_stride, n_images, width, height, color_type, strategy_and_flags,
                               max_colors, palettes, palettes ? palette_lens : nullptr, info, d_out, out_stride, d_adler);
}

int pixo_b200_png_quantize_filter(pixo_b200_ctx *ctx, const uint8_t *data, size_t data_len, uint32_t width,
                                  uint32_t height, uint32_t color_type, uint32_t strategy_and_flags,
                                  uint32_t max_colors, const uint8_t *palette, uint32_t palette_len,
                                  pixo_b200_png_reduced *info, uint8_t *out, size_t out_cap, size_t *out_len,
                                  uint32_t *adler32_out)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_png_quantize(ctx, width, height, color_type, strategy_and_flags, max_colors));
    if (!data || !out || !info || !out_len) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if ((palette == nullptr) != (palette_len == 0) || palette_len > 256)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "a given palette has 1..256 entries (palette_len %u)", palette_len);
    const size_t in_bytes = (size_t)width * height * (color_type + 1);
    if (data_len != in_bytes)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DATA_LENGTH, "Invalid data length: expected %zu bytes, got %zu",
                         in_bytes, data_len);
    uint8_t pal256[1024];
    if (palette) memcpy(pal256, palette, (size_t)palette_len * 4);
    const size_t out_bytes = (size_t)height * ((size_t)width * (color_type + 1) + 1);
    uint8_t *d_out;
    uint32_t *d_adler;   // the Adler word after the filtered stream
    auto outputs = [&](Layout &L) { d_out = L.take(out_bytes + 16), d_adler = L.take<uint32_t>(1); };
    return stage_host_call(ctx, data, in_bytes, outputs, [&](const uint8_t *d_in, HostResults &back) {
        PIXO_TRY(pixo_b200_png_quantize_filter_dev(ctx, d_in, in_bytes, 1, width, height, color_type, strategy_and_flags,
                                                   max_colors, palette ? pal256 : nullptr,
                                                   palette ? &palette_len : nullptr, info, d_out, out_bytes, d_adler));
        back = {{{out, d_out, (size_t)height * (info->row_bytes + 1), out_len, out_cap}, {adler32_out, d_adler, 4}}};
        return 0;
    });
}

uint32_t pixo_b200_adler32_combine(uint32_t adler_a, uint32_t adler_b, uint64_t len_b)
{
    const uint64_t M = 65521;
    const uint64_t a1 = adler_a & 0xFFFF, a2 = adler_a >> 16, b1 = adler_b & 0xFFFF, b2 = adler_b >> 16;
    const uint64_t s1 = (a1 + b1 + M - 1) % M;
    const uint64_t s2 = (a2 + b2 + (len_b % M) * ((a1 + M - 1) % M)) % M;
    return (uint32_t)((s2 << 16) | s1);
}

int pixo_b200_adler32_dev(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t len, uint32_t *d_out)
{
    if (!ctx || !d_out || (!d_data && len))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return launch_adler32(ctx, d_data, len, d_out);
}

int pixo_b200_adler32(pixo_b200_ctx *ctx, const uint8_t *data, size_t len, uint32_t *out)
{
    if (!ctx || !out || (!data && len))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    uint32_t *d_sum;
    auto outputs = [&](Layout &L) { d_sum = L.take<uint32_t>(1); };
    return stage_host_call(ctx, data, len, outputs, [&](const uint8_t *d_in, HostResults &back) {
        PIXO_TRY(pixo_b200_adler32_dev(ctx, d_in, len, d_sum));
        back = {{{out, d_sum, 4}}};
        return 0;
    });
}

// ---- DEFLATE ---------------------------------------------------------------------------------

// png::encode's first check (src/png/mod.rs:442-447)
static int check_level(pixo_b200_ctx *ctx, uint32_t level)
{
    if (level < 1 || level > 9)
        return set_error(ctx, PIXO_B200_ERR_INVALID_COMPRESSION_LEVEL, "Invalid compression level %u: must be 1-9", level);
    return 0;
}

// Named as pixo_b200_png_decode_to_device is, not `_dev`: like the decoders' batch call it takes host arrays (lens,
// out_lens, status) and waits for the device before it returns, where the `_dev` calls are the stream-ordered ones
int pixo_b200_deflate_zlib_on_device(pixo_b200_ctx *ctx, const uint8_t *d_streams, size_t stride, const size_t *lens,
                                     uint32_t n, uint32_t level, uint8_t *d_out, size_t out_cap_each,
                                     size_t *out_lens, int32_t *status)
{
    if (!ctx) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null context");
    PIXO_TRY(check_level(ctx, level));
    if (n && (!lens || !out_lens || !status || !d_out || !d_streams))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    // streams of a batch may not overlap: stream i is read at d_streams + i * stride
    for (uint32_t i = 0; n > 1 && i < n; i++)
        if (lens[i] > stride)
            return set_error(ctx, PIXO_B200_ERR_INVALID_DATA_LENGTH, "Invalid data length: stream %u is %zu bytes, stride %zu",
                             i, lens[i], stride);
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return deflate_zlib(ctx, d_streams, stride, lens, n, (int)level, d_out, out_cap_each, out_lens, status);
}

int pixo_b200_deflate_zlib(pixo_b200_ctx *ctx, const uint8_t *data, size_t len, uint32_t level, uint8_t *out,
                           size_t out_cap, size_t *out_len)
{
    if (!ctx) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null context");
    PIXO_TRY(check_level(ctx, level));
    if (!out_len || (!data && len) || (!out && out_cap))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    // the longest stream pixo writes: stored blocks, 5 bytes per 65 535, with the zlib header and Adler-32
    const size_t most = 2 + len + (len / 65535 + 1) * 5 + 4;
    uint8_t *d_zout;
    auto outputs = [&](Layout &L) { d_zout = L.take(most); };
    return stage_host_call(ctx, data, len, outputs, [&](const uint8_t *d_in, HostResults &back) {
        int32_t st = 0;
        PIXO_TRY(deflate_zlib(ctx, d_in, 0, &len, 1, (int)level, d_zout, most, out_len, &st));
        back = {{{out, d_zout, *out_len, out_len, out_cap}}};
        return 0;
    });
}

// ---- whole PNG files -------------------------------------------------------------------------

// encode_into's checks in pixo's order (src/png/mod.rs:437-467): the level, then those of the quantise entry points
// with OPTIMAL_COMPRESSION taken as a known flag
static int validate_png_encode(pixo_b200_ctx *ctx, uint32_t width, uint32_t height, uint32_t color_type,
                               uint32_t strategy_and_flags, uint32_t level, uint32_t max_colors)
{
    PIXO_TRY(check_level(ctx, level));
    return validate_png_quantize(ctx, width, height, color_type, strategy_and_flags & ~PIXO_B200_PNG_OPTIMAL_COMPRESSION,
                                 max_colors);
}

// The longest file of a frame: a stored-block zlib stream (2 + n + (n / 65535 + 1) * 5 + 4 bytes, the most pixo
// writes for n bytes) in IDAT chunks of 256 KiB, with the signature, IHDR and IEND; either of the unreduced rows, or,
// for RGB and RGBA, of 8-bit palette indices with the largest PLTE and tRNS
static uint64_t png_file_bound(uint32_t width, uint32_t height, uint32_t color_type)
{
    auto file = [](uint64_t n, uint64_t small) {
        const uint64_t zb = 2 + n + (n / 65535 + 1) * 5 + 4;
        return 8 + 25 + small + zb + 12 * ((zb + 262143) / 262144) + 12;
    };
    const uint64_t plain = file((uint64_t)height * ((uint64_t)width * (color_type + 1) + 1), 0);
    if (color_type != PIXO_B200_RGB && color_type != PIXO_B200_RGBA) return plain;
    return std::max(plain, file((uint64_t)height * ((uint64_t)width + 1), (12 + 768) + (12 + 256)));
}

static int refuse_optimal(pixo_b200_ctx *ctx, uint32_t strategy_and_flags)
{
    if (strategy_and_flags & PIXO_B200_PNG_OPTIMAL_COMPRESSION)
        return set_error(ctx, PIXO_B200_ERR_UNSUPPORTED, "optimal_compression (pixo's max preset) is not built");
    return 0;
}

int pixo_b200_png_encode_on_device(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride, uint32_t n_images,
                                   uint32_t width, uint32_t height, uint32_t color_type, uint32_t strategy_and_flags,
                                   uint32_t compression_level, uint32_t max_colors, const uint8_t *palettes,
                                   const uint32_t *palette_lens, uint8_t *d_out, size_t out_cap_each,
                                   size_t *out_lens, int32_t *status, pixo_b200_png_reduced *info)
{
    // the checks run before the context is needed, so that they are pixo's whether or not a device is present
    PIXO_TRY(validate_png_encode(ctx, width, height, color_type, strategy_and_flags, compression_level, max_colors));
    if (n_images && (!d_data || !d_out || !out_lens || !status))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if (palettes && !palette_lens) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "palettes without palette_lens");
    for (uint32_t i = 0; palettes && i < n_images; ++i)
        if (palette_lens[i] > 256)
            return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "palette_lens[%u] = %u not in 0..256", i, palette_lens[i]);
    const size_t in_bytes = (size_t)width * height * (color_type + 1);
    if (n_images > 1 && in_stride < in_bytes)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DATA_LENGTH, "Invalid data length: expected %zu bytes, got %zu",
                         in_bytes, in_stride);
    PIXO_TRY(refuse_optimal(ctx, strategy_and_flags));
    if (n_images == 0) return ctx ? 0 : set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    // the frames are read in passes while earlier passes' files are written
    const uintptr_t i0 = (uintptr_t)d_data, i1 = i0 + (size_t)(n_images - 1) * in_stride + in_bytes;
    const uintptr_t o0 = (uintptr_t)d_out, o1 = o0 + (size_t)n_images * out_cap_each;
    if (i0 < o1 && o0 < i1)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "the input frames and the output slots overlap");
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return png_encode(ctx, d_data, in_stride, n_images, width, height, color_type, strategy_and_flags,
                      (int)compression_level, max_colors, palettes, palettes ? palette_lens : nullptr, d_out,
                      out_cap_each, out_lens, status, info);
}

int pixo_b200_png_encode(pixo_b200_ctx *ctx, const uint8_t *data, size_t data_len, uint32_t width, uint32_t height,
                         uint32_t color_type, uint32_t strategy_and_flags, uint32_t compression_level,
                         uint32_t max_colors, const uint8_t *palette, uint32_t palette_len,
                         uint8_t *out, size_t out_cap, size_t *out_len)
{
    PIXO_TRY(validate_png_encode(ctx, width, height, color_type, strategy_and_flags, compression_level, max_colors));
    if (!data || !out_len || (!out && out_cap)) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if ((palette == nullptr) != (palette_len == 0) || palette_len > 256)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "a given palette has 1..256 entries (palette_len %u)", palette_len);
    const size_t in_bytes = (size_t)width * height * (color_type + 1);
    if (data_len != in_bytes)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DATA_LENGTH, "Invalid data length: expected %zu bytes, got %zu",
                         in_bytes, data_len);
    PIXO_TRY(refuse_optimal(ctx, strategy_and_flags));
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    uint8_t pal256[1024];
    if (palette) memcpy(pal256, palette, (size_t)palette_len * 4);
    const size_t cap = png_file_bound(width, height, color_type);
    uint8_t *d_file;
    auto outputs = [&](Layout &L) { d_file = L.take(cap); };
    return stage_host_call(ctx, data, in_bytes, outputs, [&](const uint8_t *d_in, HostResults &back) {
        size_t len = 0;
        int32_t st = 0;
        pixo_b200_png_reduced r;
        PIXO_TRY(pixo_b200_png_encode_on_device(ctx, d_in, in_bytes, 1, width, height, color_type, strategy_and_flags,
                                                compression_level, max_colors, palette ? pal256 : nullptr,
                                                palette ? &palette_len : nullptr, d_file, cap, &len, &st, &r));
        if (st)   // the slot holds the largest file, so only the stream's length can refuse the frame
            return set_error(ctx, st, "the filtered stream is %llu bytes: streams of 2^31 bytes or more are beyond "
                             "pixo's i32 positions", (unsigned long long)height * (r.row_bytes + 1));
        back = {{{out, d_file, len, out_len, out_cap}}};
        return 0;
    });
}

// ---- resize --------------------------------------------------------------------------------

// the wasm binding's enum checks (src/wasm.rs:55-67,156-166), then resize_impl's (src/resize.rs:205-250)
static int validate_resize(pixo_b200_ctx *ctx, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t color_type,
                           uint32_t algorithm)
{
    if (color_type > PIXO_B200_RGBA)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "Invalid color type: %u", color_type);
    if (algorithm > PIXO_B200_RESIZE_LANCZOS3)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "Invalid resize algorithm: %u", algorithm);
    if (sw == 0 || sh == 0)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DIMENSIONS, "Invalid image dimensions: %ux%u", sw, sh);
    if (dw == 0 || dh == 0)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DIMENSIONS, "Invalid image dimensions: %ux%u", dw, dh);
    const uint32_t mx = 1u << 24;  // src/resize.rs:30
    if (sw > mx || sh > mx || dw > mx || dh > mx)
        return set_error(ctx, PIXO_B200_ERR_IMAGE_TOO_LARGE, "Image dimensions %ux%u exceed maximum %u",
                         std::max(sw, dw), std::max(sh, dh), mx);
    return 0;
}

int pixo_b200_resize_weights(uint32_t src_size, uint32_t dst_size, uint32_t *start, uint32_t *count,
                             uint64_t *offset, float *weights, size_t weights_cap, size_t *n_weights)
{
    if (src_size == 0 || dst_size == 0)
        return set_error(nullptr, PIXO_B200_ERR_INVALID_DIMENSIONS, "Invalid size: %u -> %u", src_size, dst_size);
    if (src_size > (1u << 24) || dst_size > (1u << 24))
        return set_error(nullptr, PIXO_B200_ERR_IMAGE_TOO_LARGE, "Size %u -> %u exceeds maximum %u", src_size, dst_size,
                         1u << 24);
    if (!n_weights) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "n_weights is null");
    ResizeAxis a;
    resize_axis(src_size, dst_size, false, a);
    const size_t total = dst_size ? a.offset[dst_size - 1] + a.count[dst_size - 1] : 0;
    *n_weights = total;
    if (start) memcpy(start, a.start.data(), 4 * (size_t)dst_size);
    if (count) memcpy(count, a.count.data(), 4 * (size_t)dst_size);
    if (offset) memcpy(offset, a.offset.data(), 8 * (size_t)dst_size);
    if (!weights) return 0;
    if (weights_cap < total)
        return set_error(nullptr, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "weights capacity %zu below %zu", weights_cap, total);
    resize_axis(src_size, dst_size, true, a);
    memcpy(weights, a.w.data(), 4 * total);
    return 0;
}

int pixo_b200_resize_dev(pixo_b200_ctx *ctx, const uint8_t *d_src, size_t src_stride, uint32_t n_images,
                         uint32_t src_width, uint32_t src_height, uint32_t dst_width, uint32_t dst_height,
                         uint32_t color_type, uint32_t algorithm, uint8_t *d_dst, size_t dst_stride)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_resize(ctx, src_width, src_height, dst_width, dst_height, color_type, algorithm));
    if (!d_src || !d_dst) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    const size_t bpp = color_type + 1;
    PIXO_TRY(check_batch_strides(ctx, n_images, src_stride, (size_t)src_width * src_height * bpp, "dst_stride",
                                 dst_stride, (size_t)dst_width * dst_height * bpp));
    if (n_images == 0) return 0;
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return launch_resize(ctx, d_src, src_stride, n_images, src_width, src_height, dst_width, dst_height,
                         (uint32_t)bpp, algorithm, d_dst, dst_stride);
}

int pixo_b200_resize(pixo_b200_ctx *ctx, const uint8_t *data, size_t data_len, uint32_t src_width,
                     uint32_t src_height, uint32_t dst_width, uint32_t dst_height, uint32_t color_type,
                     uint32_t algorithm, uint8_t *out, size_t out_cap, size_t *out_len)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_resize(ctx, src_width, src_height, dst_width, dst_height, color_type, algorithm));
    if (!data || !out || !out_len) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    const size_t bpp = color_type + 1, in_bytes = (size_t)src_width * src_height * bpp;
    if (data_len != in_bytes)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DATA_LENGTH, "Invalid data length: expected %zu bytes, got %zu",
                         in_bytes, data_len);
    const size_t out_bytes = (size_t)dst_width * dst_height * bpp;
    *out_len = out_bytes;
    if (out_cap < out_bytes)
        return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu below %zu", out_cap, out_bytes);
    uint8_t *d_dst;
    auto outputs = [&](Layout &L) { d_dst = L.take(out_bytes); };
    return stage_host_call(ctx, data, in_bytes, outputs, [&](const uint8_t *d_in, HostResults &back) {
        PIXO_TRY(pixo_b200_resize_dev(ctx, d_in, in_bytes, 1, src_width, src_height, dst_width, dst_height, color_type,
                                      algorithm, d_dst, out_bytes));
        back = {{{out, d_dst, out_bytes}}};
        return 0;
    });
}

}  // extern "C"
