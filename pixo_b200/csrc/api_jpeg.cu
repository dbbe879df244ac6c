// api_jpeg.cu — the JPEG encode entry points of the C ABI: their checks, the host encode group loops, the device
// and entropy-only calls, tiled bands, header writers and progressive_file.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <thread>
#include <vector>

#include "api.hpp"
#include "jpeg_host.hpp"

using namespace pixo;

static int validate_jpeg(pixo_b200_ctx *ctx, uint32_t w, uint32_t h, uint32_t color_type,
                         uint32_t subsampling)
{
    // order follows encode_into, src/jpeg/mod.rs:333-373
    if (w == 0 || h == 0)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DIMENSIONS, "Invalid image dimensions: %ux%u", w, h);
    if (w > 65535 || h > 65535)
        return set_error(ctx, PIXO_B200_ERR_IMAGE_TOO_LARGE, "Image dimensions %ux%u exceed maximum 65535", w, h);
    if (color_type != PIXO_B200_RGB && color_type != PIXO_B200_GRAY)
        return set_error(ctx, PIXO_B200_ERR_UNSUPPORTED_COLOR, "Unsupported color type for this format");
    if (subsampling != PIXO_B200_S444 && subsampling != PIXO_B200_S420)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "unknown subsampling %u", subsampling);
    return 0;
}

extern "C" {

// encode_into validation order, src/jpeg/mod.rs:333-373: quality, then the restart interval
static int validate_options(pixo_b200_ctx *ctx, uint32_t quality, uint32_t restart_interval)
{
    if (quality == 0 || quality > 100)
        return set_error(ctx, PIXO_B200_ERR_INVALID_QUALITY, "Invalid quality %u: must be 1-100", quality);
    if (restart_interval > 65535)
        return set_error(ctx, PIXO_B200_ERR_INVALID_RESTART, "Invalid restart interval %u", restart_interval);
    return 0;
}

static void tables_from(const uint64_t *hist, bool has_chroma, HuffTables &t)
{
    // build_optimized_huffman_tables(..).unwrap_or_default(), src/jpeg/mod.rs:379-392
    if (!(hist && huff_from_histogram(hist, has_chroma, t))) huff_standard(t);
}

// A frame's tables as a DHT block (kDhtBytes: per table 16 counts + 256 values, in the order dc_lum, dc_chrom,
// ac_lum, ac_chrom) in the form the progressive stage reads; a malformed table is refused.
static int dht_prog_tables(pixo_b200_ctx *ctx, const uint8_t *dht, ProgTables *T)
{
    uint8_t bits[4][16];
    const uint8_t *vals[4];
    for (int k = 0; k < 4; ++k) {
        memcpy(bits[k], dht + k * 272, 16);
        vals[k] = dht + k * 272 + 16;
    }
    if (!prog_tables(bits, vals, T))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT,
                         "Huffman table: more than 256 values, or a code that does not fit its length");
    return 0;
}

// need: bytes of headers, scan and EOI marker
static int check_room(pixo_b200_ctx *ctx, size_t out_cap, size_t need)
{
    if (need > out_cap)
        return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu too small (need %zu)", out_cap, need);
    return 0;
}

// Ends a frame whose `body` scan bytes follow its `hdr` header bytes in out: checks that the EOI marker
// fits too, writes it and stores the frame's length.  body == (size_t)-1: the host coder ran out of room.
static int finish_frame(pixo_b200_ctx *ctx, uint8_t *out, size_t out_cap, size_t hdr, size_t body, size_t *out_len)
{
    if (body == (size_t)-1)
        return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu too small", out_cap);
    PIXO_TRY(check_room(ctx, out_cap, hdr + body + 2));
    out[hdr + body] = 0xFF;
    out[hdr + body + 1] = 0xD9;
    *out_len = hdr + body + 2;
    return 0;
}

// Coefficient records (common.cuh) of consecutive frames in one buffer: per frame the Y, Cb and Cr
// coefficient arrays, then their three extent arrays, each array 256-byte aligned, so one stride steps
// each array to the next frame's.
struct CoefLayout {
    size_t yb, cbb, yeb, ceb, each;  // bytes of the Y array, of one chroma array, of their extents, of a frame
    explicit CoefLayout(const FrameGeometry &g)
        : yb(Layout::round(g.ny * 64 * sizeof(int16_t))), cbb(Layout::round(g.nc * 64 * sizeof(int16_t))),
          yeb(Layout::round(g.ny)), ceb(Layout::round(g.nc)), each(yb + 2 * cbb + yeb + 2 * ceb) {}
    size_t stride() const { return each / sizeof(int16_t); }
    int16_t *y(void *frame) const { return reinterpret_cast<int16_t *>(frame); }
    int16_t *cb(void *frame) const { return reinterpret_cast<int16_t *>(static_cast<uint8_t *>(frame) + yb); }
    int16_t *cr(void *frame) const { return reinterpret_cast<int16_t *>(static_cast<uint8_t *>(frame) + yb + cbb); }
    CoefExtents extents(void *frame) const
    {
        uint8_t *e = static_cast<uint8_t *>(frame) + yb + 2 * cbb;
        return CoefExtents{e, e + yeb, e + yeb + ceb, each};
    }
};

// A frame's coefficient records as dense zig-zag arrays, in place (host memory): the sectors past each
// block's record become zeros.
static void expand_records(const CoefLayout &L, const FrameGeometry &g, void *frame)
{
    const CoefExtents e = L.extents(frame);
    int16_t *arr[3] = {L.y(frame), L.cb(frame), L.cr(frame)};
    const uint8_t *ext[3] = {e.y, e.cb, e.cr};
    const size_t nb[3] = {g.ny, g.nc, g.nc};
    for (int c = 0; c < (g.has_chroma ? 3 : 1); ++c)
        for (size_t b = 0; b < nb[c]; ++b) {
            const int sectors = ext[c][b];   // 1..4 sectors of 16 coefficients
            memset(arr[c] + b * 64 + sectors * 16, 0, (size_t)(4 - sectors) * 32);
        }
}

void pixo_b200_quant_tables(int quality, uint8_t lum_zz[64], uint8_t chr_zz[64], float lum[64],
                            float chr[64])
{
    quant_tables(quality, lum_zz, chr_zz, lum, chr);
}

int pixo_b200_jpeg_block_counts(uint32_t width, uint32_t height, uint32_t color_type,
                                uint32_t subsampling, size_t *ny, size_t *nc)
{
    PIXO_TRY(validate_jpeg(nullptr, width, height, color_type, subsampling));
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    if (ny) *ny = g.ny;
    if (nc) *nc = g.nc;
    return 0;
}

// Bit 0 of the trellis status word, read back after the context's stream has drained
static int trellis_status(pixo_b200_ctx *ctx, const uint32_t *d_status)
{
    PIXO_TRY(ctx->h_trellis.ensure(ctx, sizeof(uint32_t)));
    PIXO_CUDA(ctx, cudaMemcpyAsync(ctx->h_trellis.ptr, d_status, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*static_cast<const uint32_t *>(ctx->h_trellis.ptr))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT,
                         "trellis input out of range: a non-finite value or cost, a non-zero |dct| below 2^-100, or |dct / q| above 32766");
    return 0;
}

// f32 DCT scratch per piece of work: whole frames in groups that stay within kTrellisScratch (a 4K 4:2:0
// frame is ~50 MB), and a frame larger than that in bands of whole MCU rows that do.  A band's MCUs lie
// entirely inside it (only the frame's own last MCU row replicates edge rows), so a band's blocks are
// exactly the frame's, and its coefficients land at the band's first MCU in the frame's arrays.
static constexpr size_t kTrellisScratch = (size_t)256 << 20;

// COEF_TRELLIS: compute_all_coefficients(.., use_trellis = true).  Per piece the transform writes each
// block's f32 DCT to the context's scratch, then k_trellis quantises each component's blocks into the
// caller's arrays.  Queued; *d_status (the context's scratch) gets bit 0 for input k_trellis rejects.
static int trellis_pieces(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride, uint32_t n_images,
                          uint32_t width, uint32_t height, uint32_t color_type, uint32_t subsampling,
                          const float lum_q[64], const float chr_q[64], int16_t *d_y, size_t y_stride,
                          int16_t *d_cb, int16_t *d_cr, size_t c_stride, bool zigzag, uint32_t **d_status)
{
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    const bool chroma = g.has_chroma;
    const size_t row_bytes = (size_t)g.mcus_x * (g.y_per_mcu + (chroma ? 2 : 0)) * 64 * sizeof(float);  // per MCU row
    const size_t frame_bytes = row_bytes * g.mcus_y;
    const uint32_t mcu_px = g.y_per_mcu == 4 ? 16 : 8, bpp = color_type == PIXO_B200_GRAY ? 1 : 3;
    // whole frames per group, or MCU rows per band
    const uint32_t group = (uint32_t)std::max<size_t>(1, std::min<size_t>(n_images, kTrellisScratch / frame_bytes));
    const uint32_t band = frame_bytes <= kTrellisScratch
                              ? g.mcus_y
                              : (uint32_t)std::max<size_t>(1, std::min<size_t>(g.mcus_y, kTrellisScratch / row_bytes));
    const size_t piece_bytes = band < g.mcus_y ? row_bytes * band : frame_bytes * group;
    uint32_t *status;
    float *fy;
    PIXO_TRY(bind(ctx, ctx->d_trellis, [&](Layout &L) {
        status = L.take<uint32_t>(1);
        fy = L.take<float>(piece_bytes / sizeof(float));
    }));
    PIXO_CUDA(ctx, cudaMemsetAsync(status, 0, sizeof(uint32_t), ctx->stream));
    // frames [i0, i0 + nb) from MCU row m0 on, `rows` MCU rows each
    auto piece = [&](uint32_t i0, uint32_t nb, uint32_t m0, uint32_t rows) -> int {
        const uint32_t h = std::min(rows * mcu_px, height - m0 * mcu_px);
        const FrameGeometry p = make_geometry(width, h, color_type, subsampling);
        const size_t nc = chroma ? p.nc : 0;
        float *fcb = nc ? fy + (size_t)nb * p.ny * 64 : nullptr;
        float *fcr = nc ? fcb + (size_t)nb * nc * 64 : nullptr;
        const size_t y0 = (size_t)i0 * y_stride + (size_t)m0 * g.mcus_x * g.y_per_mcu * 64;
        const size_t c0 = (size_t)i0 * c_stride + (size_t)m0 * g.mcus_x * 64;
        PIXO_TRY(launch_jpeg_transform_dct(ctx, d_pixels + (size_t)i0 * pixel_stride + (size_t)m0 * mcu_px * width * bpp,
                                           pixel_stride, nb, width, h, color_type, subsampling, lum_q, chr_q, fy,
                                           p.ny * 64, fcb, fcr, nc * 64));
        PIXO_TRY(launch_trellis(ctx, fy, p.ny * 64, d_y + y0, y_stride, p.ny, nb, lum_q, 1.0f, zigzag, status));
        if (nc) {
            PIXO_TRY(launch_trellis(ctx, fcb, nc * 64, d_cb + c0, c_stride, nc, nb, chr_q, 1.0f, zigzag, status));
            PIXO_TRY(launch_trellis(ctx, fcr, nc * 64, d_cr + c0, c_stride, nc, nb, chr_q, 1.0f, zigzag, status));
        }
        return 0;
    };
    if (band == g.mcus_y) {
        for (uint32_t i0 = 0; i0 < n_images; i0 += group) PIXO_TRY(piece(i0, std::min(group, n_images - i0), 0, band));
    } else {
        for (uint32_t i = 0; i < n_images; ++i)
            for (uint32_t m0 = 0; m0 < g.mcus_y; m0 += band) PIXO_TRY(piece(i, 1, m0, band));
    }
    *d_status = status;
    return 0;
}

int pixo_b200_jpeg_coefficients_dev(pixo_b200_ctx *ctx, const uint8_t *d_pixels,
                                    size_t pixel_stride, uint32_t n_images, uint32_t width,
                                    uint32_t height, uint32_t color_type, uint32_t subsampling,
                                    const float lum_q[64], const float chr_q[64], int16_t *d_y,
                                    size_t y_stride, int16_t *d_cb, int16_t *d_cr,
                                    size_t c_stride, uint32_t flags, uint64_t *d_hist)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_jpeg(ctx, width, height, color_type, subsampling));
    if (!d_pixels || !d_y || !lum_q || !chr_q)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if (color_type != PIXO_B200_GRAY && (!d_cb || !d_cr))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null chroma buffer");
    if ((flags & PIXO_B200_COEF_TRELLIS) && d_hist)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT,
                         "COEF_TRELLIS takes no histogram (pixo's tables come from plain-rounded coefficients)");
    if (n_images == 0) return 0;
    if ((reinterpret_cast<uintptr_t>(d_y) & 15) || (y_stride & 7) ||
        (d_cb && ((reinterpret_cast<uintptr_t>(d_cb) & 15) || (reinterpret_cast<uintptr_t>(d_cr) & 15) || (c_stride & 7))))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT,
                         "coefficient buffers must be 16-byte aligned with strides multiple of 8");
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    if (flags & PIXO_B200_COEF_TRELLIS) {   // waits for the device: the input check is reported by the call
        uint32_t *status;
        PIXO_TRY(trellis_pieces(ctx, d_pixels, pixel_stride, n_images, width, height, color_type, subsampling, lum_q,
                                chr_q, d_y, y_stride, color_type == PIXO_B200_GRAY ? nullptr : d_cb,
                                color_type == PIXO_B200_GRAY ? nullptr : d_cr, c_stride,
                                (flags & PIXO_B200_COEF_ZIGZAG) != 0, &status));
        return trellis_status(ctx, status);
    }
    PIXO_TRY(launch_jpeg_transform(ctx, d_pixels, pixel_stride, n_images, width, height,
                                   color_type, subsampling, lum_q, chr_q, d_y, y_stride, d_cb,
                                   d_cr, c_stride, flags));
    if (d_hist) {
        const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
        PIXO_TRY(launch_jpeg_histogram(ctx, d_y, y_stride, d_cb, d_cr, c_stride, n_images, g.ny,
                                       g.nc, g.y_per_mcu, 0, (flags & PIXO_B200_COEF_ZIGZAG) != 0,
                                       nullptr, d_hist));
    }
    return 0;
}

// Like every host-buffer entry point: the input staged in the context's scratch, the `_dev` twin on it as
// a batch of one, the results copied out (stage_host_call)
int pixo_b200_jpeg_coefficients(pixo_b200_ctx *ctx, const uint8_t *pixels, uint32_t width,
                                uint32_t height, uint32_t color_type, uint32_t subsampling,
                                const float lum_q[64], const float chr_q[64], int16_t *y,
                                int16_t *cb, int16_t *cr, uint32_t flags, uint64_t *hist)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_jpeg(ctx, width, height, color_type, subsampling));
    if (!pixels || !y || !lum_q || !chr_q || (color_type != PIXO_B200_GRAY && (!cb || !cr)))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if ((flags & PIXO_B200_COEF_TRELLIS) && hist)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT,
                         "COEF_TRELLIS takes no histogram (pixo's tables come from plain-rounded coefficients)");
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    const size_t in_bytes = (size_t)width * height * (color_type == PIXO_B200_GRAY ? 1 : 3);
    const size_t yb = g.ny * 64 * sizeof(int16_t), cbb = g.nc * 64 * sizeof(int16_t);
    const size_t hist_bytes = kHistWords * sizeof(uint64_t);
    int16_t *dy, *dcb = nullptr, *dcr = nullptr;
    uint64_t *d_hist = nullptr;
    auto outputs = [&](Layout &L) {
        dy = L.take<int16_t>(g.ny * 64);
        if (cbb) dcb = L.take<int16_t>(g.nc * 64), dcr = L.take<int16_t>(g.nc * 64);
        if (hist) d_hist = L.take<uint64_t>(kHistWords);
    };
    return stage_host_call(ctx, pixels, in_bytes, outputs, [&](const uint8_t *d_in, HostResults &back) {
        PIXO_TRY(pixo_b200_jpeg_coefficients_dev(ctx, d_in, in_bytes, 1, width, height, color_type, subsampling, lum_q,
                                                 chr_q, dy, g.ny * 64, dcb, dcr, g.nc * 64, flags, d_hist));
        back = {{{y, dy, yb}, {cbb ? cb : nullptr, dcb, cbb}, {cbb ? cr : nullptr, dcr, cbb},
                 {hist, d_hist, hist_bytes}}};
        return 0;
    });
}

int pixo_b200_jpeg_trellis_quantize_dev(pixo_b200_ctx *ctx, const float *d_dct, size_t n_blocks, const float q[64],
                                        float lambda, int16_t *d_out, uint32_t flags)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    if (!d_dct || !q || !d_out) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    for (int k = 0; k < 64; ++k)   // every table pixo builds; the exact division is proved for these
        if (!(q[k] >= 1.0f && q[k] <= 255.0f && q[k] == (float)(int)q[k]))
            return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "quantisation table entries must be integers in 1..255");
    if (!std::isfinite(lambda)) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "lambda is not finite");
    if ((reinterpret_cast<uintptr_t>(d_dct) & 15) || (reinterpret_cast<uintptr_t>(d_out) & 15))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "block buffers must be 16-byte aligned");
    if (n_blocks == 0) return 0;
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    PIXO_TRY(ctx->d_trellis.ensure(ctx, 256));
    auto *status = static_cast<uint32_t *>(ctx->d_trellis.ptr);
    PIXO_CUDA(ctx, cudaMemsetAsync(status, 0, sizeof(uint32_t), ctx->stream));
    PIXO_TRY(launch_trellis(ctx, d_dct, 0, d_out, 0, n_blocks, 1, q, lambda, (flags & PIXO_B200_COEF_ZIGZAG) != 0,
                            status));
    return trellis_status(ctx, status);
}

// Device scan capacity per frame: a JPEG that needs more than half its raw size (noise at very
// high quality) is coded a second time with the exact size the kernel reported.
static uint64_t default_scan_cap(const pixo_b200_ctx *ctx, size_t raw_bytes)
{
    const size_t want = ctx->scan_cap_override ? ctx->scan_cap_override : (raw_bytes / 2 + 65536) / 8 * 9;
    return Layout::round(want < 1024 ? 1024 : want);
}

constexpr int kGaveUp = -1;  // recode_scan: the device stage did not finish the scan
static const char kOutOfRange[] = "coefficient out of the baseline range (|AC| <= 1023, |DC difference| <= 2047)";

// Codes one frame's scan on the device until it fits, in ctx->d_retry: the scan, then the entropy
// stage's scratch.  The first pass may be cut into segments and has `cap` bytes.  After a pass
// that did not finish, its flags decide: bit 3 (a coefficient outside the baseline range) is
// ERR_INVALID_ARGUMENT; bit 1 (a look-back chain timed out) gives up; bit 2 (a
// segment outgrew its share) runs again unsegmented; bit 0 (the scan did not fit, and the length is
// the size it needs) runs again with room for that size, unless headers, scan and EOI would no
// longer fit out_cap.  Three passes at most.  Returns 0 with the scan at the start of d_retry and
// its length in *len, kGaveUp, or an error.  It touches no other scratch of the context but
// d_raw (segmented passes), so the baseline group loop can use it while the next group's work is queued.
// ext: the transform's coefficient records (always in range); null: the caller's arrays, checked
// (launch_jpeg_entropy).
static int recode_scan(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb, const int16_t *d_cr,
                       const CoefExtents *ext, const FrameGeometry &g, const HuffTables &t, uint32_t restart_interval,
                       bool segments, size_t cap, size_t hdr, size_t out_cap, size_t *len)
{
    const size_t ent = entropy_scratch_bytes(1, g, restart_interval);
    for (int pass = 0;; ++pass) {
        uint8_t *scan, *scratch;
        PIXO_TRY(bind(ctx, ctx->d_retry, [&](Layout &L) { scan = L.take(cap), scratch = L.take(ent); }));
        uint64_t *d_len = nullptr;
        uint32_t *d_ovf = nullptr;
        PIXO_TRY(launch_jpeg_entropy(ctx, d_y, 0, d_cb, d_cr, 0, 1, g, t, restart_interval, segments, ext, scratch, scan,
                                     cap, &d_len, &d_ovf));
        uint64_t n = 0;
        uint32_t ovf = 0;
        PIXO_CUDA(ctx, cudaMemcpyAsync(&n, d_len, 8, cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaMemcpyAsync(&ovf, d_ovf, 4, cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (!ovf) {
            *len = (size_t)n;
            return 0;
        }
        if (ovf & kOvfRange) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "%s", kOutOfRange);
        if ((ovf & kOvfFault) || pass == 2) return kGaveUp;
        if (ovf & kOvfSegment) {
            segments = false;
            continue;
        }
        PIXO_TRY(check_room(ctx, out_cap, hdr + (size_t)n + 2));
        cap = Layout::round((size_t)n + 64);
    }
}

// The transform of cnt frames, pixel_stride bytes apart, into coefficient records at c (layout L)
static int transform_records(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride, uint32_t cnt,
                             const FrameGeometry &g, const float *lum, const float *chr, const CoefLayout &L, uint8_t *c)
{
    const CoefExtents ec = L.extents(c);
    return launch_jpeg_transform(ctx, d_pixels, pixel_stride, cnt, g.width, g.height, g.color_type, g.subsampling, lum,
                                 chr, L.y(c), L.stride(), g.has_chroma ? L.cb(c) : nullptr,
                                 g.has_chroma ? L.cr(c) : nullptr, L.stride(), 0, &ec);
}

// k_huff, segments allowed, over the coefficient records of cnt frames at c, in one pass: with tables t, or with
// each frame's own tables d_tabs (launch_huff_tables) when that is not null.  Frame k's scan goes to
// scan + k * scan_cap, its length and overflow flags to len[k] and ovf[k] (host or device memory, as `kind` says).
static int code_records(pixo_b200_ctx *ctx, const CoefLayout &L, uint8_t *c, uint32_t cnt, const FrameGeometry &g,
                        const HuffTables &t, const void *d_tabs, uint32_t restart_interval, uint8_t *ent, uint8_t *scan,
                        uint64_t scan_cap, uint64_t *len, uint32_t *ovf, cudaMemcpyKind kind)
{
    const size_t cs = L.stride();
    const CoefExtents ec = L.extents(c);
    uint64_t *d_len = nullptr;
    uint32_t *d_ovf = nullptr;
    PIXO_TRY(launch_jpeg_entropy(ctx, L.y(c), cs, L.cb(c), L.cr(c), cs, cnt, g, t, restart_interval, true, &ec, ent, scan,
                                 scan_cap, &d_len, &d_ovf, d_tabs));
    PIXO_CUDA(ctx, cudaMemcpyAsync(len, d_len, (size_t)cnt * 8, kind, ctx->stream));
    PIXO_CUDA(ctx, cudaMemcpyAsync(ovf, d_ovf, (size_t)cnt * 4, kind, ctx->stream));
    return 0;
}

// The tables of cnt frames' coefficient records at c, between the transform and code_records: optimize, K3's
// statistics into d_hist and each frame's tables from them (k_huff_tables) into d_dht and d_tabs; otherwise the
// standard tables' DHT blocks into d_dht when it is not null.
static int baseline_tables(pixo_b200_ctx *ctx, const CoefLayout &L, uint8_t *c, uint32_t cnt, const FrameGeometry &g,
                           uint32_t restart_interval, bool optimize, uint64_t *d_hist, uint8_t *d_dht, void *d_tabs)
{
    if (optimize) {
        const CoefExtents ec = L.extents(c);
        const size_t cs = L.stride();
        PIXO_TRY(launch_jpeg_histogram(ctx, L.y(c), cs, L.cb(c), L.cr(c), cs, cnt, g.ny, g.nc, g.y_per_mcu,
                                       restart_interval, false, &ec, d_hist));
        return launch_huff_tables(ctx, d_hist, cnt, g.has_chroma, d_dht, d_tabs);
    }
    return d_dht ? launch_huff_tables(ctx, nullptr, cnt, g.has_chroma, d_dht, nullptr) : 0;
}

// What the two group loops of the host encode share: n frames, G per group, each group's pixels uploaded on the
// copy stream into one of two input slots of d_in, in turn, while the context's stream works on the group before.
struct EncodeGroups {
    pixo_b200_ctx *ctx;
    const uint8_t *pixels;
    size_t len_each, in_stride;
    uint32_t n, G;

    uint32_t count() const { return (n + G - 1) / G; }
    uint32_t size(uint32_t gi) const { return std::min(G, n - gi * G); }
    uint8_t *input(uint32_t gi) const { return ctx->d_in.slot(gi & 1, (size_t)G * in_stride); }
    // Group gi's frames into its input slot.  Group 0 first makes both copy streams wait for whatever the caller
    // already queued on the context's stream (ev_out[0] is free until group 0's scan bytes are copied back);
    // group gi >= 2 waits until the transform of group gi - 2 has read the slot.
    int upload(uint32_t gi) const
    {
        const int slot = (int)(gi & 1);
        if (gi == 0) {
            PIXO_CUDA(ctx, cudaEventRecord(ctx->ev_out[0], ctx->stream));
            PIXO_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_out[0], 0));
            PIXO_CUDA(ctx, cudaStreamWaitEvent(ctx->d2h_stream, ctx->ev_out[0], 0));
        }
        if (gi >= 2) PIXO_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_used[slot], 0));
        for (uint32_t k = 0; k < size(gi); ++k)
            PIXO_TRY(h2d_copy(ctx, input(gi) + k * in_stride, pixels + ((size_t)gi * G + k) * len_each, len_each,
                              ctx->copy_stream));
        PIXO_CUDA(ctx, cudaEventRecord(ctx->ev_in[slot], ctx->copy_stream));
        return 0;
    }
};

// The groups of a host encode call: about 96 MB of input (4 frames at 4K, 15 at 1080p), at most 16, at
// least two groups per call: long enough for full-rate DMA and to amortise the launches, short enough that what
// no upload can hide - the last group's kernels and the read-back of its scan bytes - stays small.  Fewer while
// the baseline loop's scratch for two groups would pass 4 GiB; the progressive loop groups its frames the same way.
static EncodeGroups make_groups(pixo_b200_ctx *ctx, const uint8_t *pixels, uint32_t n, size_t len_each,
                                const FrameGeometry &g, uint32_t restart_interval)
{
    const size_t in_stride = Layout::round(len_each), coef_each = CoefLayout(g).each;
    const uint64_t scan_cap = default_scan_cap(ctx, len_each);
    uint32_t G = (uint32_t)std::min<size_t>(16, std::max<size_t>(1, (((size_t)96 << 20) + len_each / 2) / len_each));
    G = std::min(G, std::max(1u, (n + 1) / 2));
    auto group_bytes = [&](uint32_t k) {
        return 2 * (size_t)k * (in_stride + coef_each + scan_cap) + entropy_scratch_bytes(k, g, restart_interval);
    };
    while (G > 1 && group_bytes(G) > ((size_t)4 << 30)) --G;
    return EncodeGroups{ctx, pixels, len_each, in_stride, n, G};
}

// Baseline frames.  GPU: colour/DCT/quantise into coefficient records (K1/K2), when optimize symbol statistics
// (K3) and each frame's tables (k_huff_tables), k_huff; host: headers, EOI.  The H2D copy of group g+1 and the D2H
// copy of group g-1's scan bytes (d2h stream) run under the kernels of group g: the host never drains the compute
// stream between groups, it waits only for the event behind a group's lengths and tables before it queues that
// group's D2H of finished scan bytes.  A scan that does not fit is coded again on the GPU with the exact size; the
// host entropy coder is the last resort for a faulted device stage, counted in ctx->host_fallbacks.  Both use the
// frame's tables on the host: by then the next group's k_huff_tables may have overwritten the device copy.
static int encode_baseline_groups(pixo_b200_ctx *ctx, const EncodeGroups &grp, const FrameGeometry &g,
                                  uint32_t quality, uint32_t restart_interval, bool optimize, uint8_t *out,
                                  size_t out_cap_each, size_t *out_lens)
{
    float lum[64], chr[64];
    uint8_t lum_zz[64], chr_zz[64];
    quant_tables((int)quality, lum_zz, chr_zz, lum, chr);
    const CoefLayout L(g);
    const uint32_t G = grp.G;
    const uint64_t scan_cap = default_scan_cap(ctx, grp.len_each);
    uint64_t *d_hist, *h_lens[2];
    uint8_t *d_dht, *d_own, *h_dhts[2];
    uint32_t *h_ovfs[2];
    PIXO_TRY(ctx->d_coef.ensure(ctx, 2 * (size_t)G * L.each));
    PIXO_TRY(ctx->d_ent.ensure(ctx, entropy_scratch_bytes(G, g, restart_interval)));
    PIXO_TRY(ctx->d_out.ensure(ctx, 2 * (size_t)G * scan_cap));
    // d_misc: a group's statistics, its DHT blocks, its tables in k_huff's form
    PIXO_TRY(bind(ctx, ctx->d_misc, [&](Layout &M) {
        d_hist = M.take<uint64_t>((size_t)G * kHistWords);
        d_dht = M.take((size_t)G * kDhtBytes);
        d_own = M.take((size_t)G * kHuffDevBytes);
    }));
    // h_misc, per input slot: a group's lengths, overflow flags and DHT blocks, packed
    PIXO_TRY(bind(ctx, ctx->h_misc, [&](Layout &H) {
        for (int s = 0; s < 2; ++s)
            h_lens[s] = H.take<uint64_t>(G), h_ovfs[s] = H.take<uint32_t>(G), h_dhts[s] = H.take((size_t)G * kDhtBytes);
    }, 8));
    auto *d_scan = static_cast<uint8_t *>(ctx->d_out.ptr);
    void *d_tabs = optimize ? d_own : nullptr;
    auto coef_of = [&](int slot) { return ctx->d_coef.slot(slot, (size_t)G * L.each); };
    HuffTables std_t;
    huff_from_dht(dht_standard(), std_t);
    const bool out_locked = is_page_locked(out);

    // queue the kernels of group gi and the readback of its lengths and tables
    auto compute = [&](uint32_t gi) -> int {
        const uint32_t cnt = grp.size(gi);
        const int slot = (int)(gi & 1);
        uint8_t *c = coef_of(slot);
        PIXO_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_in[slot], 0));
        PIXO_TRY(transform_records(ctx, grp.input(gi), grp.in_stride, cnt, g, lum, chr, L, c));
        PIXO_CUDA(ctx, cudaEventRecord(ctx->ev_used[slot], ctx->stream));
        PIXO_TRY(baseline_tables(ctx, L, c, cnt, g, restart_interval, optimize, d_hist, optimize ? d_dht : nullptr, d_tabs));
        if (gi >= 2) PIXO_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_out[slot], 0));  // slot's previous D2H drained
        PIXO_TRY(code_records(ctx, L, c, cnt, g, std_t, d_tabs, restart_interval,
                              reinterpret_cast<uint8_t *>(ctx->d_ent.ptr), d_scan + (size_t)slot * G * scan_cap, scan_cap,
                              h_lens[slot], h_ovfs[slot], cudaMemcpyDeviceToHost));
        if (optimize)
            PIXO_CUDA(ctx, cudaMemcpyAsync(h_dhts[slot], d_dht, (size_t)cnt * kDhtBytes, cudaMemcpyDeviceToHost,
                                           ctx->stream));
        PIXO_CUDA(ctx, cudaEventRecord(ctx->ev_len[slot], ctx->stream));
        return 0;
    };

    // headers on the host, scan bytes straight from the device (d2h stream), EOI
    auto finish = [&](uint32_t gi) -> int {
        const uint32_t first = gi * G, cnt = grp.size(gi);
        const int slot = (int)(gi & 1);
        uint8_t *c = coef_of(slot);
        uint8_t *scan = d_scan + (size_t)slot * G * scan_cap;
        const uint64_t *h_len = h_lens[slot];
        const uint32_t *h_ovf = h_ovfs[slot];
        PIXO_CUDA(ctx, cudaEventSynchronize(ctx->ev_len[slot]));
        std::vector<HuffTables> tb(optimize ? cnt : 0);   // each frame's tables, from its DHT block
        for (uint32_t k = 0; k < tb.size(); ++k) huff_from_dht(h_dhts[slot] + (size_t)k * kDhtBytes, tb[k]);
        auto tables = [&](uint32_t k) -> const HuffTables & { return optimize ? tb[k] : std_t; };
        std::vector<size_t> hdr(cnt);
        bool redo = false;
        for (uint32_t k = 0; k < cnt; ++k) {
            const uint32_t img = first + k;
            uint8_t *o = out + (size_t)img * out_cap_each;
            hdr[k] = write_headers(o, g, lum_zz, chr_zz, tables(k), restart_interval);
            if (h_ovf[k]) { redo = true; continue; }
            const size_t body = (size_t)h_len[k];
            PIXO_TRY(finish_frame(ctx, o, out_cap_each, hdr[k], body, &out_lens[img]));
            if (out_locked)
                PIXO_CUDA(ctx, cudaMemcpyAsync(o + hdr[k], scan + (size_t)k * scan_cap, body, cudaMemcpyDeviceToHost,
                                               ctx->d2h_stream));
            else   // ordinary caller memory: through the pinned ring, copied out by the host pool
                PIXO_TRY(d2h_copy_sync(ctx, o + hdr[k], scan + (size_t)k * scan_cap, body, ctx->d2h_stream));
        }
        PIXO_CUDA(ctx, cudaEventRecord(ctx->ev_out[slot], ctx->d2h_stream));
        if (!redo) return 0;
        // Frames the first pass did not finish.  Their coefficients are still in this slot of
        // d_coef (the next group's transform writes the other one).
        for (uint32_t k = 0; k < cnt; ++k) {
            if (!h_ovf[k]) continue;
            const uint32_t img = first + k;
            uint8_t *o = out + (size_t)img * out_cap_each;
            uint8_t *f = c + (size_t)k * L.each;
            const HuffTables &t = tables(k);
            // bit 0: the scan did not fit (the kernel reported the size it needs); bit 2: a segment's raw
            // string did not fit its share - either way code the frame again on the GPU, unsegmented, with
            // enough room.  Bit 1 (a faulted chain) goes to the host coder.
            int rc = kGaveUp;
            size_t body = 0;
            if (!(h_ovf[k] & kOvfFault) && ctx->gpu_retry) {
                const size_t need = (h_ovf[k] & kOvfSegment) ? (size_t)scan_cap * 2 : (size_t)h_len[k];
                if (!(h_ovf[k] & kOvfSegment)) PIXO_TRY(check_room(ctx, out_cap_each, hdr[k] + need + 2));
                const CoefExtents ef = L.extents(f);
                rc = recode_scan(ctx, L.y(f), L.cb(f), L.cr(f), &ef, g, t, restart_interval, false, Layout::round(need + 64),
                                 hdr[k], out_cap_each, &body);
                if (rc != 0 && rc != kGaveUp) return rc;
            }
            if (rc == 0) {
                PIXO_TRY(finish_frame(ctx, o, out_cap_each, hdr[k], body, &out_lens[img]));
                PIXO_CUDA(ctx, cudaMemcpyAsync(o + hdr[k], ctx->d_retry.ptr, body, cudaMemcpyDeviceToHost, ctx->stream));
                PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                continue;
            }
            // last resort: the host entropy coder on the GPU's coefficient records, made dense
            ctx->host_fallbacks += 1;
            PIXO_TRY(ctx->h_out.ensure(ctx, L.each));
            auto *hc = reinterpret_cast<uint8_t *>(ctx->h_out.ptr);
            PIXO_CUDA(ctx, cudaMemcpyAsync(hc, f, L.each, cudaMemcpyDeviceToHost, ctx->stream));
            PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            expand_records(L, g, hc);
            body = entropy_encode_scan(L.y(hc), L.cb(hc), L.cr(hc), g, t, restart_interval, true, o + hdr[k],
                                       out_cap_each - hdr[k] - 2, ctx->host_threads);
            PIXO_TRY(finish_frame(ctx, o, out_cap_each, hdr[k], body, &out_lens[img]));
        }
        return 0;
    };

    PIXO_TRY(grp.upload(0));
    for (uint32_t gi = 0; gi < grp.count(); ++gi) {
        if (gi + 1 < grp.count()) PIXO_TRY(grp.upload(gi + 1));
        PIXO_TRY(compute(gi));
        if (gi > 0) PIXO_TRY(finish(gi - 1));
    }
    return finish(grp.count() - 1);
}

// A progressive pass's coefficients and tables, queued in pixo's order (encode_progressive, src/jpeg/mod.rs:872-927),
// which builds the tables from the plain-rounded coefficients before trellis overwrites them: the plain transform into
// dense arrays at c when the tables need it or no trellis follows, K3 with the restart interval (optimize),
// k_huff_tables into d_dht unless it is null, COEF_TRELLIS (*d_trellis_status: its status word, null without it).
static int progressive_coefficients(pixo_b200_ctx *ctx, const uint8_t *px, size_t pixel_stride, uint32_t cnt,
                                    const FrameGeometry &g, const float *lum, const float *chr, const CoefLayout &L,
                                    uint8_t *c, uint32_t restart_interval, bool optimize, bool trellis,
                                    uint64_t *d_hist, uint8_t *d_dht, uint32_t **d_trellis_status)
{
    const size_t cs = L.stride();
    int16_t *cb = g.has_chroma ? L.cb(c) : nullptr, *cr = g.has_chroma ? L.cr(c) : nullptr;
    if (optimize || !trellis)
        PIXO_TRY(launch_jpeg_transform(ctx, px, pixel_stride, cnt, g.width, g.height, g.color_type, g.subsampling, lum,
                                       chr, L.y(c), cs, cb, cr, cs, 0));
    if (optimize)
        PIXO_TRY(launch_jpeg_histogram(ctx, L.y(c), cs, cb, cr, cs, cnt, g.ny, g.nc, g.y_per_mcu, restart_interval,
                                       false, nullptr, d_hist));
    if (d_dht) PIXO_TRY(launch_huff_tables(ctx, optimize ? d_hist : nullptr, cnt, g.has_chroma, d_dht, nullptr));
    *d_trellis_status = nullptr;
    if (trellis)
        PIXO_TRY(trellis_pieces(ctx, px, pixel_stride, cnt, g.width, g.height, g.color_type, g.subsampling, lum, chr,
                                L.y(c), cs, cb, cr, cs, false, d_trellis_status));
    return 0;
}

// A progressive file around its 7 segments of len[s] bytes: SOF2 headers with DHT block dht's tables, per scan its SOS
// and segment, EOI.  Checks the room, then writes all but the segments (out + at[s]) and the length to *out_len.
static int progressive_layout(pixo_b200_ctx *ctx, const FrameGeometry &g, const uint8_t lum_zz[64],
                              const uint8_t chr_zz[64], const uint8_t *dht, uint32_t restart_interval,
                              const uint64_t len[7], uint8_t *out, size_t out_cap, size_t at[7], size_t *out_len)
{
    HuffTables t;
    huff_from_dht(dht, t);
    uint8_t hdr[2048];   // 281 bytes + the tables' values (at most 4 x 256)
    size_t pos = write_headers_progressive(hdr, g, lum_zz, chr_zz, t, restart_interval);
    size_t need = pos + 7 * 10 + 2;
    for (int s = 0; s < 7; ++s) need += (size_t)len[s];
    PIXO_TRY(check_room(ctx, out_cap, need));
    memcpy(out, hdr, pos);
    for (int s = 0; s < 7; ++s) {
        pos += write_sos_progressive(out + pos, s);
        at[s] = pos;
        pos += (size_t)len[s];
    }
    out[pos] = 0xFF;
    out[pos + 1] = 0xD9;
    *out_len = pos + 2;
    return 0;
}

// Progressive frames: progressive_coefficients, the 7 scans, each file around them (progressive_layout).  The stage's
// buffers are the context's, so each group is finished before the next: one coefficient slot and DHT set serve all.
static int encode_progressive_groups(pixo_b200_ctx *ctx, const EncodeGroups &grp, const FrameGeometry &g,
                                     uint32_t quality, uint32_t restart_interval, bool optimize, bool trellis,
                                     uint8_t *out, size_t out_cap_each, size_t *out_lens)
{
    float lum[64], chr[64];
    uint8_t lum_zz[64], chr_zz[64];
    quant_tables((int)quality, lum_zz, chr_zz, lum, chr);
    const CoefLayout L(g);
    const size_t cs = L.stride();
    uint64_t *d_hist;
    uint8_t *d_dht;
    PIXO_TRY(ctx->d_coef.ensure(ctx, (size_t)grp.G * L.each));
    // d_misc: a group's statistics, its DHT blocks
    PIXO_TRY(bind(ctx, ctx->d_misc, [&](Layout &M) {
        d_hist = M.take<uint64_t>((size_t)grp.G * kHistWords);
        d_dht = M.take((size_t)grp.G * kDhtBytes);
    }));
    PIXO_TRY(ctx->h_misc.ensure(ctx, (size_t)grp.G * kDhtBytes));
    auto *c = reinterpret_cast<uint8_t *>(ctx->d_coef.ptr);
    int16_t *cb = g.has_chroma ? L.cb(c) : nullptr, *cr = g.has_chroma ? L.cr(c) : nullptr;
    auto *h_dht = static_cast<const uint8_t *>(ctx->h_misc.ptr);
    // frame k's tables: its own (optimize), or the standard ones
    auto dht_of = [&](uint32_t k) { return optimize ? h_dht + (size_t)k * kDhtBytes : dht_standard(); };
    PIXO_TRY(grp.upload(0));
    for (uint32_t gi = 0; gi < grp.count(); ++gi) {
        if (gi + 1 < grp.count()) PIXO_TRY(grp.upload(gi + 1));
        // coefficients, tables and the 7 segments of every frame of the group (waits for the device)
        const uint32_t cnt = grp.size(gi);
        PIXO_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_in[gi & 1], 0));
        // DHT blocks only when optimised: the host has the standard tables without a k_huff_tables launch
        uint32_t *status;
        PIXO_TRY(progressive_coefficients(ctx, grp.input(gi), grp.in_stride, cnt, g, lum, chr, L, c, restart_interval,
                                          optimize, trellis, d_hist, optimize ? d_dht : nullptr, &status));
        PIXO_CUDA(ctx, cudaEventRecord(ctx->ev_used[gi & 1], ctx->stream));
        if (optimize)
            PIXO_CUDA(ctx, cudaMemcpyAsync(ctx->h_misc.ptr, d_dht, (size_t)cnt * kDhtBytes, cudaMemcpyDeviceToHost,
                                           ctx->stream));
        if (trellis)   // waits for the device, the DHT blocks' copy included
            PIXO_TRY(trellis_status(ctx, status));
        else if (optimize)
            PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        std::vector<ProgTables> pt(optimize ? cnt : 1);
        for (uint32_t k = 0; k < pt.size(); ++k) PIXO_TRY(dht_prog_tables(ctx, dht_of(k), &pt[k]));
        ProgSlots slots;   // in d_prog_out, sized from the measured strings
        PIXO_TRY(launch_progressive(ctx, L.y(c), cs, cb, cr, cs, cnt, g, nullptr, pt.data(), optimize, nullptr, &slots));
        // every segment's length and every frame's flags to h_prog
        uint64_t *h_len;
        uint32_t *h_ovf;
        PIXO_TRY(bind(ctx, ctx->h_prog, [&](Layout &H) {
            h_len = H.take<uint64_t>((size_t)cnt * 7);
            h_ovf = H.take<uint32_t>(cnt);
        }, 8));
        PIXO_CUDA(ctx, cudaMemcpyAsync(h_len, slots.scan_len, (size_t)cnt * 7 * 8, cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaMemcpyAsync(h_ovf, slots.overflow, (size_t)cnt * 4, cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        // each file around its segments, which come from the device
        for (uint32_t k = 0; k < cnt; ++k) {
            if (h_ovf[k]) return set_error(ctx, PIXO_B200_ERR_CUDA, "progressive splice overflowed its slot");
            const uint32_t img = gi * grp.G + k;
            uint8_t *o = out + (size_t)img * out_cap_each;
            const uint64_t *len = h_len + (size_t)k * 7;
            size_t at[7];
            PIXO_TRY(progressive_layout(ctx, g, lum_zz, chr_zz, dht_of(k), restart_interval, len, o, out_cap_each, at,
                                        &out_lens[img]));
            const uint8_t *seg = slots.out + (size_t)k * slots.cap;
            for (int s = 0; s < 7; ++s) {
                if (len[s]) PIXO_TRY(d2h_copy_sync(ctx, o + at[s], seg, (size_t)len[s], ctx->stream));
                seg += len[s];
            }
        }
    }
    return 0;
}

// The scans a host encode call writes; Refused: pixo_b200_jpeg_encode with progressive = 1
enum class Scans { Baseline, Progressive, Refused };

// The four host encode entry points: their checks, in this order, then the frames in groups through the
// baseline or the progressive loop, which leave work queued; an error return drains every stream first.
static int encode_host(pixo_b200_ctx *ctx, const uint8_t *pixels, size_t len_each, uint32_t n_images, uint32_t width,
                       uint32_t height, uint32_t color_type, uint32_t quality, uint32_t subsampling,
                       uint32_t restart_interval, bool optimize, Scans scans, bool trellis, uint8_t *out,
                       size_t out_cap_each, size_t *out_lens)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_options(ctx, quality, restart_interval));
    PIXO_TRY(validate_jpeg(ctx, width, height, color_type, subsampling));
    const size_t expected = (size_t)width * height * (color_type == PIXO_B200_GRAY ? 1 : 3);
    if (len_each != expected)
        return set_error(ctx, PIXO_B200_ERR_INVALID_DATA_LENGTH, "Invalid data length: expected %zu bytes, got %zu",
                         expected, len_each);
    if (!pixels || !out || !out_lens) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if (scans == Scans::Refused)
        return set_error(ctx, PIXO_B200_ERR_UNSUPPORTED,
                         "progressive JPEGs are encoded by pixo_b200_jpeg_encode_progressive");
    if (n_images == 0) return 0;
    if (out_cap_each < 1024 + 2)  // before any GPU work is queued
        return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu too small", out_cap_each);
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    const EncodeGroups grp = make_groups(ctx, pixels, n_images, len_each, g, restart_interval);
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    PIXO_TRY(ctx->d_in.ensure(ctx, 2 * (size_t)grp.G * grp.in_stride));
    DrainOnError drain(ctx);
    PIXO_TRY(scans == Scans::Progressive
                 ? encode_progressive_groups(ctx, grp, g, quality, restart_interval, optimize, trellis, out, out_cap_each,
                                             out_lens)
                 : encode_baseline_groups(ctx, grp, g, quality, restart_interval, optimize, out, out_cap_each, out_lens));
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->d2h_stream));
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    drain.armed = false;
    return 0;
}

int pixo_b200_jpeg_encode(pixo_b200_ctx *ctx, const uint8_t *pixels, size_t pixels_len,
                          uint32_t width, uint32_t height, uint32_t color_type, uint32_t quality,
                          uint32_t subsampling, uint32_t restart_interval,
                          uint32_t optimize_huffman, uint32_t progressive, uint32_t trellis_quant,
                          uint8_t *out, size_t out_cap, size_t *out_len)
{
    (void)trellis_quant;  // baseline encode_scan ignores use_trellis (src/jpeg/mod.rs:1408-1563)
    return encode_host(ctx, pixels, pixels_len, 1, width, height, color_type, quality, subsampling, restart_interval,
                       optimize_huffman, progressive ? Scans::Refused : Scans::Baseline, false, out, out_cap, out_len);
}

int pixo_b200_jpeg_encode_batch(pixo_b200_ctx *ctx, const uint8_t *pixels, size_t pixels_len_each,
                                uint32_t n_images, uint32_t width, uint32_t height,
                                uint32_t color_type, uint32_t quality, uint32_t subsampling,
                                uint32_t restart_interval, uint32_t optimize_huffman,
                                uint8_t *out, size_t out_cap_each, size_t *out_lens)
{
    return encode_host(ctx, pixels, pixels_len_each, n_images, width, height, color_type, quality, subsampling,
                       restart_interval, optimize_huffman, Scans::Baseline, false, out, out_cap_each, out_lens);
}

int pixo_b200_jpeg_encode_progressive(pixo_b200_ctx *ctx, const uint8_t *pixels, size_t pixels_len,
                                      uint32_t width, uint32_t height, uint32_t color_type, uint32_t quality,
                                      uint32_t subsampling, uint32_t restart_interval, uint32_t optimize_huffman,
                                      uint32_t trellis_quant, uint8_t *out, size_t out_cap, size_t *out_len)
{
    return encode_host(ctx, pixels, pixels_len, 1, width, height, color_type, quality, subsampling, restart_interval,
                       optimize_huffman, Scans::Progressive, trellis_quant, out, out_cap, out_len);
}

int pixo_b200_jpeg_encode_progressive_batch(pixo_b200_ctx *ctx, const uint8_t *pixels, size_t pixels_len_each,
                                            uint32_t n_images, uint32_t width, uint32_t height,
                                            uint32_t color_type, uint32_t quality, uint32_t subsampling,
                                            uint32_t restart_interval, uint32_t optimize_huffman,
                                            uint32_t trellis_quant, uint8_t *out, size_t out_cap_each,
                                            size_t *out_lens)
{
    return encode_host(ctx, pixels, pixels_len_each, n_images, width, height, color_type, quality, subsampling,
                       restart_interval, optimize_huffman, Scans::Progressive, trellis_quant, out, out_cap_each,
                       out_lens);
}

// Caller coefficient arrays on the device: the statistics, Huffman and progressive kernels load each
// block as 16-byte vectors, so an array that is not 16-byte aligned is refused before anything is launched.
static int check_coef_alignment(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb, const int16_t *d_cr,
                                bool has_chroma)
{
    auto mis = [](const int16_t *p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; };
    if (mis(d_y) || (has_chroma && (mis(d_cb) || mis(d_cr))))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "coefficient arrays must be 16-byte aligned");
    return 0;
}

// A pass of the progressive stage: at most the splice grid's 8192 frames, and in encode_dev_progressive no more than
// keep its raw strings (out_cap + 16 bytes per frame) and coefficient arrays each within kProgPass (one at least).
static constexpr size_t kProgPass = (size_t)512 << 20;
static constexpr uint32_t kProgPassFrames = 8192;

int pixo_b200_jpeg_progressive_scans_dev(pixo_b200_ctx *ctx, const int16_t *d_y, size_t y_stride,
                                         const int16_t *d_cb, const int16_t *d_cr, size_t c_stride,
                                         uint32_t n_frames, uint32_t width, uint32_t height, uint32_t color_type,
                                         uint32_t subsampling, const uint8_t *dht, uint8_t *d_out,
                                         size_t out_cap_each, uint64_t *d_scan_len, uint32_t *d_overflow)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_jpeg(ctx, width, height, color_type, subsampling));
    const bool chroma = color_type != PIXO_B200_GRAY;
    if (!d_y || !d_out || !d_scan_len || !d_overflow || (chroma && (!d_cb || !d_cr)))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    PIXO_TRY(check_coef_alignment(ctx, d_y, d_cb, d_cr, chroma));
    if ((y_stride & 7) || (chroma && (c_stride & 7)))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "coefficient strides must be multiples of 8 elements");
    if (n_frames > 1 && (y_stride < g.ny * 64 || (chroma && c_stride < g.nc * 64)))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT,
                         "coefficient strides must hold a frame's blocks (%zu / %zu elements)", g.ny * 64, g.nc * 64);
    ProgTables T;
    PIXO_TRY(dht_prog_tables(ctx, dht ? dht : dht_standard(), &T));
    if (n_frames == 0) return 0;
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    // The pass from frame i0 on.  A call of more than one pass is checked first (dst null: the measuring half alone),
    // so that a rejected coefficient leaves every output untouched.
    const int16_t *cb = chroma ? d_cb : nullptr, *cr = chroma ? d_cr : nullptr;
    auto pass = [&](uint32_t i0, ProgSlots *dst) {
        auto at = [&](const int16_t *a, size_t stride) { return a ? a + (size_t)i0 * stride : nullptr; };
        return launch_progressive(ctx, at(d_y, y_stride), y_stride, at(cb, c_stride), at(cr, c_stride), c_stride,
                                  std::min(kProgPassFrames, n_frames - i0), g, nullptr, &T, false, nullptr, dst);
    };
    if (n_frames > kProgPassFrames)
        for (uint32_t i0 = 0; i0 < n_frames; i0 += kProgPassFrames) PIXO_TRY(pass(i0, nullptr));
    for (uint32_t i0 = 0; i0 < n_frames; i0 += kProgPassFrames) {
        ProgSlots dst{d_out + (size_t)i0 * out_cap_each, out_cap_each, d_scan_len + (size_t)i0 * 7, d_overflow + i0};
        PIXO_TRY(pass(i0, &dst));
    }
    return 0;
}

int pixo_b200_jpeg_encode_dev_opts(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride,
                                   uint32_t n_images, uint32_t width, uint32_t height, uint32_t color_type,
                                   uint32_t quality, uint32_t subsampling, uint32_t restart_interval,
                                   uint32_t optimize_huffman, uint8_t *d_scan, size_t scan_cap_each,
                                   uint64_t *d_scan_len, uint32_t *d_overflow, uint8_t *d_dht)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_options(ctx, quality, restart_interval));
    PIXO_TRY(validate_jpeg(ctx, width, height, color_type, subsampling));
    if (!d_pixels || !d_scan || !d_scan_len || !d_overflow)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if (n_images == 0) return 0;
    if (n_images > 65535) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "at most 65535 frames per call");
    if (scan_cap_each % 4 || (reinterpret_cast<uintptr_t>(d_scan) & 15))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "scan buffer must be 16-byte aligned, capacity multiple of 4");
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    float lum[64], chr[64];
    quant_tables((int)quality, nullptr, nullptr, lum, chr);
    const CoefLayout L(g);
    const bool optimize = optimize_huffman != 0;
    // optimize: every frame's statistics, then its tables in k_huff's form, in d_misc
    uint64_t *d_hist = nullptr;
    void *d_tabs = nullptr;
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    PIXO_TRY(ctx->d_coef.ensure(ctx, (size_t)n_images * L.each));
    PIXO_TRY(ctx->d_ent.ensure(ctx, entropy_scratch_bytes(n_images, g, restart_interval)));
    if (optimize)
        PIXO_TRY(bind(ctx, ctx->d_misc, [&](Layout &M) {
            d_hist = M.take<uint64_t>((size_t)n_images * kHistWords);
            d_tabs = M.take((size_t)n_images * kHuffDevBytes);
        }));
    auto *c = reinterpret_cast<uint8_t *>(ctx->d_coef.ptr);
    PIXO_TRY(transform_records(ctx, d_pixels, pixel_stride, n_images, g, lum, chr, L, c));
    HuffTables t;
    huff_standard(t);
    PIXO_TRY(baseline_tables(ctx, L, c, n_images, g, restart_interval, optimize, d_hist, d_dht, d_tabs));
    return code_records(ctx, L, c, n_images, g, t, d_tabs, restart_interval, reinterpret_cast<uint8_t *>(ctx->d_ent.ptr),
                        d_scan, scan_cap_each, d_scan_len, d_overflow, cudaMemcpyDeviceToDevice);
}

int pixo_b200_jpeg_encode_dev_progressive(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride,
                                          uint32_t n_images, uint32_t width, uint32_t height, uint32_t color_type,
                                          uint32_t quality, uint32_t subsampling, uint32_t restart_interval,
                                          uint32_t optimize_huffman, uint32_t trellis_quant, uint8_t *d_out,
                                          size_t out_cap_each, uint64_t *d_scan_len, uint32_t *d_overflow,
                                          uint8_t *d_dht)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_options(ctx, quality, restart_interval));
    PIXO_TRY(validate_jpeg(ctx, width, height, color_type, subsampling));
    if (!d_pixels || !d_out || !d_scan_len || !d_overflow)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if (n_images == 0) return 0;
    if (n_images > 65535) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "at most 65535 frames per call");
    if ((reinterpret_cast<uintptr_t>(d_scan_len) & 7) || (reinterpret_cast<uintptr_t>(d_overflow) & 3))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "d_scan_len must be 8-byte aligned, d_overflow 4-byte aligned");
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    const bool optimize = optimize_huffman != 0, trellis = trellis_quant != 0;
    float lum[64], chr[64];
    quant_tables((int)quality, nullptr, nullptr, lum, chr);
    const CoefLayout L(g);
    const size_t cs = L.stride();
    const size_t raw_each = Layout::round(out_cap_each + 16);
    const uint32_t pass = (uint32_t)std::min<size_t>(
        std::min<size_t>(n_images, kProgPassFrames), std::max<size_t>(1, std::min(kProgPass / raw_each, kProgPass / L.each)));
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    PIXO_TRY(ctx->d_coef.ensure(ctx, (size_t)pass * L.each));
    // d_misc: a pass's statistics (optimize), its DHT blocks when the caller keeps none
    uint64_t *d_hist = nullptr;
    uint8_t *dht_own = nullptr;
    if (optimize || !d_dht)
        PIXO_TRY(bind(ctx, ctx->d_misc, [&](Layout &M) {
            if (optimize) d_hist = M.take<uint64_t>((size_t)pass * kHistWords);
            if (!d_dht) dht_own = M.take((size_t)pass * kDhtBytes);
        }));
    auto *c = reinterpret_cast<uint8_t *>(ctx->d_coef.ptr);
    int16_t *cb = g.has_chroma ? L.cb(c) : nullptr, *cr = g.has_chroma ? L.cr(c) : nullptr;
    for (uint32_t i0 = 0; i0 < n_images; i0 += pass) {
        const uint32_t cnt = std::min(pass, n_images - i0);
        uint8_t *dht = d_dht ? d_dht + (size_t)i0 * kDhtBytes : dht_own;
        uint32_t *status;
        PIXO_TRY(progressive_coefficients(ctx, d_pixels + (size_t)i0 * pixel_stride, pixel_stride, cnt, g, lum, chr, L, c,
                                          restart_interval, optimize, trellis, d_hist, dht, &status));
        ProgSlots dst{d_out + (size_t)i0 * out_cap_each, out_cap_each, d_scan_len + (size_t)i0 * 7, d_overflow + i0};
        PIXO_TRY(launch_progressive(ctx, L.y(c), cs, cb, cr, cs, cnt, g, dht, nullptr, false, status, &dst));
    }
    return 0;
}

int pixo_b200_jpeg_encode_dev(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride,
                              uint32_t n_images, uint32_t width, uint32_t height,
                              uint32_t color_type, uint32_t quality, uint32_t subsampling,
                              uint8_t *d_scan, size_t scan_cap_each, uint64_t *d_scan_len,
                              uint32_t *d_overflow)
{
    return pixo_b200_jpeg_encode_dev_opts(ctx, d_pixels, pixel_stride, n_images, width, height, color_type, quality,
                                          subsampling, 0, 0, d_scan, scan_cap_each, d_scan_len, d_overflow, nullptr);
}

// Host coefficient arrays: baseline Huffman tables code DC differences of category <= 11 and AC values
// of category <= 10 (what an 8-bit forward DCT can produce); anything else has no code.  seed: the DC
// predictors before block 0 (a band of a tiled frame), or null.
static int check_range(pixo_b200_ctx *ctx, const int16_t *y, const int16_t *cb, const int16_t *cr,
                       const FrameGeometry &g, uint32_t restart_interval, const int32_t *seed)
{
    if (!coefficients_in_range(y, g.ny, restart_interval, g.y_per_mcu, seed ? seed[0] : 0) ||
        (g.has_chroma && (!coefficients_in_range(cb, g.nc, restart_interval, 1, seed ? seed[1] : 0) ||
                          !coefficients_in_range(cr, g.nc, restart_interval, 1, seed ? seed[2] : 0))))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "%s", kOutOfRange);
    return 0;
}

int pixo_b200_jpeg_entropy_encode(pixo_b200_ctx *ctx, const int16_t *y, const int16_t *cb,
                                  const int16_t *cr, uint32_t width, uint32_t height,
                                  uint32_t color_type, uint32_t quality, uint32_t subsampling,
                                  uint32_t restart_interval, uint32_t optimize_huffman,
                                  uint8_t *out, size_t out_cap, size_t *out_len)
{
    PIXO_TRY(validate_options(ctx, quality, restart_interval));
    PIXO_TRY(validate_jpeg(ctx, width, height, color_type, subsampling));
    if (!y || !out || !out_len || (color_type != PIXO_B200_GRAY && (!cb || !cr)))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    PIXO_TRY(check_range(ctx, y, cb, cr, g, restart_interval, nullptr));
    if (out_cap < 1024 + 2)
        return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu too small", out_cap);
    uint64_t hist[536];
    if (optimize_huffman) host_histogram(y, cb, cr, g, restart_interval, hist);
    HuffTables t;
    tables_from(optimize_huffman ? hist : nullptr, g.has_chroma, t);
    uint8_t lum_zz[64], chr_zz[64];
    quant_tables((int)quality, lum_zz, chr_zz, nullptr, nullptr);
    const size_t hdr = write_headers(out, g, lum_zz, chr_zz, t, restart_interval);
    int threads = ctx ? ctx->host_threads : (int)std::thread::hardware_concurrency();
    const size_t body = entropy_encode_scan(y, cb, cr, g, t, restart_interval, false, out + hdr, out_cap - hdr - 2,
                                            threads < 1 ? 1 : threads);
    return finish_frame(ctx, out, out_cap, hdr, body, out_len);
}

int pixo_b200_jpeg_entropy_encode_dev(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                      const int16_t *d_cr, uint32_t width, uint32_t height,
                                      uint32_t color_type, uint32_t quality, uint32_t subsampling,
                                      uint32_t restart_interval, uint32_t optimize_huffman,
                                      uint8_t *out, size_t out_cap, size_t *out_len)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_options(ctx, quality, restart_interval));
    PIXO_TRY(validate_jpeg(ctx, width, height, color_type, subsampling));
    if (!d_y || !out || !out_len || (color_type != PIXO_B200_GRAY && (!d_cb || !d_cr)))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if (out_cap < 1024 + 2)
        return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu too small", out_cap);
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    PIXO_TRY(check_coef_alignment(ctx, d_y, d_cb, d_cr, g.has_chroma));
    uint8_t lum_zz[64], chr_zz[64];
    quant_tables((int)quality, lum_zz, chr_zz, nullptr, nullptr);
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint8_t *dht = dht_standard();
    if (optimize_huffman) {   // K3, k_huff_tables, the DHT block back to the host
        uint64_t *d_hist;
        uint8_t *d_dht;
        PIXO_TRY(bind(ctx, ctx->d_misc, [&](Layout &M) { d_hist = M.take<uint64_t>(kHistWords), d_dht = M.take(kDhtBytes); }));
        PIXO_TRY(ctx->h_misc.ensure(ctx, kDhtBytes));
        PIXO_TRY(launch_jpeg_histogram(ctx, d_y, 0, d_cb, d_cr, 0, 1, g.ny, g.nc, g.y_per_mcu, restart_interval,
                                       false, nullptr, d_hist));
        PIXO_TRY(launch_huff_tables(ctx, d_hist, 1, g.has_chroma, d_dht, nullptr));
        PIXO_CUDA(ctx, cudaMemcpyAsync(ctx->h_misc.ptr, d_dht, kDhtBytes, cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        dht = static_cast<const uint8_t *>(ctx->h_misc.ptr);
    }
    HuffTables t;
    huff_from_dht(dht, t);
    const size_t hdr = write_headers(out, g, lum_zz, chr_zz, t, restart_interval);
    // The device scan buffer follows the size a JPEG of this geometry normally has, not the caller's
    // worst-case capacity (tens of GB for a gigapixel frame); a scan that needs more is coded again
    // with the exact size the kernel reported.
    const size_t raw = (size_t)width * height * (color_type == PIXO_B200_GRAY ? 1 : 3);
    const size_t scan_cap = std::min<size_t>((out_cap - hdr - 2) & ~(size_t)15, (size_t)default_scan_cap(ctx, raw));
    size_t body = 0;
    const int rc = recode_scan(ctx, d_y, d_cb, d_cr, nullptr, g, t, restart_interval, true, scan_cap, hdr, out_cap, &body);
    if (rc == kGaveUp) return set_error(ctx, PIXO_B200_ERR_CUDA, "device entropy stage did not finish");
    PIXO_TRY(rc);
    PIXO_TRY(finish_frame(ctx, out, out_cap, hdr, body, out_len));
    PIXO_CUDA(ctx, cudaMemcpyAsync(out + hdr, ctx->d_retry.ptr, body, cudaMemcpyDeviceToHost, ctx->stream));
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

// ---- one frame tiled over several GPUs -----------------------------------------------------------

int pixo_b200_jpeg_band_last_dc(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                const int16_t *d_cr, size_t ny, size_t nc, int32_t last_dc[3])
{
    if (!ctx || !last_dc) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    int16_t v[3] = {0, 0, 0};
    if (ny && d_y) PIXO_CUDA(ctx, cudaMemcpyAsync(&v[0], d_y + (ny - 1) * 64, 2, cudaMemcpyDeviceToHost, ctx->stream));
    if (nc && d_cb) PIXO_CUDA(ctx, cudaMemcpyAsync(&v[1], d_cb + (nc - 1) * 64, 2, cudaMemcpyDeviceToHost, ctx->stream));
    if (nc && d_cr) PIXO_CUDA(ctx, cudaMemcpyAsync(&v[2], d_cr + (nc - 1) * 64, 2, cudaMemcpyDeviceToHost, ctx->stream));
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < 3; ++k) last_dc[k] = v[k];
    return 0;
}

int pixo_b200_jpeg_band_histogram_dev(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                      const int16_t *d_cr, uint32_t width, uint32_t band_height,
                                      uint32_t color_type, uint32_t subsampling,
                                      const int32_t dc_seed[3], uint64_t *d_hist)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_jpeg(ctx, width, band_height, color_type, subsampling));
    if (!d_y || !d_hist || (color_type != PIXO_B200_GRAY && (!d_cb || !d_cr)))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    const FrameGeometry g = make_geometry(width, band_height, color_type, subsampling);
    PIXO_TRY(check_coef_alignment(ctx, d_y, d_cb, d_cr, g.has_chroma));
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return launch_jpeg_histogram(ctx, d_y, 0, d_cb, d_cr, 0, 1, g.ny, g.nc, g.y_per_mcu, 0, false, nullptr, d_hist,
                                 dc_seed);
}

int pixo_b200_jpeg_band_entropy_dev(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                    const int16_t *d_cr, uint32_t width, uint32_t band_height,
                                    uint32_t color_type, uint32_t subsampling,
                                    const int32_t dc_seed[3], const uint64_t *hist, uint8_t *d_raw,
                                    size_t raw_cap, uint64_t *nbits, uint32_t *tail7)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_jpeg(ctx, width, band_height, color_type, subsampling));
    if (!d_y || !d_raw || !nbits || !tail7 || (color_type != PIXO_B200_GRAY && (!d_cb || !d_cr)))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if ((raw_cap & 3) || (reinterpret_cast<uintptr_t>(d_raw) & 15))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "raw buffer must be 16-byte aligned, capacity multiple of 4");
    const FrameGeometry g = make_geometry(width, band_height, color_type, subsampling);
    PIXO_TRY(check_coef_alignment(ctx, d_y, d_cb, d_cr, g.has_chroma));
    HuffTables t;
    tables_from(hist, g.has_chroma, t);
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    // the stream-ordered flow into a small device scratch, read back
    struct Totals {
        uint64_t bits_tail[2];   // the band's bit count, its last 7 bits
        uint32_t flags;          // k_band_totals ORs into these
    };
    PIXO_TRY(ctx->d_misc.ensure(ctx, sizeof(Totals)));
    PIXO_TRY(ctx->h_misc.ensure(ctx, sizeof(Totals)));
    auto *d = static_cast<Totals *>(ctx->d_misc.ptr);
    auto *h = static_cast<Totals *>(ctx->h_misc.ptr);
    // a segment that outgrew its share (bit 0 of a segmented pass): the band again, as one string
    for (bool segments = true;; segments = false) {
        PIXO_CUDA(ctx, cudaMemsetAsync(&d->flags, 0, sizeof d->flags, ctx->stream));
        PIXO_TRY(launch_band_entropy(ctx, d_y, d_cb, d_cr, g, t, dc_seed, nullptr, segments, d_raw, raw_cap,
                                     d->bits_tail, &d->flags));
        PIXO_CUDA(ctx, cudaMemcpyAsync(h, d, sizeof(Totals), cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (!(segments && h->flags == kOvfNoFit && ctx->bands[d_raw].S > 1)) break;
    }
    const uint32_t ovf = h->flags;
    *nbits = h->bits_tail[0];
    *tail7 = (uint32_t)h->bits_tail[1];
    if (ovf & kOvfRange) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "%s", kOutOfRange);
    if (ovf & kOvfFault) return set_error(ctx, PIXO_B200_ERR_CUDA, "device entropy stage did not finish (flags %u)", ovf);
    if (ovf) return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "raw capacity %zu too small (need %llu)", raw_cap,
                              (unsigned long long)((h->bits_tail[0] + 7) / 8));
    return 0;
}

int pixo_b200_jpeg_band_splice_dev(pixo_b200_ctx *ctx, const uint8_t *d_raw, uint64_t nbits,
                                   uint64_t start_bit, uint32_t tail_in, uint32_t is_last_band,
                                   uint8_t *d_out, size_t out_cap, uint64_t *out_len)
{
    if (!ctx || !d_out || !out_len || (!d_raw && nbits))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (nbits == 0) {   // an empty band owns no byte of the stream
        *out_len = 0;
        return 0;
    }
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    // the stream-ordered flow into a small device scratch, read back
    struct Spliced {
        uint64_t len;
        uint32_t flags;   // OR-ed into
    };
    PIXO_TRY(ctx->d_misc.ensure(ctx, sizeof(Spliced)));
    PIXO_TRY(ctx->h_misc.ensure(ctx, sizeof(Spliced)));
    auto *d = static_cast<Spliced *>(ctx->d_misc.ptr);
    auto *h = static_cast<Spliced *>(ctx->h_misc.ptr);
    PIXO_CUDA(ctx, cudaMemsetAsync(d, 0, sizeof(Spliced), ctx->stream));
    PIXO_TRY(launch_band_splice(ctx, d_raw, start_bit, tail_in, is_last_band != 0, nullptr, d_out, out_cap, &d->len,
                                &d->flags));
    PIXO_CUDA(ctx, cudaMemcpyAsync(h, d, sizeof(Spliced), cudaMemcpyDeviceToHost, ctx->stream));
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h->flags) return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "splice output capacity %zu too small", out_cap);
    *out_len = h->len;
    return 0;
}

int pixo_b200_jpeg_band_entropy_dev_async(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                          const int16_t *d_cr, uint32_t width, uint32_t band_height,
                                          uint32_t color_type, uint32_t subsampling,
                                          const int32_t *d_dc_seed, const uint64_t *hist, uint8_t *d_raw,
                                          size_t raw_cap, uint64_t *d_bits_tail, uint32_t *d_flags)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_TRY(validate_jpeg(ctx, width, band_height, color_type, subsampling));
    if (!d_y || !d_raw || !d_dc_seed || !d_bits_tail || !d_flags || (color_type != PIXO_B200_GRAY && (!d_cb || !d_cr)))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if ((raw_cap & 3) || (reinterpret_cast<uintptr_t>(d_raw) & 15))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "raw buffer must be 16-byte aligned, capacity multiple of 4");
    const FrameGeometry g = make_geometry(width, band_height, color_type, subsampling);
    PIXO_TRY(check_coef_alignment(ctx, d_y, d_cb, d_cr, g.has_chroma));
    HuffTables t;
    tables_from(hist, g.has_chroma, t);
    if (raw_cap < band_raw_bytes(g))
        return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "raw capacity %zu too small (need %zu)", raw_cap,
                         band_raw_bytes(g));
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return launch_band_entropy(ctx, d_y, d_cb, d_cr, g, t, nullptr, d_dc_seed, true, d_raw, raw_cap, d_bits_tail,
                               d_flags);
}

int pixo_b200_jpeg_band_splice_dev_async(pixo_b200_ctx *ctx, const uint8_t *d_raw, const uint64_t *d_offset,
                                         uint8_t *d_out, size_t out_cap, uint64_t *d_out_len,
                                         uint32_t *d_flags)
{
    if (!ctx || !d_raw || !d_offset || !d_out || !d_out_len || !d_flags)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return launch_band_splice(ctx, d_raw, 0, 0, false, d_offset, d_out, out_cap, d_out_len, d_flags);
}

// The progressive scans of one band (pixo_b200_jpeg_band_dev_progressive*): a band's arrays, 16-byte aligned where it
// has blocks, inside the frame's
static int check_prog_band(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb, const int16_t *d_cr, size_t ny,
                           size_t nc, uint64_t y_base, uint64_t c_base)
{
    if ((ny && !d_y) || (nc && (!d_cb || !d_cr))) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    PIXO_TRY(check_coef_alignment(ctx, ny ? d_y : nullptr, d_cb, d_cr, nc > 0));
    // enc_of ((index + 1) << 1 | init) must fit 32 bits
    if (y_base + ny >= 0x7FFFFFFFull || c_base + nc >= 0x7FFFFFFFull || y_base > 0x7FFFFFFFull || c_base > 0x7FFFFFFFull)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "progressive band: too many blocks per component");
    return 0;
}

int pixo_b200_jpeg_band_dev_progressive_summary(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                                const int16_t *d_cr, size_t ny, size_t nc, uint64_t y_base,
                                                uint64_t c_base, int32_t last_dc[3], uint32_t last_enc[4])
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    if (!last_dc || !last_enc) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_TRY(check_prog_band(ctx, d_y, d_cb, d_cr, ny, nc, y_base, c_base));
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    ProgBandSummary sum;
    PIXO_TRY(launch_progressive_band_summary(ctx, d_y, d_cb, d_cr, ny, nc, y_base, c_base, &sum));
    for (int k = 0; k < 3; ++k) last_dc[k] = sum.last_dc[k];
    for (int k = 0; k < 4; ++k) last_enc[k] = sum.last_enc[k];
    return 0;
}

int pixo_b200_jpeg_band_dev_progressive(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                        const int16_t *d_cr, size_t ny, size_t nc, uint64_t y_base, uint64_t c_base,
                                        uint64_t frame_ny, uint64_t frame_nc, const int32_t dc_seed[3],
                                        const uint32_t ac_carry[4], const uint64_t *d_hist, uint8_t *d_dht,
                                        uint8_t *d_raw, size_t raw_cap, size_t *raw_need, uint64_t nbits[7],
                                        uint32_t tail7[7])
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    if (!dc_seed || !ac_carry || !raw_need || !nbits || !tail7)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_TRY(check_prog_band(ctx, d_y, d_cb, d_cr, ny, nc, y_base, c_base));
    if (y_base + ny > frame_ny || c_base + nc > frame_nc)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "progressive band: blocks outside the frame");
    if ((ny || nc) && !d_raw) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if ((reinterpret_cast<uintptr_t>(d_raw) & 15) || (reinterpret_cast<uintptr_t>(d_hist) & 7))
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "d_raw must be 16-byte aligned, d_hist 8-byte aligned");
    ProgBand B;
    B.ny = ny; B.nc = nc; B.y_base = y_base; B.c_base = c_base; B.frame_ny = frame_ny; B.frame_nc = frame_nc;
    for (int k = 0; k < 3; ++k) {
        if (dc_seed[k] < -16383 || dc_seed[k] > 16383)
            return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "DC seed %d out of the progressive range", dc_seed[k]);
        B.dc_seed[k] = dc_seed[k];
    }
    for (int k = 0; k < 4; ++k) {   // a carry names a block before the band: (index + 1) <= the band's first index
        if ((ac_carry[k] >> 1) > (k < 2 ? y_base : c_base))
            return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "AC carry %u lies past the band's first block", ac_carry[k]);
        B.ac_carry[k] = ac_carry[k];
    }
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    return launch_progressive_band(ctx, d_y, d_cb, d_cr, B, d_hist, d_dht, d_raw, raw_cap, raw_need, nbits, tail7);
}

int pixo_b200_jpeg_band_dev_progressive_splice(pixo_b200_ctx *ctx, const uint8_t *d_raw, uint32_t scan, uint64_t nbits,
                                               uint64_t start_bit, uint32_t tail_in, uint32_t is_last_band,
                                               uint8_t *d_out, size_t out_cap, uint64_t *out_len)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    if (scan >= 7) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "scan %u: a progressive frame has 7", scan);
    if (nbits == 0) {   // the band owns no byte of this scan; it still returns with the stream drained, as the
                        // other band calls do
        if (!d_out || !out_len) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
        PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
        PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *out_len = 0;
        return 0;
    }
    const auto it = ctx->prog_bands.find(d_raw);
    if (it == ctx->prog_bands.end())
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "this raw buffer was not coded by pixo_b200_jpeg_band_dev_progressive");
    return pixo_b200_jpeg_band_splice_dev(ctx, d_raw + (size_t)scan * it->second, nbits, start_bit, tail_in, is_last_band,
                                          d_out, out_cap, out_len);
}

int pixo_b200_jpeg_band_entropy(const int16_t *y, const int16_t *cb, const int16_t *cr, uint32_t width,
                                uint32_t band_height, uint32_t color_type, uint32_t subsampling,
                                const int32_t dc_seed[3], const uint64_t *hist, uint8_t *raw,
                                size_t raw_cap, uint64_t *nbits, uint32_t *tail7)
{
    PIXO_TRY(validate_jpeg(nullptr, width, band_height, color_type, subsampling));
    if (!y || !raw || !nbits || !tail7 || (color_type != PIXO_B200_GRAY && (!cb || !cr)))
        return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    const FrameGeometry g = make_geometry(width, band_height, color_type, subsampling);
    PIXO_TRY(check_range(nullptr, y, cb, cr, g, 0, dc_seed));
    HuffTables t;
    tables_from(hist, g.has_chroma, t);
    const uint64_t n = band_encode_raw(y, cb, cr, g, t, dc_seed, raw, raw_cap, tail7);
    if (n == (uint64_t)-1) return set_error(nullptr, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "raw capacity %zu too small", raw_cap);
    *nbits = n;
    return 0;
}

int pixo_b200_jpeg_band_histogram(const int16_t *y, const int16_t *cb, const int16_t *cr, uint32_t width,
                                  uint32_t band_height, uint32_t color_type, uint32_t subsampling,
                                  const int32_t dc_seed[3], uint64_t hist[536])
{
    PIXO_TRY(validate_jpeg(nullptr, width, band_height, color_type, subsampling));
    if (!y || !hist || (color_type != PIXO_B200_GRAY && (!cb || !cr)))
        return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    const FrameGeometry g = make_geometry(width, band_height, color_type, subsampling);
    PIXO_TRY(check_range(nullptr, y, cb, cr, g, 0, dc_seed));
    host_histogram(y, cb, cr, g, 0, hist, dc_seed);
    return 0;
}

int pixo_b200_jpeg_band_splice(const uint8_t *raw, uint64_t nbits, uint64_t start_bit, uint32_t tail_in,
                               uint32_t is_last_band, uint8_t *out, size_t out_cap, size_t *out_len)
{
    if (!out || !out_len || (!raw && nbits)) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    const size_t n = band_splice(raw, nbits, (uint32_t)(start_bit & 7), tail_in, is_last_band != 0, out, out_cap);
    if (n == (size_t)-1) return set_error(nullptr, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "splice output capacity %zu too small", out_cap);
    *out_len = n;
    return 0;
}

int pixo_b200_jpeg_write_headers(uint32_t width, uint32_t height, uint32_t color_type, uint32_t quality,
                                 uint32_t subsampling, uint32_t restart_interval, const uint64_t *hist,
                                 uint8_t *out, size_t out_cap, size_t *out_len)
{
    PIXO_TRY(validate_options(nullptr, quality, restart_interval));
    PIXO_TRY(validate_jpeg(nullptr, width, height, color_type, subsampling));
    if (!out || !out_len) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if (out_cap < 1024) return set_error(nullptr, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu too small", out_cap);
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    uint8_t lum_zz[64], chr_zz[64];
    quant_tables((int)quality, lum_zz, chr_zz, nullptr, nullptr);
    HuffTables t;
    tables_from(hist, g.has_chroma, t);
    *out_len = write_headers(out, g, lum_zz, chr_zz, t, restart_interval);
    return 0;
}

int pixo_b200_jpeg_write_headers_dht(uint32_t width, uint32_t height, uint32_t color_type, uint32_t quality,
                                     uint32_t subsampling, uint32_t restart_interval, const uint8_t *dht,
                                     uint8_t *out, size_t out_cap, size_t *out_len)
{
    PIXO_TRY(validate_options(nullptr, quality, restart_interval));
    PIXO_TRY(validate_jpeg(nullptr, width, height, color_type, subsampling));
    if (!dht || !out || !out_len) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    ProgTables check;
    PIXO_TRY(dht_prog_tables(nullptr, dht, &check));
    if (out_cap < 1024) return set_error(nullptr, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu too small", out_cap);
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    uint8_t lum_zz[64], chr_zz[64];
    quant_tables((int)quality, lum_zz, chr_zz, nullptr, nullptr);
    HuffTables t;
    huff_from_dht(dht, t);
    uint8_t hdr[2048];   // 281 bytes + the tables' values (at most 4 x 256)
    const size_t n = write_headers(hdr, g, lum_zz, chr_zz, t, restart_interval);
    if (n > out_cap)
        return set_error(nullptr, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu too small (need %zu)", out_cap, n);
    memcpy(out, hdr, n);
    *out_len = n;
    return 0;
}

int pixo_b200_jpeg_progressive_file(uint32_t width, uint32_t height, uint32_t color_type, uint32_t quality,
                                    uint32_t subsampling, uint32_t restart_interval, const uint8_t *dht,
                                    const uint8_t *segments, const uint64_t scan_len[7], uint8_t *out, size_t out_cap,
                                    size_t *out_len)
{
    PIXO_TRY(validate_options(nullptr, quality, restart_interval));
    PIXO_TRY(validate_jpeg(nullptr, width, height, color_type, subsampling));
    if (!scan_len || !out || !out_len) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    if (!dht) dht = dht_standard();
    ProgTables check;
    PIXO_TRY(dht_prog_tables(nullptr, dht, &check));
    uint64_t body = 0;
    for (int s = 0; s < 7; ++s) {
        if (scan_len[s] > out_cap)
            return set_error(nullptr, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu too small", out_cap);
        body += scan_len[s];
    }
    if (body && !segments) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "null buffer");
    const FrameGeometry g = make_geometry(width, height, color_type, subsampling);
    uint8_t lum_zz[64], chr_zz[64];
    quant_tables((int)quality, lum_zz, chr_zz, nullptr, nullptr);
    size_t at[7];
    PIXO_TRY(progressive_layout(nullptr, g, lum_zz, chr_zz, dht, restart_interval, scan_len, out, out_cap, at, out_len));
    for (int s = 0; s < 7; ++s) {
        if (scan_len[s]) memcpy(out + at[s], segments, (size_t)scan_len[s]);
        segments += scan_len[s];
    }
    return 0;
}

}  // extern "C"
