// common.cuh — context object, error plumbing and small device helpers shared by the kernels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/pixo_b200.h"

namespace pixo {

constexpr int kHistWords = 536;  // dc_lum[12] dc_chrom[12] ac_lum[256] ac_chrom[256]
// A frame's four Huffman tables (dc_lum, dc_chrom, ac_lum, ac_chrom) as DHT data, 16 counts + 256 values each,
// and in the form k_huff reads them (HuffDev, jpeg_entropy.cu)
constexpr size_t kDhtBytes = 4 * 272;
constexpr size_t kHuffDevBytes = 1632;

// natural index of zig-zag position i (src/jpeg/quantize.rs:18-22); with a compile-time i the
// kernels' reorders are static register renaming
__host__ __device__ constexpr int zz_nat(int i)
{
    constexpr int t[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                           12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                           35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                           58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
    return t[i];
}

// Coefficient records, the format the transform hands the encode paths' K3 and k_huff: a block's 64
// coefficients in zig-zag order in its 128-byte slot, of which only the 32-byte sectors up to the one
// holding the last non-zero coefficient are written (sector 0, with the DC that the next block predicts
// from, always), plus one byte per block in an extent array: the number of sectors written, 1..4.
// Bytes past the last written sector are undefined; a reader loads the record's 2 * sectors 16-byte
// pieces and takes the rest as zeros.  Extent arrays of the Y, Cb and Cr coefficient arrays, `stride`
// bytes between images:
struct CoefExtents {
    uint8_t *y, *cb, *cr;
    size_t stride;
};

// Bits of the entropy stage's per-frame (or per-band) overflow word; their values are public
// (include/pixo_b200.h)
constexpr uint32_t kOvfNoFit = 1u;     // the scan did not fit its capacity; its length is the size it needs
constexpr uint32_t kOvfFault = 2u;     // a look-back chain timed out
constexpr uint32_t kOvfSegment = 4u;   // a segment's raw string outgrew its share
constexpr uint32_t kOvfRange = 8u;     // a coefficient outside the baseline range
constexpr uint32_t kOvfInput = 16u;    // input the trellis or the progressive stage cannot carry

// Reusable scratch of a context: device memory (Buffer<false>, DevBuf) or page-locked host memory
// (Buffer<true>, PinnedBuf), two types so that one cannot be passed where the other is meant.  Freed
// with the context.
template <bool Pinned>
struct Buffer {
    void *ptr = nullptr;
    size_t cap = 0;
    Buffer() = default;
    Buffer(const Buffer &) = delete;
    Buffer &operator=(const Buffer &) = delete;
    ~Buffer()
    {
        if (ptr) Pinned ? cudaFreeHost(ptr) : cudaFree(ptr);
    }
    // at least `bytes`: a smaller buffer is freed, once the context's stream has drained, and
    // allocated again with room to grow
    int ensure(pixo_b200_ctx *ctx, size_t bytes);
    // slot i of a buffer used as an array of equal slots, `stride` bytes each
    uint8_t *slot(size_t i, size_t stride) const { return static_cast<uint8_t *>(ptr) + i * stride; }
};
using DevBuf = Buffer<false>;
using PinnedBuf = Buffer<true>;

// A few persistent host threads per context for the one host-side job that is worth spreading:
// copying a caller's ordinary (pageable) memory into / out of the pinned staging ring while the DMA
// engine drains it.  Created on first use; the threads sleep on a condition variable between calls.
class HostPool {
public:
    explicit HostPool(int nthreads);
    ~HostPool();
    // fn(job) for job in [0, njobs), on the pool's threads and the caller; returns when all are done
    void run(int njobs, const std::function<void(int)> &fn);

private:
    void worker();
    std::vector<std::thread> threads_;
    std::mutex m_;
    std::condition_variable cv_work_, cv_done_;
    const std::function<void(int)> *fn_ = nullptr;
    std::atomic<int> next_{0};
    int njobs_ = 0, active_ = 0;
    uint64_t generation_ = 0;
    bool stop_ = false;
};

// The layout of a scratch buffer: regions appended in order, each taking whole 256-byte units, so that
// every region starts 256-byte aligned.  A stage describes its regions once and runs that description
// twice: without a base, to count the bytes to ensure, and on the buffer, to bind its pointers (see bind).
// Small host read-back areas pack their regions in 8-byte units instead (`unit`).
class Layout {
public:
    explicit Layout(void *base = nullptr, size_t unit = 256) : base_(static_cast<uint8_t *>(base)), unit_(unit) {}
    // the next region, room for `count` T; null while counting
    template <class T = uint8_t>
    T *take(size_t count)
    {
        T *p = base_ ? reinterpret_cast<T *>(base_ + size_) : nullptr;
        end_ = size_ + count * sizeof(T);
        size_ = (end_ + unit_ - 1) / unit_ * unit_;
        return p;
    }
    size_t size() const { return size_; }   // bytes taken so far, the last region's too
    size_t end() const { return end_; }     // where the last region's own bytes end: what a buffer must hold
    // the bytes a region of `bytes` takes, and the most whole units `bytes` holds
    static size_t round(size_t bytes) { return (bytes + 255) / 256 * 256; }
    static size_t floor(size_t bytes) { return bytes / 256 * 256; }

private:
    uint8_t *base_;
    size_t unit_;
    size_t size_ = 0, end_ = 0;
};

// Images cut into S segments, each coded as a raw bit string of its own and spliced afterwards
// (see jpeg_entropy.cu, k_seg_*).  Sizes only: the scratch and the raw area are bound where they are used.
struct SegPlan {
    uint32_t n, S;
    uint64_t seg_mcus, last_mcus, bpm;
    size_t raw_cap;                 // bytes per segment
    uint32_t max_tiles;             // per image
};

// Huffman tables of the progressive scans as get_code_from_table sees them: (code << 8) | length per
// symbol, pixo's fallback (0, 4) for a symbol the table does not hold.  DC categories 0..15.
struct ProgTables {
    uint32_t dc[2][16];
    uint32_t ac[2][256];
};

// Where the progressive scans of n frames go: frame i's 7 stuffed segments back to back at out + i * cap, their
// lengths at scan_len + i * 7, its flags at overflow[i] (device memory)
struct ProgSlots {
    uint8_t *out = nullptr;
    uint64_t cap = 0;
    uint64_t *scan_len = nullptr;
    uint32_t *overflow = nullptr;
};

// One band of a frame's MCU rows for the progressive scans (pixo_b200_jpeg_band_dev_progressive): its blocks of
// each component, the frame index of its first, the frame's blocks (frame_nc 0: gray), and what the frame's earlier
// bands leave - the DC predictors and, per AC scan (Y 1-10, Y 11-63, Cb, Cr), the carry of the EOB run
struct ProgBand {
    uint64_t ny, nc, y_base, c_base, frame_ny, frame_nc;
    int dc_seed[3];
    uint32_t ac_carry[4];
};

// What a band leaves the later ones: its last DC per component, its largest enc_of per AC scan, and status bit 0
// for a coefficient outside -16383..16383
struct ProgBandSummary {
    uint32_t last_enc[4];
    int32_t last_dc[3];
    uint32_t status;
};

// What a context has set on one kernel.  Function attributes belong to the device, and every context
// sets the same values, so contexts sharing a device never undo each other's settings.
struct KernelAttrs {
    size_t smem_limit = 0;      // cudaFuncAttributeMaxDynamicSharedMemorySize as set
    int blocks_per_sm = 0;      // occupancy query of the transform's persistent kernels, 0: not asked
    bool carveout_set = false;  // cudaFuncAttributePreferredSharedMemoryCarveout
};

}  // namespace pixo

struct pixo_b200_ctx {
    int device = 0;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;  // H2D of the next group of frames
    cudaStream_t d2h_stream = nullptr;   // D2H of finished scan bytes
    int sm_count = 0;
    int host_threads = 0;
    uint64_t launches = 0;
    uint64_t host_fallbacks = 0;   // frames finished by the host entropy coder (see encode_baseline_groups)
    size_t scan_cap_override = 0;  // device scan bytes per frame; 0 = the built-in heuristic
    bool gpu_retry = true;         // re-run k_huff with the exact size when the heuristic was too small
    std::string err;
    // reusable scratch
    pixo::DevBuf d_in, d_misc, d_out, d_ent, d_coef, d_retry, d_raw;
    pixo::DevBuf d_hwin;                        // k_huff: every warp's assembled unit, from its phase A to its phase B
    pixo::DevBuf d_red, d_red_idx, d_red_img;   // PNG reduction: statistics, palette indices, reduced rows
    pixo::DevBuf d_quant, d_quant_img;          // PNG quantisation: sample sort, then palettes / tables / indices
    pixo::DevBuf d_trellis;                     // JPEG trellis: status word + f32 DCT blocks
    pixo::DevBuf d_prog, d_prog_raw, d_prog_out;   // JPEG progressive scans: per-block state, raw strings,
                                                   // the splice's scratch (and the host loop's frame slots)
    pixo::DevBuf d_resize, d_resize_tmp;   // resize: Lanczos3 weight tables; the u8 intermediate (bounded)
    pixo::DevBuf d_jdec;                   // JPEG decode: a pass's records, tables and scans, coefficients, planes
    pixo::DevBuf d_pdec;                   // PNG decode: a pass's records, chunks and streams, rings, inflated rows
    pixo::DevBuf d_lz, d_zemit;            // DEFLATE: a pass's streams, tokens and hash state; its coded streams
    pixo::DevBuf d_png_filt, d_png_z;      // PNG encode: a pass's filtered streams; their zlib streams
    pixo::DevBuf d_png_box;                // PNG encode: a pass's container upload (files, CRC words, small chunks)
    pixo::PinnedBuf h_in, h_out, h_misc, h_red, h_quant;
    pixo::PinnedBuf h_trellis, h_prog;     // the trellis status; the progressive scans' bit counts / lengths
    pixo::PinnedBuf h_resize[2];           // Lanczos3 weight tables on their way to d_resize, in turn
    // host encode, per input slot: pixels uploaded, read by the transform, scan bytes copied back, lengths on host
    cudaEvent_t ev_in[2] = {}, ev_used[2] = {}, ev_out[2] = {}, ev_len[2] = {};
    std::vector<cudaEvent_t> stage_events;  // one per pinned staging slot of h2d_copy
    cudaEvent_t switch_event = nullptr;     // pixo_b200_ctx_set_stream: the new stream waits for the old one
    cudaEvent_t resize_events[2] = {};      // the last copy out of h_resize[i] has run
    uint64_t resize_uploads = 0;            // Lanczos3 table uploads so far (h_resize[resize_uploads % 2] is next)
    std::unique_ptr<pixo::HostPool> pool;   // see HostPool
    // How the bands coded by pixo_b200_jpeg_band_entropy_dev(_async) were cut into segments, keyed by
    // the caller's raw buffer (which holds the segments' strings, bit counts and tails until the splice).
    std::unordered_map<const void *, pixo::SegPlan> bands;
    // The bands coded by pixo_b200_jpeg_band_dev_progressive: bytes between their scans' splice areas (each one of
    // `bands`), keyed by the caller's raw buffer
    std::unordered_map<const void *, size_t> prog_bands;
    std::unordered_map<const void *, pixo::KernelAttrs> kernels;   // keyed by the kernel's host function

    pixo_b200_ctx() = default;
    ~pixo_b200_ctx();   // destroys the streams and events; the scratch frees itself
};

namespace pixo {

int set_error(pixo_b200_ctx *ctx, int code, const char *fmt, ...);
int cuda_fail(pixo_b200_ctx *ctx, cudaError_t e, const char *what);

#define PIXO_CUDA(ctx, call)                                            \
    do {                                                                \
        cudaError_t e__ = (call);                                       \
        if (e__ != cudaSuccess) return ::pixo::cuda_fail(ctx, e__, #call); \
    } while (0)

#define PIXO_TRY(expr)                 \
    do {                               \
        int rc__ = (expr);             \
        if (rc__ != 0) return rc__;    \
    } while (0)

// Ensure `buf` holds the regions `describe(Layout &)` takes, then bind them: describe runs twice, without a
// base to count them and on the buffer to set the pointers it assigns.
template <bool Pinned, class F>
int bind(pixo_b200_ctx *ctx, Buffer<Pinned> &buf, F &&describe, size_t unit = 256)
{
    Layout count(nullptr, unit);
    describe(count);
    PIXO_TRY(buf.ensure(ctx, count.end()));
    Layout L(buf.ptr, unit);
    describe(L);
    return 0;
}

// Dynamic shared memory of a launch: `bytes`, and `limit`, what the kernel's maximum is raised to.  A
// kernel launched with varying sizes passes one fixed limit, so that no context lowers it under another.
struct Smem {
    size_t bytes, limit;
    Smem(size_t b) : bytes(b), limit(b) {}
    Smem(size_t b, size_t l) : bytes(b), limit(l) {}
};

// Raise `kernel`'s dynamic shared memory maximum to `limit` unless this context already has
inline int allow_smem(pixo_b200_ctx *ctx, const void *kernel, size_t limit)
{
    size_t &set = ctx->kernels[kernel].smem_limit;
    if (set >= limit) return 0;
    PIXO_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit));
    set = limit;
    return 0;
}

// Every kernel of the library is launched here: on the context's stream, counted (the count is
// pixo_b200_ctx_launch_count) and checked.
template <class... P, class... A>
int launch(pixo_b200_ctx *ctx, void (*kernel)(P...), dim3 grid, dim3 block, Smem smem, A &&...args)
{
    if (smem.bytes) PIXO_TRY(allow_smem(ctx, reinterpret_cast<const void *>(kernel), smem.limit));
    kernel<<<grid, block, smem.bytes, ctx->stream>>>(std::forward<A>(args)...);
    ctx->launches++;
    PIXO_CUDA(ctx, cudaGetLastError());
    return 0;
}

// ---- launchers implemented in the .cu files ----
// ext: write coefficient records and their extents (flags is then ignored)
int launch_jpeg_transform(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride,
                          uint32_t n_images, uint32_t w, uint32_t h, uint32_t color_type,
                          uint32_t subsampling, const float *lum_q, const float *chr_q,
                          int16_t *d_y, size_t y_stride, int16_t *d_cb, int16_t *d_cr,
                          size_t c_stride, uint32_t flags, const CoefExtents *ext = nullptr);
// the same transform writing each block's unquantised f32 DCT (natural order, 64 floats; 4:2:0 chroma:
// the DCT of the averaged block), strides in floats: the input of launch_trellis
int launch_jpeg_transform_dct(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride, uint32_t n_images,
                              uint32_t w, uint32_t h, uint32_t color_type, uint32_t subsampling,
                              const float *lum_q, const float *chr_q, float *d_y, size_t y_stride, float *d_cb,
                              float *d_cr, size_t c_stride);
// k_trellis (jpeg_trellis.cu) on nb blocks of each of n_frames frames (strides in elements); q: host table,
// natural order.  Sets bit 0 of *d_status for input it rejects (see jpeg_trellis.cu).
int launch_trellis(pixo_b200_ctx *ctx, const float *d_src, size_t src_stride, int16_t *d_dst, size_t dst_stride,
                   uint64_t nb, uint32_t n_frames, const float q[64], float lambda, bool zigzag, uint32_t *d_status);
// ext: the arrays are coefficient records (zigzag_in is then ignored)
int launch_jpeg_histogram(pixo_b200_ctx *ctx, const int16_t *d_y, size_t y_stride,
                          const int16_t *d_cb, const int16_t *d_cr, size_t c_stride,
                          uint32_t n_images, size_t ny, size_t nc, uint32_t blocks_y_per_mcu,
                          uint32_t restart_interval, bool zigzag_in, const CoefExtents *ext, uint64_t *d_hist,
                          const int *dc_seed = nullptr);
int launch_png_filter_rows(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride, uint32_t n_images,
                           uint32_t width, uint32_t height, size_t row_bytes, uint32_t bpp, uint32_t strategy,
                           uint8_t *d_out, size_t out_stride, uint32_t *d_adler, const uint8_t *d_above,
                           uint32_t rule_height);
int launch_adler32(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t len, uint32_t *d_out);
// pixo_b200_png_reduce_filter_dev after validation (png_reduce.cu)
int png_reduce_filter(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride, uint32_t n_images,
                      uint32_t width, uint32_t height, uint32_t color_type, uint32_t strategy_and_flags,
                      pixo_b200_png_reduced *info, uint8_t *d_out, size_t out_stride, uint32_t *d_adler);
// pixo_b200_png_quantize_filter_dev after validation (png_quantize.cu); palettes / palette_lens are host
// memory and may be null
int png_quantize_filter(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride, uint32_t n_images,
                        uint32_t width, uint32_t height, uint32_t color_type, uint32_t strategy_and_flags,
                        uint32_t max_colors, const uint8_t *palettes, const uint32_t *palette_lens,
                        pixo_b200_png_reduced *info, uint8_t *d_out, size_t out_stride, uint32_t *d_adler);
// pixo_b200_resize_dev after validation (resize.cu): n frames of bpp bytes per pixel, algorithm 0 Nearest,
// 1 Bilinear, 2 Lanczos3
int launch_resize(pixo_b200_ctx *ctx, const uint8_t *d_src, size_t src_stride, uint32_t n, uint32_t sw, uint32_t sh,
                  uint32_t dw, uint32_t dh, uint32_t bpp, uint32_t algorithm, uint8_t *d_dst, size_t dst_stride);
// pixo_b200_deflate_zlib_on_device after validation (png_deflate.cu): level 1-9, host lens / out_lens / status
int deflate_zlib(pixo_b200_ctx *ctx, const uint8_t *d_streams, size_t stride, const size_t *lens, uint32_t n, int level,
                 uint8_t *d_out, size_t out_cap_each, size_t *out_lens, int32_t *status);
// pixo_b200_png_encode_on_device after validation (png_encode.cu): n frames -> n whole PNG files, host arrays;
// info may be null.  Waits for the device.
int png_encode(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride, uint32_t n, uint32_t width,
               uint32_t height, uint32_t color_type, uint32_t strategy_and_flags, int level, uint32_t max_colors,
               const uint8_t *palettes, const uint32_t *palette_lens, uint8_t *d_out, size_t out_cap_each,
               size_t *out_lens, int32_t *status, pixo_b200_png_reduced *info);

struct FrameGeometry;
struct HuffTables;
size_t entropy_scratch_bytes(uint32_t n, const FrameGeometry &g, uint32_t restart_interval);
// ext: the arrays are the transform's coefficient records; null: the caller's dense natural-order
// arrays, whose coefficients are checked against the baseline range.  d_tabs: n frames' own tables as
// launch_huff_tables writes them (t is then unused); null: t for every frame.
int launch_jpeg_entropy(pixo_b200_ctx *ctx, const int16_t *d_y, size_t y_stride, const int16_t *d_cb,
                        const int16_t *d_cr, size_t c_stride, uint32_t n, const FrameGeometry &g,
                        const HuffTables &t, uint32_t restart_interval, bool allow_segments,
                        const CoefExtents *ext, uint8_t *d_scratch, uint8_t *d_out, uint64_t out_cap,
                        uint64_t **d_out_len, uint32_t **d_overflow, const void *d_tabs = nullptr);
// k_huff_tables (jpeg_entropy.cu): the Huffman tables of n frames from their statistics (kHistWords each;
// d_hist null: the standard tables), as pixo_b200_jpeg_write_headers builds them from a histogram, to d_dht
// (kDhtBytes each) and d_tabs (kHuffDevBytes each, launch_jpeg_entropy's d_tabs); either may be null
int launch_huff_tables(pixo_b200_ctx *ctx, const uint64_t *d_hist, uint32_t n, bool has_chroma, uint8_t *d_dht,
                       void *d_tabs);
int launch_band_entropy(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb, const int16_t *d_cr,
                        const FrameGeometry &g, const HuffTables &t, const int dc_seed[3], const int *d_dc_seed,
                        bool allow_segments, uint8_t *d_raw, uint64_t raw_cap, uint64_t *d_bits_tail,
                        uint32_t *d_flags);
int launch_band_splice(pixo_b200_ctx *ctx, const uint8_t *d_raw, uint64_t base_bit, uint32_t base_tail, bool last,
                       const uint64_t *d_base, uint8_t *d_out, uint64_t out_cap, uint64_t *d_out_len,
                       uint32_t *d_flags);
// bytes a band's raw buffer needs for the band as one string of the usual size, with its trailer
size_t band_raw_bytes(const FrameGeometry &g);
// The raw area of a SegPlan: the segments' strings, then their bit counts and tails (the trailer)
struct SegRaw {
    uint8_t *strings;
    unsigned long long *bits, *tails;
    size_t total, trailer;   // bytes of the area, of the trailer
};
SegRaw seg_raw(const SegPlan &p, void *base);
size_t seg_scratch_bytes(const SegPlan &p);   // the device scratch of its coding and splice
// n whole raw strings of raw_cap bytes each, spliced on their own (no segments)
SegPlan splice_plan(uint32_t n, size_t raw_cap);
// The splice of a whole-string plan (S == 1) that writes an image only when all of it fits: a string whose
// stuffed bytes exceed out_cap gets overflow bit 0, its length in d_out_len and nothing in d_out.  bounds:
// [n][nr + 1] bit offsets into each string, multiples of 8, the last its bit count; range_len ([n][nr]) receives
// the stuffed bytes between consecutive bounds of every string that has bytes.
int launch_splice_bounded(pixo_b200_ctx *ctx, const SegPlan &sp, uint8_t *seg_scratch, const uint8_t *raw_area,
                          uint8_t *d_out, uint64_t out_cap, uint64_t *d_out_len, uint32_t *d_overflow,
                          const unsigned long long *bounds, uint32_t nr, uint64_t *range_len);

// progressive scans (jpeg_progressive.cu)
bool prog_tables(const uint8_t bits[4][16], const uint8_t *const vals[4], ProgTables *T);
// The 7 scans of n whole frames into *dst (the coefficients, DHT blocks and trellis status of an encode come from
// api_jpeg.cu's progressive_coefficients).  Tables and the raw strings:
//  - d_dht: frame i's from its DHT block at d_dht + i * kDhtBytes, queued without a wait; a frame's raw string
//    is as long as its slot (dst->cap + 16 bytes), and a frame whose raw bytes exceed dst->cap is left out
//    (overflow bit 0).  d_trellis_status (or null) is folded into the frames' flags.
//  - otherwise the host's T (n when per_frame, else 1), and one wait for the bit counts, read back as
//    launch_progressive_band reads its own: a coefficient out of range is refused before anything is written,
//    and each raw string is as long as the longest frame's, so only the splice decides the fit.  dst null:
//    nothing is coded; dst->out null: per-frame slots of twice the longest string, which every frame fits, in
//    d_prog_out, set in *dst.
int launch_progressive(pixo_b200_ctx *ctx, const int16_t *d_y, size_t y_stride, const int16_t *d_cb,
                       const int16_t *d_cr, size_t c_stride, uint32_t n, const FrameGeometry &g, const uint8_t *d_dht,
                       const ProgTables *T, bool per_frame, const uint32_t *d_trellis_status, ProgSlots *dst);
// one band of a frame tiled over several GPUs (pixo_b200_jpeg_band_dev_progressive, _summary)
int launch_progressive_band_summary(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb, const int16_t *d_cr,
                                    uint64_t ny, uint64_t nc, uint64_t y_base, uint64_t c_base, ProgBandSummary *out);
int launch_progressive_band(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb, const int16_t *d_cr,
                            const ProgBand &B, const uint64_t *d_hist, uint8_t *d_dht_out, uint8_t *d_raw,
                            size_t raw_cap, size_t *raw_need, uint64_t nbits[7], uint32_t tail7[7]);

}  // namespace pixo
