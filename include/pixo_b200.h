/*
 * pixo_b200.h — C ABI of libpixo_b200.so: the H100 (sm_90a) replacement for the data-parallel
 * stages of leerob/pixo's JPEG and PNG encoders.
 *
 * pixo (v0.4.1 @ 437bf63) has no FFI of its own; its only dispatch seam is src/simd/mod.rs
 * (row-granular, 15 KB calls — far too small for a GPU).  This boundary therefore sits one
 * level up, at the reference functions that already take a whole image (SURVEY.md §8b).
 * Each entry point cites the reference interface it replaces (file:line in the pixo tree).
 * INTEGRATION.md shows the Rust `extern "C"` binding and the call-site patch.
 *
 * Conventions
 *  - plain pointers and sizes only; the caller owns every buffer; the library never retains
 *    or frees caller memory.  `_dev` variants take device pointers and run in order on the
 *    context's stream: after the work queued on it before the call, before the work queued after.
 *    These return with their work still queued (a call that grows the context's scratch first
 *    waits for the stream once, to free the smaller buffer):
 *      jpeg_coefficients_dev (without PIXO_B200_COEF_TRELLIS), jpeg_encode_dev, jpeg_encode_dev_opts,
 *      jpeg_encode_dev_progressive, png_filter_dev,
 *      png_filter_rows_dev, adler32_dev, resize_dev, jpeg_band_histogram_dev,
 *      jpeg_band_entropy_dev_async, jpeg_band_splice_dev_async.
 *    (resize_dev with Lanczos3 stages its weight tables in one of the context's two pinned buffers,
 *    in turn, and first waits until the copy out of that buffer, two Lanczos3 calls back, has run.)
 *    These wait for the work queued before them, and for part of their own, before they return,
 *    because a result they read back decides what they do next or is a host output (the last
 *    kernels or copies of progressive_scans_dev, reduce_filter_dev and quantize_filter_dev are
 *    still queued when they return):
 *      jpeg_coefficients_dev with PIXO_B200_COEF_TRELLIS, jpeg_trellis_quantize_dev,
 *      jpeg_progressive_scans_dev, jpeg_entropy_encode_dev, jpeg_band_last_dc,
 *      jpeg_band_entropy_dev, jpeg_band_splice_dev, jpeg_band_dev_progressive_summary,
 *      jpeg_band_dev_progressive, jpeg_band_dev_progressive_splice, png_reduce_filter_dev,
 *      png_quantize_filter_dev.
 *    The `_on_device` calls (deflate_zlib_on_device, png_encode_on_device) and the decoders' `_to_device` calls
 *    take host arrays for their per-item results and wait for the device before they return.
 *    The others take host pointers and return after the result is in `out`.
 *  - every function returns a pixo_b200_status (0 = ok).  pixo_b200_last_error(ctx) gives the
 *    message a Rust shim would wrap in Error::CompressionError(String) (src/error.rs:41).
 *    Validation errors mirror the reference's own checks (src/jpeg/mod.rs:333-373,
 *    src/png/mod.rs:442-467).
 *  - there is NO CPU fallback: without a CUDA device every compute entry point fails with
 *    PIXO_B200_ERR_CUDA.
 *  - a context owns one CUDA stream plus reusable device/pinned scratch (mirrors the
 *    encode_into buffer-reuse convention, src/jpeg/mod.rs:375-376).  One context per host
 *    thread; contexts are independent and may target different GPUs.
 */
#ifndef PIXO_B200_H
#define PIXO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PIXO_B200_VERSION 0x000100

typedef struct pixo_b200_ctx pixo_b200_ctx;

typedef enum {
    PIXO_B200_OK = 0,
    PIXO_B200_ERR_INVALID_QUALITY = 1,     /* Error::InvalidQuality          src/error.rs */
    PIXO_B200_ERR_INVALID_DIMENSIONS = 2,  /* Error::InvalidDimensions */
    PIXO_B200_ERR_IMAGE_TOO_LARGE = 3,     /* Error::ImageTooLarge */
    PIXO_B200_ERR_UNSUPPORTED_COLOR = 4,   /* Error::UnsupportedColorType */
    PIXO_B200_ERR_INVALID_DATA_LENGTH = 5, /* Error::InvalidDataLength */
    PIXO_B200_ERR_INVALID_RESTART = 6,     /* Error::InvalidRestartInterval */
    PIXO_B200_ERR_INVALID_ARGUMENT = 7,    /* null pointer, unknown enum value ... */
    PIXO_B200_ERR_OUTPUT_TOO_SMALL = 8,    /* caller's output capacity insufficient */
    PIXO_B200_ERR_UNSUPPORTED = 9,         /* option outside the hot path (progressive) */
    PIXO_B200_ERR_CUDA = 10,               /* CUDA runtime/driver failure (no device, launch) */
    PIXO_B200_ERR_OOM = 11,                /* device or pinned allocation failed */
    PIXO_B200_ERR_INVALID_DECODE = 12,     /* Error::InvalidDecode: malformed or corrupt input to a decoder */
    PIXO_B200_ERR_UNSUPPORTED_DECODE = 13, /* Error::UnsupportedDecode: valid input a decoder does not handle */
    PIXO_B200_ERR_INVALID_COMPRESSION_LEVEL = 14  /* Error::InvalidCompressionLevel: a level outside 1-9 */
} pixo_b200_status;

/* pixo::ColorType repr(u8) — src/color.rs:8-18 */
enum { PIXO_B200_GRAY = 0, PIXO_B200_GRAY_ALPHA = 1, PIXO_B200_RGB = 2, PIXO_B200_RGBA = 3 };
/* pixo::jpeg::Subsampling — src/jpeg/mod.rs:96-102 */
enum { PIXO_B200_S444 = 0, PIXO_B200_S420 = 1 };
/* pixo::png::FilterStrategy, declaration order — src/png/mod.rs:345-364 */
enum {
    PIXO_B200_FILTER_NONE = 0, PIXO_B200_FILTER_SUB = 1, PIXO_B200_FILTER_UP = 2,
    PIXO_B200_FILTER_AVERAGE = 3, PIXO_B200_FILTER_PAETH = 4, PIXO_B200_FILTER_MINSUM = 5,
    PIXO_B200_FILTER_ADAPTIVE = 6, PIXO_B200_FILTER_ADAPTIVE_FAST = 7,
    PIXO_B200_FILTER_BIGRAMS = 8
};

/* flags for pixo_b200_jpeg_coefficients* (ZIGZAG also for pixo_b200_jpeg_trellis_quantize_dev) */
#define PIXO_B200_COEF_ZIGZAG 1u  /* emit each block in zig-zag order (quantize.rs:107-113) */
#define PIXO_B200_COEF_TRELLIS 2u /* trellis-quantise: compute_all_coefficients(.., use_trellis = true) */

/* ---- context ---------------------------------------------------------------------------- */
int pixo_b200_version(void);
/* number of visible CUDA devices (0 when none / no driver) */
int pixo_b200_device_count(void);
int pixo_b200_ctx_create(int device, pixo_b200_ctx **out);
void pixo_b200_ctx_destroy(pixo_b200_ctx *ctx);
/* last error message of this context (thread's last error when ctx == NULL); never NULL */
const char *pixo_b200_last_error(const pixo_b200_ctx *ctx);
/* adopt an external CUDA stream (cudaStream_t) for all work of this context; NULL restores
 * the context's own stream.  Work queued before the switch is ordered before work queued after it:
 * the new stream waits, on the device, for the old one's work so far (the host does not wait), so
 * the context's scratch, pixo_b200_ctx_sync, pixo_b200_download and pixo_b200_ctx_destroy stay
 * correct across the switch.  Switching to the current stream does nothing.  An adopted stream must
 * stay valid until the context has switched away from it (the switch records an event on it) or has
 * been destroyed (pixo_b200_ctx_sync and pixo_b200_ctx_destroy synchronise it). */
int pixo_b200_ctx_set_stream(pixo_b200_ctx *ctx, void *cuda_stream);
void *pixo_b200_ctx_stream(pixo_b200_ctx *ctx);
int pixo_b200_ctx_sync(pixo_b200_ctx *ctx);
/* kernels launched by this context since creation (every launch is one of this library's own
 * kernels; memcpy/memset are not counted) */
uint64_t pixo_b200_ctx_launch_count(const pixo_b200_ctx *ctx);
/* number of host threads the host-side entropy coder may use (default: hardware threads) */
int pixo_b200_ctx_set_host_threads(pixo_b200_ctx *ctx, int n);
/* Observability of the one place host code can finish device work.  The GPU entropy stage writes
 * each frame's scan into a device buffer sized by a heuristic (half the raw frame + 64 KiB, x 9/8);
 * a frame that needs more is coded again on the GPU with the exact size (the kernel reports it),
 * and only if that is switched off, or the device stage reports a fault, does the host coder
 * finish the frame from the same GPU coefficient arrays.  host_fallbacks counts those frames
 * since the context was created (0 in normal operation).
 * set_scan_capacity: bytes_per_frame 0 restores the heuristic; gpu_retry 0 disables the second
 * GPU pass (test hook: a tiny capacity with gpu_retry 0 forces the host coder). */
uint64_t pixo_b200_ctx_host_fallbacks(const pixo_b200_ctx *ctx);
int pixo_b200_ctx_set_scan_capacity(pixo_b200_ctx *ctx, size_t bytes_per_frame, int gpu_retry);

/* device / pinned memory helpers so a Rust caller need not link the CUDA runtime */
int pixo_b200_dev_alloc(pixo_b200_ctx *ctx, size_t bytes, void **dptr);
int pixo_b200_dev_free(pixo_b200_ctx *ctx, void *dptr);
int pixo_b200_host_alloc_pinned(pixo_b200_ctx *ctx, size_t bytes, void **hptr);
int pixo_b200_host_free_pinned(pixo_b200_ctx *ctx, void *hptr);
int pixo_b200_upload(pixo_b200_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes);
int pixo_b200_download(pixo_b200_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes);

/* ---- JPEG ------------------------------------------------------------------------------- */

/* QuantizationTables::with_quality — src/jpeg/quantize.rs:42-89.
 * lum_zz/chr_zz: zig-zag order u8 (what DQT carries); lum/chr: natural order f32 (arithmetic).
 * Any output pointer may be NULL.  Host-only, no device needed. */
void pixo_b200_quant_tables(int quality, uint8_t lum_zz[64], uint8_t chr_zz[64], float lum[64],
                            float chr[64]);

/* Block counts of the coefficient arrays: ny Y blocks, nc blocks per chroma component
 * (src/jpeg/mod.rs:1055-1125). */
int pixo_b200_jpeg_block_counts(uint32_t width, uint32_t height, uint32_t color_type,
                                uint32_t subsampling, size_t *ny, size_t *nc);

/* Replaces compute_all_coefficients — src/jpeg/mod.rs:932-966 (and the per-MCU transform
 * work inlined in encode_scan :1408-1563 and build_optimized_huffman_tables :684-824):
 * extract_block/extract_mcu_420 (:1565-1656) -> color::rgb_to_ycbcr (src/color.rs:60-77) ->
 * dct::dct_2d (src/jpeg/dct.rs:614-700) -> quantize_dct (:970): quantize_block
 * (src/jpeg/quantize.rs:99-105), or with PIXO_B200_COEF_TRELLIS trellis::trellis_quantize
 * (src/jpeg/trellis.rs:67-208, lambda None) as use_trellis = true selects (pixo's max preset).
 * y: ny*64, cb/cr: nc*64 int16 (cb/cr ignored for Gray), natural order unless
 * PIXO_B200_COEF_ZIGZAG, blocks in the reference's MCU order (4:2:0: Y TL,TR,BL,BR per MCU).
 * hist (optional, may be NULL): 536 u64 = dc_lum[12] dc_chrom[12] ac_lum[256] ac_chrom[256],
 * the count_block statistics of src/jpeg/mod.rs:826-860 with no restart interval.  hist must be
 * NULL with PIXO_B200_COEF_TRELLIS (PIXO_B200_ERR_INVALID_ARGUMENT): pixo builds its tables from
 * plain-rounded coefficients, which a call without the flag returns.  Other flag bits are ignored.
 * With PIXO_B200_COEF_TRELLIS the _dev variant waits for the device before it returns. */
int pixo_b200_jpeg_coefficients(pixo_b200_ctx *ctx, const uint8_t *pixels, uint32_t width,
                                uint32_t height, uint32_t color_type, uint32_t subsampling,
                                const float lum_q[64], const float chr_q[64], int16_t *y,
                                int16_t *cb, int16_t *cr, uint32_t flags, uint64_t *hist);

/* Same, device pointers, asynchronous on the context's stream.  `n_images` frames of identical
 * geometry: frame i reads d_pixels + i*pixel_stride and writes d_y + i*y_stride (int16
 * elements), d_cb/d_cr + i*c_stride.  d_hist (optional): n_images*536 u64, zeroed by the call. */
int pixo_b200_jpeg_coefficients_dev(pixo_b200_ctx *ctx, const uint8_t *d_pixels,
                                    size_t pixel_stride, uint32_t n_images, uint32_t width,
                                    uint32_t height, uint32_t color_type, uint32_t subsampling,
                                    const float lum_q[64], const float chr_q[64], int16_t *d_y,
                                    size_t y_stride, int16_t *d_cb, int16_t *d_cr,
                                    size_t c_stride, uint32_t flags, uint64_t *d_hist);

/* Replaces trellis::trellis_quantize (src/jpeg/trellis.rs:67-208) for a batch of blocks, with the
 * same kernel PIXO_B200_COEF_TRELLIS runs.  d_dct: n_blocks x 64 f32 DCT coefficients (natural order,
 * device, 16-byte aligned); q: 64 f32 quantiser entries (natural order, host; integers 1..255);
 * lambda: pixo's Option<f32>, 1.0f for None (trellis_quantize_adaptive's formula, trellis.rs:304-321,
 * picks it from the quality).  d_out: n_blocks x 64 int16 (device, 16-byte aligned), natural order
 * unless PIXO_B200_COEF_ZIGZAG.  Waits for the device.  PIXO_B200_ERR_INVALID_ARGUMENT for input
 * this kernel does not carry: a non-finite coefficient or cost, a non-zero |dct| below 2^-100, or
 * |dct / q| above 32766 (where the reference's i16 candidates saturate or overflow); the output is
 * then unspecified. */
int pixo_b200_jpeg_trellis_quantize_dev(pixo_b200_ctx *ctx, const float *d_dct, size_t n_blocks,
                                        const float q[64], float lambda, int16_t *d_out,
                                        uint32_t flags);

/* Replaces pixo::jpeg::encode_into — src/jpeg/mod.rs:328-447 (baseline: encode_scan :1408).
 * GPU: colour/subsample/DCT/quantise, symbol statistics when optimize_huffman, Huffman bit
 * packing with 0xFF stuffing and restart markers (huffman.rs:423-481, src/bits.rs:195-290,
 * mod.rs:1423-1445); host: headers (:449-648) and Huffman table construction
 * (src/jpeg/huffman.rs:100-391).  Byte-identical to the reference.  Only the scan bytes come
 * back over PCIe.  restart_interval 0 = None.  progressive is outside this path
 * (PIXO_B200_ERR_UNSUPPORTED when non-zero: progressive files come from
 * pixo_b200_jpeg_encode_progressive); trellis_quant is accepted and ignored, exactly as
 * the reference's baseline encode_scan ignores use_trellis (src/jpeg/mod.rs:1408-1563 always
 * calls quantize_block). */
int pixo_b200_jpeg_encode(pixo_b200_ctx *ctx, const uint8_t *pixels, size_t pixels_len,
                          uint32_t width, uint32_t height, uint32_t color_type, uint32_t quality,
                          uint32_t subsampling, uint32_t restart_interval,
                          uint32_t optimize_huffman, uint32_t progressive, uint32_t trellis_quant,
                          uint8_t *out, size_t out_cap, size_t *out_len);

/* Batch of n_images frames of identical geometry and options (frame i at pixels + i*len).
 * Transfers and kernels of different frames overlap.  out: n_images
 * slots of out_cap_each bytes; out_lens[i] receives each JPEG's length. */
int pixo_b200_jpeg_encode_batch(pixo_b200_ctx *ctx, const uint8_t *pixels, size_t pixels_len_each,
                                uint32_t n_images, uint32_t width, uint32_t height,
                                uint32_t color_type, uint32_t quality, uint32_t subsampling,
                                uint32_t restart_interval, uint32_t optimize_huffman,
                                uint8_t *out, size_t out_cap_each, size_t *out_lens);

/* pixo::jpeg::encode_into with options.progressive (src/jpeg/mod.rs:395-410, encode_progressive
 * :872-927): the same file pixo writes - SOI, APP0, DQT, SOF2, DHT, DRI when restart_interval != 0,
 * then the 7 scans of simple_progressive_script (Y DC, Cb DC, Cr DC, Y 1-10, Y 11-63, Cb 1-63,
 * Cr 1-63, Ah = Al = 0), each an SOS and its entropy-coded segment, then EOI.  pixo's quirks are kept:
 * every scan walks its component's array in compute_all_coefficients order (MCU order for 4:2:0 Y),
 * DC predictors are never reset, DRI is written but no RST marker, the optimised tables come from the
 * plain-rounded baseline statistics (restart interval included) also under trellis_quant, EOB runs
 * whose symbol a table lacks get the (0, 4) fallback code, and a gray frame still gets the (empty)
 * chroma scans.  These files are pixo's, not always conformant JPEGs.  GPU: transform, statistics,
 * COEF_TRELLIS when trellis_quant, and the progressive scan stage (stuffed segments); host: headers and
 * tables.  Same errors as pixo_b200_jpeg_encode; PIXO_B200_ERR_CUDA for a device fault (no host twin). */
int pixo_b200_jpeg_encode_progressive(pixo_b200_ctx *ctx, const uint8_t *pixels, size_t pixels_len,
                                      uint32_t width, uint32_t height, uint32_t color_type, uint32_t quality,
                                      uint32_t subsampling, uint32_t restart_interval, uint32_t optimize_huffman,
                                      uint32_t trellis_quant, uint8_t *out, size_t out_cap, size_t *out_len);
int pixo_b200_jpeg_encode_progressive_batch(pixo_b200_ctx *ctx, const uint8_t *pixels, size_t pixels_len_each,
                                            uint32_t n_images, uint32_t width, uint32_t height,
                                            uint32_t color_type, uint32_t quality, uint32_t subsampling,
                                            uint32_t restart_interval, uint32_t optimize_huffman,
                                            uint32_t trellis_quant, uint8_t *out, size_t out_cap_each,
                                            size_t *out_lens);

/* The progressive scan stage on caller coefficient arrays (device memory, compute_all_coefficients'
 * layout: natural order, frame i at d_y + i*y_stride, d_cb/d_cr + i*c_stride, strides in int16
 * elements, multiples of 8 and at least a frame's blocks when n_frames > 1; arrays 16-byte aligned;
 * d_cb/d_cr ignored for gray).  Per frame the 7 stuffed, 1-padded segments back to back at
 * d_out + i*out_cap_each, lengths in d_scan_len[i*7 + s] (the size needed, also when it did not fit);
 * d_overflow[i] bit 0: they did not fit out_cap_each and nothing was written for that frame.
 * dht: 4 x (16 counts + 256 values), order dc_lum, dc_chrom, ac_lum, ac_chrom (the file's DHT), NULL =
 * the standard tables.  PIXO_B200_ERR_INVALID_ARGUMENT, with nothing written, for a coefficient outside
 * -16383..16383 (every DC difference then fits int16 and every category is <= 15), a table with more
 * than 256 values or a code that does not fit its length, or a layout above.  Waits for the device to
 * measure the scans; the splice into d_out is queued on the context's stream. */
int pixo_b200_jpeg_progressive_scans_dev(pixo_b200_ctx *ctx, const int16_t *d_y, size_t y_stride,
                                         const int16_t *d_cb, const int16_t *d_cr, size_t c_stride,
                                         uint32_t n_frames, uint32_t width, uint32_t height, uint32_t color_type,
                                         uint32_t subsampling, const uint8_t *dht, uint8_t *d_out,
                                         size_t out_cap_each, uint64_t *d_scan_len, uint32_t *d_overflow);

/* Device-resident variant of the whole hot path (asynchronous on the context's stream):
 * frame i at d_pixels + i*pixel_stride -> entropy-coded scan bytes (what encode_scan appends
 * between the SOS header and EOI, src/jpeg/mod.rs:1408-1563) at d_scan + i*scan_cap_each, byte
 * count in d_scan_len[i] (the size needed, also when it did not fit); d_overflow[i] != 0 when the
 * frame was not finished: bit 0 scan_cap_each was too small, bit 1 a device fault (spin limit), bit 2 a
 * segment of a frame that is coded in segments (few large frames) outgrew its internal buffer - does
 * not happen for JPEGs smaller than their raw pixels; pixo_b200_jpeg_encode* handle all three.  Baseline, standard Huffman tables, no restart interval:
 * the same as pixo_b200_jpeg_encode_dev_opts(.., 0, 0, .., NULL), which also takes a restart interval and
 * optimised tables (pixo's balanced preset).
 * Headers/EOI are the caller's (pixo_b200_jpeg_encode* add them). */
int pixo_b200_jpeg_encode_dev(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride,
                              uint32_t n_images, uint32_t width, uint32_t height,
                              uint32_t color_type, uint32_t quality, uint32_t subsampling,
                              uint8_t *d_scan, size_t scan_cap_each, uint64_t *d_scan_len,
                              uint32_t *d_overflow);

/* pixo_b200_jpeg_encode_dev with pixo's remaining baseline options: restart_interval (0 = None; RSTn
 * markers in the scan, src/jpeg/mod.rs:1423-1445) and optimize_huffman (every frame gets the tables
 * build_optimized_huffman_tables(..).unwrap_or_default() gives its own statistics, src/jpeg/mod.rs:379-392,
 * built on the GPU).  Same arguments, checks and overflow bits as pixo_b200_jpeg_encode_dev, and queued on the
 * context's stream like it: the statistics, the tables and the scans never wait for the host.
 * d_dht (device, may be NULL): n_images x 1088 bytes, frame i's tables at d_dht + i*1088 as 4 x (16 counts +
 * 256 values, unused values 0) in the order dc_lum, dc_chrom, ac_lum, ac_chrom - the layout
 * pixo_b200_jpeg_progressive_scans_dev takes - standard ones unless optimize_huffman.  A file is
 * pixo_b200_jpeg_write_headers_dht(frame i's tables), the scan bytes, then EOI (0xFF 0xD9). */
int pixo_b200_jpeg_encode_dev_opts(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride,
                                   uint32_t n_images, uint32_t width, uint32_t height, uint32_t color_type,
                                   uint32_t quality, uint32_t subsampling, uint32_t restart_interval,
                                   uint32_t optimize_huffman, uint8_t *d_scan, size_t scan_cap_each,
                                   uint64_t *d_scan_len, uint32_t *d_overflow, uint8_t *d_dht);

/* pixo's max preset for device frames: pixo_b200_jpeg_encode_progressive_batch's scans without a host in the
 * loop.  Frame i at d_pixels + i*pixel_stride -> its 7 stuffed, 1-padded segments (simple_progressive_script's
 * scans, in order) back to back at d_out + i*out_cap_each, their lengths in d_scan_len[i*7 + s] and, when d_dht
 * (device, may be NULL) is given, the tables they were coded with at d_dht + i*1088 (pixo_b200_jpeg_encode_dev_opts'
 * layout; standard ones unless optimize_huffman).  Segments and tables are exactly what
 * pixo_b200_jpeg_encode_progressive_batch writes for the same pixels and options, quirks included (see
 * pixo_b200_jpeg_encode_progressive); pixo_b200_jpeg_progressive_file(frame i's tables, its segments, its
 * lengths) is that call's file.
 * Queued on the context's stream like pixo_b200_jpeg_encode_dev_opts: nothing waits for the device except growth
 * of the context's scratch.  What the host entry point learns by waiting is a bit of d_overflow[i]:
 *   bit 0   the segments did not fit out_cap_each; nothing was written in the frame's slot, and d_scan_len holds
 *           lengths whose sum is enough for a second call (the exact ones when the frame's raw bits fit the slot,
 *           twice each segment's unstuffed bytes otherwise)
 *   bit 4   input the trellis or the progressive stage cannot carry (a frame of 8-bit pixels never reaches it); set on
 *           every frame coded in the same pass, with nothing written in their slots
 * Checks, in this order, each before anything is launched: quality and restart_interval (as pixo_b200_jpeg_encode),
 * the geometry, null d_pixels / d_out / d_scan_len / d_overflow (PIXO_B200_ERR_INVALID_ARGUMENT), n_images 0 returns
 * at once, more than 65535 frames and a d_scan_len not 8-byte aligned or a d_overflow not 4-byte aligned are
 * PIXO_B200_ERR_INVALID_ARGUMENT.  d_pixels and d_out may sit at any byte.  Frames go through in passes of at most
 * 8192, each holding a raw string of out_cap_each + 16 bytes per frame and the frames' coefficients in the context's
 * scratch, at most 512 MiB of each (one frame at least); see DESIGN.md section 7. */
int pixo_b200_jpeg_encode_dev_progressive(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride,
                                          uint32_t n_images, uint32_t width, uint32_t height, uint32_t color_type,
                                          uint32_t quality, uint32_t subsampling, uint32_t restart_interval,
                                          uint32_t optimize_huffman, uint32_t trellis_quant, uint8_t *d_out,
                                          size_t out_cap_each, uint64_t *d_scan_len, uint32_t *d_overflow,
                                          uint8_t *d_dht);

/* Entropy-code caller-provided coefficient arrays (host) into a baseline JPEG: the host half of
 * pixo_b200_jpeg_encode on its own (src/jpeg/mod.rs:395-447,1408-1563 consuming arrays shaped
 * like compute_all_coefficients' result).  Host-only, no device needed.
 * Coefficients outside the baseline range - an AC value with |v| > 1023, or a DC difference (int16
 * wrapping, against the previous block of the component, 0 after a restart) with |d| > 2047 - have no
 * Huffman code: every entry point that takes caller coefficients returns
 * PIXO_B200_ERR_INVALID_ARGUMENT for them (the stream-ordered ones set bit 3 of d_flags). */
int pixo_b200_jpeg_entropy_encode(pixo_b200_ctx *ctx, const int16_t *y, const int16_t *cb,
                                  const int16_t *cr, uint32_t width, uint32_t height,
                                  uint32_t color_type, uint32_t quality, uint32_t subsampling,
                                  uint32_t restart_interval, uint32_t optimize_huffman,
                                  uint8_t *out, size_t out_cap, size_t *out_len);

/* The same for coefficient arrays that live on the DEVICE (natural order, the layout
 * pixo_b200_jpeg_coefficients_dev writes): optimised-table statistics (K3) and the Huffman /
 * stuffing / restart stage (k_huff) run on the GPU, only the scan bytes come back; out receives
 * the complete JPEG.  This is what a frame tiled over several GPUs uses once its bands'
 * coefficients have been gathered on one of them (SURVEY.md section 8e).
 * d_y, and d_cb / d_cr unless Gray, must be 16-byte aligned (the kernels load whole blocks as
 * 16-byte vectors): PIXO_B200_ERR_INVALID_ARGUMENT otherwise, before anything is launched.  The
 * same holds for pixo_b200_jpeg_band_histogram_dev and pixo_b200_jpeg_band_entropy_dev(_async). */
int pixo_b200_jpeg_entropy_encode_dev(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                      const int16_t *d_cr, uint32_t width, uint32_t height,
                                      uint32_t color_type, uint32_t quality, uint32_t subsampling,
                                      uint32_t restart_interval, uint32_t optimize_huffman,
                                      uint8_t *out, size_t out_cap, size_t *out_len);

/* ---- one frame tiled over several GPUs (SURVEY.md section 8e, BASELINE config C4) --------------
 * The reference's analogue is compute_all_coefficients_parallel (src/jpeg/mod.rs:1137-1215, rayon
 * over MCU rows) followed by the sequential encode_scan.  Here every GPU owns a contiguous band of
 * MCU rows and runs the WHOLE path on it; only finished scan bytes are gathered:
 *   1. transform: pixo_b200_jpeg_coefficients_dev on the band's pixel rows (a band starts on an
 *      MCU row, so it is an image of its own: no halo; the frame's bottom clamp falls in the last band);
 *   2. the DC predictors cross bands: band r starts from band r-1's last DC per component
 *      (pixo_b200_jpeg_band_last_dc; one tiny all-gather);
 *   3. [optimize_huffman] pixo_b200_jpeg_band_histogram_dev, statistics summed over the bands
 *      (all-reduce of 536 u64), identical tables on every rank;
 *   4. pixo_b200_jpeg_band_entropy_dev: the band's Huffman code as a raw bit string (no 0xFF
 *      stuffing, no padding: both depend on the bit offset, which is not known yet) plus its bit
 *      count and last 7 bits (second tiny all-gather -> every band's bit offset in the frame's stream
 *      and the bits it inherits in its first byte);
 *   5. pixo_b200_jpeg_band_splice_dev: shift to the bit offset, complete the shared first byte, stuff
 *      0xFF -> 0xFF00 (src/bits.rs:245-259), 1-pad the frame's last byte (:261-272).  A band owns the
 *      stream bytes whose LAST bit it wrote;
 *   6. rank 0 writes pixo_b200_jpeg_write_headers, the bands' bytes in band order, EOI.
 * No restart interval on this path (every interval would need its own offset exchange).
 * The `_dev` calls return after their host outputs are valid.  Host twins (no device needed) take
 * host arrays: they serve the CPU-only tests and a host that merely assembles. */
int pixo_b200_jpeg_band_last_dc(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                const int16_t *d_cr, size_t ny, size_t nc, int32_t last_dc[3]);
int pixo_b200_jpeg_band_histogram_dev(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                      const int16_t *d_cr, uint32_t width, uint32_t band_height,
                                      uint32_t color_type, uint32_t subsampling,
                                      const int32_t dc_seed[3], uint64_t *d_hist /* 536, device */);
/* (pixo_b200_jpeg_band_histogram_dev does not wait for the device, so it cannot report coefficients
 * outside the baseline range: it counts them in the nearest category, and the band's
 * pixo_b200_jpeg_band_entropy_dev(_async) rejects them.) */
/* hist (host, optional): the frame's summed statistics -> optimised tables (standard when NULL or
 * when they cannot be built, as the reference's unwrap_or_default does).  d_raw: 16-byte aligned,
 * raw_cap a multiple of 4; it must stay untouched until the band has been spliced.  A raw_cap of at
 * least the band's pixel bytes + 1 MiB lets a long band be coded as several independent segments
 * (shorter look-back chains); with less room the band is coded as one string, in what raw_cap leaves
 * after 512 bytes for its bit count and tail.  A segment gets about its pixel bytes; a dense band
 * whose segments outgrow that is coded again as one string in the same call.  A string that does not
 * fit returns PIXO_B200_ERR_OUTPUT_TOO_SMALL with *nbits = the bits it needs; a second call whose
 * raw_cap holds those bits' bytes rounded up to a multiple of 256, plus the 512, succeeds. */
int pixo_b200_jpeg_band_entropy_dev(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                    const int16_t *d_cr, uint32_t width, uint32_t band_height,
                                    uint32_t color_type, uint32_t subsampling,
                                    const int32_t dc_seed[3], const uint64_t *hist, uint8_t *d_raw,
                                    size_t raw_cap, uint64_t *nbits, uint32_t *tail7);
/* d_raw: a buffer this context coded with pixo_b200_jpeg_band_entropy_dev(_async); nbits: the count
 * that returned (0: an empty band, which owns no byte; d_raw may then be NULL).  start_bit: bits of the
 * frame's stream before this band; tail_in: the last (start_bit % 8) of them. */
int pixo_b200_jpeg_band_splice_dev(pixo_b200_ctx *ctx, const uint8_t *d_raw, uint64_t nbits,
                                   uint64_t start_bit, uint32_t tail_in, uint32_t is_last_band,
                                   uint8_t *d_out, size_t out_cap, uint64_t *out_len);
/* Stream-ordered variants: everything that crosses a band boundary stays in DEVICE memory, so a
 * rank can queue transform -> (NCCL all-gather of predictors) -> coding -> (all-gather of bits) ->
 * splice without a single host synchronisation; only the final byte count is read back.
 *   d_dc_seed:   int32[3] in device memory (written by an earlier operation on the stream)
 *   d_bits_tail: uint64[2] out, {bit count, last 7 bits}
 *   d_offset:    uint64[3] in, {start_bit, the last 7 bits of the stream before this band, is_last_band}
 *   d_flags:     uint32, OR-ed: bit 0 a capacity was too small, bit 1 device fault, bit 3 a coefficient
 *                outside the baseline range (caller zeroes it)
 * raw_cap must be at least the band's pixel bytes + 1 MiB.  A dense band coded in segments can set bit 0
 * with that room (see pixo_b200_jpeg_band_entropy_dev, which recodes it as one string). */
int pixo_b200_jpeg_band_entropy_dev_async(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                          const int16_t *d_cr, uint32_t width, uint32_t band_height,
                                          uint32_t color_type, uint32_t subsampling,
                                          const int32_t *d_dc_seed, const uint64_t *hist, uint8_t *d_raw,
                                          size_t raw_cap, uint64_t *d_bits_tail, uint32_t *d_flags);
int pixo_b200_jpeg_band_splice_dev_async(pixo_b200_ctx *ctx, const uint8_t *d_raw, const uint64_t *d_offset,
                                         uint8_t *d_out, size_t out_cap, uint64_t *d_out_len,
                                         uint32_t *d_flags);
/* The progressive scans of one band (pixo's max preset, pixo_b200_jpeg_encode_progressive's scans and quirks).  A band
 * of whole MCU rows is a contiguous range of each component's array (4:2:0 Y in MCU order too), so it is given as
 * ny Y and nc chroma blocks starting at the frame's Y block y_base and chroma block c_base (the blocks of the bands
 * before it).  Per scan a band needs from the bands before it:
 *   - DC scans: the DC predictor of its first block, the last DC of the nearest earlier band with blocks of that
 *     component in the arrays being coded (0 for none; predictors are never reset);
 *   - AC scans (Y 1-10, Y 11-63, Cb 1-63, Cr 1-63): the EOB run pending at its start, given as the carry
 *     max((index + 1) << 1 | init) over the earlier bands' last_enc (0 for none): init is 1 when that block's last
 *     non-zero lies below the scan's Se.  0x7FFF flushes then fall where pixo's frame-wide count puts them, and the
 *     flush at the scan's end belongs to the band that holds the scan's last block;
 *   - its start bit in each scan's stream, and the bits it inherits in the stream's first byte (see below).
 * Every array is natural order, 16-byte aligned where the band has blocks of it; d_cb / d_cr are ignored when nc
 * is 0.  Coefficients outside -16383..16383 return PIXO_B200_ERR_INVALID_ARGUMENT, with nothing written.  These
 * calls wait for the device.  No restart interval on this path (pixo's max preset sets none).
 *
 * summary: the band's last DC per component (0 without blocks) and, per AC scan, its largest
 * ((frame index + 1) << 1 | init) over its non-empty blocks (0: none), from the arrays being coded. */
int pixo_b200_jpeg_band_dev_progressive_summary(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                                const int16_t *d_cr, size_t ny, size_t nc, uint64_t y_base,
                                                uint64_t c_base, int32_t last_dc[3], uint32_t last_enc[4]);
/* The band's 7 scans as raw bit strings (no 0xFF stuffing, no padding) in d_raw, their bit counts in nbits and their
 * last 7 bits (fewer when the string is shorter; the last bit in bit 0) in tail7.  frame_ny / frame_nc: the frame's
 * block counts (frame_nc 0: a gray frame, whose chroma scans are empty).  dc_seed / ac_carry: see above (ac_carry in
 * the order Y 1-10, Y 11-63, Cb, Cr).  d_hist (device, may be NULL): the frame's 536 summed statistics of the
 * PLAIN-rounded coefficients (pixo_b200_jpeg_band_histogram_dev of every band, seeded with the plain arrays' DC
 * predictors) -> optimised tables built on the device as pixo_b200_jpeg_encode_dev_progressive builds them; NULL:
 * the standard tables.  d_dht (device, may be NULL) receives those tables (1088 bytes, the layout
 * pixo_b200_jpeg_progressive_file takes), also for a band without blocks.  d_raw: 16-byte aligned, untouched by
 * other work until the band's scans have been spliced; NULL allowed for a band without blocks.  *raw_need receives
 * the bytes d_raw must hold (0 without blocks); below that the call returns PIXO_B200_ERR_OUTPUT_TOO_SMALL with
 * nbits set and nothing else written, and a second call with raw_cap >= *raw_need succeeds. */
int pixo_b200_jpeg_band_dev_progressive(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb,
                                        const int16_t *d_cr, size_t ny, size_t nc, uint64_t y_base, uint64_t c_base,
                                        uint64_t frame_ny, uint64_t frame_nc, const int32_t dc_seed[3],
                                        const uint32_t ac_carry[4], const uint64_t *d_hist, uint8_t *d_dht,
                                        uint8_t *d_raw, size_t raw_cap, size_t *raw_need, uint64_t nbits[7],
                                        uint32_t tail7[7]);
/* Scan `scan` (0..6, simple_progressive_script's order) of a band coded into d_raw, as
 * pixo_b200_jpeg_band_splice_dev splices a baseline band: nbits = that scan's count (0: the band owns no byte of the
 * scan; d_raw may then be NULL), start_bit = the scan's bits in the bands before it, tail_in = the last
 * (start_bit % 8) of those bits (they may come from several bands when some wrote fewer than 7), is_last_band = no
 * later band writes a bit of this scan (this band 1-pads its end).  The 7 segments of pixo_b200_jpeg_progressive_file
 * are, per scan, the bands' spliced bytes in band order. */
int pixo_b200_jpeg_band_dev_progressive_splice(pixo_b200_ctx *ctx, const uint8_t *d_raw, uint32_t scan, uint64_t nbits,
                                               uint64_t start_bit, uint32_t tail_in, uint32_t is_last_band,
                                               uint8_t *d_out, size_t out_cap, uint64_t *out_len);
int pixo_b200_jpeg_band_entropy(const int16_t *y, const int16_t *cb, const int16_t *cr, uint32_t width,
                                uint32_t band_height, uint32_t color_type, uint32_t subsampling,
                                const int32_t dc_seed[3], const uint64_t *hist, uint8_t *raw,
                                size_t raw_cap, uint64_t *nbits, uint32_t *tail7);
int pixo_b200_jpeg_band_histogram(const int16_t *y, const int16_t *cb, const int16_t *cr, uint32_t width,
                                  uint32_t band_height, uint32_t color_type, uint32_t subsampling,
                                  const int32_t dc_seed[3], uint64_t hist[536]);
int pixo_b200_jpeg_band_splice(const uint8_t *raw, uint64_t nbits, uint64_t start_bit, uint32_t tail_in,
                               uint32_t is_last_band, uint8_t *out, size_t out_cap, size_t *out_len);
/* SOI .. SOS of the frame (src/jpeg/mod.rs:395-430,449-648); out_cap >= 1024.  Host-only. */
int pixo_b200_jpeg_write_headers(uint32_t width, uint32_t height, uint32_t color_type, uint32_t quality,
                                 uint32_t subsampling, uint32_t restart_interval, const uint64_t *hist,
                                 uint8_t *out, size_t out_cap, size_t *out_len);
/* The same headers with the Huffman tables given as DHT data (host, 1088 bytes, the layout
 * pixo_b200_jpeg_encode_dev_opts writes to d_dht): a file's headers for exactly the tables its scan was
 * coded with.  Tables built from hist give the bytes pixo_b200_jpeg_write_headers(.., hist, ..) gives.
 * PIXO_B200_ERR_INVALID_ARGUMENT for a table of more than 256 values or with a code that does not fit its
 * length; out_cap >= 1024, and >= the headers' length (at most 281 bytes + the tables' values).  Host-only. */
int pixo_b200_jpeg_write_headers_dht(uint32_t width, uint32_t height, uint32_t color_type, uint32_t quality,
                                     uint32_t subsampling, uint32_t restart_interval, const uint8_t *dht,
                                     uint8_t *out, size_t out_cap, size_t *out_len);

/* A whole progressive file from one frame's scans (host memory): SOI, APP0, DQT, SOF2, DHT of `dht` (1088 bytes in
 * pixo_b200_jpeg_encode_dev_opts' layout, NULL = the standard tables), DRI when restart_interval != 0, then per
 * scan s of simple_progressive_script its SOS and scan_len[s] bytes of `segments` (the 7 segments back to back, as
 * pixo_b200_jpeg_encode_dev_progressive and pixo_b200_jpeg_progressive_scans_dev leave them in a slot), then EOI.
 * For the segments and tables of pixo_b200_jpeg_encode_progressive it is the file that call writes.  The tables are
 * checked as pixo_b200_jpeg_write_headers_dht checks them; PIXO_B200_ERR_OUTPUT_TOO_SMALL when out_cap is below the
 * file's length.  Host-only. */
int pixo_b200_jpeg_progressive_file(uint32_t width, uint32_t height, uint32_t color_type, uint32_t quality,
                                    uint32_t subsampling, uint32_t restart_interval, const uint8_t *dht,
                                    const uint8_t *segments, const uint64_t scan_len[7], uint8_t *out, size_t out_cap,
                                    size_t *out_len);

/* ---- PNG -------------------------------------------------------------------------------- */

/* Replaces filter::apply_filters_with_row_bytes — src/png/filter.rs:64-206 (+ the rayon path
 * apply_filters_parallel :574-608), i.e. filter_{sub,up,average,paeth} (src/simd/mod.rs:159-236,
 * normative scalar src/simd/fallback.rs:100-159), score_filter (:93-98), adaptive_filter
 * (filter.rs:302-393), adaptive_filter_fast (:474-527), bigrams_filter (:410-471).
 * Semantics follow the default-feature build (`parallel` on): area <= 4096 forces Sub; for
 * height <= 32 AdaptiveFast is sticky on row 0's winner (:147-166).
 * out: height*(row_bytes+1).  adler32_out (optional): Adler-32 of `out`
 * (src/compress/adler32.rs:11-47), computed on the device in the same pass.
 * strategy may be OR-ed with PIXO_B200_PNG_OPTIMIZE_ALPHA: the pre-pass encode() runs before
 * filtering when PngOptions::optimize_alpha is set (maybe_optimize_alpha, src/png/mod.rs:633-671:
 * colour bytes of fully transparent pixels become 0; bytes_per_pixel 4 = Rgba, 2 = GrayAlpha,
 * other pixel sizes are left alone) is applied on the fly while the rows are read. */
#define PIXO_B200_PNG_OPTIMIZE_ALPHA 0x100u
int pixo_b200_png_filter(pixo_b200_ctx *ctx, const uint8_t *data, uint32_t width,
                         uint32_t height, size_t row_bytes, uint32_t bytes_per_pixel,
                         uint32_t strategy, uint8_t *out, uint32_t *adler32_out);

/* Device-pointer, batched variant (asynchronous).  Frame i: d_data + i*in_stride ->
 * d_out + i*out_stride; d_adler (optional): n_images u32.  Frames must not overlap: with
 * n_images > 1, in_stride < height*row_bytes returns PIXO_B200_ERR_INVALID_DATA_LENGTH and
 * out_stride < height*(row_bytes+1) returns PIXO_B200_ERR_OUTPUT_TOO_SMALL.  Any alignment. */
int pixo_b200_png_filter_dev(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride,
                             uint32_t n_images, uint32_t width, uint32_t height,
                             size_t row_bytes, uint32_t bytes_per_pixel, uint32_t strategy,
                             uint8_t *d_out, size_t out_stride, uint32_t *d_adler);

/* One image's rows in bands (SURVEY.md section 8e: filters read the RAW previous row, so a band
 * only needs the one raw row above it - an overlapping read, not an exchange).  d_rows: band_rows
 * rows of the image starting at some row r0; d_row_above: the raw row r0-1 (NULL for r0 == 0 =
 * zeros, src/png/filter.rs:112-117); image_height: rows of the WHOLE image (the strategy pre-rules
 * of apply_filters_with_row_bytes look at the whole image).  d_out: band_rows*(row_bytes+1);
 * d_adler (optional): Adler-32 of this band's slice of the filtered stream, started from the
 * initial state; combine the bands' values in order (s1 = s1A + s1B - 1, s2 = s2A + s2B +
 * lenB*(s1A - 1) mod 65521 - pixo_b200_adler32_combine). */
int pixo_b200_png_filter_rows_dev(pixo_b200_ctx *ctx, const uint8_t *d_rows, const uint8_t *d_row_above,
                                  uint32_t width, uint32_t image_height, uint32_t band_rows,
                                  size_t row_bytes, uint32_t bytes_per_pixel, uint32_t strategy,
                                  uint8_t *d_out, uint32_t *d_adler);
/* Adler-32 of A ++ B from adler32(A), adler32(B) and len(B).  Host-only. */
uint32_t pixo_b200_adler32_combine(uint32_t adler_a, uint32_t adler_b, uint64_t len_b);

/* Lossless colour-type and palette reduction ahead of the filter: what pixo's balanced and max presets
 * do in encode_into before DEFLATE (src/png/mod.rs:521-568).  Flags for the strategy word of
 * pixo_b200_png_reduce_filter* only (pixo_b200_png_filter* keep rejecting them):
 *   REDUCE_COLOR_TYPE  PngOptions::reduce_color_type  RGB/RGBA -> Gray (1/2/4/8 bits), RGB, GrayAlpha
 *   REDUCE_PALETTE     PngOptions::reduce_palette     RGB/RGBA with <= 256 colours -> indexed */
#define PIXO_B200_PNG_REDUCE_COLOR_TYPE 0x200u
#define PIXO_B200_PNG_REDUCE_PALETTE 0x400u

/* The reduced image (ReducedImage, src/png/mod.rs:673-680): what write_ihdr, PLTE and tRNS need. */
typedef struct {
    uint8_t color_type_byte;       /* IHDR colour type: 0 Gray, 2 RGB, 3 indexed, 4 GrayAlpha, 6 RGBA */
    uint8_t bit_depth;             /* IHDR bit depth: 1, 2, 4 or 8 */
    uint8_t effective_color_type;  /* PIXO_B200_GRAY..RGBA as maybe_optimize_alpha sees it (indexed: RGB) */
    uint8_t bytes_per_pixel;       /* of the filter (1 for indexed and sub-byte gray) */
    uint32_t palette_len;          /* PLTE entries, 0 = no PLTE */
    uint32_t trns_len;             /* tRNS entries: palette_len when some alpha is below 255, else 0
                                      (src/png/mod.rs:535-545) */
    uint32_t reserved;
    uint64_t row_bytes;            /* bytes of a reduced row; the filtered stream has height*(row_bytes+1) */
    uint8_t palette[256][4];       /* RGBA, PLTE order (the modified Zeng order) */
} pixo_b200_png_reduced;

/* Replaces maybe_reduce_color_type -> maybe_optimize_alpha -> filter::apply_filters_with_row_bytes in
 * encode_into (src/png/mod.rs:521-568): maybe_reduce_color_type :683-836, build_palette :838-900,
 * optimize_palette_order / mzeng_reindex / apply_most_popular_first :909-1120, all_gray_rgb /
 * analyze_rgba :1122-1147, reduce_gray_bit_depth / palette_bit_depth / pack_bits_rows
 * (src/png/bit_depth.rs).  The GPU finds the colours, the gray / opaque properties and the palette
 * statistics, packs the reduced rows and filters them with the same kernels as pixo_b200_png_filter;
 * the host orders the <= 256 palette entries.  strategy_and_flags: a filter strategy OR-ed with
 * PIXO_B200_PNG_OPTIMIZE_ALPHA (applied to the REDUCED rows when their effective colour type is RGBA
 * or GrayAlpha) and the two REDUCE flags.  Validation as encode_into (src/png/mod.rs:442-467).
 * out: height*(info->row_bytes+1) bytes (PIXO_B200_ERR_OUTPUT_TOO_SMALL with *out_len = the size
 * needed otherwise); adler32_out (optional): Adler-32 of the filtered stream. */
int pixo_b200_png_reduce_filter(pixo_b200_ctx *ctx, const uint8_t *data, size_t data_len, uint32_t width,
                                uint32_t height, uint32_t color_type, uint32_t strategy_and_flags,
                                pixo_b200_png_reduced *info, uint8_t *out, size_t out_cap, size_t *out_len,
                                uint32_t *adler32_out);
/* Batch of device-resident frames of one input geometry: frame i at d_data + i*in_stride, its filtered
 * stream (height*(info[i].row_bytes+1) bytes) at d_out + i*out_stride, out_stride >= height*(width*bpp+1);
 * d_adler (optional): n_images u32.  Frames of one batch may reduce differently.  Returns once info[] is
 * valid (the palette ordering is host work between GPU passes); the filter and its Adler-32 are still
 * asynchronous on the context's stream. */
int pixo_b200_png_reduce_filter_dev(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride,
                                    uint32_t n_images, uint32_t width, uint32_t height, uint32_t color_type,
                                    uint32_t strategy_and_flags, pixo_b200_png_reduced *info, uint8_t *d_out,
                                    size_t out_stride, uint32_t *d_adler);

/* Lossy palette quantisation ahead of the filter: what encode_into does when PngOptions::quantization
 * selects it (src/png/mod.rs:469-511, QuantizationOptions :70-100).  Flags for the strategy word of
 * pixo_b200_png_quantize_filter* only (every other entry point keeps rejecting them):
 *   QUANTIZE_AUTO   QuantizationMode::Auto   quantise RGB/RGBA when should_quantize_auto says so
 *   QUANTIZE_FORCE  QuantizationMode::Force  quantise every RGB/RGBA image
 *   DITHER          QuantizationOptions::dithering (Floyd-Steinberg on RGB, alpha kept)
 * Neither mode flag is QuantizationMode::Off; both together are an error. */
#define PIXO_B200_PNG_QUANTIZE_AUTO 0x800u
#define PIXO_B200_PNG_QUANTIZE_FORCE 0x1000u
#define PIXO_B200_PNG_DITHER 0x2000u

/* Replaces encode_into's choice between quantize_image -> encode_indexed_into (src/png/mod.rs:469-511,
 * 1505-1701, 1814-1886) and the lossless reduction path (pixo_b200_png_reduce_filter, which frames that do
 * not quantise take with the same OPTIMIZE_ALPHA / REDUCE_* flags).  A quantised frame is described as
 * colour type 3, bit depth 8, bytes_per_pixel 1, row_bytes = width, effective colour type RGB; palette in
 * pixo's order (median-cut box order after k-means, or key order when the image has at most max_colors
 * histogram colours) and trns_len the length maybe_trim_transparency keeps (0: no tRNS).  Its 8-bit index
 * rows are filtered with the strategy encode_indexed_into uses (Adaptive, AdaptiveFast, MinSum and Bigrams
 * become None).  max_colors: QuantizationOptions::max_colors (a u16; above 256 acts as 256, 0 is legal).
 * palette (optional, RGBA, 1..256 entries): the palette pixo's median_cut_palette produced, mapped exactly
 * as quantize_image maps one (6-6-6 table, then the plain map or the dither).  Without it, an image whose
 * histogram samples hold more than 8192 colours returns PIXO_B200_ERR_UNSUPPORTED: pixo keeps the 8192
 * most frequent with an unstable sort whose tie order decides the palette and is not restated here.
 * out / out_len / adler32_out as pixo_b200_png_reduce_filter. */
int pixo_b200_png_quantize_filter(pixo_b200_ctx *ctx, const uint8_t *data, size_t data_len, uint32_t width,
                                  uint32_t height, uint32_t color_type, uint32_t strategy_and_flags,
                                  uint32_t max_colors, const uint8_t *palette, uint32_t palette_len,
                                  pixo_b200_png_reduced *info, uint8_t *out, size_t out_cap, size_t *out_len,
                                  uint32_t *adler32_out);
/* Batch of device-resident frames, as pixo_b200_png_reduce_filter_dev; a batch may mix frames that
 * quantise with frames that do not.  palettes (optional, HOST memory): n_images x 256 x 4 bytes with
 * palette_lens[i] entries for frame i, 0 = design it.  Any n_images: the quantised frames are mapped and
 * filtered in passes of a few thousand, so the context's scratch does not grow with the batch.  Returns
 * once info[] is valid. */
int pixo_b200_png_quantize_filter_dev(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride,
                                      uint32_t n_images, uint32_t width, uint32_t height, uint32_t color_type,
                                      uint32_t strategy_and_flags, uint32_t max_colors, const uint8_t *palettes,
                                      const uint32_t *palette_lens, pixo_b200_png_reduced *info, uint8_t *d_out,
                                      size_t out_stride, uint32_t *d_adler);

/* ---- resize ----------------------------------------------------------------------------- */

/* pixo::resize::ResizeAlgorithm, numbered as the wasm binding numbers it (src/wasm.rs:156-166) */
enum { PIXO_B200_RESIZE_NEAREST = 0, PIXO_B200_RESIZE_BILINEAR = 1, PIXO_B200_RESIZE_LANCZOS3 = 2 };

/* Replaces pixo::resize::resize_into — src/resize.rs:180-602: Nearest (:299-330), Bilinear (:333-389) and
 * separable Lanczos3 (:391-602, a u8 intermediate of src_height x dst_width pixels between the passes),
 * byte-identical, for Gray, GrayAlpha, RGB and RGBA (the output has the input's colour type).  Errors in
 * this order: PIXO_B200_ERR_INVALID_ARGUMENT for an unknown colour type or algorithm (resizeImage's
 * checks, src/wasm.rs:183-201), then resize_impl's (src/resize.rs:205-250): a zero source, then a zero
 * destination dimension PIXO_B200_ERR_INVALID_DIMENSIONS; any dimension above 1 << 24
 * PIXO_B200_ERR_IMAGE_TOO_LARGE; data_len != src_width*src_height*bpp PIXO_B200_ERR_INVALID_DATA_LENGTH.
 * Then out_cap below dst_width*dst_height*bpp returns PIXO_B200_ERR_OUTPUT_TOO_SMALL with *out_len = the
 * size needed.  Where f32 rounding makes pixo's Bilinear index one pixel past the source (a side above
 * 2^23; pixo panics there) the last pixel is read. */
int pixo_b200_resize(pixo_b200_ctx *ctx, const uint8_t *data, size_t data_len, uint32_t src_width,
                     uint32_t src_height, uint32_t dst_width, uint32_t dst_height, uint32_t color_type,
                     uint32_t algorithm, uint8_t *out, size_t out_cap, size_t *out_len);
/* Batch of device-resident frames of one geometry, asynchronous on the context's stream: frame i at
 * d_src + i*src_stride (src_width*src_height*bpp bytes, rows packed) -> d_dst + i*dst_stride.  Any
 * alignment and any n_images.  Frames must not overlap: with n_images > 1, src_stride below a source
 * frame returns PIXO_B200_ERR_INVALID_DATA_LENGTH and dst_stride below a destination frame
 * PIXO_B200_ERR_OUTPUT_TOO_SMALL.  Nothing is launched unless the call is valid.  Lanczos3's weight tables
 * are computed on the host and uploaded on the stream from the context's pinned buffers; its intermediate stays within 256 MiB of device scratch (larger
 * frames go in bands of destination rows).  The output is packed pixels, what
 * pixo_b200_jpeg_encode_dev and pixo_b200_png_filter_dev read. */
int pixo_b200_resize_dev(pixo_b200_ctx *ctx, const uint8_t *d_src, size_t src_stride, uint32_t n_images,
                         uint32_t src_width, uint32_t src_height, uint32_t dst_width, uint32_t dst_height,
                         uint32_t color_type, uint32_t algorithm, uint8_t *d_dst, size_t dst_stride);
/* Lanczos3's contribution table for one axis (precompute_contributions, src/resize.rs:416-456), as the
 * resizers use it: destination index d reads source indices start[d] .. start[d]+count[d]-1 with weights
 * weights[offset[d] ..], normalised f32 computed with pixo's own sinf (the libm port of musl's, which the
 * wasm build runs).  *n_weights receives the total; start/count/offset (dst_size entries each) and weights
 * may be NULL; weights_cap below the total returns PIXO_B200_ERR_OUTPUT_TOO_SMALL after the other
 * arrays are written.  Host-only, no device needed. */
int pixo_b200_resize_weights(uint32_t src_size, uint32_t dst_size, uint32_t *start, uint32_t *count,
                             uint64_t *offset, float *weights, size_t weights_cap, size_t *n_weights);

/* ---- baseline JPEG decoding ------------------------------------------------------------ */

/* Replaces pixo::decode::decode_jpeg — src/decode/jpeg.rs:214-740 with bit_reader.rs:141-256 and idct.rs — pixel for
 * pixel, on every input it accepts: truncated, corrupt and RSTn-bearing scans included (a read failure ends the scan,
 * and the blocks never stored stay 0 in the component planes, as there).  Errors are pixo's, decided in pixo's order:
 * PIXO_B200_ERR_INVALID_DECODE (Error::InvalidDecode) or PIXO_B200_ERR_UNSUPPORTED_DECODE (Error::UnsupportedDecode,
 * e.g. "progressive JPEG not supported"), with pixo's Display text ("Decode error: ...", "Unsupported: ...") as the
 * error string.  One difference: an SOS with no components before any SOF0, on which pixo panics, is
 * PIXO_B200_ERR_INVALID_DECODE ("SOS with no frame components").  The output is packed Gray (color_type
 * PIXO_B200_GRAY) or RGB (PIXO_B200_RGB), width * height * (1 or 3) bytes. */

/* Host only, no device needed: the geometry and colour type decode_jpeg would return, or its error (the string is
 * pixo_b200_last_error(NULL) on this thread).  Returns 0 exactly when decode_jpeg returns Ok.  width, height and
 * color_type may be NULL. */
int pixo_b200_jpeg_decode_info(const uint8_t *data, size_t len, uint32_t *width, uint32_t *height,
                               uint32_t *color_type);
/* One file to host memory.  pixels_cap below the frame returns PIXO_B200_ERR_OUTPUT_TOO_SMALL with the geometry
 * set.  Waits for the device. */
int pixo_b200_jpeg_decode(pixo_b200_ctx *ctx, const uint8_t *data, size_t len, uint8_t *pixels, size_t pixels_cap,
                          uint32_t *width, uint32_t *height, uint32_t *color_type);
/* n files in host memory -> decoded frames in device memory: file i's frame at d_out + out_offsets[i] (the caller
 * sizes them with pixo_b200_jpeg_decode_info; any byte alignment).  status[i] receives 0 or file i's error code
 * before the call returns; a file that fails is skipped and nothing is written for it.  The headers are parsed on
 * the host; the scans are uploaded and decoded on the context's stream, and the call returns with that work queued
 * (the files may be reused at once).  Every file's scan is decoded sequentially by one GPU thread; the files of a
 * batch run in parallel, one per warp.  3 launches per pass (scan, IDCT, colour); passes hold at most 65 536 files
 * and about 1 GiB of device scratch.  A file needs 192 bytes of scratch per 8x8 block of its component planes (the
 * frame as its SOF0 declares it, rounded up to whole MCUs, i.e. about 3 bytes per sample) plus its scan bytes; a
 * file larger than the pass limit goes alone, and one larger than the device can hold returns PIXO_B200_ERR_OOM
 * (frames of earlier passes may then have been written).  Null arrays, or a null d_out with n > 0, return
 * PIXO_B200_ERR_INVALID_ARGUMENT before anything is read. */
int pixo_b200_jpeg_decode_to_device(pixo_b200_ctx *ctx, const uint8_t *const *files, const size_t *lens, uint32_t n,
                                    uint8_t *d_out, const size_t *out_offsets, int32_t *status);

/* ---- PNG decoding ------------------------------------------------------------------------- */

/* Replaces pixo::decode::decode_png — src/decode/png.rs:101-626 with inflate.rs:46-513 and bit_reader.rs:10-135 —
 * pixel for pixel, with pixo's error for every file it refuses, decided in pixo's order: the chunk walk (truncated
 * chunk, then each chunk's CRC, IHDR length and colour type), the checks after it, the zlib header, inflate with
 * pixo's Huffman tables as from_lengths builds them (no completeness check; later symbols win the 9-bit lookup),
 * Adler-32 over every byte produced, the size, the first row with an invalid filter type, then a missing PLTE.
 * Errors: PIXO_B200_ERR_INVALID_DECODE (Error::InvalidDecode), PIXO_B200_ERR_UNSUPPORTED_DECODE (Adam7, preset
 * dictionary), PIXO_B200_ERR_INVALID_DIMENSIONS (a zero side) and PIXO_B200_ERR_IMAGE_TOO_LARGE (a side above
 * 2^24), with pixo's Display text as the error string.  The frame is packed: Gray, GrayAlpha, RGB or RGBA as pixo
 * returns it (16-bit samples keep their high byte, sub-8-bit gray is bit-replicated, tRNS is ignored for gray and
 * RGB, and indexed is RGBA only when tRNS holds a value other than 255), width * height * channels bytes: the layout
 * pixo_b200_resize_dev and the device encoders read.  A chunk type that is not valid UTF-8 is shown as pixo shows
 * it (U+FFFD); a NUL in it ends the C string. */

/* Host only, no device needed: the geometry and colour type decode_png would return, or the error it decides
 * before inflating (the string is pixo_b200_last_error(NULL) on this thread).  One exception: the IDAT chunks' CRCs
 * are checked only in a file the host refuses for another reason, so a file whose only fault is an IDAT CRC (or is
 * found while inflating) returns 0 here.  *producible is 0 when the IDAT data cannot produce the frame's rows
 * (height * (1 + scanline bytes) above 1032 bytes per DEFLATE byte plus 65 535: every symbol takes a bit, a 258-byte
 * match two), so that decoding is certain to fail and no frame need be allocated for the file.  width, height,
 * color_type and producible may be NULL. */
int pixo_b200_png_decode_info(const uint8_t *data, size_t len, uint32_t *width, uint32_t *height,
                              uint32_t *color_type, int32_t *producible);
/* One file to host memory.  pixels_cap below the frame returns PIXO_B200_ERR_OUTPUT_TOO_SMALL with the geometry
 * set, except for a file that is not producible (see above): it is decoded for its error alone, with no frame
 * allocated and no output capacity needed.  Waits for the device. */
int pixo_b200_png_decode(pixo_b200_ctx *ctx, const uint8_t *data, size_t len, uint8_t *pixels, size_t pixels_cap,
                         uint32_t *width, uint32_t *height, uint32_t *color_type);
/* n files in host memory -> decoded frames in device memory: file i's frame at d_out + out_offsets[i] (sized with
 * pixo_b200_png_decode_info; any byte alignment).  status[i] receives 0 or file i's error code; a file that fails
 * is skipped and nothing is written for it.  The chunks are walked on the host; the IDAT payloads are uploaded and
 * decoded on the context's stream, and the call waits for the device once per pass, so status is final and the
 * frames are written (in stream order) when it returns.  Per pass: k_png_crc (every IDAT chunk's CRC-32, over many
 * CTAs), k_png_inflate (one warp per zlib stream, longest first), k_png_unfilter (a wavefront of 32-row groups,
 * writing 8-bit Gray / GrayAlpha / RGB / RGBA frames directly) and, when the pass holds sub-8-bit, 16-bit or indexed
 * files, k_png_expand: 3 or 4 launches.  Passes hold at most 65 536 files and about 1 GiB of device scratch; a file
 * needs its IDAT bytes plus min(expected size, 1032 * DEFLATE bytes + 65 535) for its inflated rows (a header that
 * claims more than its stream can produce costs only what the stream can produce), and one larger than the pass
 * limit goes alone; one larger than the device can hold returns PIXO_B200_ERR_OOM (frames of earlier passes may
 * then have been written).  Null arrays, or a null d_out with n > 0, return PIXO_B200_ERR_INVALID_ARGUMENT before
 * anything is read. */
int pixo_b200_png_decode_to_device(pixo_b200_ctx *ctx, const uint8_t *const *files, const size_t *lens, uint32_t n,
                                   uint8_t *d_out, const size_t *out_offsets, int32_t *status);

/* Replaces compress::adler32::adler32 — src/compress/adler32.rs:11-47 (dispatch
 * src/simd/mod.rs:72-90).  Host buffer in, checksum out. */
int pixo_b200_adler32(pixo_b200_ctx *ctx, const uint8_t *data, size_t len, uint32_t *out);
/* device buffer; result written to d_out (device u32), asynchronous */
int pixo_b200_adler32_dev(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t len, uint32_t *d_out);

/* Replaces compress::deflate::deflate_zlib_packed (src/compress/deflate.rs:1074) at levels 1-9: the zlib stream
 * pixo writes for `data`, byte for byte (one DEFLATE block, stored, fixed or dynamic, as compress_packed_zlib
 * chooses).  A level outside 1-9 returns PIXO_B200_ERR_INVALID_COMPRESSION_LEVEL ("Invalid compression level {n}:
 * must be 1-9", pixo's png::encode check).  *out_len receives the stream's length; when it exceeds out_cap the call
 * returns PIXO_B200_ERR_OUTPUT_TOO_SMALL and writes nothing.  Inputs of 2^31 bytes or more (beyond pixo's i32
 * positions) return PIXO_B200_ERR_UNSUPPORTED. */
int pixo_b200_deflate_zlib(pixo_b200_ctx *ctx, const uint8_t *data, size_t len, uint32_t level, uint8_t *out,
                           size_t out_cap, size_t *out_len);
/* n device streams, stream i at d_streams + i * stride, lens[i] bytes (host array), each to its slot at
 * d_out + i * out_cap_each.  out_lens[i] and status[i] (host arrays) receive each stream's length and 0, or
 * PIXO_B200_ERR_OUTPUT_TOO_SMALL for a stream longer than its slot, which is then left untouched.  Streams are
 * parsed one warp each, longest first, in passes of about 1 GiB of token scratch (a longer stream goes alone); the
 * call waits once per pass for the symbol counts and for the pass's coding, and returns with the work done.  Level
 * and length errors as pixo_b200_deflate_zlib, before anything is launched; null arrays or d_out return
 * PIXO_B200_ERR_INVALID_ARGUMENT, and a stream longer than stride in a batch of more than one returns
 * PIXO_B200_ERR_INVALID_DATA_LENGTH.  Named like pixo_b200_png_decode_to_device, not `_dev`: it takes host arrays and
 * waits for the device before it returns, where the `_dev` calls are the stream-ordered ones listed above. */
int pixo_b200_deflate_zlib_on_device(pixo_b200_ctx *ctx, const uint8_t *d_streams, size_t stride, const size_t *lens,
                                     uint32_t n, uint32_t level, uint8_t *d_out, size_t out_cap_each,
                                     size_t *out_lens, int32_t *status);

/* ---- whole PNG files ---------------------------------------------------------------------- */

/* PngOptions::optimal_compression (pixo's max preset).  Accepted only by the two encode calls, which refuse it. */
#define PIXO_B200_PNG_OPTIMAL_COMPRESSION 0x4000u

/* Replaces pixo::png::encode_into (src/png/mod.rs:437-630, and encode_indexed_into :1814-1886 for frames that
 * quantise) at pixo's fast and balanced presets: one host image -> one complete PNG file in `out`, byte for byte
 * pixo's (the default, parallel build's filter choice).  strategy_and_flags, max_colors and palette / palette_len
 * mean what they mean for pixo_b200_png_quantize_filter: without a QUANTIZE flag the frame takes the reduction path,
 * and without a REDUCE flag either it is only filtered (preset 0).  compression_level: PngOptions::compression_level,
 * the DEFLATE level (pixo_b200_deflate_zlib).  The file is the signature, IHDR, PLTE and tRNS when the frame has a
 * palette (a quantised frame's tRNS trimmed as pixo trims it), the zlib stream in IDAT chunks of 256 KiB, and IEND.
 * pixo's strip_metadata has no flag: pixo never writes tEXt, zTXt, iTXt or tIME, so on its own output
 * strip_metadata_chunks changes nothing.  Errors in pixo's order, before anything is launched: a level outside 1-9
 * PIXO_B200_ERR_INVALID_COMPRESSION_LEVEL; then pixo_b200_png_quantize_filter's checks (dimensions, size above 2^24,
 * colour type, flags, AUTO with FORCE, max_colors, the palette, data_len); then PIXO_B200_PNG_OPTIMAL_COMPRESSION
 * returns PIXO_B200_ERR_UNSUPPORTED.  A filtered stream of 2^31 bytes or more returns PIXO_B200_ERR_UNSUPPORTED;
 * more than 8192 sampled colours without a palette returns it as pixo_b200_png_quantize_filter does.  *out_len
 * receives the file's length; above out_cap the call returns PIXO_B200_ERR_OUTPUT_TOO_SMALL and writes nothing.
 * The checks need no context: with ctx NULL they run in the same order, and a call that passes them returns
 * PIXO_B200_ERR_INVALID_ARGUMENT ("ctx is null"). */
int pixo_b200_png_encode(pixo_b200_ctx *ctx, const uint8_t *data, size_t data_len, uint32_t width, uint32_t height,
                         uint32_t color_type, uint32_t strategy_and_flags, uint32_t compression_level,
                         uint32_t max_colors, const uint8_t *palette, uint32_t palette_len,
                         uint8_t *out, size_t out_cap, size_t *out_len);

/* n device frames of one geometry (frame i at d_data + i*in_stride) -> n complete PNG files, file i in the slot at
 * d_out + i*out_cap_each, any byte alignment.  palettes / palette_lens (HOST memory, optional) and info (optional,
 * n entries) as pixo_b200_png_quantize_filter_dev.  out_lens[i] and status[i] (host arrays) receive each file's
 * length and 0; the length is known before anything is written, so a slot too small gets
 * PIXO_B200_ERR_OUTPUT_TOO_SMALL, keeps the length it needs in out_lens[i], and is left untouched.  A frame whose
 * filtered stream is 2^31 bytes or more gets PIXO_B200_ERR_UNSUPPORTED (out_lens[i] 0) and an untouched slot; the
 * other frames are still written.  Checks as pixo_b200_png_encode, with in_stride below a frame in a batch of more
 * than one PIXO_B200_ERR_INVALID_DATA_LENGTH, and input frames overlapping the output slots
 * PIXO_B200_ERR_INVALID_ARGUMENT, all before anything is launched.  The frames go in passes whose unreduced
 * filtered streams total about 1 GiB (a larger frame goes alone), on the context's stream: the filter stage
 * (pixo_b200_png_quantize_filter_dev's launches), DEFLATE (pixo_b200_deflate_zlib_on_device's: k_lz77 and
 * k_deflate_emit per pass of its own), then k_png_idat (the zlib streams into their IDAT chunks with each chunk's
 * CRC-32, in 4 KiB pieces over many CTAs) and k_png_idat_finish (the small chunks, the CRCs and IEND) when the pass
 * writes a file.  The call waits for the device once per stage and pass and returns with every file written.  A
 * frame that quantises with more than 8192 sampled colours and no palette fails the call with
 * PIXO_B200_ERR_UNSUPPORTED, as pixo_b200_png_quantize_filter_dev; files of earlier passes may then have been
 * written.  The extra scratch is the pass's unreduced filtered streams and their stored-block zlib bounds. */
int pixo_b200_png_encode_on_device(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride, uint32_t n_images,
                                   uint32_t width, uint32_t height, uint32_t color_type, uint32_t strategy_and_flags,
                                   uint32_t compression_level, uint32_t max_colors, const uint8_t *palettes,
                                   const uint32_t *palette_lens, uint8_t *d_out, size_t out_cap_each,
                                   size_t *out_lens, int32_t *status, pixo_b200_png_reduced *info);

#ifdef __cplusplus
}
#endif
#endif /* PIXO_B200_H */
