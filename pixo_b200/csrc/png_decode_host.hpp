// png_decode_host.hpp — host half of the PNG decoder (pixo::decode::decode_png): the chunk walk with pixo's checks,
// messages and order, the zlib header, and the per-file records the kernels read (png_decode_host.cpp).  The IDAT
// CRCs, inflate, unfiltering and sample expansion run on the device (png_decode.cu).
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "decode_host.hpp"
#include "png_host.hpp"   // PIXO_HOST_DEVICE

namespace pixo {

// The CRC-32 of PNG chunks (reflected 0xEDB88320).  crc32_update runs the register over bytes without the final
// inversion; crc32_shift(r, n) is the register r advanced over n zero bytes, so that the register over A || B
// from any start s is crc32_shift(reg(s, A), |B|) ^ reg(0, B).  k_png_crc combines its pieces with crc32_shift.
uint32_t crc32_update(uint32_t reg, const uint8_t *p, size_t n);

// a * b modulo the CRC polynomial, bit 31 holding x^0 (the reflected order the register uses)
PIXO_HOST_DEVICE inline uint32_t crc_mulmod(uint32_t a, uint32_t b)
{
    uint32_t p = 0;
    for (uint32_t m = 1u << 31; m; m >>= 1) {
        if (a & m) p ^= b;
        b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}

PIXO_HOST_DEVICE inline uint32_t crc32_shift(uint32_t reg, uint64_t nbytes)
{
    // x^(8 * nbytes) by squaring: x2n holds x^(2^k) for the bits of 8 * nbytes
    uint32_t x2n = 1u << 30, f = 1u << 31;   // x^1, x^0
    for (int k = 0; k < 3; ++k) x2n = crc_mulmod(x2n, x2n);
    for (; nbytes; nbytes >>= 1) {
        if (nbytes & 1) f = crc_mulmod(x2n, f);
        x2n = crc_mulmod(x2n, x2n);
    }
    return crc_mulmod(f, reg);
}

#ifdef __CUDACC__
// The pieces of a chunk's CRC-32 on the device (k_png_crc checks them, k_png_idat writes them): the CTA fills the
// 256-entry table in shared memory (a __syncthreads must follow), then a thread runs the register over its piece.
__device__ __forceinline__ void crc32_table(uint32_t *tab)
{
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = i;
        for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ 0xEDB88320u : c >> 1;
        tab[i] = c;
    }
}

__device__ __forceinline__ uint32_t crc32_piece(const uint32_t *tab, const uint8_t *__restrict__ p, uint64_t n)
{
    uint32_t reg = 0;
    for (uint64_t i = 0; i < n; ++i) reg = (reg >> 8) ^ tab[(reg ^ __ldg(p + i)) & 0xFF];
    return reg;
}
#endif

// One file after the host's share of decode_png (src/decode/png.rs:101-263 and the zlib header of
// inflate_zlib_with_size, src/decode/inflate.rs:294-320)
struct PdecParsed {
    DecodeStatus status;
    uint32_t width = 0, height = 0;
    uint8_t depth = 0, ctype = 0;   // IHDR bit depth and PNG colour type (0, 2, 3, 4, 6)
    bool has_plte = false;
    std::vector<uint8_t> plte, trns;
    // IDAT chunks met before the walk stopped: byte offset of each payload in the file, its length and stored CRC
    std::vector<uint64_t> idat_off;
    std::vector<uint32_t> idat_len, idat_crc;
    uint64_t idat_total = 0;
    uint64_t expected = 0;      // calculate_expected_size: height * (1 + scanline bytes)
    uint64_t sb = 0;            // scanline bytes (without the filter byte)
    uint32_t bpp = 0;           // the unfilter's bytes per pixel (1 for indexed and sub-8-bit gray)
    uint32_t out_channels = 0;  // of the decoded frame
    uint32_t out_ct = 0;        // pixo_b200 colour type of the decoded frame
    uint64_t out_bytes() const { return (uint64_t)width * height * out_channels; }
    // the most bytes the DEFLATE data (IDAT bytes less the 2-byte header and the 4-byte Adler-32) can produce:
    // every symbol takes at least one bit, so a match of 258 bytes takes at least 2
    uint64_t produce_bound() const { return 1032 * (idat_total - 6) + 65535; }
    // false when the stream cannot produce the rows: decode_png is then certain to fail (size mismatch, or an
    // earlier inflate error), and no frame need be allocated for the file
    bool producible() const { return expected <= produce_bound(); }
    uint64_t scratch() const { return producible() ? expected : produce_bound(); }
    // frames of 8-bit Gray, GrayAlpha, RGB and RGBA are the unfiltered rows themselves
    bool direct() const { return depth == 8 && ctype != 3; }
};

// Everything decode_png decides before it inflates: p.status is clear when the file reaches the DEFLATE data.  The
// IDAT CRCs are left to the device, except in a file refused here: that one is walked again with them checked, each
// at its place in the walk, so that an IDAT chunk that fails before the error found is reported first, as in pixo.
void parse(const uint8_t *data, size_t len, PdecParsed &p);

}  // namespace pixo

struct pixo_b200_ctx;
namespace pixo {
// Decodes n parsed files (all without error) on the context's stream: file i's frame to d_out + out_off[i].  data[i]
// is the file.  Waits for the device once per pass and sets res[i] to what the device decided: clear, or the first
// failure in pixo's order after the host's checks.  Passes of bounded scratch.
int launch_decode(pixo_b200_ctx *ctx, const PdecParsed *const *files, const uint8_t *const *data, uint32_t n,
                  const uint64_t *out_off, uint8_t *d_out, DecodeStatus *res);
}  // namespace pixo
