// jpeg_decode_host.hpp — host half of the baseline JPEG decoder (pixo::decode::decode_jpeg): marker parsing with
// pixo's checks and messages, the decode tables, and the entropy range (jpeg_decode_host.cpp).  The kernels are in
// jpeg_decode.cu.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "decode_host.hpp"

namespace pixo {

// HuffmanTable as HuffmanTable::build makes it (src/decode/jpeg.rs:77-147): the 8-bit lookup (value | length << 8,
// 0: take the slow path), max_code / val_offset per length, and where its values start in the values area
struct JdecHuff {
    uint16_t lookup[256];
    int32_t max_code[17];
    int32_t val_offset[17];
    uint32_t nvalues;
    uint32_t values;   // byte offset into the pass's values area
};

// One file of a decode pass as the kernels read it
struct JdecFile {
    uint64_t src, src_len;        // the entropy bytes: offset into the pass's byte area, length (find_entropy_end)
    uint64_t coef[3];             // each component's coefficient plane: offset in blocks into the coefficient area
    uint64_t plane[3];            // each component's u8 plane: byte offset into the plane area
    uint64_t plane_len[3];        // bytes of each plane
    uint64_t out;                 // byte offset of the decoded frame in the caller's buffer
    uint32_t width, height, mcu_w, mcu_h;
    uint32_t ncomp, restart, max_h, max_v, bpm;   // bpm: blocks per MCU
    uint32_t h[3], v[3], first[3];                // sampling factors; a component's first block within the MCU
    uint32_t dc[3], ac[3];                        // the components' tables: index into the pass's table area
    alignas(16) uint16_t quant[3][64];            // the components' quantisation tables, zig-zag order
};

// A file after its headers, up to the first SOS
struct JdecParsed {
    DecodeStatus status;
    uint32_t width = 0, height = 0, ncomp = 0, restart = 0, max_h = 1, max_v = 1;
    uint8_t h[3] = {}, v[3] = {}, q[3] = {}, dc[3] = {}, ac[3] = {};
    uint16_t quant[4][64] = {};
    JdecHuff tab[8] = {};                  // DC 0-3, AC 4-7; `values` indexes vals[i]
    std::vector<uint8_t> vals[8];
    size_t entropy = 0, entropy_len = 0;   // the scan's bytes in the file
    uint32_t out_ct = 0;                   // pixo_b200 colour type of the decoded frame: Gray or RGB
    uint32_t mcu_w() const { return (width + max_h * 8 - 1) / (max_h * 8); }
    uint32_t mcu_h() const { return (height + max_v * 8 - 1) / (max_v * 8); }
    uint64_t plane_w(int c) const { return (uint64_t)mcu_w() * h[c] * 8; }
    uint64_t plane_h(int c) const { return (uint64_t)mcu_h() * v[c] * 8; }
    uint64_t blocks() const;          // all components' blocks
    uint64_t out_bytes() const { return (uint64_t)width * height * (ncomp == 1 ? 1 : 3); }
    bool producible() const { return true; }   // every file that parses has its frame decoded
};

// Parses data as JpegDecoder::decode does up to the scan (src/decode/jpeg.rs:214-484), with pixo's errors in
// pixo's order, and finds the scan's entropy range (find_entropy_end, :653-671)
void parse(const uint8_t *data, size_t len, JdecParsed &p);
size_t jdec_entropy_end(const uint8_t *data, size_t len);

}  // namespace pixo

struct pixo_b200_ctx;
namespace pixo {
// Decodes n parsed files (all without error) on the context's stream: file i's frame to d_out + out_off[i], packed
// Gray or RGB.  data[i] is the file; its scan's bytes are copied out before the call returns.  Passes of bounded
// scratch.  res is never written: every error of decode_jpeg is decided on the host.
int launch_decode(pixo_b200_ctx *ctx, const JdecParsed *const *files, const uint8_t *const *data, uint32_t n,
                  const uint64_t *out_off, uint8_t *d_out, DecodeStatus *res);
}  // namespace pixo
