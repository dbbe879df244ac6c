// jpeg_host.hpp — host half of the JPEG path: quantisation tables, headers, Huffman table
// construction and the baseline entropy coder that consumes the GPU's coefficient arrays.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <vector>

namespace pixo {

struct FrameGeometry {
    uint32_t width = 0, height = 0;
    uint32_t color_type = 2;   // PIXO_B200_RGB
    uint32_t subsampling = 1;  // PIXO_B200_S420
    uint32_t mcus_x = 0, mcus_y = 0;
    uint32_t y_per_mcu = 1;    // 4 for 4:2:0, else 1
    bool has_chroma = true;
    size_t ny = 0, nc = 0;     // blocks per component array
    size_t total_mcus() const { return (size_t)mcus_x * mcus_y; }
};
FrameGeometry make_geometry(uint32_t w, uint32_t h, uint32_t color_type, uint32_t subsampling);

// with_quality, src/jpeg/quantize.rs:42-89
void quant_tables(int quality, uint8_t lum_zz[64], uint8_t chr_zz[64], float lum[64],
                  float chr[64]);

struct HuffTables {
    // order: dc_lum, dc_chrom, ac_lum, ac_chrom (DHT ids 0x00,0x01,0x10,0x11)
    uint8_t bits[4][16];
    uint8_t vals[4][256];
    int nvals[4];
    uint16_t code[4][256];
    uint8_t len[4][256];
};
void huff_standard(HuffTables &t);
// HuffmanTables::optimized_from_counts, src/jpeg/huffman.rs:167-205.  false == None.
bool huff_from_histogram(const uint64_t hist[536], bool has_chroma, HuffTables &t);
// Tables from DHT data: per table 16 counts + 256 values, in the order dc_lum, dc_chrom, ac_lum, ac_chrom.
// Each table must hold at most 256 values (prog_tables checks that).
void huff_from_dht(const uint8_t dht[1088], HuffTables &t);
// The standard tables (huff_standard) as DHT data
const uint8_t *dht_standard();

// SOI..SOS (src/jpeg/mod.rs:395-430,449-648).  Returns bytes written (<= 1024).
size_t write_headers(uint8_t *out, const FrameGeometry &g, const uint8_t lum_zz[64],
                     const uint8_t chr_zz[64], const HuffTables &t, uint32_t restart_interval);

// Progressive files (encode_into with options.progressive, src/jpeg/mod.rs:395-410): SOI..DRI with SOF2,
// and the SOS of scan 0..6 of simple_progressive_script (write_sos_progressive, :650-683: one component,
// table selector 0x00 for Y and 0x11 for chroma, Ah = Al = 0; gray frames get the chroma SOS too).
size_t write_headers_progressive(uint8_t *out, const FrameGeometry &g, const uint8_t lum_zz[64],
                                 const uint8_t chr_zz[64], const HuffTables &t, uint32_t restart_interval);
size_t write_sos_progressive(uint8_t *out, int scan);   // 10 bytes

// encode_scan (src/jpeg/mod.rs:1408-1563) over precomputed coefficient arrays (natural or
// zig-zag order), multi-threaded over MCU segments; byte-identical to the sequential
// reference.  Returns bytes written, or (size_t)-1 when `cap` is too small.
size_t entropy_encode_scan(const int16_t *y, const int16_t *cb, const int16_t *cr,
                           const FrameGeometry &g, const HuffTables &t,
                           uint32_t restart_interval, bool zigzag_in, uint8_t *out, size_t cap,
                           int threads);

// histogram of a frame on the host (used by the host-only entropy API)
void host_histogram(const int16_t *y, const int16_t *cb, const int16_t *cr,
                    const FrameGeometry &g, uint32_t restart_interval, uint64_t hist[536],
                    const int *seed = nullptr);

// A frame tiled over several GPUs (SURVEY.md section 8e): one band's raw bit string and its splice
// into the frame's scan (host versions of k_huff<RAW> / k_seg_*).
uint64_t band_encode_raw(const int16_t *y, const int16_t *cb, const int16_t *cr, const FrameGeometry &g,
                         const HuffTables &t, const int seed[3], uint8_t *out, size_t cap, uint32_t *tail7);
size_t band_splice(const uint8_t *raw, uint64_t nbits, uint32_t phase, uint32_t tail_in, bool last,
                   uint8_t *out, size_t cap);

// true when every AC coefficient has category <= 10 and every DC difference (previous block of
// the same component, reset at restart boundaries; `seed` before block 0) category <= 11
bool coefficients_in_range(const int16_t *blocks, size_t nblocks, uint32_t restart_interval, uint32_t per_mcu,
                           int seed = 0);

// run fn(job) for job in [0, n) on up to `threads` std::threads
void parallel_jobs(int n, int threads, void (*fn)(int, void *), void *arg);

}  // namespace pixo
