// png_encode.cu — whole PNG files on the device: pixo::png::encode_into at presets 0 and 1 (src/png/mod.rs:437-630,
// and encode_indexed_into :1814-1886 for frames that quantise), byte-identical, for batches of device frames.  The
// frames go in passes of about 1 GiB of unreduced filtered bytes; each pass runs
//   the filter stage    png_quantize_filter (png_quantize.cu) into the pass's filtered streams, info[] on the host
//   DEFLATE             deflate_zlib (png_deflate.cu) at the compression level into the pass's zlib streams, with
//                       their exact lengths on the host
//   host                each file's exact length and status, and its signature, IHDR, PLTE and tRNS with their
//                       CRC-32s, packed into one upload with the starting words of the IDAT CRCs
//   k_png_idat          one thread per 4 KiB piece of a zlib stream: its warp copies the pieces into their IDAT
//                       payloads in the caller's slots; the thread runs the CRC register over its piece and folds
//                       it into its chunk's word with crc32_shift, as k_png_crc checks them (png_decode.cu)
//   k_png_idat_finish   one warp per file: the small chunks, each IDAT chunk's length, type and CRC, and IEND
// so a pass adds the stage's launches, DEFLATE's two per internal pass and, when it writes a file, these two.
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "decode_host.hpp"
#include "png_decode_host.hpp"

namespace pixo {

namespace {

constexpr uint64_t kIdatChunk = 256 * 1024;   // write_idat_chunks' chunk size (src/png/mod.rs:606-616)
constexpr uint32_t kIdatPiece = 4096;          // bytes a k_png_idat thread copies and runs the register over
constexpr int kIdatThreads = 256;
constexpr uint64_t kMaxStream = (uint64_t)1 << 31;   // deflate_zlib's limit: pixo's i32 positions

// One file of a pass as the container kernels read it
struct IdatFile {
    const uint8_t *z;     // its zlib stream (16-byte aligned, readable up to the next multiple of 16)
    uint8_t *dst;         // the caller's slot
    uint64_t zlen;
    uint64_t pre;         // signature, IHDR, PLTE and tRNS: offset into the pass's prefix bytes
    uint32_t pre_len;
    uint32_t chunk0;      // its first IDAT chunk's CRC word
};

__device__ __forceinline__ uint8_t *payload_at(const IdatFile &F, uint64_t at)
{
    return F.dst + F.pre_len + at / kIdatChunk * (kIdatChunk + 12) + 8 + at % kIdatChunk;
}

__global__ void __launch_bounds__(kIdatThreads)
k_png_idat(const IdatFile *__restrict__ files, const uint64_t *__restrict__ piece_prefix, uint32_t n, uint64_t npieces,
           uint32_t *__restrict__ acc)
{
    __shared__ uint32_t tab[256];
    crc32_table(tab);
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, g0 = g - lane;
    const uint32_t f = g < npieces ? item_of(piece_prefix, n, g) : 0;
    // the warp's pieces, one after the other: 16-byte loads from the stream, byte stores at any alignment
    for (uint32_t j = 0; j < 32 && g0 + j < npieces; ++j) {
        const IdatFile F = files[__shfl_sync(~0u, f, j)];
        const uint64_t at = (g0 + j - __ldg(piece_prefix + __shfl_sync(~0u, f, j))) * kIdatPiece;
        const uint32_t len = (uint32_t)min((uint64_t)kIdatPiece, F.zlen - at);
        uint8_t *d = payload_at(F, at);
        for (uint32_t v = lane; 16 * v < len; v += 32) {
            const uint4 q = __ldg(reinterpret_cast<const uint4 *>(F.z + at) + v);
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
            const uint32_t e = min(16u, len - 16 * v);
#pragma unroll
            for (uint32_t b = 0; b < 16; ++b)
                if (b < e) d[16 * v + b] = (uint8_t)(w[b / 4] >> (8 * (b % 4)));
        }
    }
    if (g >= npieces) return;
    const IdatFile F = files[f];
    const uint64_t at = (g - __ldg(piece_prefix + f)) * kIdatPiece;
    const uint64_t k = at / kIdatChunk, clen = min(kIdatChunk, F.zlen - k * kIdatChunk);
    const uint64_t len = min((uint64_t)kIdatPiece, F.zlen - at);
    const uint32_t reg = crc32_piece(tab, F.z + at, len);
    atomicXor(acc + F.chunk0 + k, crc32_shift(reg, clen - at % kIdatChunk - len));
}

__device__ __forceinline__ void put_be32(uint8_t *p, uint32_t v)
{
    p[0] = (uint8_t)(v >> 24), p[1] = (uint8_t)(v >> 16), p[2] = (uint8_t)(v >> 8), p[3] = (uint8_t)v;
}

// acc holds each chunk's register over "IDAT" and its payload once k_png_idat has run; the CRC is its inversion
__global__ void __launch_bounds__(kIdatThreads)
k_png_idat_finish(const IdatFile *__restrict__ files, uint32_t n, const uint8_t *__restrict__ pre,
                  const uint32_t *__restrict__ acc)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n) return;
    const IdatFile F = files[i];
    for (uint32_t b = lane; b < F.pre_len; b += 32) F.dst[b] = pre[F.pre + b];
    const uint64_t nch = (F.zlen + kIdatChunk - 1) / kIdatChunk;
    for (uint64_t k = lane; k < nch; k += 32) {
        const uint64_t clen = min(kIdatChunk, F.zlen - k * kIdatChunk);
        uint8_t *c = payload_at(F, k * kIdatChunk) - 8;
        put_be32(c, (uint32_t)clen);
        put_be32(c + 4, 0x49444154u);   // "IDAT"
        put_be32(c + 8 + clen, acc[F.chunk0 + k] ^ 0xFFFFFFFFu);
    }
    // IEND: length 0, "IEND", CRC AE 42 60 82
    const uint64_t kIend0 = 0x444E454900000000ull, kIend1 = 0x826042AEull;
    if (lane < 12)
        F.dst[F.pre_len + F.zlen + 12 * nch + lane] = (uint8_t)(lane < 8 ? kIend0 >> (8 * lane) : kIend1 >> (8 * (lane - 8)));
}

// write_chunk (src/png/chunk.rs:10) of a small chunk, on the host
void put_chunk(std::vector<uint8_t> &out, const char *type, const uint8_t *data, size_t len)
{
    const uint8_t be[4] = {(uint8_t)(len >> 24), (uint8_t)(len >> 16), (uint8_t)(len >> 8), (uint8_t)len};
    out.insert(out.end(), be, be + 4);
    const size_t t = out.size();
    out.insert(out.end(), type, type + 4);
    out.insert(out.end(), data, data + len);
    const uint32_t crc = crc32_update(0xFFFFFFFFu, out.data() + t, 4 + len) ^ 0xFFFFFFFFu;
    const uint8_t c[4] = {(uint8_t)(crc >> 24), (uint8_t)(crc >> 16), (uint8_t)(crc >> 8), (uint8_t)crc};
    out.insert(out.end(), c, c + 4);
}

// encode_into's signature, IHDR (write_ihdr, src/png/mod.rs:592-604), PLTE and tRNS for one reduced frame
void file_prefix(const pixo_b200_png_reduced &r, uint32_t width, uint32_t height, std::vector<uint8_t> &out)
{
    static const uint8_t kSig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    out.insert(out.end(), kSig, kSig + 8);
    const uint8_t ihdr[13] = {(uint8_t)(width >> 24), (uint8_t)(width >> 16), (uint8_t)(width >> 8), (uint8_t)width,
                              (uint8_t)(height >> 24), (uint8_t)(height >> 16), (uint8_t)(height >> 8),
                              (uint8_t)height, r.bit_depth, r.color_type_byte, 0, 0, 0};
    put_chunk(out, "IHDR", ihdr, 13);
    if (r.palette_len) {
        uint8_t plte[768], trns[256];
        for (uint32_t k = 0; k < r.palette_len; ++k) memcpy(plte + 3 * k, r.palette[k], 3);
        put_chunk(out, "PLTE", plte, 3 * (size_t)r.palette_len);
        for (uint32_t k = 0; k < r.trns_len; ++k) trns[k] = r.palette[k][3];
        if (r.trns_len) put_chunk(out, "tRNS", trns, r.trns_len);
    }
}

}  // namespace

int png_encode(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride, uint32_t n, uint32_t width,
               uint32_t height, uint32_t color_type, uint32_t strategy_and_flags, int level, uint32_t max_colors,
               const uint8_t *palettes, const uint32_t *palette_lens, uint8_t *d_out, size_t out_cap_each,
               size_t *out_lens, int32_t *status, pixo_b200_png_reduced *info)
{
    // every frame's slot for its filtered stream holds the unreduced stream
    const uint64_t fb = (uint64_t)height * ((uint64_t)width * (color_type + 1) + 1);
    const uint64_t fstride = (fb + 15) / 16 * 16;
    std::vector<uint64_t> charge(n, fb);
    std::vector<const uint64_t *> ptrs(n);
    for (uint32_t i = 0; i < n; ++i) ptrs[i] = &charge[i];
    std::vector<pixo_b200_png_reduced> own(info ? 0 : n);
    if (!info) info = own.data();
    for (uint32_t p0 = 0, p1; p0 < n; p0 = p1) {
        p1 = pass_end(ptrs.data(), p0, n, [](uint64_t c) { return c; });
        const uint32_t m = p1 - p0;
        uint8_t *filt;
        PIXO_TRY(bind(ctx, ctx->d_png_filt, [&](Layout &L) { filt = L.take(m * fstride); }));
        PIXO_TRY(png_quantize_filter(ctx, d_data + (size_t)p0 * in_stride, in_stride, m, width, height, color_type,
                                     strategy_and_flags, max_colors, palettes ? palettes + (size_t)p0 * 1024 : nullptr,
                                     palettes ? palette_lens + p0 : nullptr, info + p0, filt, fstride, nullptr));
        // DEFLATE codes the streams below 2^31 bytes; a longer one is passed as empty and its frame refused
        std::vector<size_t> lens(m), zlens(m);
        std::vector<int32_t> zst(m);
        uint64_t most = 0;
        bool any = false;
        for (uint32_t i = 0; i < m; ++i) {
            const uint64_t L = (uint64_t)height * (info[p0 + i].row_bytes + 1);
            status[p0 + i] = L >= kMaxStream ? PIXO_B200_ERR_UNSUPPORTED : 0;
            out_lens[p0 + i] = 0;
            lens[i] = status[p0 + i] ? 0 : L;
            most = std::max<uint64_t>(most, lens[i]);
            any |= !status[p0 + i];
        }
        if (!any) continue;
        const uint64_t zstride = (2 + most + (most / 65535 + 1) * 5 + 4 + 15) / 16 * 16;   // the stored-block bound
        uint8_t *zs;
        PIXO_TRY(bind(ctx, ctx->d_png_z, [&](Layout &L) { zs = L.take(m * zstride); }));
        PIXO_TRY(deflate_zlib(ctx, filt, fstride, lens.data(), m, level, zs, zstride, zlens.data(), zst.data()));
        // each file's exact length, then its small chunks
        std::vector<IdatFile> files;
        std::vector<uint64_t> prefix{0};
        std::vector<uint32_t> acc;
        std::vector<uint8_t> pre;
        const uint8_t kIdat[4] = {'I', 'D', 'A', 'T'};
        const uint32_t s0 = crc32_update(0xFFFFFFFFu, kIdat, 4);
        for (uint32_t i = 0; i < m; ++i) {
            const uint32_t f = p0 + i;
            if (status[f]) continue;
            if (zst[i]) return set_error(ctx, PIXO_B200_ERR_CUDA, "frame %u: its zlib stream outgrew the stored-block bound", f);
            const pixo_b200_png_reduced &r = info[f];
            const uint64_t nch = (zlens[i] + kIdatChunk - 1) / kIdatChunk;
            const uint64_t pre_len = 8 + 25 + (r.palette_len ? 12 + 3 * (uint64_t)r.palette_len : 0) +
                                     (r.palette_len && r.trns_len ? 12 + (uint64_t)r.trns_len : 0);
            out_lens[f] = pre_len + zlens[i] + 12 * nch + 12;
            if (out_lens[f] > out_cap_each) {
                status[f] = PIXO_B200_ERR_OUTPUT_TOO_SMALL;
                continue;
            }
            IdatFile F{zs + i * zstride, d_out + (size_t)f * out_cap_each, zlens[i], pre.size(), (uint32_t)pre_len,
                       (uint32_t)acc.size()};
            file_prefix(r, width, height, pre);
            for (uint64_t k = 0; k < nch; ++k)
                acc.push_back(crc32_shift(s0, std::min(kIdatChunk, zlens[i] - k * kIdatChunk)));
            files.push_back(F);
            prefix.push_back(prefix.back() + (zlens[i] + kIdatPiece - 1) / kIdatPiece);
        }
        if (files.empty()) continue;
        const uint32_t k = (uint32_t)files.size();
        // one upload: the files, the piece prefix sums, the CRC words and the prefix bytes
        IdatFile *d_files;
        uint64_t *d_prefix;
        uint32_t *d_acc;
        uint8_t *d_pre;
        auto describe = [&](Layout &L) {
            d_files = L.take<IdatFile>(k), d_prefix = L.take<uint64_t>(k + 1);
            d_acc = L.take<uint32_t>(acc.size()), d_pre = L.take(pre.size());
        };
        Layout count;
        describe(count);
        std::vector<uint8_t> image(count.end());
        Layout H(image.data());
        describe(H);
        memcpy(d_files, files.data(), k * sizeof(IdatFile));
        memcpy(d_prefix, prefix.data(), (k + 1) * 8);
        memcpy(d_acc, acc.data(), acc.size() * 4);
        memcpy(d_pre, pre.data(), pre.size());
        PIXO_TRY(bind(ctx, ctx->d_png_box, describe));
        PIXO_CUDA(ctx, cudaMemcpyAsync(d_files, image.data(), image.size(), cudaMemcpyHostToDevice, ctx->stream));
        const uint64_t pieces = prefix.back();
        PIXO_TRY(launch(ctx, k_png_idat, dim3((unsigned)((pieces + kIdatThreads - 1) / kIdatThreads)),
                        dim3(kIdatThreads), 0, d_files, d_prefix, k, pieces, d_acc));
        PIXO_TRY(launch(ctx, k_png_idat_finish, dim3((k + kIdatThreads / 32 - 1) / (kIdatThreads / 32)),
                        dim3(kIdatThreads), 0, d_files, k, d_pre, d_acc));
    }
    // the files are written when the call returns
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

}  // namespace pixo
