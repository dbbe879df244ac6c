// jpeg_transform.cu — fused colour -> (4:2:0 subsample) -> 8x8 forward DCT -> quantise kernels.
//
// Restates, bit-for-bit, the per-MCU work of pixo's
//   extract_block / extract_mcu_420   src/jpeg/mod.rs:1565-1656
//   color::rgb_to_ycbcr               src/color.rs:60-77
//   dct::dct_2d / aan_dct_1d          src/jpeg/dct.rs:591-700   (binary32, no FMA, fixed order)
//   quantize::quantize_block          src/jpeg/quantize.rs:99-105
//   quantize::zigzag_reorder          src/jpeg/quantize.rs:107-113 (optional, free: register renaming)
// and emits the arrays compute_all_coefficients (src/jpeg/mod.rs:932-966) returns.
//
// Design (H100): one thread owns one 8x8 block entirely in registers (both 1-D passes are plain
// register arithmetic on pairs of rows / columns, no shuffles).  K1 (4:2:0) runs persistent warp-autonomous
// workers fed by TMA; a warp colour-converts with dp4a straight out of its shared-memory pixel
// tile, exchanges packed 2x2 chroma sums through a swizzled warp-private buffer, and writes
// coefficients through a swizzled stage with 512-byte coalesced warp stores.  HBM traffic is
// the algorithmic 3 B/px in + 3 B/px out.
#include <cuda.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"

namespace pixo {
namespace {

// ---- strict binary32 arithmetic: one rounding per op, never contracted ------------------
#define FADD(a, b) __fadd_rn((a), (b))
#define FSUB(a, b) __fsub_rn((a), (b))
#define FMUL(a, b) __fmul_rn((a), (b))

// AAN constants, src/jpeg/dct.rs:591-608 (same decimal literals)
#define AAN_A1 0.70710678118654752440f
#define AAN_A2 0.5411961f
#define AAN_A3 0.70710678118654752440f
#define AAN_A4 1.3065629f
#define AAN_A5 0.38268343f
#define AAN_S0 0.3535534f
#define AAN_S1 0.2548978f
#define AAN_S2 0.2705981f
#define AAN_S3 0.3006724f
#define AAN_S4 0.3535534f
#define AAN_S5 0.4499881f
#define AAN_S6 0.6532815f
#define AAN_S7 1.2814578f

// ---- colour conversion on packed bytes ---------------------------------------------------
__device__ __forceinline__ int dp4a_us(uint32_t a_u8x4, uint32_t b_s8x4, int c)
{
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a_u8x4), "r"(b_s8x4), "r"(c));
    return d;
}

// u8 -> f32 minus `bias` without I2F: bits 0x4B0000vv are the float 2^23 + vv.
__device__ __forceinline__ float byte1_to_float_minus(uint32_t s, float magic)
{
    return FSUB(__uint_as_float(__byte_perm(s, 0x4B000000u, 0x7651)), magic);
}

__device__ __forceinline__ uint4 ldg_stream(const uint4 *p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// Stage a ROWS x (TILE_PX*BPP)-byte strip of the image in shared memory.  Pixels outside the
// image replicate the last column / row (clamp happens in source space, before any colour
// maths, as in extract_block: src/jpeg/mod.rs:1579-1580,1625-1626).
template <int BPP, int ROWS, int TILE_PX, int NT>
__device__ __forceinline__ void load_tile(uint8_t *__restrict__ smem,
                                          const uint8_t *__restrict__ img, uint32_t w,
                                          uint32_t h, uint32_t x0, uint32_t y0, int tid)
{
    constexpr int TB = TILE_PX * BPP;
    static_assert(TB % 16 == 0, "tile row must be a whole number of 16-byte chunks");
    const size_t pitch = (size_t)w * BPP;
    const uint8_t *col0 = img + (size_t)x0 * BPP;
    const bool fast = (x0 + TILE_PX <= w) && (pitch % 16 == 0) &&
                      ((reinterpret_cast<uintptr_t>(col0) & 15) == 0);
    if (fast) {
        constexpr int CH = TB / 16;
        constexpr int TOTAL = ROWS * CH;
#pragma unroll 4
        for (int idx = tid; idx < TOTAL; idx += NT) {
            const int r = idx / CH, k = idx - r * CH;
            const uint32_t sy = min(y0 + (uint32_t)r, h - 1);
            const uint4 val = ldg_stream(reinterpret_cast<const uint4 *>(col0 + sy * pitch) + k);
            reinterpret_cast<uint4 *>(smem + r * TB)[k] = val;
        }
        return;
    }
    const uint32_t inside_px = min((uint32_t)TILE_PX, w - x0);
    const int lin = (int)inside_px * BPP;
    const uint8_t *img_lo = img;
    const uint8_t *img_hi = img + pitch * h;
    // Unaligned pitch, tile fully inside the image in x: every row is TB bytes at an arbitrary
    // byte phase.  Fetch eight rows' worth of aligned word pairs back to back (one exposed
    // memory latency per batch instead of one per row), then funnel-shift into place.
    if (x0 + TILE_PX <= w) {
        constexpr int NW = TB / 4;                 // words per tile row
        constexpr int WPL = (NW + NT - 1) / NT;    // words per thread per row
        const uint32_t y_last = min(y0 + (uint32_t)ROWS - 1, h - 1);
        const uint8_t *first = col0 + min(y0, h - 1) * pitch - 3;
        const uint8_t *last = col0 + y_last * pitch + TB + 8;
        if (first >= img_lo && last <= img_hi) {
#pragma unroll
            for (int rb = 0; rb < ROWS; rb += 8) {
                uint32_t lo[8][WPL], hi[8][WPL];
#pragma unroll
                for (int rr = 0; rr < 8; ++rr) {
                    const uint32_t sy = min(y0 + (uint32_t)(rb + rr), h - 1);
                    const uint8_t *src = col0 + sy * pitch;
                    const uint32_t *a0 = reinterpret_cast<const uint32_t *>(src - (reinterpret_cast<uintptr_t>(src) & 3));
#pragma unroll
                    for (int i = 0; i < WPL; ++i) {
                        const int k = tid + i * NT;
                        if (k < NW) { lo[rr][i] = __ldg(a0 + k); hi[rr][i] = __ldg(a0 + k + 1); }
                    }
                }
#pragma unroll
                for (int rr = 0; rr < 8; ++rr) {
                    const uint32_t sy = min(y0 + (uint32_t)(rb + rr), h - 1);
                    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(col0 + sy * pitch) & 3) * 8;
#pragma unroll
                    for (int i = 0; i < WPL; ++i) {
                        const int k = tid + i * NT;
                        if (k < NW) reinterpret_cast<uint32_t *>(smem + (rb + rr) * TB)[k] = __funnelshift_r(lo[rr][i], hi[rr][i], sh);
                    }
                }
            }
            return;
        }
    }
    for (int r = 0; r < ROWS; ++r) {
        const uint32_t sy = min(y0 + (uint32_t)r, h - 1);
        const uint8_t *src = col0 + sy * pitch;
        uint8_t *dst = smem + r * TB;
        const int nwords = lin >> 2;
        const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3) * 8;
        for (int k = tid; k < nwords; k += NT) {
            const uint8_t *p = src + 4 * k;
            const uint8_t *a0 = p - (sh >> 3);
            uint32_t val;
            if (a0 >= img_lo && a0 + 8 <= img_hi) {
                const uint32_t lo = __ldg(reinterpret_cast<const uint32_t *>(a0));
                const uint32_t hi = sh ? __ldg(reinterpret_cast<const uint32_t *>(a0) + 1) : 0u;
                val = __funnelshift_r(lo, hi, sh);
            } else {
                val = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) |
                      ((uint32_t)p[3] << 24);
            }
            reinterpret_cast<uint32_t *>(dst)[k] = val;
        }
        for (int i = (nwords << 2) + tid; i < lin; i += NT) dst[i] = src[i];
        const uint8_t *last = src + (inside_px - 1) * BPP;
        for (int i = lin + tid; i < TB; i += NT) dst[i] = last[i % BPP];
    }
}

// =========================================================================================
// Lane-pair block pipeline.  Each thread carries two independent 8-vectors (two rows, or two
// columns) through the DCT side by side.  Hopper has no packed FP32 instructions, so every pair
// operation is two scalar binary32 instructions with an explicit rounding mode (add/sub/mul.rn,
// fma.rn, add.rz, fma.rm): ptxas never contracts those, and each lane performs exactly one IEEE
// binary32 rounding per reference operation.
// =========================================================================================
struct f2 {
    float lo, hi;
};

__device__ __forceinline__ f2 pk(float lo, float hi) { return f2{lo, hi}; }
__device__ __forceinline__ void upk(f2 v, float &lo, float &hi)
{
    lo = v.lo;
    hi = v.hi;
}
__device__ __forceinline__ void upk_u(f2 v, uint32_t &lo, uint32_t &hi)
{
    lo = __float_as_uint(v.lo);
    hi = __float_as_uint(v.hi);
}
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return f2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f2 sub2(f2 a, f2 b) { return f2{__fsub_rn(a.lo, b.lo), __fsub_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return f2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c)
{
    return f2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)};
}
__device__ __forceinline__ f2 add2_rz(f2 a, f2 b) { return f2{__fadd_rz(a.lo, b.lo), __fadd_rz(a.hi, b.hi)}; }
__device__ __forceinline__ f2 fma2_rm(f2 a, f2 b, f2 c)
{
    return f2{__fmaf_rd(a.lo, b.lo, c.lo), __fmaf_rd(a.hi, b.hi, c.hi)};
}
#define K2(c) pk((c), (c))

// Multiply both lanes by a constant: the row pass's post-scale, whose two results land directly
// in the registers of the column-pair layout (no transpose moves).
__device__ __forceinline__ void mulc(f2 a, float c, float &lo, float &hi)
{
    float x, y;
    upk(a, x, y);
    lo = FMUL(x, c);
    hi = FMUL(y, c);
}
// aan_dct_1d (src/jpeg/dct.rs:648-700) on two independent 8-vectors at once; returns the eight
// outputs *before* the S[k] post-scale (o[k]), which the caller applies.
__device__ __forceinline__ void aan_1d_x2_core(const f2 (&d)[8], f2 (&o)[8])
{
#define MULC(a, c) mul2((a), K2(c))
    const f2 tmp0 = add2(d[0], d[7]), tmp7 = sub2(d[0], d[7]);
    const f2 tmp1 = add2(d[1], d[6]), tmp6 = sub2(d[1], d[6]);
    const f2 tmp2 = add2(d[2], d[5]), tmp5 = sub2(d[2], d[5]);
    const f2 tmp3 = add2(d[3], d[4]), tmp4 = sub2(d[3], d[4]);

    const f2 tmp10 = add2(tmp0, tmp3), tmp13 = sub2(tmp0, tmp3);
    const f2 tmp11 = add2(tmp1, tmp2), tmp12 = sub2(tmp1, tmp2);

    o[0] = add2(tmp10, tmp11);
    o[4] = sub2(tmp10, tmp11);
    const f2 z1 = MULC(add2(tmp12, tmp13), AAN_A1);
    o[2] = add2(tmp13, z1);
    o[6] = sub2(tmp13, z1);

    const f2 u10 = add2(tmp4, tmp5), u11 = add2(tmp5, tmp6), u12 = add2(tmp6, tmp7);
    const f2 z5 = MULC(sub2(u10, u12), AAN_A5);
    const f2 z2 = add2(MULC(u10, AAN_A2), z5);
    const f2 z4 = add2(MULC(u12, AAN_A4), z5);
    const f2 z3 = MULC(u11, AAN_A3);
    const f2 z11 = add2(tmp7, z3), z13 = sub2(tmp7, z3);

    o[5] = add2(z13, z2);
    o[3] = sub2(z13, z2);
    o[1] = add2(z11, z4);
    o[7] = sub2(z11, z4);
#undef MULC
}

// One table entry per output word (two adjacent natural-order coefficients):
// (-d_lo, -d_hi, r_lo, r_hi) with r = RN(1/d).
struct __align__(16) QPair {
    float nd_lo, nd_hi, r_lo, r_hi;
};

// The quantiser's table, passed as a kernel parameter and copied to shared memory once per CTA:
// 32 entries per component table, one per output word.
struct QPairTab {
    QPair t[2][32];  // [0] luminance, [1] chrominance (x4 folded in for 4:2:0, see fill_qpair_tab)
};

// dct_2d (src/jpeg/dct.rs:614-646) + quantize_block (src/jpeg/quantize.rs:99-105) on a block
// held as row pairs R[i][c] = (v[2i][c], v[2i+1][c]); writes 64 int16 (8 x 16 B).
//   x / d      : q0 = x*r; q = fma(fma(q0, -d, x), r, q0) == RN(x/d)     (tools/verify_div.c)
//   round      : w = RZ(q + 0.5); m = floor(sign(q) * w) via fma.rm with 1.5*2^23;
//                result = m for q >= 0, ~m for q < 0  == round-half-away(q)  (derivation in DESIGN.md;
//                tests/test_transform_edges_gpu.py runs ties, their neighbours and 0.49999997)
// `out` is the block's 128-byte slot in a warp-private shared-memory stage; its eight 16-byte
// chunks are written at chunk index (k ^ swz) so that the lanes of a quarter warp hit distinct
// banks (the caller then copies the stage out with fully coalesced 512-byte warp stores).
// The table is read from shared memory (32 LDS.128 per block) because constant-bank tables with
// static offsets would need one copy of the transform per table, and a run-time index into the
// constant bank gives per-thread loads.

// row pass on row pairs; the post-scale is done lane by lane so the results land in the
// column-pair layout C[r][j] = (V[r][2j], V[r][2j+1]) without transposes
__device__ __forceinline__ void dct_rows_x2(f2 (&R)[4][8], f2 (&C)[8][4])
{
    constexpr float SK[8] = {AAN_S0, AAN_S1, AAN_S2, AAN_S3, AAN_S4, AAN_S5, AAN_S6, AAN_S7};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        f2 o[8];
        aan_1d_x2_core(R[i], o);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float a0, a1, b0, b1;
            mulc(o[2 * j], SK[2 * j], a0, a1);          // (V[2i][2j],   V[2i+1][2j])
            mulc(o[2 * j + 1], SK[2 * j + 1], b0, b1);  // (V[2i][2j+1], V[2i+1][2j+1])
            C[2 * i][j] = pk(a0, b0);
            C[2 * i + 1][j] = pk(a1, b1);
        }
    }
}

// What the transform writes per block: natural order, zig-zag order (both all 64 coefficients), or
// a coefficient record (zig-zag order, cut after the sector of the last non-zero coefficient, plus
// its extent: see CoefExtents in common.cuh), or - kDct, the trellis quantiser's input - the block's
// unquantised f32 DCT in natural order (256 bytes), written straight from registers to global memory.
enum CoefOut { kNatural, kZigzag, kRecords, kDct };

// column pass on column pairs, quantising each pair of columns as soon as it is transformed;
// tab(i) returns table entry i (one per output word).  kRecords: *eout = the block's record extent
// (32-byte sectors up to the last non-zero one: an OR over each sector's words, a few instructions).
// kDct: no quantiser; the DCT times `dscale` (a power of two, so exact) goes to dout (null: nowhere).
template <int OUT, typename TabFn>
__device__ __forceinline__ void dct_cols_quant_store_x2(f2 (&C)[8][4], TabFn tab, uint4 *__restrict__ out,
                                                        const int swz, uint8_t *eout, float *dout, float dscale)
{
    constexpr bool ZIGZAG = OUT != kNatural;
    constexpr float SK[8] = {AAN_S0, AAN_S1, AAN_S2, AAN_S3, AAN_S4, AAN_S5, AAN_S6, AAN_S7};
    if constexpr (OUT == kDct) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const f2 in[8] = {C[0][j], C[1][j], C[2][j], C[3][j], C[4][j], C[5][j], C[6][j], C[7][j]};
            f2 o[8];
            aan_1d_x2_core(in, o);
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const f2 x = mul2(mul2(o[r], K2(SK[r])), K2(dscale));
                if (dout) *reinterpret_cast<float2 *>(dout + r * 8 + 2 * j) = make_float2(x.lo, x.hi);
            }
        }
        return;
    }
    uint32_t W[32];
    const f2 half2 = K2(0.5f), magic2 = K2(12582912.0f);  // 1.5 * 2^23
    uint32_t kSign, kOne;  // in registers so copysign(1.0, q) is ONE lop3: (q & sign) | one
    asm("mov.b32 %0, 0x80000000;" : "=r"(kSign));
    asm("mov.b32 %0, 0x3F800000;" : "=r"(kOne));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        QPair T[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) T[r] = tab(r * 4 + j);
        const f2 in[8] = {C[0][j], C[1][j], C[2][j], C[3][j], C[4][j], C[5][j], C[6][j], C[7][j]};
        f2 o[8];
        aan_1d_x2_core(in, o);
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const f2 nd = pk(T[r].nd_lo, T[r].nd_hi), rc = pk(T[r].r_lo, T[r].r_hi);
            const f2 x = mul2(o[r], K2(SK[r]));   // post-scale: feeds only a multiply / fma addend
            const f2 q0 = mul2(x, rc);
            const f2 e = fma2(q0, nd, x);
            const f2 q = fma2(e, rc, q0);
            uint32_t ql, qh;
            upk_u(q, ql, qh);
            uint32_t sl, sh;
            asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(sl) : "r"(ql), "r"(kSign), "r"(kOne));
            asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(sh) : "r"(qh), "r"(kSign), "r"(kOne));
            const f2 sg = pk(__uint_as_float(sl), __uint_as_float(sh));
            const f2 w = add2_rz(q, half2);
            const f2 tt = fma2_rm(w, sg, magic2);
            uint32_t tl, th, neg;
            upk_u(tt, tl, th);
            asm("prmt.b32 %0, %1, %2, %3;" : "=r"(neg) : "r"(ql), "r"(qh), "r"(0xFFBBu));
            W[r * 4 + j] = __byte_perm(tl, th, 0x5410) ^ neg;
        }
    }
    uint32_t Z[32];   // the output words in the order they are stored
#pragma unroll
    for (int k = 0; k < 8; ++k) {
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            if (ZIGZAG) {
                const int i0 = zz_nat(k * 8 + m * 2), i1 = zz_nat(k * 8 + m * 2 + 1);
                Z[k * 4 + m] = __byte_perm(W[i0 >> 1], W[i1 >> 1],
                                           ((i0 & 1) ? 0x0032 : 0x0010) | ((i1 & 1) ? 0x7600 : 0x5400));
            } else {
                Z[k * 4 + m] = W[k * 4 + m];
            }
        }
        out[k ^ swz] = make_uint4(Z[k * 4], Z[k * 4 + 1], Z[k * 4 + 2], Z[k * 4 + 3]);
    }
    if (OUT == kRecords) {
        uint32_t o[4] = {0, 0, 0, 0};   // OR of sector 1..3's words
#pragma unroll
        for (int i = 8; i < 32; ++i) o[i >> 3] |= Z[i];
        *eout = (uint8_t)(o[3] ? 4 : o[2] ? 3 : o[1] ? 2 : 1);
    }
}

// chroma_u MUST be warp-uniform (the callers derive it from a warp vote, so the branch is one).
template <int OUT>
__device__ __forceinline__ void dct_quant_store_x2(f2 (&R)[4][8], const QPairTab *qs, const bool chroma_u,
                                                   uint4 *__restrict__ out, const int swz, uint8_t *eout,
                                                   float *dout = nullptr, float dscale = 1.0f)
{
    f2 C[8][4];
    dct_rows_x2(R, C);
    const QPair *t = qs->t[chroma_u ? 1 : 0];
    dct_cols_quant_store_x2<OUT>(C, [&](int i) { return t[i]; }, out, swz, eout, dout, dscale);
}

// Copy a warp's 32-slot stage (4 KB, swizzled as above) to global memory: instruction j moves
// slots 4j..4j+3, i.e. 512 contiguous bytes per warp store.  dst_of(s): slot s's destination, or
// null when it has none.  kRecords: ext[s] is slot s's record extent in sectors (the warp's 32
// extents, 4-byte aligned in shared memory); only the sectors of a slot's record are written, and the
// extents go out as one 32-byte warp store to edst_of(s) (null: none).
template <int OUT, typename SwzFn, typename DstFn, typename EDstFn>
__device__ __forceinline__ void flush_stage(const uint4 *__restrict__ stage, const uint8_t *ext, int lane,
                                            SwzFn swz_of, DstFn dst_of, EDstFn edst_of)
{
    __syncwarp();
    uint32_t e[8];   // kRecords: word j holds the extents of slots 4j..4j+3; this lane's is byte lane >> 3
    if (OUT == kRecords) {
        const uint4 a = reinterpret_cast<const uint4 *>(ext)[0], b = reinterpret_cast<const uint4 *>(ext)[1];
        e[0] = a.x; e[1] = a.y; e[2] = a.z; e[3] = a.w; e[4] = b.x; e[5] = b.y; e[6] = b.z; e[7] = b.w;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int s = j * 4 + (lane >> 3), k = lane & 7;
        const uint4 v = stage[s * 8 + (k ^ swz_of(s))];
        uint4 *d = dst_of(s);
        if (OUT != kRecords) {
            if (d) d[k] = v;
        } else {
            // piece k lies in sector k >> 1.  A predicated store: left to itself, ptxas branches around
            // the stage read and the address arithmetic of every skipped piece.
            const uint32_t keep = (d != nullptr) & ((uint32_t)(k >> 1) < __byte_perm(e[j], 0, 0x4440 + (lane >> 3)));
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %5, 0;\n\t"
                         "@p st.global.v4.u32 [%0], {%1, %2, %3, %4};\n\t}"
                         :: "l"(d + k), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(keep) : "memory");
        }
    }
    if (OUT == kRecords) {
        uint8_t *ed = edst_of(lane);
        if (ed) *ed = ext[lane];
    }
    __syncwarp();
}

// ---- TMA / mbarrier plumbing ---------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void *dst, const void *tmap, int x, int y, int z,
                                            uint64_t *bar)
{
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes "
        "[%0], [%1, {%2, %3, %4}], [%5];" ::"r"(smem_u32(dst)),
        "l"(tmap), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar))
        : "memory");
}

// =========================================================================================
// K1: RGB, 4:2:0.  Persistent, warp-autonomous: every warp is an independent worker that owns
// a private 12 KB pixel buffer, a 4 KB chroma exchange buffer and an mbarrier, and loops over
// "units" of 16 MCUs (256 x 16 px) of one MCU row:
//     wait for the unit's pixels (TMA)           -> 2 x (32 Y blocks: colour + DCT + quant)
//     issue the TMA load of the warp's next unit -> 32 chroma blocks (16 Cb + 16 Cr)
// so each lane runs exactly three block pipelines per unit, no CTA-wide barrier exists, and
// the next unit's pixels stream in underneath the chroma pass.  Interior units of
// 16-byte-pitched images arrive by one 3-D cp.async.bulk.tensor (TMA); bottom-edge units
// (row replication) and unaligned images use the warp-cooperative clamped loader.
// =========================================================================================
constexpr int K1_WARPS = 4;
constexpr int K1_THREADS = K1_WARPS * 32;
// 2, not 3: on the H100 the 255-register build does not spill and runs 32 4K frames in 0.58 ms against
// 0.61 ms at 3 CTAs per SM (168 registers, spills); the grid follows the occupancy query.
constexpr int K1_MIN_BLOCKS = 2;
constexpr int K1_MCUS = 16;             // MCUs per unit, staged as two half tiles of 8 MCUs
constexpr int K1_HB = 8 * 16 * 3;        // 384 bytes per half-tile row
constexpr int K1_HALF_BYTES = 16 * K1_HB;  // 6 KB; also hosts that half's 4 KB output stage
constexpr int K1_TILE_BYTES = 2 * K1_HALF_BYTES;

struct K1Params {
    const uint8_t *pixels;
    size_t pixel_stride;
    uint32_t w, h, mcus_x, mcus_y, units_x, n_images;
    int16_t *y, *cb, *cr;            // kDct: float arrays (and the strides count floats)
    size_t y_stride, c_stride;
    CoefExtents e;                   // kRecords only
    uint32_t use_tma;
};

struct __align__(128) K1WarpSmem {
    uint8_t tile[2][K1_HALF_BYTES];  // pixels of MCUs 0-7 / 8-15; reused as output stage once read
    uint32_t csum[K1_MCUS * 64];     // chroma quad sums; reused as the chroma pass's output stage
    __align__(16) uint8_t ext[32];   // kRecords: the stage's record extents, by slot
    uint64_t bar;
};

struct __align__(128) K1Smem {
    K1WarpSmem w[K1_WARPS];
    QPairTab q;
};

// 8 RGB pixels in six words -> the eight raw 4-byte windows (r,g,b,next r) the dot products read
__device__ __forceinline__ void rgb_windows8(const uint32_t (&w)[6], uint32_t (&win)[8])
{
    win[0] = w[0];
    win[1] = __funnelshift_r(w[0], w[1], 24);
    win[2] = __funnelshift_r(w[1], w[2], 16);
    win[3] = w[2] >> 8;
    win[4] = w[3];
    win[5] = __funnelshift_r(w[3], w[4], 24);
    win[6] = __funnelshift_r(w[4], w[5], 16);
    win[7] = w[5] >> 8;
}

// One RGB row of a Y block (8 px in six words): Y - 128 as float for each pixel and the packed
// chroma terms P = [(256 - cb) | 0xFF00, (256 - cr) | 0xFF00] clamped per colour.rs.
//   y        = (77r + 150g + 29b + 128) >> 8
//   256 - cb = byte 1 of (43r + 85g - 128b - 32641)     [cb = ((-43r-85g+128b+128)>>8)+128]
//   256 - cr = byte 1 of (-128r + 107g + 21b - 32641)
// All three dot products read the raw 4-byte window (r,g,b,next r) with a zero 4th weight.
__device__ __forceinline__ void ycc_row8(const uint32_t (&w)[6], float (&yv)[8], uint32_t (&hs)[4])
{
    uint32_t win[8];
    rgb_windows8(w, win);
    uint32_t pp[8];
#pragma unroll
    for (int x = 0; x < 8; ++x) {
        const uint32_t ys = __dp4a(win[x], 0x001D964Du, 128u);
        const int ucb = dp4a_us(win[x], 0x0080552Bu, -32641);
        const int ucr = dp4a_us(win[x], 0x00156B80u, -32641);
        yv[x] = __uint_as_float(__byte_perm(ys, 0x4B000000u, 0x7651));  // 2^23 + y
        pp[x] = __vmaxu2(__byte_perm((uint32_t)ucb, (uint32_t)ucr, 0x7531), 0xFF01FF01u);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) hs[k] = pp[2 * k] + pp[2 * k + 1];
}

// Warp-cooperative version of load_tile: ROWS x (TILE_PX*3) bytes with edge replication.
// (kept out of line: it only runs for edge units and unaligned images, and inlining it twice
// into the persistent loop costs instruction-cache room the TMA path needs)
template <int ROWS, int TILE_PX>
__device__ __noinline__ void warp_load_tile_rgb(uint8_t *__restrict__ smem,
                                                   const uint8_t *__restrict__ img, uint32_t w,
                                                   uint32_t h, uint32_t x0, uint32_t y0, int lane)
{
    load_tile<3, ROWS, TILE_PX, 32>(smem, img, w, h, x0, y0, lane);
}

template <int OUT>
__global__ void __launch_bounds__(K1_THREADS, K1_MIN_BLOCKS)
k_jpeg_420(const __grid_constant__ K1Params P, const __grid_constant__ QPairTab qp,
           const __grid_constant__ CUtensorMap tmap)
{
    extern __shared__ __align__(128) uint8_t smem_raw[];
    K1Smem &S = *reinterpret_cast<K1Smem *>(smem_raw);
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    K1WarpSmem &WS = S.w[warp];
    for (int i = tid; i < 64; i += K1_THREADS) S.q.t[i >> 5][i & 31] = qp.t[i >> 5][i & 31];
    const QPairTab *QS = &S.q;

    if (lane == 0) {
        mbar_init(&WS.bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // Unit coordinates (image, MCU row, unit in the row) advance by a constant stride: the step is
    // decomposed once, so the loop carries no division (a 64-bit u / units_per_img would put two
    // copies of a ~100-instruction routine in the hot loop).
    const uint32_t units_per_img = P.mcus_y * P.units_x;
    const uint64_t nunits = (uint64_t)units_per_img * P.n_images;
    const uint32_t stride = gridDim.x * K1_WARPS;
    const uint32_t d_ux = stride % P.units_x, d_t = stride / P.units_x;
    const uint32_t d_my = d_t % P.mcus_y, d_img = d_t / P.mcus_y;
    uint32_t phase = 0;

    auto advance = [&](uint32_t &img, uint32_t &my, uint32_t &ux) {
        ux += d_ux;
        if (ux >= P.units_x) { ux -= P.units_x; ++my; }
        my += d_my;
        if (my >= P.mcus_y) { my -= P.mcus_y; ++img; }
        img += d_img;
    };
    auto unit_by_tma = [&](uint32_t my) { return P.use_tma && (my * 16 + 16 <= P.h); };
    auto issue_tma = [&](uint32_t img_, uint32_t my_, uint32_t ux_) {
        if (unit_by_tma(my_)) {   // both halves under ONE barrier phase (one arrival, 12 KB)
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(&WS.bar, K1_TILE_BYTES);
            tma_load_3d(WS.tile[0], &tmap, (int)(ux_ * (2 * K1_HB / 8)), (int)(my_ * 16), (int)img_, &WS.bar);
            tma_load_3d(WS.tile[1], &tmap, (int)(ux_ * (2 * K1_HB / 8) + K1_HB / 8), (int)(my_ * 16), (int)img_, &WS.bar);
        }
    };
    // synchronously load half `half` of the current unit (edge rows / unaligned images)
    auto load_half = [&](uint32_t img_, uint32_t my_, uint32_t ux_, int half) {
        const uint8_t *image = P.pixels + (size_t)img_ * P.pixel_stride;
        const uint32_t x0 = ux_ * (K1_MCUS * 16) + half * 128;
        if (x0 < P.w) warp_load_tile_rgb<16, 128>(WS.tile[half], image, P.w, P.h, x0, my_ * 16, lane);
        __syncwarp();
    };

    uint64_t u = (uint64_t)blockIdx.x * K1_WARPS + warp;
    uint32_t img, my, ux;
    {
        const uint32_t u0 = blockIdx.x * K1_WARPS + warp;   // < stride <= 2^32
        img = u0 / units_per_img;
        const uint32_t rem = u0 - img * units_per_img;
        my = rem / P.units_x;
        ux = rem - my * P.units_x;
    }
    if (u < nunits && lane == 0) issue_tma(img, my, ux);

    for (; u < nunits; u += stride) {
        if (unit_by_tma(my)) {
            mbar_wait(&WS.bar, phase);
            phase ^= 1;
        } else {
            load_half(img, my, ux, 0);
            load_half(img, my, ux, 1);
        }
        uint32_t img_n = img, my_n = my, ux_n = ux;   // the warp's next unit: prefetched below, current next time round
        advance(img_n, my_n, ux_n);
        const uint32_t mcu0 = ux * K1_MCUS;
        const uint32_t n_mcu = min((uint32_t)K1_MCUS, P.mcus_x - mcu0);
        const size_t mcu_base = (size_t)my * P.mcus_x + mcu0;

#pragma unroll 1
        for (int job = 0; job < 3; ++job) {
            // a warp vote, so that ptxas knows the flag is uniform (see dct_quant_store_x2)
            const bool chroma_u = __ballot_sync(0xffffffffu, job == 2) != 0u;
            f2 R[4][8];
            uint4 *stage;   // this warp's 32 x 128-byte output stage for the job
            int slot, swz;
            if (!chroma_u) {
                // ---- 32 Y blocks (8 MCUs) + their packed chroma quad sums ----
                const int by = lane >> 4, l16 = lane & 15;
                const int par = l16 >> 3, k8 = l16 & 7;
                const int mj = (k8 >> 1) * 2 + par;   // MCU within the job; same parity per quarter warp
                const int mcu = job * 8 + mj;
                const int bx = k8 & 1;
                const uint8_t *base = WS.tile[job] + (by * 8) * K1_HB + (mj * 2 + bx) * 24;
                uint4 *cdst = reinterpret_cast<uint4 *>(WS.csum) + mcu * 16;
                // No guard for MCUs past the right edge: those lanes convert whatever bytes their tile
                // columns hold (zero fill / stale pixels - any bytes are fine) and their stage slots and
                // chroma sums are never flushed: one straight-line, warp-convergent path.
#pragma unroll
                for (int rp = 0; rp < 4; ++rp) {
                    float y0[8], y1[8];
                    uint32_t h0[4], h1[4];
                    {
                        const uint2 *p = reinterpret_cast<const uint2 *>(base + (rp * 2) * K1_HB);
                        const uint2 a = p[0], b = p[1], c = p[2];
                        const uint32_t wds[6] = {a.x, a.y, b.x, b.y, c.x, c.y};
                        ycc_row8(wds, y0, h0);
                    }
                    {
                        const uint2 *p = reinterpret_cast<const uint2 *>(base + (rp * 2 + 1) * K1_HB);
                        const uint2 a = p[0], b = p[1], c = p[2];
                        const uint32_t wds[6] = {a.x, a.y, b.x, b.y, c.x, c.y};
                        ycc_row8(wds, y1, h1);
                    }
#pragma unroll
                    for (int x = 0; x < 8; ++x)  // (2^23 + y) - (2^23 + 128) = y - 128, exact
                        R[rp][x] = sub2(pk(y0[x], y1[x]), K2(8388736.0f));
                    const int logical = (by * 4 + rp) * 2 + bx;
                    cdst[logical ^ (mcu & 7)] =
                        make_uint4(h0[0] + h1[0], h0[1] + h1[1], h0[2] + h1[2], h0[3] + h1[3]);
                }
                __syncwarp();  // every lane is done with this half tile
                stage = reinterpret_cast<uint4 *>(WS.tile[job]);  // the consumed half becomes the stage
                slot = mj * 4 + by * 2 + bx;                  // = block index within the job's 32
                swz = ((slot >> 3) << 1) | (slot & 1);        // distinct across a quarter warp
            } else {
                if (lane == 0 && u + stride < nunits) issue_tma(img_n, my_n, ux_n);   // both half tiles were flushed
                // ---- lanes 0-15: Cb of MCU lane, lanes 16-31: Cr of MCU lane-16 ----
                const int comp = lane >> 4, mcu = lane & 15;
                const uint4 *csrc = reinterpret_cast<const uint4 *>(WS.csum) + mcu * 16;
                const uint32_t sel = comp == 0 ? 0x7610u : 0x7632u;
                // low half = 65536 - sum(cb), high half = 65539 - sum(cr)  (see ycc_row8);
                // block value = 4 * (sum * 0.25 - 128) = sum - 512  (src/jpeg/mod.rs:1642-1653)
                const float bias = comp == 0 ? 8453632.0f : 8453635.0f;  // 2^23 + 65536(+3) - 512
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float v0[8], v1[8];
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int l0 = (2 * i) * 2 + hh, l1 = (2 * i + 1) * 2 + hh;
                        const uint4 s0 = csrc[l0 ^ (mcu & 7)];
                        const uint4 s1 = csrc[l1 ^ (mcu & 7)];
                        const uint32_t a[4] = {s0.x, s0.y, s0.z, s0.w};
                        const uint32_t b[4] = {s1.x, s1.y, s1.z, s1.w};
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            v0[hh * 4 + k] = __uint_as_float(__byte_perm(a[k], 0x4B000000u, sel));
                            v1[hh * 4 + k] = __uint_as_float(__byte_perm(b[k], 0x4B000000u, sel));
                        }
                    }
#pragma unroll
                    for (int x = 0; x < 8; ++x) R[i][x] = sub2(K2(bias), pk(v0[x], v1[x]));
                }
                __syncwarp();  // every lane has read its chroma sums: the buffer becomes the stage
                stage = reinterpret_cast<uint4 *>(WS.csum);
                slot = lane;                                  // 0-15 Cb, 16-31 Cr
                swz = slot & 7;
            }
            // The transform runs in every lane (edge lanes work on garbage and their slots are never
            // flushed): the quantiser's table reads are uniform-datapath loads, which exist only in
            // warp-convergent code.
            if constexpr (OUT == kDct) {
                // the block's f32 DCT straight to its slot; the chroma block holds 4x the averaged
                // block (quad sums), so its DCT is scaled by 0.25, exactly
                float *dout = nullptr;
                if (!chroma_u) {
                    if (job * 8u + (slot >> 2) < n_mcu)
                        dout = reinterpret_cast<float *>(P.y) + (size_t)img * P.y_stride + ((mcu_base + job * 8) * 4 + slot) * 64;
                } else if ((uint32_t)(lane & 15) < n_mcu) {
                    dout = reinterpret_cast<float *>(lane < 16 ? P.cb : P.cr) + (size_t)img * P.c_stride +
                           (mcu_base + (lane & 15)) * 64;
                }
                dct_quant_store_x2<OUT>(R, QS, chroma_u, stage + slot * 8, swz, &WS.ext[slot], dout,
                                        chroma_u ? 0.25f : 1.0f);
                continue;
            }
            dct_quant_store_x2<OUT>(R, QS, chroma_u, stage + slot * 8, swz, &WS.ext[slot]);
            if (!chroma_u) {
                const size_t b0 = (mcu_base + job * 8) * 4;   // the job's first Y block
                uint4 *ybase = reinterpret_cast<uint4 *>(P.y + (size_t)img * P.y_stride + b0 * 64);
                const uint32_t first = job * 8;
                flush_stage<OUT>(
                    stage, WS.ext, lane, [](int s) { return ((s >> 3) << 1) | (s & 1); },
                    [&](int s) -> uint4 * { return first + (s >> 2) < n_mcu ? ybase + s * 8 : nullptr; },
                    [&](int s) -> uint8_t * {   // called for kRecords only: P.e is set
                        return first + (s >> 2) < n_mcu ? P.e.y + ((size_t)img * P.e.stride + b0 + s) : nullptr;
                    });
            } else {
                uint4 *cbb = reinterpret_cast<uint4 *>(P.cb + (size_t)img * P.c_stride + mcu_base * 64);
                uint4 *crb = reinterpret_cast<uint4 *>(P.cr + (size_t)img * P.c_stride + mcu_base * 64);
                flush_stage<OUT>(
                    stage, WS.ext, lane, [](int s) { return s & 7; },
                    [&](int s) -> uint4 * {
                        return (uint32_t)(s & 15) < n_mcu ? (s < 16 ? cbb : crb) + (s & 15) * 8 : nullptr;
                    },
                    [&](int s) -> uint8_t * {   // kRecords only
                        return (uint32_t)(s & 15) < n_mcu
                                   ? (s < 16 ? P.e.cb : P.e.cr) + ((size_t)img * P.e.stride + mcu_base + (s & 15))
                                   : nullptr;
                    });
            }
        }
        img = img_n; my = my_n; ux = ux_n;
    }
}

// =========================================================================================
// K2: RGB 4:4:4 (warp-autonomous, below) and Gray (64 threads, CTA = 64 blocks of one block
// row; every warp owns 32 consecutive blocks, runs the same packed block pipeline as K1 and
// flushes its 4 KB stage with coalesced stores).
// =========================================================================================
constexpr int GRAY_BLOCKS = 64;

// 8 RGB pixels in six words (see rgb_windows8) -> Y - 128 as float
__device__ __forceinline__ void y_row8(const uint32_t (&w)[6], float (&v)[8])
{
    uint32_t win[8];
    rgb_windows8(w, win);
#pragma unroll
    for (int x = 0; x < 8; ++x)
        v[x] = byte1_to_float_minus(__dp4a(win[x], 0x001D964Du, 128u), 8388736.0f);
}
// ... -> Cb - 128 / Cr - 128 as float; wgt = 0x0080552B (Cb) or 0x00156B80 (Cr), see ycc_row8
__device__ __forceinline__ void c_row8(const uint32_t (&w)[6], uint32_t wgt, float (&v)[8])
{
    uint32_t win[8];
    rgb_windows8(w, win);
#pragma unroll
    for (int x = 0; x < 8; ++x) {
        // byte 1 of u = 256 - c (c = cb or cr before the clamp); c <= 255 <=> u >= -65280
        const int u = max(dp4a_us(win[x], wgt, -32641), -65280);
        v[x] = FSUB(8388736.0f, __uint_as_float(__byte_perm((uint32_t)u, 0x4B000000u, 0x7651)));  // c - 128
    }
}

// K2 (4:4:4), on K1's skeleton: persistent warp-autonomous workers, no CTA barrier.  A unit is
// 32 blocks of one block row (256 x 8 pixels, 6 KB), fetched by one 3-D TMA into one of the
// warp's TWO tile buffers - the next unit's pixels stream in while this one is transformed (all
// three component passes read the same RGB tile, so it cannot double as the output stage the way
// K1's half tiles do).  Lane = block; pass c converts the lane's 8x8 pixels to component c and
// runs the packed DCT/quantiser; the warp's 4 KB stage goes out as 512-byte coalesced stores.
constexpr int K444_WARPS = 4;
constexpr int K444_THREADS = K444_WARPS * 32;
constexpr int K444_ROW_B = 32 * 8 * 3;           // 768 bytes per tile row
constexpr int K444_TILE_BYTES = 8 * K444_ROW_B;  // 6 KB
// 2, not 3: at 168 registers ptxas demotes a block array to local memory; on the H100 the 4:4:4
// kernel takes 0.93 ms per 32 4K frames at 2 CTAs per SM against 0.99-1.00 ms at 3.
constexpr int K444_MIN_BLOCKS = 2;

struct __align__(128) K444WarpSmem {
    uint8_t tile[2][K444_TILE_BYTES];
    uint4 stage[256];
    __align__(16) uint8_t ext[32];   // kRecords: the stage's record extents
    uint64_t bar[2];
};

struct __align__(128) K444Smem {
    K444WarpSmem w[K444_WARPS];
    QPairTab q;
};

// K1Params with mcus_x / mcus_y = blocks per row / block rows, units_x = units per block row
template <int OUT>
__global__ void __launch_bounds__(K444_THREADS, K444_MIN_BLOCKS)
k_jpeg_444(const __grid_constant__ K1Params P, const __grid_constant__ QPairTab qp,
           const __grid_constant__ CUtensorMap tmap)
{
    extern __shared__ __align__(128) uint8_t smem_raw[];
    K444Smem &S = *reinterpret_cast<K444Smem *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    K444WarpSmem &WS = S.w[warp];
    for (int i = tid; i < 64; i += K444_THREADS) S.q.t[i >> 5][i & 31] = qp.t[i >> 5][i & 31];
    const QPairTab *QS = &S.q;
    if (lane == 0) {
        mbar_init(&WS.bar[0], 1);
        mbar_init(&WS.bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const uint32_t units_per_img = P.mcus_y * P.units_x;   // no division in the loop: see k_jpeg_420
    const uint64_t nunits = (uint64_t)units_per_img * P.n_images;
    const uint32_t stride = gridDim.x * K444_WARPS;
    const uint32_t d_ux = stride % P.units_x, d_t = stride / P.units_x;
    const uint32_t d_by = d_t % P.mcus_y, d_img = d_t / P.mcus_y;
    uint32_t phase = 0;  // bit b = parity to wait for on bar[b]

    auto advance = [&](uint32_t &img, uint32_t &by, uint32_t &ux) {
        ux += d_ux;
        if (ux >= P.units_x) { ux -= P.units_x; ++by; }
        by += d_by;
        if (by >= P.mcus_y) { by -= P.mcus_y; ++img; }
        img += d_img;
    };
    auto unit_by_tma = [&](uint32_t by) { return P.use_tma && (by * 8 + 8 <= P.h); };
    auto issue_tma = [&](uint32_t img_, uint32_t by_, uint32_t ux_, int b) {
        if (unit_by_tma(by_)) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(&WS.bar[b], K444_TILE_BYTES);
            tma_load_3d(WS.tile[b], &tmap, (int)(ux_ * (K444_ROW_B / 8)), (int)(by_ * 8), (int)img_, &WS.bar[b]);
        }
    };

    uint64_t u = (uint64_t)blockIdx.x * K444_WARPS + warp;
    uint32_t img, by, ux;
    {
        const uint32_t u0 = blockIdx.x * K444_WARPS + warp;
        img = u0 / units_per_img;
        const uint32_t rem = u0 - img * units_per_img;
        by = rem / P.units_x;
        ux = rem - by * P.units_x;
    }
    int b = 0;
    if (u < nunits && lane == 0) issue_tma(img, by, ux, 0);
    for (; u < nunits; u += stride, b ^= 1) {
        uint32_t img_n = img, by_n = by, ux_n = ux;
        advance(img_n, by_n, ux_n);
        if (lane == 0 && u + stride < nunits) issue_tma(img_n, by_n, ux_n, b ^ 1);  // that buffer was released below
        if (unit_by_tma(by)) {
            mbar_wait(&WS.bar[b], (phase >> b) & 1u);
            phase ^= 1u << b;
        } else {
            const uint8_t *image = P.pixels + (size_t)img * P.pixel_stride;
            warp_load_tile_rgb<8, 256>(WS.tile[b], image, P.w, P.h, ux * 256, by * 8, lane);
            __syncwarp();
        }
        const uint32_t bx0 = ux * 32;
        // Lanes past the right edge transform whatever their 24-byte columns of the tile hold (the
        // tile is always 32 blocks wide) and are dropped by the flush: the whole pass is
        // warp-convergent, which the quantiser's uniform-datapath table reads need.
        const uint8_t *base = WS.tile[b] + lane * 24;
        auto row_words = [&](int r, uint32_t (&wds)[6]) {
            const uint2 *p = reinterpret_cast<const uint2 *>(base + r * K444_ROW_B);
            const uint2 a = p[0], c1 = p[1], c2 = p[2];
            wds[0] = a.x; wds[1] = a.y; wds[2] = c1.x; wds[3] = c1.y; wds[4] = c2.x; wds[5] = c2.y;
        };
        const size_t b0 = (size_t)by * P.mcus_x + bx0;   // the unit's first block
        auto flush = [&](int16_t *arr, uint8_t *earr) {   // earr: the extents (kRecords only)
            uint4 *dbase = reinterpret_cast<uint4 *>(arr + b0 * 64);
            flush_stage<OUT>(
                WS.stage, WS.ext, lane, [](int s) { return s & 7; },
                [&](int s) -> uint4 * { return bx0 + s < P.mcus_x ? dbase + s * 8 : nullptr; },
                [&](int s) -> uint8_t * { return bx0 + s < P.mcus_x ? earr + s : nullptr; });
        };
#pragma unroll 1
        for (int comp = 0; comp < 3; ++comp) {
            const bool chroma_u = __ballot_sync(0xffffffffu, comp != 0) != 0u;   // uniform, and ptxas can tell
            f2 R[4][8];
            // the component is decided once per pass, not per pixel: straight-line fills
            if (!chroma_u) {
#pragma unroll
                for (int rp = 0; rp < 4; ++rp) {
                    float v0[8], v1[8];
                    uint32_t wa[6], wb[6];
                    row_words(rp * 2, wa); row_words(rp * 2 + 1, wb);
                    y_row8(wa, v0); y_row8(wb, v1);
#pragma unroll
                    for (int x = 0; x < 8; ++x) R[rp][x] = pk(v0[x], v1[x]);
                }
            } else {
                const uint32_t wgt = comp == 1 ? 0x0080552Bu : 0x00156B80u;
#pragma unroll
                for (int rp = 0; rp < 4; ++rp) {
                    float v0[8], v1[8];
                    uint32_t wa[6], wb[6];
                    row_words(rp * 2, wa); row_words(rp * 2 + 1, wb);
                    c_row8(wa, wgt, v0); c_row8(wb, wgt, v1);
#pragma unroll
                    for (int x = 0; x < 8; ++x) R[rp][x] = pk(v0[x], v1[x]);
                }
            }
            if constexpr (OUT == kDct) {   // the block's f32 DCT straight to its slot
                float *arr = reinterpret_cast<float *>(comp == 0 ? P.y : (comp == 1 ? P.cb : P.cr)) +
                             (size_t)img * (comp == 0 ? P.y_stride : P.c_stride);
                dct_quant_store_x2<OUT>(R, QS, chroma_u, WS.stage + lane * 8, lane & 7, &WS.ext[lane],
                                        bx0 + lane < P.mcus_x ? arr + (b0 + lane) * 64 : nullptr);
                continue;
            }
            dct_quant_store_x2<OUT>(R, QS, chroma_u, WS.stage + lane * 8, lane & 7, &WS.ext[lane]);
            uint8_t *earr = nullptr;
            if (OUT == kRecords)
                earr = (comp == 0 ? P.e.y : (comp == 1 ? P.e.cb : P.e.cr)) + ((size_t)img * P.e.stride + b0);
            flush(comp == 0 ? P.y + (size_t)img * P.y_stride : (comp == 1 ? P.cb : P.cr) + (size_t)img * P.c_stride, earr);
        }
        __syncwarp();  // every lane is done with tile[b]: the TMA issued next iteration may refill it
        img = img_n; by = by_n; ux = ux_n;
    }
}

template <int OUT>
__global__ void __launch_bounds__(64)
k_jpeg_gray(const uint8_t *__restrict__ pixels, size_t pixel_stride, uint32_t w, uint32_t h,
            uint32_t blocks_x, uint32_t tiles_x, int16_t *__restrict__ yout, size_t y_stride,
            uint8_t *__restrict__ yext, size_t e_stride, const __grid_constant__ QPairTab qp)
{
    constexpr int TB = GRAY_BLOCKS * 8;  // 512
    __shared__ __align__(16) uint8_t tile[8 * TB];
    __shared__ __align__(16) uint4 stage[2][256];
    __shared__ __align__(16) uint8_t ext[2][32];   // kRecords: the stages' record extents
    __shared__ QPairTab qsm;
    for (int i = threadIdx.x; i < 64; i += 64) qsm.t[i >> 5][i & 31] = qp.t[i >> 5][i & 31];
    const QPairTab *QS = &qsm;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tx = blockIdx.x % tiles_x;
    const uint32_t brow = blockIdx.x / tiles_x;
    const uint32_t img = blockIdx.y;
    const uint8_t *image = pixels + (size_t)img * pixel_stride;
    load_tile<1, 8, GRAY_BLOCKS * 8, 64>(tile, image, w, h, tx * (GRAY_BLOCKS * 8), brow * 8, tid);
    __syncthreads();
    const int j = tid;
    const uint32_t b0 = tx * GRAY_BLOCKS;
    {   // every lane (the tile is fully defined: load_tile replicates past the right edge; the flush drops them)
        f2 R[4][8];
#pragma unroll
        for (int rp = 0; rp < 4; ++rp) {
            const uint2 a = *reinterpret_cast<const uint2 *>(tile + (rp * 2) * TB + j * 8);
            const uint2 b = *reinterpret_cast<const uint2 *>(tile + (rp * 2 + 1) * TB + j * 8);
            const uint32_t wa[2] = {a.x, a.y}, wb[2] = {b.x, b.y};
#pragma unroll
            for (int x = 0; x < 8; ++x) {
                // gray as f32 - 128.0, src/jpeg/mod.rs:1584-1589
                const float f0 = __uint_as_float(__byte_perm(wa[x >> 2], 0x4B000000u, 0x7650 + (x & 3)));
                const float f1 = __uint_as_float(__byte_perm(wb[x >> 2], 0x4B000000u, 0x7650 + (x & 3)));
                R[rp][x] = sub2(pk(f0, f1), K2(8388736.0f));
            }
        }
        if constexpr (OUT == kDct) {   // the block's f32 DCT straight to its slot (yout is a float array)
            const uint32_t blk = b0 + j;
            dct_quant_store_x2<OUT>(R, QS, false, stage[warp] + lane * 8, lane & 7, &ext[warp][lane],
                                    blk < blocks_x ? reinterpret_cast<float *>(yout) + (size_t)img * y_stride +
                                                         ((size_t)brow * blocks_x + blk) * 64
                                                   : nullptr);
            return;
        }
        dct_quant_store_x2<OUT>(R, QS, false, stage[warp] + lane * 8, lane & 7, &ext[warp][lane]);
    }
    const uint32_t first = b0 + warp * 32;
    const size_t bfirst = (size_t)brow * blocks_x + first;
    uint4 *dbase = reinterpret_cast<uint4 *>(yout + (size_t)img * y_stride + bfirst * 64);
    flush_stage<OUT>(
        stage[warp], ext[warp], lane, [](int s) { return s & 7; },
        [&](int s) -> uint4 * { return first + s < blocks_x ? dbase + s * 8 : nullptr; },
        [&](int s) -> uint8_t * {   // kRecords only
            return first + s < blocks_x ? yext + ((size_t)img * e_stride + bfirst + s) : nullptr;
        });
}

// =========================================================================================
// K3: symbol pre-scan statistics (count_block, src/jpeg/mod.rs:826-860): per-table histograms
// of DC categories and AC (run,size) symbols over a frame, from the coefficient arrays.
// The DC predictor chain is just "previous block of the same component in scan order", which
// is the previous element of the component's array; it resets at restart boundaries
// (src/jpeg/mod.rs:1433-1443).  One thread per block; smem histograms, one global flush.
// =========================================================================================
__device__ __forceinline__ int category16(int v)
{
    const int a = v < 0 ? -v : v;
    return 32 - __clz(a);  // 0 for 0
}

// IN: the arrays' CoefOut format; kRecords reads the extents in E.
template <int IN>
__global__ void __launch_bounds__(256)
k_jpeg_hist(const int16_t *__restrict__ ycoef, size_t y_stride, const int16_t *__restrict__ cbcoef,
            const int16_t *__restrict__ crcoef, size_t c_stride, const CoefExtents E, size_t ny, size_t nc,
            uint32_t blocks_y_per_mcu, uint32_t restart_interval,
            unsigned long long *__restrict__ hist, const int seed_y, const int seed_cb, const int seed_cr)
{
    __shared__ uint32_t sh[kHistWords];
    for (int i = threadIdx.x; i < kHistWords; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const uint32_t img = blockIdx.y;
    const size_t total = ny + 2 * nc;
    for (size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x; b < total;
         b += (size_t)gridDim.x * blockDim.x) {
        const int16_t *arr;
        const uint8_t *earr;
        size_t idx;
        bool lum;
        uint32_t per_mcu;
        int seed;  // predictor before block 0: non-zero only for a band of a tiled frame
        if (b < ny) { arr = ycoef + (size_t)img * y_stride; earr = E.y; idx = b; lum = true; per_mcu = blocks_y_per_mcu; seed = seed_y; }
        else if (b < ny + nc) { arr = cbcoef + (size_t)img * c_stride; earr = E.cb; idx = b - ny; lum = false; per_mcu = 1; seed = seed_cb; }
        else { arr = crcoef + (size_t)img * c_stride; earr = E.cr; idx = b - ny - nc; lum = false; per_mcu = 1; seed = seed_cr; }
        const uint4 *src = reinterpret_cast<const uint4 *>(arr + idx * 64);
        // a record's pieces past its last written sector are undefined: zeros instead
        const int np = IN == kRecords ? 2 * __ldg(earr + ((size_t)img * E.stride + idx)) : 8;
        uint32_t wv[32];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const uint4 t = k < np ? __ldg(src + k) : make_uint4(0, 0, 0, 0);
            wv[k * 4] = t.x; wv[k * 4 + 1] = t.y; wv[k * 4 + 2] = t.z; wv[k * 4 + 3] = t.w;
        }
        // DC difference against the previous block of this component
        const size_t mcu = idx / per_mcu;
        const bool first_in_mcu = (idx % per_mcu) == 0;
        const bool reset = restart_interval && first_in_mcu && (mcu % restart_interval) == 0;
        const int prev = reset ? 0 : (idx ? (int)arr[(idx - 1) * 64] : seed);
        const int dc = (int)(int16_t)(wv[0] & 0xFFFF);
        const int diff = (int)(int16_t)(dc - prev);
        // categories past the baseline tables (DC > 11, AC > 10) are clamped to stay inside their
        // bins; such input is rejected by the entropy stage that follows (overflow bit 3)
        atomicAdd(&sh[(lum ? 0 : 12) + min(category16(diff), 11)], 1u);
        // AC: walk coefficients in zig-zag order
        uint32_t *ac = sh + (lum ? 24 : 280);
        int run = 0;
#pragma unroll
        for (int i = 1; i < 64; ++i) {
            const int nat = IN != kNatural ? i : zz_nat(i);
            const uint32_t word = wv[nat >> 1];
            const int c = (int)(int16_t)((nat & 1) ? (word >> 16) : (word & 0xFFFF));
            if (c == 0) {
                ++run;
            } else {
                if (run >= 16) { atomicAdd(&ac[0xF0], (uint32_t)(run >> 4)); run &= 15; }
                atomicAdd(&ac[(run << 4) | min(category16(c), 10)], 1u);
                run = 0;
            }
        }
        if (run > 0) atomicAdd(&ac[0], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kHistWords; i += blockDim.x)
        if (sh[i]) atomicAdd(&hist[(size_t)img * kHistWords + i], (unsigned long long)sh[i]);
}

// Table entries (-d, -d', r, r') per output word, r = RN(1/d) (see dct_quant_store_x2).
// chr_scale: the chroma block handed to the DCT is `chr_scale` x the reference's block (4 for
// 4:2:0, whose x0.25 is folded in here: power-of-two scaling commutes exactly with every rounding
// in the pipeline).
void fill_qpair_tab(const float *lum_q, const float *chr_q, float chr_scale, QPairTab *qp)
{
    for (int c = 0; c < 2; ++c) {
        const float *d = c ? chr_q : lum_q;
        const float sc = c ? chr_scale : 1.0f;
        for (int w = 0; w < 32; ++w) {
            volatile float r0 = 1.0f / d[2 * w], r1 = 1.0f / d[2 * w + 1];  // RN(1/d), kept out of x87/fast-math paths
            QPair e;
            e.nd_lo = -(d[2 * w] * sc);
            e.nd_hi = -(d[2 * w + 1] * sc);
            e.r_lo = r0 / sc;
            e.r_hi = r1 / sc;
            qp->t[c][w] = e;
        }
    }
}

}  // namespace

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *,
                                  const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn tensor_map_encoder()
{
    static const EncodeTiledFn fn = []() -> EncodeTiledFn {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess) {
            cudaGetLastError();
            return nullptr;
        }
        return reinterpret_cast<EncodeTiledFn>(p);
    }();
    return fn;
}

// 3-D view of a batch of interleaved-RGB frames for TMA: (8-byte words per row, rows, frames).
bool make_rgb_tensor_map(CUtensorMap *tm, const uint8_t *pixels, size_t pixel_stride, uint32_t n,
                         uint32_t w, uint32_t h, uint32_t box_words, uint32_t box_rows)
{
    const size_t pitch = (size_t)w * 3;
    if (pitch % 16 != 0 || (reinterpret_cast<uintptr_t>(pixels) & 15) != 0) return false;
    if (n > 1 && pixel_stride % 16 != 0) return false;
    EncodeTiledFn enc = tensor_map_encoder();
    if (!enc) return false;
    const cuuint64_t gdim[3] = {pitch / 8, h, n};
    const cuuint64_t gstr[2] = {pitch, n > 1 ? pixel_stride : pitch * h};
    const cuuint32_t box[3] = {box_words, box_rows, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 3, const_cast<uint8_t *>(pixels), gdim, gstr, box,
               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// k_jpeg_420, or k_jpeg_444 when `s444`: persistent kernels with one unit per warp in flight, so the
// grid is as many CTAs as fit on the device (the occupancy query, asked once per context, kernel and
// output format) and no more than the units need.
int launch_rgb_transform(pixo_b200_ctx *ctx, bool s444, int out, const uint8_t *px, size_t pixel_stride,
                         uint32_t n, uint32_t w, uint32_t h, int16_t *y, size_t y_stride, int16_t *cb,
                         int16_t *cr, size_t c_stride, const CoefExtents &e, const QPairTab &qt)
{
    // 4:2:0 walks MCUs of 16x16 px, 16 to a unit; 4:4:4 walks 8x8 blocks, 32 to a unit
    const uint32_t px_per = s444 ? 8 : 16, per_unit = s444 ? 32 : K1_MCUS;
    K1Params P;
    P.pixels = px; P.pixel_stride = pixel_stride; P.w = w; P.h = h;
    P.mcus_x = (w + px_per - 1) / px_per; P.mcus_y = (h + px_per - 1) / px_per;
    P.units_x = (P.mcus_x + per_unit - 1) / per_unit;
    P.n_images = n; P.y = y; P.cb = cb; P.cr = cr; P.y_stride = y_stride; P.c_stride = c_stride; P.e = e;
    alignas(64) CUtensorMap tm;
    memset(&tm, 0, sizeof tm);
    // one TMA box: half a 4:2:0 unit (8 MCUs) or a whole 4:4:4 unit, px_per rows
    P.use_tma = make_rgb_tensor_map(&tm, px, pixel_stride, n, w, h, (s444 ? K444_ROW_B : K1_HB) / 8, px_per) ? 1u : 0u;
    const int warps = s444 ? K444_WARPS : K1_WARPS;
    const size_t smem = s444 ? sizeof(K444Smem) : sizeof(K1Smem);
    void (*const k420[4])(K1Params, QPairTab, CUtensorMap) = {k_jpeg_420<kNatural>, k_jpeg_420<kZigzag>,
                                                               k_jpeg_420<kRecords>, k_jpeg_420<kDct>};
    void (*const k444[4])(K1Params, QPairTab, CUtensorMap) = {k_jpeg_444<kNatural>, k_jpeg_444<kZigzag>,
                                                               k_jpeg_444<kRecords>, k_jpeg_444<kDct>};
    auto kern = s444 ? k444[out] : k420[out];
    int &bps = ctx->kernels[reinterpret_cast<const void *>(kern)].blocks_per_sm;
    if (!bps) {
        PIXO_TRY(allow_smem(ctx, reinterpret_cast<const void *>(kern), smem));
        int nb = 0;
        PIXO_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, warps * 32, smem));
        bps = nb > 0 ? nb : 1;
    }
    const uint64_t nunits = (uint64_t)P.mcus_y * P.units_x * n;
    const uint64_t grid = std::min<uint64_t>((uint64_t)ctx->sm_count * bps, (nunits + warps - 1) / warps);
    return launch(ctx, kern, (unsigned)grid, warps * 32, smem, P, qt, tm);
}

// The extents of the frames from image i0 on (none: dense arrays)
CoefExtents extents_from(const CoefExtents *e, size_t i0)
{
    if (!e) return CoefExtents{nullptr, nullptr, nullptr, 0};
    const size_t o = i0 * e->stride;
    return CoefExtents{e->y + o, e->cb ? e->cb + o : nullptr, e->cr ? e->cr + o : nullptr, e->stride};
}

// launch_jpeg_transform / launch_jpeg_transform_dct: `out` is the CoefOut format; the arrays hold int16
// coefficients, or floats for kDct (strides in elements either way)
int transform(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride, uint32_t n_images, uint32_t w,
              uint32_t h, uint32_t color_type, uint32_t subsampling, const float *lum_q, const float *chr_q,
              int out, void *d_y_, size_t y_stride, void *d_cb_, void *d_cr_, size_t c_stride, const CoefExtents *ext)
{
    QPairTab qt;
    fill_qpair_tab(lum_q, chr_q, (color_type != PIXO_B200_GRAY && subsampling == PIXO_B200_S420) ? 4.0f : 1.0f, &qt);
    const size_t esz = out == kDct ? sizeof(float) : sizeof(int16_t);
    auto at = [esz](void *base, size_t elems) -> int16_t * {   // element offset in the arrays' own type
        return base ? reinterpret_cast<int16_t *>(static_cast<uint8_t *>(base) + elems * esz) : nullptr;
    };
    // the exact-division identity is proved for integer divisors 1..255 only
    for (int i = 0; i < 64; ++i) {
        const float a = lum_q[i], b = chr_q[i];
        if (!(a >= 1.0f && a <= 255.0f && a == (float)(int)a && b >= 1.0f && b <= 255.0f &&
              b == (float)(int)b))
            return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT,
                             "quantisation table entries must be integers in 1..255");
    }
    // frames per launch: grid.y of the gray kernel and the 32-bit unit coordinates of K1 / K2 (a
    // frame has fewer than 2^24 units: 65 535^2 px / (256 x 8))
    const uint64_t units_max = (uint64_t)((w + 7) / 8 + 31) / 32 * ((h + 7) / 8);   // K2's units; K1 has fewer
    const uint32_t per_launch = (uint32_t)std::min<uint64_t>(65535, 0xFFFFFFFFull / (units_max ? units_max : 1));
    for (uint32_t i0 = 0; i0 < n_images; i0 += per_launch) {
        const uint32_t nb = n_images - i0 < per_launch ? n_images - i0 : per_launch;
        const uint8_t *px = d_pixels + (size_t)i0 * pixel_stride;
        int16_t *y = at(d_y_, (size_t)i0 * y_stride);
        int16_t *cb = at(d_cb_, (size_t)i0 * c_stride);
        int16_t *cr = at(d_cr_, (size_t)i0 * c_stride);
        const CoefExtents e = extents_from(ext, i0);
        if (color_type == PIXO_B200_GRAY) {
            const uint32_t bx = (w + 7) / 8, by = (h + 7) / 8;
            const uint32_t tiles_x = (bx + GRAY_BLOCKS - 1) / GRAY_BLOCKS;
            dim3 grid(tiles_x * by, nb);
            void (*const kg[4])(const uint8_t *, size_t, uint32_t, uint32_t, uint32_t, uint32_t, int16_t *, size_t,
                                uint8_t *, size_t, QPairTab) = {k_jpeg_gray<kNatural>, k_jpeg_gray<kZigzag>,
                                                                 k_jpeg_gray<kRecords>, k_jpeg_gray<kDct>};
            PIXO_TRY(launch(ctx, kg[out], grid, 64, 0, px, pixel_stride, w, h, bx, tiles_x, y, y_stride, e.y, e.stride, qt));
        } else {
            PIXO_TRY(launch_rgb_transform(ctx, subsampling == PIXO_B200_S444, out, px, pixel_stride, nb, w, h, y,
                                          y_stride, cb, cr, c_stride, e, qt));
        }
    }
    return 0;
}

}  // namespace

int launch_jpeg_transform(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride,
                          uint32_t n_images, uint32_t w, uint32_t h, uint32_t color_type,
                          uint32_t subsampling, const float *lum_q, const float *chr_q,
                          int16_t *d_y, size_t y_stride, int16_t *d_cb, int16_t *d_cr,
                          size_t c_stride, uint32_t flags, const CoefExtents *ext)
{
    const int out = ext ? kRecords : (flags & PIXO_B200_COEF_ZIGZAG) ? kZigzag : kNatural;
    return transform(ctx, d_pixels, pixel_stride, n_images, w, h, color_type, subsampling, lum_q, chr_q, out, d_y,
                     y_stride, d_cb, d_cr, c_stride, ext);
}

int launch_jpeg_transform_dct(pixo_b200_ctx *ctx, const uint8_t *d_pixels, size_t pixel_stride, uint32_t n_images,
                              uint32_t w, uint32_t h, uint32_t color_type, uint32_t subsampling,
                              const float *lum_q, const float *chr_q, float *d_y, size_t y_stride, float *d_cb,
                              float *d_cr, size_t c_stride)
{
    return transform(ctx, d_pixels, pixel_stride, n_images, w, h, color_type, subsampling, lum_q, chr_q, kDct, d_y,
                     y_stride, d_cb, d_cr, c_stride, nullptr);
}

int launch_jpeg_histogram(pixo_b200_ctx *ctx, const int16_t *d_y, size_t y_stride,
                          const int16_t *d_cb, const int16_t *d_cr, size_t c_stride,
                          uint32_t n_images, size_t ny, size_t nc, uint32_t blocks_y_per_mcu,
                          uint32_t restart_interval, bool zigzag_in, const CoefExtents *ext, uint64_t *d_hist,
                          const int *dc_seed)
{
    const int s0 = dc_seed ? dc_seed[0] : 0, s1 = dc_seed ? dc_seed[1] : 0, s2 = dc_seed ? dc_seed[2] : 0;
    PIXO_CUDA(ctx, cudaMemsetAsync(d_hist, 0, (size_t)n_images * kHistWords * sizeof(uint64_t),
                                   ctx->stream));
    const size_t total = ny + 2 * nc;
    uint32_t gx = (uint32_t)((total + 255) / 256);
    const uint32_t cap = (uint32_t)ctx->sm_count * 8;
    if (gx > cap) gx = cap;
    if (gx == 0) gx = 1;
    for (uint32_t i0 = 0; i0 < n_images; i0 += 65535) {
        const uint32_t nb = n_images - i0 < 65535 ? n_images - i0 : 65535;
        dim3 grid(gx, nb);
        auto *hist = reinterpret_cast<unsigned long long *>(d_hist + (size_t)i0 * kHistWords);
        const int16_t *y = d_y + (size_t)i0 * y_stride;
        const int16_t *cb = d_cb ? d_cb + (size_t)i0 * c_stride : nullptr;
        const int16_t *cr = d_cr ? d_cr + (size_t)i0 * c_stride : nullptr;
        const CoefExtents e = extents_from(ext, i0);
        void (*const kh[3])(const int16_t *, size_t, const int16_t *, const int16_t *, size_t, CoefExtents, size_t, size_t,
                            uint32_t, uint32_t, unsigned long long *, int, int, int) = {
            k_jpeg_hist<kNatural>, k_jpeg_hist<kZigzag>, k_jpeg_hist<kRecords>};
        const int in = ext ? kRecords : zigzag_in ? kZigzag : kNatural;
        PIXO_TRY(launch(ctx, kh[in], grid, 256, 0, y, y_stride, cb, cr, c_stride, e, ny, nc, blocks_y_per_mcu,
                        restart_interval, hist, s0, s1, s2));
    }
    return 0;
}

}  // namespace pixo
