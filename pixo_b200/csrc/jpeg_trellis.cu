// jpeg_trellis.cu — k_trellis: pixo's trellis quantiser (src/jpeg/trellis.rs:67-296) for a batch of
// 8x8 blocks, bit for bit.
//
// The reference runs a Viterbi search per block over the 63 AC positions in zig-zag order: at most 8
// states (cost, zero run) survive each step, every state spawns up to 5 candidate values, children with
// the same (value, zero run) merge, a stable sort by cost keeps the cheapest 8, and the cheapest final
// state (EOB cost added where a zero run is open) is backtracked.  The candidates depend only on the
// coefficient, so the children of one step fall into a fixed set of at most 12 slots:
//     slot 0       the zero child of parent 0
//     slots 1..4   the non-zero candidates c1..c4 (zero run 0): each merges over ALL parents
//     slots 5..11  the zero children of parents 1..7, merged with an earlier parent of the same new run
// in exactly the order the reference inserts them, so (cost, slot) orders the children as the stable
// sort does.  A merge keeps the first minimum (the reference replaces only on a strictly smaller cost).
//
// Design (H100): one thread per block, the state list in registers (every loop over states, candidates
// and slots is unrolled, so all indices are static), and per thread in shared memory the block's 63 AC
// coefficients in zig-zag order plus one 64-bit back-pointer word per step (8 states x (slot, parent)).
// A thread reads and writes only its own columns, so the kernel has no barrier.  All arithmetic is
// binary32 with one rounding per operation (__fadd_rn / __fmul_rn, never contracted); the quotients
// coef / q use the transform's exact 3-op division (tools/verify_div.c: equal to the IEEE quotient for
// every integer divisor 1..255 away from underflow), which needs no slow-path call.
#include "common.cuh"

namespace pixo {
namespace {

constexpr int TR_THREADS = 64;
constexpr int TR_COL = TR_THREADS + 1;   // padded row of the coefficient / result array (bank spread)
// pixo's i16 casts saturate, and its `ceil + 1` / `floor - 1` candidate overflows i16 past this bound:
// inputs with |dct / q| above it are rejected (status bit 0) instead of guessed
constexpr float TR_FQ_MAX = 32766.0f;
// non-zero coefficients below this magnitude are rejected too: the exact division holds away from underflow
constexpr float TR_X_MIN = 7.888609052e-31f;   // 2^-100

// zig-zag position of natural index k (inverse of zz_nat)
__host__ __device__ constexpr int nat_zz(int k)
{
    constexpr int t[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42,
                           3,  8,  12, 17, 25, 30, 41, 43, 9,  11, 18, 24, 31, 40, 44, 53,
                           10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60,
                           21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};
    return t[k];
}

struct TrellisShared {
    float coef[63 * TR_COL];                 // [zz - 1][thread]: AC coefficients, then the chosen values
    unsigned long long rec[63][TR_THREADS];  // [step][thread]: byte s = (slot << 3) | parent of state s
    float rate[16 * 16];                     // estimate_ac_rate(run, cat) for a non-zero value
    float qz[64], rz[64];                    // the quantiser and its reciprocals in zig-zag order
};

// estimate_ac_huffman_length + value bits (trellis.rs:246-279), binary32 as the reference rounds it
__device__ __forceinline__ float ac_rate(int run, int cat)
{
    const int rs = (run << 4) | cat;
    float huff;
    switch (rs) {
    case 0x01: huff = 2.0f; break;
    case 0x02: huff = 2.5f; break;
    case 0x03: huff = 3.0f; break;
    case 0x04: huff = 4.0f; break;
    case 0x11: huff = 3.0f; break;
    case 0x12: huff = 4.0f; break;
    case 0x21: huff = 4.0f; break;
    default: huff = __fadd_rn(__fadd_rn(3.0f, __fmul_rn((float)run, 0.5f)), __fmul_rn((float)cat, 0.3f));
    }
    return __fadd_rn(huff, (float)cat);
}

// x / d for an integer d in 1..255 with r = RN(1/d): q0 = x*r; RN(x/d) = fma(fma(-q0, d, x), r, q0)
__device__ __forceinline__ float qdiv(float x, float d, float r)
{
    const float q0 = __fmul_rn(x, r);
    return __fmaf_rn(__fmaf_rn(-q0, d, x), r, q0);
}

__device__ __forceinline__ int category(int v)
{
    const int a = v < 0 ? -v : v;
    return 32 - __clz(a);
}

// generate_candidates (trellis.rs:210-244) without the leading 0: up to four distinct non-zero values
__device__ __forceinline__ int candidates(float fq, int (&c)[4])
{
    const int rounded = (int)roundf(fq), fl = (int)floorf(fq), ce = (int)ceilf(fq);
    int n = 0;
    c[0] = c[1] = c[2] = c[3] = 0;
    auto push = [&](int v) {
        if (v != 0 && v != c[0] && v != c[1] && v != c[2]) {
            if (n == 0) c[0] = v; else if (n == 1) c[1] = v; else if (n == 2) c[2] = v; else c[3] = v;
            ++n;
        }
    };
    push(fl);
    push(rounded);
    push(ce);
    if (fabsf(fq) > 1.5f) push(fq >= 0.0f ? ce + 1 : fl - 1);   // never a duplicate: beyond ceil / floor
    return n;
}

// One block per thread.  Block i of frame f: J.src + f * src_stride + i * 64 (natural order f32), result
// to J.dst + f * dst_stride + i * 64 (int16, natural order or zig-zag when ZZ).
struct TrellisJob {
    const float *src;
    size_t src_stride;
    int16_t *dst;
    size_t dst_stride;
    uint64_t nb;        // blocks per frame
    uint32_t n_frames;
    float lambda;
    float q[64];        // natural order, integers 1..255
    float r[64];        // RN(1 / q)
};

template <bool ZZ>
__global__ void __launch_bounds__(TR_THREADS, 1)
k_trellis(const __grid_constant__ TrellisJob J, uint32_t *__restrict__ status)
{
    extern __shared__ __align__(16) uint8_t tr_smem[];
    TrellisShared &S = *reinterpret_cast<TrellisShared *>(tr_smem);
    const int tid = threadIdx.x;
    for (int i = tid; i < 256; i += TR_THREADS) S.rate[i] = (i & 15) ? ac_rate(i >> 4, i & 15) : 0.0f;
    if (tid == 0) {   // static indices: a run-time index into the parameter would copy it to local memory
#pragma unroll
        for (int t = 0; t < 64; ++t) { S.qz[t] = J.q[zz_nat(t)]; S.rz[t] = J.r[zz_nat(t)]; }
    }
    __syncthreads();
    const uint64_t b = (uint64_t)blockIdx.x * TR_THREADS + tid;
    if (b >= J.nb * J.n_frames) return;
    const uint64_t f = b / J.nb, i = b - f * J.nb;
    const float4 *src = reinterpret_cast<const float4 *>(J.src + f * J.src_stride + i * 64);
    bool bad = false;

    // the block's AC coefficients to shared memory in zig-zag order; every input is checked here
    float dc = 0.0f;
#pragma unroll
    for (int k4 = 0; k4 < 16; ++k4) {
        const float4 v = __ldg(src + k4);
        const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            const int k = k4 * 4 + m;
            const float fq = qdiv(e[m], J.q[k], J.r[k]);
            bad |= !(fabsf(e[m]) <= 3.402823466e38f) || (e[m] != 0.0f && fabsf(e[m]) < TR_X_MIN) ||
                   !(fabsf(fq) <= TR_FQ_MAX);
            if (k == 0) dc = fq;
            else S.coef[(nat_zz(k) - 1) * TR_COL + tid] = e[m];
        }
    }
    const float lambda = J.lambda;
    const float INF = __int_as_float(0x7f800000);

    // state list: cost and zero run of states 0..n-1
    float cost[8];
    int run[8];
    int n = 1;
    cost[0] = 0.0f; run[0] = 0;
#pragma unroll
    for (int s = 1; s < 8; ++s) { cost[s] = INF; run[s] = 0; }

#pragma unroll 1
    for (int t = 1; t < 64; ++t) {
        const float coef = S.coef[(t - 1) * TR_COL + tid], q = S.qz[t];
        const float fq = qdiv(coef, q, S.rz[t]);
        int c[4];
        const int nc = candidates(fq, c);
        // distortions (coef - cand * q)^2, cand 0 first
        const float dz0 = __fsub_rn(coef, __fmul_rn(0.0f, q));
        const float lz = __fmul_rn(lambda, __fmul_rn(dz0, dz0));
        float lc[4];
        int cat[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float d = __fsub_rn(coef, __fmul_rn((float)c[j], q));
            lc[j] = __fmul_rn(lambda, __fmul_rn(d, d));
            cat[j] = category(c[j]);
        }
        // zero children: new run and cost per parent
        float zc[8];
        int zr[8];
#pragma unroll
        for (int p = 0; p < 8; ++p) {
            const int nr = run[p] + 1;
            const bool zrl = nr >= 16;
            zr[p] = zrl ? 0 : nr;
            zc[p] = __fadd_rn(__fadd_rn(cost[p], zrl ? 10.0f : 0.0f), lz);
        }
        // the 12 slots: cost, parent, valid
        float E[12];
        int P[12];
        bool V[12];
#pragma unroll
        for (int p = 0; p < 8; ++p) {
            const int slot = p == 0 ? 0 : 4 + p;
            bool leader = p < n;
#pragma unroll
            for (int o = 0; o < p; ++o) leader &= !(o < n && zr[o] == zr[p]);
            float best = zc[p];
            int bp = p;
#pragma unroll
            for (int o = p + 1; o < 8; ++o)
                if (o < n && zr[o] == zr[p] && zc[o] < best) { best = zc[o]; bp = o; }
            E[slot] = leader ? best : INF;
            P[slot] = bp;
            V[slot] = leader;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float best = INF;
            int bp = 0;
#pragma unroll
            for (int p = 0; p < 8; ++p) {
                const float e = __fadd_rn(__fadd_rn(cost[p], S.rate[(run[p] << 4) | cat[j]]), lc[j]);
                if (p < n && (p == 0 || e < best)) { best = e; bp = p; }
            }
            V[1 + j] = j < nc;
            E[1 + j] = j < nc ? best : INF;
            P[1 + j] = bp;
        }
        // stable sort by cost, keep 8: a slot's new index is its rank by (cost, slot)
        int rank[12];
        int nv = 0;
#pragma unroll
        for (int a = 0; a < 12; ++a) {
            bad |= V[a] && !(E[a] < INF);
            nv += V[a];
            int r = 0;
#pragma unroll
            for (int o = 0; o < 12; ++o)
                if (o != a) r += V[o] && (E[o] < E[a] || (E[o] == E[a] && o < a));
            rank[a] = r;
        }
        n = nv < 8 ? nv : 8;
        unsigned long long word = 0;
#pragma unroll
        for (int s = 0; s < 8; ++s) {
            float nc_ = INF;
            int nr_ = 0;
            unsigned long long by = 0;
#pragma unroll
            for (int a = 0; a < 12; ++a) {
                if (V[a] && rank[a] == s) {
                    nc_ = E[a];
                    nr_ = (a >= 1 && a <= 4) ? 0 : zr[a == 0 ? 0 : a - 4];
                    by = (unsigned long long)((a << 3) | P[a]);
                }
            }
            cost[s] = nc_;
            run[s] = nr_;
            word |= by << (8 * s);
        }
        S.rec[t - 1][tid] = word;
    }

    // EOB cost where a zero run is open, then the first minimum
    int best_s = 0;
    float best = INF;
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const float e = run[s] > 0 ? __fadd_rn(cost[s], 4.0f) : cost[s];
        if (s < n && (s == 0 || e < best)) { best = e; best_s = s; }
    }
    // backtrack; each step's value replaces its coefficient in shared memory
    int s = best_s;
#pragma unroll 1
    for (int t = 63; t >= 1; --t) {
        const unsigned long long word = S.rec[t - 1][tid];
        const int by = (int)((word >> (8 * s)) & 0xFF);
        const int slot = by >> 3;
        int v = 0;
        if (slot >= 1 && slot <= 4) {
            const float coef = S.coef[(t - 1) * TR_COL + tid];
            int c[4];
            candidates(qdiv(coef, S.qz[t], S.rz[t]), c);
            v = slot == 1 ? c[0] : slot == 2 ? c[1] : slot == 3 ? c[2] : c[3];
        }
        S.coef[(t - 1) * TR_COL + tid] = __int_as_float(v);
        s = by & 7;
    }
    if (bad) atomicOr(status, 1u);

    // (dct[0] / q[0]).round() as i16, then the block out as 8 x 16 bytes
    const int dcv = (int)roundf(dc);
    uint4 *dst = reinterpret_cast<uint4 *>(J.dst + f * J.dst_stride + i * 64);
    auto val = [&](int k) -> uint32_t {   // k: output position
        const int z = ZZ ? k : nat_zz(k);
        const int v = z == 0 ? dcv : __float_as_int(S.coef[(z - 1) * TR_COL + tid]);
        return (uint32_t)v & 0xFFFFu;
    };
#pragma unroll
    for (int k8 = 0; k8 < 8; ++k8) {
        uint32_t w[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) w[m] = val(k8 * 8 + m * 2) | (val(k8 * 8 + m * 2 + 1) << 16);
        dst[k8] = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

}  // namespace

// Blocks of `n_frames` frames, `nb` per frame, through k_trellis.  Only enqueues: status bit 0 is set
// (never cleared) for input the trellis rejects; the caller clears and reads it.
int launch_trellis(pixo_b200_ctx *ctx, const float *d_src, size_t src_stride, int16_t *d_dst, size_t dst_stride,
                   uint64_t nb, uint32_t n_frames, const float q[64], float lambda, bool zigzag, uint32_t *d_status)
{
    const uint64_t total = nb * n_frames;
    if (total == 0) return 0;
    TrellisJob J;
    J.src = d_src; J.src_stride = src_stride; J.dst = d_dst; J.dst_stride = dst_stride;
    J.nb = nb; J.n_frames = n_frames; J.lambda = lambda;
    for (int k = 0; k < 64; ++k) {
        J.q[k] = q[k];
        volatile float r = 1.0f / q[k];   // RN(1/q), kept out of x87 / fast-math paths
        J.r[k] = r;
    }
    auto kern = zigzag ? k_trellis<true> : k_trellis<false>;
    const uint64_t grid = (total + TR_THREADS - 1) / TR_THREADS;
    if (grid > 0x7FFFFFFFull) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "too many blocks for one call");
    return launch(ctx, kern, (unsigned)grid, TR_THREADS, sizeof(TrellisShared), J, d_status);
}

}  // namespace pixo
