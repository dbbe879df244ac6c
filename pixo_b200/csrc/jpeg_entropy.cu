// jpeg_entropy.cu — baseline Huffman entropy coding of the quantised coefficient arrays ON the
// GPU (SURVEY.md §8f rank 1), so that only finished scan bytes cross PCIe.
//
// Restates the bit stream of pixo's sequential coder byte for byte:
//   encode_block            src/jpeg/huffman.rs:423-481 (DC diff, (run,size) symbols, ZRL, EOB)
//   category / encode_value src/jpeg/huffman.rs:394-418
//   BitWriterMsb            src/bits.rs:195-290 (MSB-first, 0xFF -> 0xFF00 stuffing, 1-padding)
//   encode_scan             src/jpeg/mod.rs:1408-1563 (scan order: Y..,Cb,Cr per MCU)
//
// One kernel, one pass over the coefficients (k_huff).  The DC predictor of a block is the
// previous block of the same component in the coefficient array, so every block's code is
// independent of the others; only its POSITION in the stream is not.  The kernel is persistent
// and every warp works alone (warp-level synchronisation only): it draws a unit of 96
// consecutive blocks (scan order, whole MCUs) of one image from a ticket counter, then
//   1. codes them in three passes of one block per lane, each pass of one component, every block
//      once into a private shared-memory slot; a 64-bit non-zero mask drives the symbol loop, so the
//      loop runs once per non-zero coefficient and there is a single, small copy of the symbol code.
//      The encode paths hand over the transform's coefficient records (CoefExtents, common.cuh):
//      the lane loads the block's extent, then only the 32-byte sectors the transform wrote, already
//      in zig-zag order.  Caller arrays (the CHECK instantiations) are dense and in natural order:
//      the zig-zag reorder happens in registers on the way in.  Either way the mask is computed from
//      the words;
//   2. the 96 bit lengths are scanned in scan order; the unit total enters a decoupled look-back
//      chain (one status word per unit: bit count + the unit's last 7 bits), which yields the
//      unit's bit offset in the image's stream and the partial byte it inherits;
//   3. the slots are funnel-shifted into a shared window aligned to the stream's 32-bit words;
//   4. the unit owns every byte whose last bit it wrote.  It counts its 0xFF bytes, a second
//      look-back chain turns those counts into the number of stuffed zeros before the unit, and
//      the assembled bytes, parked meanwhile in a per-warp global buffer, are copied out with the
//      0x00s inserted, 16 bytes per store.
// One ticket, two look-backs and one window sweep serve 96 blocks.  Tickets are dispensed
// unit-major across the images of a batch, so their chains advance side by side.  Restart intervals
// (handle_restart, src/jpeg/mod.rs:1423-1445) run here too: every interval is a bit stream of its
// own (units never straddle one, chain 1 restarts with it, its last unit pads and appends the
// RSTn marker), while chain 2 - every byte written so far - runs across the whole image.
#include <type_traits>

#include "common.cuh"
#include "jpeg_host.hpp"

namespace pixo {
namespace {

// Huffman tables as the symbol loop wants them: one word per symbol,
//   entry = (code << (32 - len)) | (len + cat),   cat = symbol & 15 (AC) or the DC category
// i.e. the code left-aligned in the upper half-word and the total field width (code + amplitude
// bits) in the low five bits.
// AC entries sit at word  run * 12 + (cat - 1)  (cat 1..10): the 32 entries a warp asks for most
// (run < 8, cat <= 4) fall into 32 different shared-memory banks, so the per-symbol lookup is
// conflict-free for typical blocks (the plain run * 16 + cat layout put runs 0/2/4/6 on the same
// banks).  ZRL and EOB follow the grid.
constexpr int AC_STRIDE = 12, AC_ZRL = 190, AC_EOB = 191, AC_WORDS = 192;
struct HuffDev {
    uint32_t dc[2][12];
    uint32_t ac[2][AC_WORDS];
};
static_assert(sizeof(HuffDev) == kHuffDevBytes, "common.cuh sizes the per-frame tables by kHuffDevBytes");
// One component's half of a HuffDev (dc[k], ac[k]): what a warp of k_huff<.., TABLES> keeps of its frame's tables
struct HuffHalf {
    uint32_t dc[12];
    uint32_t ac[AC_WORDS];
};
struct FrameTables {   // k_huff<.., TABLES>'s tables: frame i's at tabs[i]
    const HuffDev *tabs;
};

struct EntParams {
    const int16_t *y, *cb, *cr;    // CHECK: blocks in natural order, as compute_all_coefficients returns them;
                                   // else the transform's coefficient records, with their extents in e
    size_t y_stride, c_stride;     // int16 elements between images
    CoefExtents e;
    uint32_t bpm;                  // blocks per MCU in scan order: 6 (4:2:0), 3 (4:4:4), 1 (gray)
    uint32_t y_per_mcu;            // 4, 1, 1
    uint32_t nblocks;              // per image, scan order
    uint32_t nunits;               // per image
    uint32_t rst_mcus;             // restart interval in MCUs, 0 = none (a unit never straddles an interval)
    uint32_t rst_blocks;           // ... in blocks
    uint32_t upi;                  // units per full interval
    uint32_t nimages;
    unsigned long long *st_bits;   // [n][nunits] look-back chain 1: stream bits
    unsigned long long *st_ff;     // [n][nunits] look-back chain 2: 0xFF bytes
    uint32_t *ticket;              // unit dispenser (launch order == dependency order)
    uint8_t *out;                  // [n][out_cap]
    uint64_t out_cap;
    uint64_t *out_len;             // [n] final byte count
    // RAW + segments: every image is cut into seg_per_img runs of whole MCUs, each coded as a bit
    // string of its own ("pseudo image" q = image * seg_per_img + segment: status words, raw buffer,
    // bit count and tail are all indexed by q); k_seg_* splice them afterwards.  0/1 = not segmented.
    uint32_t seg_per_img;
    uint32_t nblocks_last;         // blocks of an image's last segment (the others have nblocks)
    size_t seg_y_stride, seg_c_stride;   // int16 elements between the segments of an image
    uint8_t *win;                  // !RAW: [grid * HUFF_WARPS][GWIN_B] each warp's assembled unit, from phase A to B
    const int *dc_seed_dev;        // the same three predictors in device memory (stream-ordered callers), or null
    int dc_seed[3];                // DC predictors (Y, Cb, Cr) before block 0: 0 for a whole image, the previous
                                   // band's last DCs when the arrays are one band of a frame tiled over several GPUs
    unsigned long long *out_tail;  // RAW only: [n] the stream's last 7 bits
    uint32_t *overflow;            // [n] bit 0: out_cap was exceeded (out_len = the size needed); bit 1: a chain timed out;
                                   // bit 3: a coefficient outside the baseline range (see code_block)
};

constexpr int CB = 32;             // blocks coded side by side == one warp
static_assert(CB * 4 == 128, "the slot word stride is spelled out in code_block's PTX");
constexpr int NPASS = 3;           // passes of 32 blocks per unit
constexpr int UB = NPASS * CB;     // blocks per unit: 16 MCUs of 4:2:0, 32 of 4:4:4, 96 gray blocks
constexpr int HUFF_WARPS = 4;      // warps per CTA (they only share the tables)
constexpr int HUFF_CTAS_PER_SM = 5;
constexpr int SLOT_W = 16;         // words of a block's code kept in shared memory (16: 512 bits)
constexpr int MAX_W = 54;          // worst case: 27 + 63 * 26 = 1665 bits
constexpr int SUB_W = 256;         // window words per emitted piece (32 bytes per lane)
constexpr int SUB_B = SUB_W * 4;
constexpr int WIN_W = 1024;        // stream words assembled per round (the stage: a q80 noise unit, ~2.8 KB, in one)
constexpr int WIN_B = WIN_W * 4;
constexpr int SBUF_B = 2 * SUB_B + 48;    // stuffed bytes of a piece + alignment slack + the head pad
constexpr int GWIN_B = 20 * SUB_B;        // a warp's assembled unit in global memory, whole pieces
static_assert(UB * 1665 / 8 + 8 <= GWIN_B, "the longest unit (every block 1665 bits) + its head and padding bytes");
static_assert(WIN_B % SUB_B == 0 && GWIN_B % WIN_B == 0, "rounds hold whole pieces, the parked unit whole rounds");
constexpr uint32_t SPIN_LIMIT = 1u << 22;
constexpr int LB_GROUPS = 4;       // look-back window: 32 * LB_GROUPS predecessors per step

constexpr unsigned long long ST_AGG = 1ull << 62, ST_PFX = 2ull << 62;
constexpr unsigned long long ST_VAL = (1ull << 55) - 1;

__device__ __forceinline__ unsigned long long ld_status(const unsigned long long *p)
{
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_status(unsigned long long *p, unsigned long long v)
{
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long pack_status(unsigned long long flag, uint32_t tail,
                                                          unsigned long long value)
{
    return flag | ((unsigned long long)(tail & 0x7F) << 55) | (value & ST_VAL);
}

// Exclusive prefix over units [0, chunk) of one image (whole warp; decoupled look-back, 128
// predecessors per step, four per lane).  tail_in = the 7-bit tail published by unit chunk-1.
// Returns the prefix in the low 55 bits, tail_in in bits 55..61, bit 62 = the chain timed out.
// (Inlined at both call sites.)
__device__ __forceinline__ unsigned long long look_back(const unsigned long long *st, int chunk, int lane)
{
    unsigned long long excl = 0;
    uint32_t tl = 0, spins = 0;
    bool first = true, fault = false;
    int base = chunk - 1;
    // Chunks finish roughly in ticket order: wait (one lane, sleeping) until the nearest
    // predecessor has published, then the wide scan below almost never has to retry.
    if (lane == 0) {
        while ((ld_status(st + base) >> 62) == 0) {
            if (++spins > SPIN_LIMIT) break;
            __nanosleep(100);
        }
    }
    __syncwarp();
    while (base >= 0) {
        unsigned long long v[LB_GROUPS];
        const unsigned long long *p = st + (base - lane);
#pragma unroll
        for (int k = 0; k < LB_GROUPS; ++k) v[k] = base - lane - 32 * k >= 0 ? ld_status(p - 32 * k) : ST_PFX;
        unsigned long long step = 0;
        bool retry = false, done = false;
#pragma unroll
        for (int k = 0; k < LB_GROUPS; ++k) {
            const uint32_t flag = (uint32_t)(v[k] >> 62);
            const uint32_t inv = __ballot_sync(0xffffffffu, flag == 0);
            const uint32_t pm = __ballot_sync(0xffffffffu, flag == 2);
            const int stop = pm ? __ffs(pm) - 1 : 32;           // nearest inclusive prefix, if any
            if (inv & ((2u << min(stop, 31)) - 1u)) { retry = true; break; }
            // aggregates are small (a unit's bits / bytes, < 2^18): one 32-bit warp reduction
            step += __reduce_add_sync(0xffffffffu, lane < stop ? (uint32_t)v[k] : 0u);
            if (pm) { step += __shfl_sync(0xffffffffu, v[k], stop) & ST_VAL; done = true; break; }
        }
        if (retry) {
            if (++spins > SPIN_LIMIT) { fault = true; break; }
            __nanosleep(20);
            continue;
        }
        excl += step;
        if (first) { tl = __shfl_sync(0xffffffffu, (uint32_t)(v[0] >> 55) & 0x7Fu, 0); first = false; }
        if (done) break;
        base -= 32 * LB_GROUPS;
    }
    return (excl & ST_VAL) | ((unsigned long long)tl << 55) | (fault ? 1ull << 62 : 0ull);
}

// bits 0..15 -> even positions, bits 16..31 -> odd positions (outer perfect shuffle)
__device__ __forceinline__ uint32_t interleave16(uint32_t x)
{
    uint32_t t;
    t = (x ^ (x >> 8)) & 0x0000FF00u; x ^= t ^ (t << 8);
    t = (x ^ (x >> 4)) & 0x00F000F0u; x ^= t ^ (t << 4);
    t = (x ^ (x >> 2)) & 0x0C0C0C0Cu; x ^= t ^ (t << 2);
    t = (x ^ (x >> 1)) & 0x22222222u; x ^= t ^ (t << 1);
    return x;
}

// 0x80 in every byte of w that equals 0xFF
__device__ __forceinline__ uint32_t ff_bytes(uint32_t w)
{
    return ((w & 0x7F7F7F7Fu) + 0x01010101u) & w & 0x80808080u;
}

// ---- the symbol loop -------------------------------------------------------------------------
__device__ __forceinline__ int lds_s16(uint32_t a)
{
    int v;
    asm volatile("ld.shared.s16 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t a)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v)
{
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v));
}
__device__ __forceinline__ uint32_t msb_index(uint32_t v)  // FLO: 31 - clz, v != 0
{
    uint32_t r;
    asm("bfind.u32 %0, %1;" : "=r"(r) : "r"(v));
    return r;
}

// Codes one block (encode_block, src/jpeg/huffman.rs:423-481) into 32-bit words
//   word k -> shared [sa_slot + k * CB * 4] for k < SLOT_W; SPILL: later words -> spill[k - SLOT_W],
//   !SPILL: later words are dropped (the caller sees the length and runs the SPILL variant).
// Pending bits are kept left-aligned in `acc`; a symbol arrives left-aligned too (vl, n bits).
// Returns the block's length in bits; *acc_out = the last, partial word (left-aligned).
// CHECK (caller coefficients; pixels cannot produce anything else): a DC difference of category > 11
// or an AC value of category > 10 has no baseline code, so its category is clamped (no table is read
// outside its entries, the length stays <= MAX_W words) and *bad is set; the caller reports the block
// instead of using its bits.  Off, the loop is a few instructions per symbol shorter.
template <bool SPILL, bool CHECK>
__device__ __forceinline__ uint32_t code_block(uint32_t M0, uint32_t M1, int diff, const uint32_t *dctab,
                                               uint32_t sa_ac, uint32_t sa_stage, uint32_t sa_slot,
                                               uint32_t *spill, uint32_t *acc_out, bool *bad)
{
    uint32_t acc = 0, filled = 0;
    uint32_t sp = sa_slot;
    const uint32_t sp_end = sa_slot + SLOT_W * CB * 4;
    auto put = [&](uint32_t vl, uint32_t n) {
        if (!SPILL) {  // branch-free: a full word is stored under a predicate
            asm volatile(
                "{\n\t"
                ".reg .pred p, q;\n\t"
                ".reg .b32 t, hi, lo, tot;\n\t"
                "shr.b32 t, %4, %1;\n\t"
                "or.b32 hi, %0, t;\n\t"
                "shf.r.wrap.b32 lo, 0, %4, %1;\n\t"   // vl << (32 - filled); 0 when filled == 0
                "add.u32 tot, %1, %5;\n\t"
                "setp.ge.u32 p, tot, 32;\n\t"
                "setp.lt.and.u32 q, %2, %3, p;\n\t"
                "@q st.shared.u32 [%2], hi;\n\t"
                "@p add.u32 %2, %2, 128;\n\t"
                "selp.b32 %0, lo, hi, p;\n\t"
                "and.b32 %1, tot, 31;\n\t"
                "}"
                : "+r"(acc), "+r"(filled), "+r"(sp)
                : "r"(sp_end), "r"(vl), "r"(n));
            return;
        }
        const uint32_t hi = acc | (vl >> filled);
        const uint32_t lo = __funnelshift_r(0u, vl, filled);  // vl << (32 - filled); 0 when filled == 0
        const uint32_t total = filled + n;
        if (total >= 32u) {
            if (sp < sp_end) sts_u32(sp, hi);
            else if (SPILL) spill[(sp - sp_end) / (CB * 4)] = hi;
            sp += CB * 4;
            acc = lo;
        } else {
            acc = hi;
        }
        filled = total & 31u;
    };
    {   // DC difference
        const uint32_t a = (uint32_t)abs(diff);
        const uint32_t cat = CHECK ? min(32u - (uint32_t)__clz(a), 11u) : 32u - (uint32_t)__clz(a);
        const uint32_t e = dctab[cat];
        const uint32_t amp = a ^ (((1u << cat) - 1u) & (uint32_t)(diff >> 31));
        const uint32_t n = e & 31u;
        put((e & 0xFFFF0000u) | (n ? amp << (32u - n) : 0u), n);
    }
    const uint32_t zrl = lds_u32(sa_ac + AC_ZRL * 4), eob = lds_u32(sa_ac + AC_EOB * 4);
    uint32_t nprev = ~0u;  // -(previous position) - 1
    uint32_t amax = CHECK ? (uint32_t)abs(diff) >> 11 : 0u;   // non-zero: a value has no code (DC > 2047, AC > 1023)
    // (no constants live across the loop: at 80 registers ptxas re-materialises them every
    // iteration - the single-bit mask comes from BMSK, the amplitude mask from a shifted sign)
    const uint32_t sa_ac_top = sa_ac + 31u * 4u;   // entry of (run, cat) = sa_ac_top + run*48 - clz(|c|)*4
#pragma unroll 1
    for (int half = 0; half < 2; ++half) {
        uint32_t mb = __brev(half ? M1 : (M0 & ~1u));  // scan order == descending bit index
        const uint32_t top = half * 32 + 31;
        while (mb) {
            const uint32_t f = msb_index(mb);
            uint32_t bit;
            asm("bmsk.clamp.b32 %0, %1, 1;" : "=r"(bit) : "r"(f));   // 1 << f
            mb ^= bit;
            const uint32_t pos = top - f;
            uint32_t run = pos + nprev;
            nprev = ~pos;
            // coefficient pos sits at stage word pos >> 1, half-word pos & 1:
            // address = stage + pos * 64 - (pos & 1) * 62, spelled as two multiply-adds
            uint32_t caddr;
            asm("{\n\t.reg .b32 h, x;\n\tand.b32 h, %1, 1;\n\tmad.lo.u32 x, %1, 64, %2;\n\tmad.lo.u32 %0, h, -62, x;\n\t}"
                : "=r"(caddr) : "r"(pos), "r"(sa_stage));
            const int c = lds_s16(caddr);
#pragma unroll 1
            while (run >= 16u) { put(zrl & 0xFFFF0000u, zrl & 31u); run -= 16u; }  // rare: keep it small
            const uint32_t a = (uint32_t)abs(c);
            if (CHECK) amax |= a >> 10;
            const uint32_t lz = CHECK ? max((uint32_t)__clz((int)a), 22u) : (uint32_t)__clz((int)a);   // 32 - cat
            const uint32_t e = lds_u32(sa_ac_top + run * (AC_STRIDE * 4u) - lz * 4u);
            const uint32_t amp = a ^ ((uint32_t)(c >> 31) >> lz);     // c >= 0: c; c < 0: (c - 1) masked to cat bits
            const uint32_t n = e & 31u;
            put((e & 0xFFFF0000u) | __funnelshift_r(0u, amp, n), n);   // amp << (32 - n), 2 <= n <= 26
        }
    }
    if (nprev != ~63u) put(eob & 0xFFFF0000u, eob & 31u);
    *acc_out = acc;
    *bad = amax != 0;
    return ((sp - sa_slot) / (CB * 4)) * 32u + filled;
}

// warp-wide exclusive scan; *total = sum over the warp
__device__ __forceinline__ uint32_t warp_scan(uint32_t x, int lane, uint32_t *total)
{
    uint32_t inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t n = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += n;
    }
    *total = __shfl_sync(0xffffffffu, inc, 31);
    return inc - x;
}

// Shared memory of one warp.  The coefficient stage is dead once a unit's blocks are coded; the
// blocks' lengths and offsets (scan order), the stream window of phase A and the stuffed bytes of
// phase B reuse it.
struct WarpMem {
    uint32_t slot[NPASS][SLOT_W * CB];     // slot[p]: the codes of pass p, word k of lane l at k * CB + l
    union {
        uint32_t stage[32 * CB];           // one pass's coefficients, word j of lane l at j * CB + l
        uint32_t tl[2 * UB];               // [0, UB): (length << 7) | last 7 bits, then [UB, 2 UB): bit offsets
        uint32_t obuf[WIN_W];
        uint8_t sbuf[SBUF_B];
    };
};

// What a warp remembers about a unit between its phases (lane-private unless noted).
struct UnitState {
    uint32_t unit, img;    // uniform
    uint32_t L[NPASS];     // this lane's block of pass p: code length,
    uint32_t o_t[NPASS];   // ... bit offset inside the unit,
    int nwt[NPASS];        // ... words it occupies
    uint32_t Lc, ctail;    // uniform: unit bits, its last 7 bits
    unsigned long long Pc; // uniform: bits before the unit (after phase A)
    uint32_t tailin;       // uniform: the 7 bits before the unit
    uint32_t own;          // uniform: output bytes the unit writes (owned + stuffed zeros + RSTn marker)
    uint32_t marker;       // uniform: 0xD0..0xD7 when the unit closes a restart interval, else 0
    bool first, last, final_; // uniform: first / last unit of its bit stream (image or interval); last of the image
    bool fault;
    bool skip;             // uniform: the unit lies past the end of a short last segment: nothing to do
};

// Persistent kernel; every WARP works on its own: it draws units of 96 blocks (whole MCUs of one
// image, in scan order) from the ticket counter and takes each through three phases with
// warp-level synchronisation only,
//   W  code the blocks into slots, publish the unit's bit count               (chain 1)
//   A  look back for the bit offset, assemble + count 0xFF, publish the count  (chain 2)
//   B  look back for the stuffed-byte offset, emit
// software-pipelined as  A(j) W(j+1) B(j):  a look-back runs a phase after the value it depends
// on was published by this warp's neighbours in the chain, so it seldom has to wait for them.
// A assembles the unit once, in windows of WIN_B bytes in shared memory, and parks the bytes in the
// warp's piece of P.win (L2-resident: a few KB per warp), where B reads them back while W(j+1)
// reuses the slots and the stage.
//
// W codes a unit in three passes of one block per lane, each pass of one component (so the
// Huffman table is the same across the warp and the lanes' symbol loops are of similar length):
//   4:2:0  Y of MCUs 0-7 | Y of MCUs 8-15 | Cb (lanes 0-15), Cr (lanes 16-31) of MCUs 0-15
//   4:4:4  Y | Cb | Cr of MCUs 0-31
//   gray   blocks 0-31 | 32-63 | 64-95
// The blocks' bit offsets come from a scan over the 96 lengths in scan order, so the assembly
// puts every block where the sequential coder would.
//
// RAW (the segments of a long image, or of a band of a frame that is tiled over several GPUs): the
// string starts at a bit of the stream that is not known yet, so nothing that depends on
// byte alignment can happen here.  Phase A writes the UNSTUFFED bytes of the local string
// (bit 0 = its first bit, the last partial byte zero-filled, no 1-padding) straight from the
// assembled windows, phase B and chain 2 do not exist, and the final unit reports the string's
// bit count and its last 7 bits.  k_seg_* below splice such strings into scan bytes once their
// bit offsets are known.
// CHECK: see code_block; a block with a coefficient outside the baseline range sets overflow bit 3.
// TABLES: every frame has tables of its own, Tp.tabs[frame] (k_huff_tables; a segment's frame is q / seg_per_img).  A warp keeps the half of them that its current pass codes with (HuffHalf, 816 bytes) and
// loads it again when the frame or the component changes: a whole HuffDev per warp would take the CTA to
// 47.5 KB of shared memory, and five CTAs per SM would no longer fit.
template <bool RAW, bool CHECK, bool TABLES>
__global__ void __launch_bounds__(32 * HUFF_WARPS, HUFF_CTAS_PER_SM)
k_huff(const __grid_constant__ EntParams P, const __grid_constant__ std::conditional_t<TABLES, FrameTables, HuffDev> Tp)
{
    __shared__ std::conditional_t<TABLES, HuffHalf[HUFF_WARPS], HuffDev> T;
    __shared__ __align__(16) WarpMem wmem[HUFF_WARPS];
    static_assert(SBUF_B <= sizeof(((WarpMem *)0)->stage), "the stuffed bytes must fit the stage");

    const int lane = threadIdx.x & 31;
    if constexpr (!TABLES) {
        for (int i = threadIdx.x; i < (int)(sizeof(HuffDev) / 4); i += blockDim.x)
            reinterpret_cast<uint32_t *>(&T)[i] = reinterpret_cast<const uint32_t *>(&Tp)[i];
        __syncthreads();
    }
    uint32_t tab_key = ~0u;   // TABLES: frame * 2 + half of the warp's copy (uniform)
    WarpMem &M = wmem[threadIdx.x >> 5];
    uint32_t *const obuf = M.obuf;
    uint8_t *const sbuf = M.sbuf;
    uint8_t *const gwin = RAW ? nullptr : P.win + ((size_t)blockIdx.x * HUFF_WARPS + (threadIdx.x >> 5)) * GWIN_B;
    const uint32_t sa_stage = (uint32_t)__cvta_generic_to_shared(M.stage) + 4u * lane;
    const uint32_t total_units = P.nunits * P.nimages;
    uint32_t spill[NPASS][MAX_W - SLOT_W];  // words beyond SLOT_W (long blocks): local memory

    // ---- W: code the unit's blocks into the slots, publish the bit count ------------------------------
    auto phase_w = [&](uint32_t id, UnitState &C) {
        // unit-major dispensing: the n images' chains advance side by side
        C.unit = id / P.nimages;
        C.img = id - C.unit * P.nimages;
        C.fault = false;
        // the unit's place: with a restart interval every interval is its own bit stream
        // (handle_restart, src/jpeg/mod.rs:1423-1445) and is cut into units separately
        uint32_t s0, iend, interval = 0;
        uint32_t nblk = P.nblocks;
        size_t y_off = (size_t)C.img * P.y_stride, c_off = (size_t)C.img * P.c_stride;
        size_t ey_off = (size_t)C.img * P.e.stride, ec_off = ey_off;   // the same blocks' extents
        bool seg_prev = false;     // block 0 continues the previous segment's DC chain
        if (RAW && P.seg_per_img > 1) {
            const uint32_t ii = C.img / P.seg_per_img, seg = C.img - ii * P.seg_per_img;
            y_off = (size_t)ii * P.y_stride + (size_t)seg * P.seg_y_stride;
            c_off = (size_t)ii * P.c_stride + (size_t)seg * P.seg_c_stride;
            ey_off = (size_t)ii * P.e.stride + (size_t)seg * (P.seg_y_stride / 64);
            ec_off = (size_t)ii * P.e.stride + (size_t)seg * (P.seg_c_stride / 64);
            if (seg == P.seg_per_img - 1) nblk = P.nblocks_last;
            seg_prev = seg != 0;
        }
        C.skip = false;
        if (P.rst_blocks) {
            interval = C.unit / P.upi;
            const uint32_t sub = C.unit - interval * P.upi;
            s0 = interval * P.rst_blocks + sub * UB;
            iend = (uint32_t)min((unsigned long long)(interval + 1) * P.rst_blocks, (unsigned long long)nblk);
            C.first = sub == 0;
        } else {
            s0 = C.unit * UB;
            iend = nblk;
            C.first = C.unit == 0;
        }
        if (s0 >= iend) { C.skip = true; return; }   // short last segment: no such unit
        C.last = s0 + UB >= iend;
        C.final_ = C.last && iend == nblk;
        C.marker = (C.last && !C.final_) ? 0xD0u + (interval & 7u) : 0u;
        // units, intervals and segments are whole MCUs: a short unit has empty lanes
        const uint32_t nv = min((uint32_t)UB, iend - s0);
        const uint32_t bpm = P.bpm, ypm = P.y_per_mcu, mu0 = s0 / bpm;
        uint32_t srel[NPASS], t7[NPASS];
#pragma unroll 1
        for (int p = 0; p < NPASS; ++p) {
            uint32_t mm, kk, comp;   // this lane's block: MCU inside the unit, place inside the MCU, component
            if (ypm == 4) {
                if (p < 2) { mm = 8 * p + (lane >> 2); kk = lane & 3; comp = 0; }
                else { mm = lane & 15; kk = 4 + (lane >> 4); comp = 1 + (lane >> 4); }
            } else if (bpm == 3) {
                mm = lane; kk = p; comp = p;
            } else {
                mm = 32 * p + lane; kk = 0; comp = 0;
            }
            const uint32_t sr = mm * bpm + kk;   // scan position inside the unit
            const bool valid = sr < nv;
            uint32_t *const slot = M.slot[p];
            uint32_t L = 0, tail7 = 0;
            int nwt = 0;
            if (__any_sync(0xffffffffu, valid)) {   // (a short last unit may leave a whole pass empty)
                if constexpr (TABLES) {   // the pass's half of its frame's tables (comp ? 1 : 0 is the same in every lane)
                    const uint32_t half = comp ? 1u : 0u;
                    const uint32_t key = ((RAW && P.seg_per_img > 1) ? C.img / P.seg_per_img : C.img) * 2u + half;
                    if (key != tab_key) {
                        const uint32_t *src = reinterpret_cast<const uint32_t *>(Tp.tabs + (key >> 1));
                        uint32_t *dst = reinterpret_cast<uint32_t *>(&T[threadIdx.x >> 5]);
                        __syncwarp();   // every lane is done with the previous half
                        for (int i = lane; i < 12 + AC_WORDS; i += 32)
                            dst[i] = __ldg(src + (i < 12 ? half * 12 + i : 24 + half * AC_WORDS + (i - 12)));
                        __syncwarp();
                        tab_key = key;
                    }
                }
                const uint32_t m = mu0 + mm;
                const int16_t *arr;
                const uint8_t *earr;   // !CHECK: the array's extents (P.e is null otherwise)
                size_t idx, eidx;
                int seed;
                if (comp == 0) { arr = P.y + y_off; earr = P.e.y; idx = (size_t)m * ypm + kk; eidx = ey_off + idx; seed = P.dc_seed[0]; }
                else if (comp == 1) { arr = P.cb + c_off; earr = P.e.cb; idx = m; eidx = ec_off + idx; seed = P.dc_seed[1]; }
                else { arr = P.cr + c_off; earr = P.e.cr; idx = m; eidx = ec_off + idx; seed = P.dc_seed[2]; }
                // The DC predictor is the previous block of the same component, which the lane to the
                // left codes in this pass - except at lane 0 and at the first Cr lane of 4:2:0: those
                // load it (or reset it: a restart interval's first MCU, src/jpeg/mod.rs:1433-1443).
                const bool from_left = lane != 0 && !(ypm == 4 && p == 2 && lane == 16);
                int prev_ld = 0;
                if (valid && !from_left) {
                    const bool dc_reset = P.rst_mcus && C.first && mm == 0;
                    // (a later segment's first block follows the previous segment's last one in the same array)
                    if (P.dc_seed_dev && idx == 0 && !seg_prev) seed = P.dc_seed_dev[comp];
                    prev_ld = dc_reset ? 0 : ((idx || seg_prev) ? arr[((long long)idx - 1) * 64] : seed);
                }
                int dc = 0;
                uint32_t M0 = 0, M1 = 0;
                if (valid) {
                    const uint4 *src = reinterpret_cast<const uint4 *>(arr + idx * 64);
                    uint32_t w[32];  // the block in zig-zag order: word j = coefficients zz(2j), zz(2j+1)
                    if (CHECK) {
                        uint32_t n[32];  // the caller's block: natural order, two coefficients per word
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            const uint4 v = __ldg(src + q);
                            n[q * 4] = v.x; n[q * 4 + 1] = v.y; n[q * 4 + 2] = v.z; n[q * 4 + 3] = v.w;
                        }
                        dc = (int)(int16_t)(n[0] & 0xFFFF);
                        // zig-zag reorder (zigzag_reorder, src/jpeg/quantize.rs:107-113) on the way into the
                        // stage; all indices are compile-time
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int i0 = zz_nat(2 * j), i1 = zz_nat(2 * j + 1);
                            w[j] = __byte_perm(n[i0 >> 1], n[i1 >> 1],
                                               ((i0 & 1) ? 0x0032 : 0x0010) | ((i1 & 1) ? 0x7600 : 0x5400));
                        }
#pragma unroll
                        for (int j = 0; j < 32; ++j) M.stage[j * CB + lane] = w[j];
                    } else {
                        // the transform's record, already in zig-zag order: its written sectors (sector 0 is
                        // always there, so its load does not wait for the extent), zeros for the rest.  The
                        // symbol loop reads only the stage words of non-zero coefficients, so only the
                        // record's words are staged.
                        const int np = 2 * __ldg(earr + eidx);
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            const uint4 v = (q < 2 || q < np) ? __ldg(src + q) : make_uint4(0, 0, 0, 0);
                            w[q * 4] = v.x; w[q * 4 + 1] = v.y; w[q * 4 + 2] = v.z; w[q * 4 + 3] = v.w;
                        }
                        dc = (int)(int16_t)(w[0] & 0xFFFF);
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            if (q < 2 || q < np) {
#pragma unroll
                                for (int t = 0; t < 4; ++t) M.stage[(q * 4 + t) * CB + lane] = w[q * 4 + t];
                            }
                        }
                    }
                    asm volatile("" ::: "memory");  // the stage is read back through ld.shared below
                    {   // bit i = zig-zag coefficient i != 0
                        uint32_t e0 = 0, e1 = 0;
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            e0 += __vminu2(w[j], 0x00010001u) * (1u << j);       // disjoint bits: + is |
                            e1 += __vminu2(w[16 + j], 0x00010001u) * (1u << j);
                        }
                        M0 = interleave16(e0); M1 = interleave16(e1);
                    }
                }
                const int left = __shfl_up_sync(0xffffffffu, dc, 1);
                const int diff = (int)(int16_t)(dc - (from_left ? left : prev_ld));
                if (valid) {
                    const int tbl = comp ? 1 : 0;   // the same in every lane of the pass
                    const uint32_t *dctab;
                    uint32_t sa_ac;
                    if constexpr (TABLES) {
                        dctab = T[threadIdx.x >> 5].dc;
                        sa_ac = (uint32_t)__cvta_generic_to_shared(&T[threadIdx.x >> 5].ac[0]);
                    } else {
                        dctab = T.dc[tbl];
                        sa_ac = (uint32_t)__cvta_generic_to_shared(&T.ac[tbl][0]);
                    }
                    const uint32_t sa_slot = (uint32_t)__cvta_generic_to_shared(slot) + 4u * lane;
                    uint32_t acc;
                    bool bad;
                    L = code_block<false, CHECK>(M0, M1, diff, dctab, sa_ac, sa_stage, sa_slot, spill[p], &acc, &bad);
                    if (L > SLOT_W * 32u)  // long block: run again, keeping the words past the slot in local memory
                        L = code_block<true, CHECK>(M0, M1, diff, dctab, sa_ac, sa_stage, sa_slot, spill[p], &acc, &bad);
                    if (CHECK && bad) atomicOr(&P.overflow[C.img], kOvfRange);
                    asm volatile("" ::: "memory");  // slot words were written through st.shared
                    const int nw = (int)(L >> 5), filled = (int)(L & 31u);
                    nwt = nw;
                    if (filled) {
                        if (nw < SLOT_W) slot[nw * CB + lane] = acc; else spill[p][nw - SLOT_W] = acc;
                        nwt = nw + 1;
                    }
                    const uint32_t lastw = nw == 0 ? 0u : (nw - 1 < SLOT_W ? slot[(nw - 1) * CB + lane] : spill[p][nw - 1 - SLOT_W]);
                    tail7 = __funnelshift_rc(acc, lastw, 32 - filled) & 0x7Fu;
                }
            }
            if (p == 0) { C.L[0] = L; C.nwt[0] = nwt; t7[0] = tail7; srel[0] = sr; }
            else if (p == 1) { C.L[1] = L; C.nwt[1] = nwt; t7[1] = tail7; srel[1] = sr; }
            else { C.L[2] = L; C.nwt[2] = nwt; t7[2] = tail7; srel[2] = sr; }
        }
        __syncwarp();  // every lane is done with the stage
        // the bit offsets: an exclusive scan over the 96 lengths in scan order, positions 3l..3l+2 in lane l
        uint32_t *const tl = M.tl, *const off = M.tl + UB;
#pragma unroll
        for (int p = 0; p < NPASS; ++p) tl[srel[p]] = (C.L[p] << 7) | t7[p];
        __syncwarp();
        const uint32_t l0 = tl[3 * lane] >> 7, l1 = tl[3 * lane + 1] >> 7, l2 = tl[3 * lane + 2] >> 7;
        const uint32_t ex = warp_scan(l0 + l1 + l2, lane, &C.Lc);
        off[3 * lane] = ex; off[3 * lane + 1] = ex + l0; off[3 * lane + 2] = ex + l0 + l1;
        uint32_t ctail = 0;
        if (lane == 0) {  // the unit's last 7 bits (a block has >= 2 bits: at most 4 steps)
            int got = 0;
            for (int k = (int)nv - 1; k >= 0 && got < 7; --k) {
                const uint32_t x = tl[k];
                const int take = min((int)(x >> 7), 7 - got);
                ctail |= (x & ((1u << take) - 1u)) << got;
                got += take;
            }
            st_status(P.st_bits + (size_t)C.img * P.nunits + C.unit,
                      pack_status(C.first ? ST_PFX : ST_AGG, ctail, C.Lc));
        }
        __syncwarp();
#pragma unroll
        for (int p = 0; p < NPASS; ++p) C.o_t[p] = off[srel[p]];
        C.ctail = __shfl_sync(0xffffffffu, ctail, 0);
        C.Pc = 0;
        C.tailin = 0;
        C.own = 0;
        __syncwarp();
    };

    // ---- stuffed bytes of one piece (this lane's 32 bytes in wv) -> sbuf -> global ----------------
    // a, b: the unit's owned byte range inside the piece; ffb / Fr: 0xFF bytes before this
    // lane's 32 bytes / in the whole piece; G: output index of the piece's first owned byte.
    // mk: RSTn marker byte to append after the piece's bytes (0 = none).
    auto emit_window = [&](const UnitState &C, const uint32_t (&wv)[8], uint32_t ffb, uint32_t Fr, int a, int b,
                           unsigned long long G, uint32_t mk) {
        uint8_t *outp = P.out + (size_t)C.img * P.out_cap;
        const uint32_t nr0 = (uint32_t)max(b - a, 0) + Fr;
        const uint32_t nr = nr0 + (mk ? 2u : 0u);
        const uint32_t shb = (uint32_t)((reinterpret_cast<uintptr_t>(outp) + G) & 15u);
        // Every lane with owned bytes emits its whole 32-byte piece (bytes outside the owned
        // range land outside the part of sbuf that is copied out); sbuf index 16 + shb is
        // the unit's first owned byte of this piece.
        if (32 * lane < b) {
            uint32_t dst = 16u + shb + (uint32_t)(32 * lane) - (uint32_t)a + ffb;
            // A lane without a 0xFF among its 32 bytes (all of them on smooth content, ~7 of 8 on
            // noise) writes them as ALIGNED words whatever its byte offset: word k = the tail of
            // little-endian word k-1 and the head of word k (one funnel shift), plus at most three
            // single bytes at either end - all predicated, the same instruction sequence in every
            // lane.  7 word + <= 6 byte stores instead of 32 byte stores.  A lane that holds a 0xFF
            // goes byte by byte.
            uint32_t anyff = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) anyff |= ff_bytes(wv[j]);
            if (anyff == 0) {
                uint32_t m[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) m[j] = __byte_perm(wv[j], 0, 0x0123);   // memory order
                const uint32_t al = dst & 3u, sh8 = 8u * al;
                uint8_t *base = sbuf + (dst - al);                 // aligned
                uint32_t *wbase = reinterpret_cast<uint32_t *>(base);
#pragma unroll
                for (int k = 1; k < 8; ++k) wbase[k] = __funnelshift_l(m[k - 1], m[k], sh8);
                if (al == 0) {
                    wbase[0] = m[0];
                } else {
                    // head: bytes al..3 of word 0 <- the low 4 - al bytes of m[0]
                    base[3] = (uint8_t)(m[0] >> (24u - sh8));
                    if (al < 3) base[2] = (uint8_t)(m[0] >> (16u - sh8));
                    if (al < 2) base[1] = (uint8_t)m[0];
                    // tail: bytes 0..al-1 of word 8 <- the top al bytes of m[7]
                    base[32] = (uint8_t)(m[7] >> (32u - sh8));
                    if (al > 1) base[33] = (uint8_t)(m[7] >> (40u - sh8));
                    if (al > 2) base[34] = (uint8_t)(m[7] >> 24);
                }
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const uint32_t w = wv[j];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const uint32_t byte = (w >> (24 - 8 * i)) & 0xFFu;
                        sbuf[dst++] = (uint8_t)byte;
                        if (byte == 0xFFu) sbuf[dst++] = 0;
                    }
                }
            }
        }
        __syncwarp();
        if (mk) {  // 0xFF 0xDn, not subject to stuffing; after the barrier: the last lane's spare bytes land here too
            if (lane == 0) { sbuf[16u + shb + nr0] = 0xFF; sbuf[16u + shb + nr0 + 1] = (uint8_t)mk; }
            __syncwarp();
        }
        if (G + nr <= P.out_cap) {
            uint8_t *gdst = outp + G - shb;  // 16-byte aligned
            const uint32_t end = shb + nr;
            const uint32_t full_lo = (shb + 15u) >> 4, full_hi = end >> 4;  // whole 16-byte pieces
            const uint8_t *sb = sbuf + 16;
            for (uint32_t c16 = full_lo + lane; c16 < full_hi; c16 += 32)
                *reinterpret_cast<uint4 *>(gdst + c16 * 16) = *reinterpret_cast<const uint4 *>(sb + c16 * 16);
            // ragged head (lanes 0-15) and tail (lanes 16-31), one byte per lane
            const uint32_t hb = (uint32_t)lane < 16u ? shb + lane : max(full_hi, full_lo) * 16u + (lane - 16u);
            const bool in_head = (uint32_t)lane < 16u && hb < min(full_lo * 16u, end);
            const bool in_tail = lane >= 16 && full_hi >= full_lo && hb < end;
            if (in_head || in_tail) gdst[hb] = sb[hb];
        } else if (lane == 0) {
            atomicOr(&P.overflow[C.img], kOvfNoFit);
        }
        __syncwarp();  // sbuf is rewritten by the next piece, or by the next unit's stage
    };

    // ---- A: the unit's stream, window by window: assemble, then per 1 KB piece count its 0xFF bytes
    // and park the piece in gwin (RAW: write its unstuffed bytes).  Returns the 0xFF count.
    auto sweep = [&](UnitState &C) -> uint32_t {
        const uint32_t q0 = (uint32_t)C.Pc & 31u;         // bit offset of the unit inside window word 0
        const uint32_t endbit = q0 + C.Lc;                // window bit index one past the unit
        const uint32_t padc = (C.last && !RAW) ? ((8u - (endbit & 7u)) & 7u) : 0u;   // 1-padding (bits.rs:261-272)
        const int ob0 = (int)(q0 >> 3);                   // owned window bytes [ob0, ob1)
        const int ob1 = (int)(RAW ? ((C.last ? endbit + 7u : endbit) >> 3) : (endbit >> 3) + (padc ? 1u : 0u));
        const int nrounds = max(1, (ob1 + WIN_B - 1) / WIN_B);
        const int wtop = (int)((endbit + padc + 31u) >> 5);   // window words written, over all rounds
        uint32_t Fsum = 0;
#pragma unroll 1
        for (int r = 0; r < nrounds; ++r) {
            const int wlo = r * WIN_W, wb0 = r * WIN_B;
            const int nsub = max(1, (min(wtop - wlo, WIN_W) + SUB_W - 1) / SUB_W);   // pieces this round holds
            for (int i = lane; i < nsub * SUB_W / 4; i += 32) reinterpret_cast<uint4 *>(obuf)[i] = make_uint4(0, 0, 0, 0);
            __syncwarp();
#pragma unroll
            for (int p = 0; p < NPASS; ++p) {   // the lane's three blocks, each funnel-shifted to its place
                const uint32_t *const slot = M.slot[p];
                const uint32_t *const spl = spill[p];
                const uint32_t D = q0 + C.o_t[p];
                const int d0 = (int)(D >> 5), sh = (int)(D & 31u);
                const int nd = C.L[p] ? (int)((sh + C.L[p] + 31u) >> 5) : 0;   // destination words
                const int nwt = C.nwt[p];
                const int kb = max(0, wlo - d0), ke = min(nd, wlo + WIN_W - d0);
                uint32_t prev = 0;
                if (nwt <= SLOT_W) {  // the usual case: every word is in the slot
                    if (kb > 0 && kb <= nwt) prev = slot[(kb - 1) * CB + lane];
                    for (int k = kb; k < ke; ++k) {
                        const uint32_t cur = k < nwt ? slot[k * CB + lane] : 0u;
                        const uint32_t v = __funnelshift_r(cur, prev, sh);
                        uint32_t *dst = obuf + (d0 + k - wlo);
                        if (k == 0 || k == nd - 1) atomicOr(dst, v); else *dst = v;
                        prev = cur;
                    }
                } else {
                    if (kb > 0 && kb <= nwt) prev = (kb - 1) < SLOT_W ? slot[(kb - 1) * CB + lane] : spl[kb - 1 - SLOT_W];
                    for (int k = kb; k < ke; ++k) {
                        uint32_t cur = 0;
                        if (k < nwt) cur = k < SLOT_W ? slot[k * CB + lane] : spl[k - SLOT_W];
                        const uint32_t v = __funnelshift_r(cur, prev, sh);
                        uint32_t *dst = obuf + (d0 + k - wlo);
                        if (k == 0 || k == nd - 1) atomicOr(dst, v); else *dst = v;
                        prev = cur;
                    }
                }
            }
            if (lane == 0) {
                const uint32_t q = q0 & 7u;  // inherited bits of the straddling first byte
                if (r == 0 && q) atomicOr(&obuf[0], (C.tailin & ((1u << q) - 1u)) << (32u - q0));
                const int pw = (int)(endbit >> 5) - wlo;
                if (padc && pw >= 0 && pw < WIN_W)
                    atomicOr(&obuf[pw], ((1u << padc) - 1u) << (32u - (endbit & 31u) - padc));
            }
            __syncwarp();
#pragma unroll 1
            for (int s = 0; s < nsub; ++s) {
                // Count the 0xFF bytes in this lane's 32 bytes.  No bounds: a window byte the unit
                // does not own is either untouched (0) or the unfinished last byte, whose low bits
                // are still 0 - never 0xFF.
                const int pb0 = wb0 + s * SUB_B;             // unit byte index of the piece's byte 0
                uint32_t wv[8];
                {
                    const uint4 x = reinterpret_cast<const uint4 *>(obuf + s * SUB_W)[2 * lane];
                    const uint4 y = reinterpret_cast<const uint4 *>(obuf + s * SUB_W)[2 * lane + 1];
                    wv[0] = x.x; wv[1] = x.y; wv[2] = x.z; wv[3] = x.w; wv[4] = y.x; wv[5] = y.y; wv[6] = y.z; wv[7] = y.w;
                }
                if (RAW) {
                    // piece byte i is byte (Pc >> 5) * 4 + pb0 + i of the band's raw string
                    const int a = max(ob0 - pb0, 0), b = min(ob1 - pb0, SUB_B);
                    uint8_t *outp = P.out + (size_t)C.img * P.out_cap;
                    const unsigned long long wbase = (C.Pc >> 5) * 4ull + (unsigned long long)pb0;
                    if (wbase + (unsigned long long)max(b, 0) <= P.out_cap) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const int i0 = 32 * lane + 4 * j;
                            if (i0 >= a && i0 + 4 <= b) {
                                *reinterpret_cast<uint32_t *>(outp + wbase + i0) = __byte_perm(wv[j], 0, 0x0123);
                            } else if (i0 + 4 > a && i0 < b) {
#pragma unroll
                                for (int t = 0; t < 4; ++t)
                                    if (i0 + t >= a && i0 + t < b) outp[wbase + i0 + t] = (uint8_t)(wv[j] >> (24 - 8 * t));
                            }
                        }
                    } else if (lane == 0) {
                        atomicOr(&P.overflow[C.img], kOvfNoFit);
                    }
                    continue;
                }
                uint32_t cnt = 0;
#pragma unroll
                for (int j = 0; j < 8; ++j) cnt += __popc(ff_bytes(wv[j]));
                Fsum += __reduce_add_sync(0xffffffffu, cnt);
                uint4 *g = reinterpret_cast<uint4 *>(gwin + pb0) + 2 * lane;   // read back by this lane in B
                g[0] = make_uint4(wv[0], wv[1], wv[2], wv[3]);
                g[1] = make_uint4(wv[4], wv[5], wv[6], wv[7]);
            }
            __syncwarp();  // obuf is rewritten by the next round, or by the next unit's stage
        }
        C.own = (uint32_t)(ob1 - ob0) + Fsum + (C.marker ? 2u : 0u);
        return Fsum;
    };

    // ---- B: the parked pieces, stuffed, to the output from byte gbase on ---------------------------------
    auto emit = [&](UnitState &C, unsigned long long gbase) {
        const uint32_t q0 = (uint32_t)C.Pc & 31u, endbit = q0 + C.Lc;
        const uint32_t padc = C.last ? ((8u - (endbit & 7u)) & 7u) : 0u;
        const int ob0 = (int)(q0 >> 3), ob1 = (int)((endbit >> 3) + (padc ? 1u : 0u));
        const int npieces = max(1, (ob1 + SUB_B - 1) / SUB_B);
        unsigned long long G = gbase;
#pragma unroll 1
        for (int s = 0; s < npieces; ++s) {
            const int pb0 = s * SUB_B;
            const uint4 *g = reinterpret_cast<const uint4 *>(gwin + pb0) + 2 * lane;
            const uint4 x = g[0], y = g[1];
            const uint32_t wv[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
            uint32_t cnt = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) cnt += __popc(ff_bytes(wv[j]));
            uint32_t Fr;
            const uint32_t ffb = warp_scan(cnt, lane, &Fr);
            const int a = max(ob0 - pb0, 0), b = min(ob1 - pb0, SUB_B);
            emit_window(C, wv, ffb, Fr, a, b, G, s == npieces - 1 ? C.marker : 0u);
            G += (unsigned long long)(max(b - a, 0) + (int)Fr);
        }
        if (lane == 0 && C.final_) {
            P.out_len[C.img] = G;
            if (G > P.out_cap) atomicOr(&P.overflow[C.img], kOvfNoFit);
        }
    };

    // ---- A: bit offset from chain 1, then the unit's 0xFF count into chain 2 ------------------------
    auto phase_a = [&](UnitState &C) {
        if (C.skip) return;
        unsigned long long *st1 = P.st_bits + (size_t)C.img * P.nunits;
        unsigned long long *st2 = P.st_ff + (size_t)C.img * P.nunits;
        if (!C.first) {
            const unsigned long long lb = look_back(st1, (int)C.unit, lane);
            C.Pc = lb & ST_VAL;
            C.tailin = (uint32_t)(lb >> 55) & 0x7Fu;
            C.fault |= (lb >> 62) != 0;
            if (lane == 0) st_status(st1 + C.unit, pack_status(ST_PFX, C.ctail, C.Pc + C.Lc));
        }
        sweep(C);
        if (RAW) {
            if (lane == 0 && C.final_) {
                P.out_len[C.img] = C.Pc + C.Lc;       // BITS
                P.out_tail[C.img] = C.ctail;
                if (((C.Pc + C.Lc + 7) >> 3) > P.out_cap) atomicOr(&P.overflow[C.img], kOvfNoFit);
            }
            if (lane == 0 && C.fault) atomicOr(&P.overflow[C.img], kOvfFault);
            return;
        }
        if (lane == 0) st_status(st2 + C.unit, pack_status(C.unit == 0 ? ST_PFX : ST_AGG, 0, C.own));
    };
    // ---- B: stuffed-byte offset from chain 2, then the bytes ------------------------------------------
    auto phase_b = [&](UnitState &C) {
        if (RAW || C.skip) return;
        unsigned long long *st2 = P.st_ff + (size_t)C.img * P.nunits;
        unsigned long long ffx = 0;
        if (C.unit) {
            const unsigned long long lb = look_back(st2, (int)C.unit, lane);
            ffx = lb & ST_VAL;
            C.fault |= (lb >> 62) != 0;
            if (lane == 0) st_status(st2 + C.unit, pack_status(ST_PFX, 0, ffx + C.own));
        }
        emit(C, ffx);   // chain 2 counts every byte written before this unit
        if (lane == 0 && C.fault) atomicOr(&P.overflow[C.img], kOvfFault);
    };

    UnitState cur, pend;
    bool have_pend = false;
    for (;;) {
        uint32_t id = 0;
        if (lane == 0) id = atomicAdd(P.ticket, 1u);
        id = __shfl_sync(0xffffffffu, id, 0);
        const bool have = id < total_units;
        if (have_pend) phase_a(pend);
        if (have) phase_w(id, cur);
        if (have_pend) phase_b(pend);
        if (!have) break;
        pend = cur;
        have_pend = true;
    }
}

// ---- a frame's Huffman tables from its statistics ---------------------------------------------------
// huff_from_histogram (jpeg_host.cpp), that is pixo's optimized_from_counts / build_code_lengths /
// build_bits_vals (src/jpeg/huffman.rs:167-205,288-391), on the device.  One CTA per frame; warp k builds
// table k (dc_lum, dc_chrom, ac_lum, ac_chrom).  pixo pops a min-heap on (frequency, node index), the
// leaves numbered in ascending symbol order and merged nodes after them.  Merged frequencies come out
// non-decreasing with increasing indices, so merging two queues - the leaves sorted by (count, symbol) and
// the merged nodes in the order they are made, a leaf winning a tie - pops the same nodes.  The warp ranks
// the leaves; one lane runs the (at most 255) merges and the merged nodes' depths.  A leaf's length is its
// depth + 1 (pixo's convention) and a table with a length above 16 fails; a single symbol gets length 1.
// vals are in (length, symbol) order and the codes canonical (assign_codes).  A failed luma table makes
// all four tables standard, a failed chroma table only itself; gray frames take the standard chroma tables.
struct HuffStd {   // the standard tables (huff_standard), what a table falls back to
    uint8_t dht[kDhtBytes];
    HuffDev dev;
};

struct TableMem {  // one warp's table
    unsigned long long cnt[256];   // the statistics, by symbol
    unsigned long long sf[256];    // the leaves' counts in (count, symbol) order
    unsigned long long mf[256];    // the merged nodes' frequencies, in the order they are made
    uint16_t lpar[256], mpar[256], mdep[256];   // parent of a sorted leaf, of a merged node; a merged node's depth
    uint8_t ssym[256];             // the symbol of a sorted leaf
    uint8_t len[256];              // code length by symbol, 0: not in the table
    uint8_t vals[256];
    uint32_t words[12 + AC_WORDS]; // k_huff's entries (HuffHalf's layout; a DC table fills the first 12)
    int nlen[17], start[17], first[17], seen[17];   // per length: symbols, first vals index, first code, placed
};

__global__ void __launch_bounds__(128) k_huff_tables(const unsigned long long *hist, uint32_t has_chroma,
                                                     const __grid_constant__ HuffStd S, uint8_t *dht, HuffDev *dev)
{
    __shared__ TableMem tm[4];
    __shared__ int ok[4];
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t f = blockIdx.x;
    const unsigned full = 0xffffffffu, below = (1u << lane) - 1u;
    TableMem &t = tm[k];
    const int nsym = k < 2 ? 12 : 256;
    bool good = hist != nullptr && (has_chroma || k == 0 || k == 2);   // (uniform in the warp)
    if (good) {
        const unsigned long long *h = hist + (size_t)f * kHistWords + (k == 0 ? 0 : k == 1 ? 12 : k == 2 ? 24 : 280);
        for (int s = lane; s < 256; s += 32) {
            t.cnt[s] = s < nsym ? h[s] : 0ull;
            t.len[s] = 0;
            t.vals[s] = 0;
        }
        for (int i = lane; i < 12 + AC_WORDS; i += 32) t.words[i] = 0;
        if (lane < 17) { t.nlen[lane] = 0; t.seen[lane] = 0; }
        __syncwarp();
        // each lane ranks symbols lane + 32 j among the leaves by (count, symbol)
        unsigned long long c[8];
        int r[8], m = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) { c[j] = t.cnt[lane + 32 * j]; r[j] = 0; }
        for (int s = 0; s < nsym; ++s) {
            const unsigned long long x = t.cnt[s];
            if (!x) continue;
#pragma unroll
            for (int j = 0; j < 8; ++j) r[j] += (x < c[j] || (x == c[j] && s < lane + 32 * j)) ? 1 : 0;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            m += __popc(__ballot_sync(full, c[j] != 0));
            if (c[j]) { t.sf[r[j]] = c[j]; t.ssym[r[j]] = (uint8_t)(lane + 32 * j); }
        }
        __syncwarp();
        if (m == 0) {
            good = false;
        } else if (m == 1) {
            if (lane == 0) t.len[t.ssym[0]] = 1;
        } else {
            if (lane == 0) {
                int li = 0, mi = 0;   // next leaf, next merged node to pop; merged nodes [0, j) exist
                for (int j = 0; j < m - 1; ++j) {
                    unsigned long long sum = 0;
                    for (int two = 0; two < 2; ++two) {
                        if (li < m && (mi >= j || t.sf[li] <= t.mf[mi])) { sum += t.sf[li]; t.lpar[li++] = (uint16_t)j; }
                        else { sum += t.mf[mi]; t.mpar[mi++] = (uint16_t)j; }
                    }
                    t.mf[j] = sum;
                }
                t.mdep[m - 2] = 0;   // the root; a parent is made after its children
                for (int j = m - 3; j >= 0; --j) t.mdep[j] = (uint16_t)(t.mdep[t.mpar[j]] + 1);
            }
            __syncwarp();
            bool longer = false;
            for (int i = lane; i < m; i += 32) {
                const int L = t.mdep[t.lpar[i]] + 2;   // the leaf's depth + 1
                longer |= L > 16;
                t.len[t.ssym[i]] = (uint8_t)min(L, 255);
            }
            if (__any_sync(full, longer)) good = false;
        }
        if (good) {
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int s = lane + 32 * j;
                if (s < nsym && t.len[s]) atomicAdd(&t.nlen[t.len[s]], 1);
            }
            __syncwarp();
            if (lane == 0) {
                int st = 0, code = 0;
                t.start[0] = t.first[0] = 0;
                for (int l = 1; l <= 16; ++l) {
                    t.start[l] = st;
                    t.first[l] = code;
                    st += t.nlen[l];
                    code = (code + t.nlen[l]) << 1;
                }
            }
            __syncwarp();
#pragma unroll 1
            for (int j = 0; j < 8; ++j) {   // in symbol order: vals by (length, symbol)
                const int s = lane + 32 * j;
                const int L = s < nsym ? t.len[s] : 0;
                const uint32_t same = __match_any_sync(full, L);
                const int pos = t.start[L] + t.seen[L] + __popc(same & below);
                __syncwarp();
                if (L && (same & below) == 0) t.seen[L] += __popc(same);
                __syncwarp();
                if (!L) continue;
                t.vals[pos] = (uint8_t)s;
                const uint32_t code = (uint32_t)(t.first[L] + (pos - t.start[L])) << (32 - L);
                if (k < 2) {
                    t.words[s] = code | (uint32_t)(L + s);
                } else {   // make_huff_dev's AC layout
                    const int cat = s & 15, run = s >> 4;
                    const int w = s == 0x00 ? AC_EOB : s == 0xF0 ? AC_ZRL : (cat >= 1 && cat <= 10) ? run * AC_STRIDE + cat - 1 : -1;
                    if (w >= 0) t.words[12 + w] = code | (uint32_t)(L + cat);
                }
            }
        }
    }
    if (lane == 0) ok[k] = good;
    __syncthreads();
    const bool own = ok[0] && ok[2] && good;
    if (dht) {
        uint8_t *o = dht + (size_t)f * kDhtBytes + k * 272;
        for (int i = lane; i < 272; i += 32)
            o[i] = own ? (i < 16 ? (uint8_t)t.nlen[i + 1] : t.vals[i - 16]) : S.dht[k * 272 + i];
    }
    if (dev) {
        uint32_t *o = k < 2 ? dev[f].dc[k] : dev[f].ac[k - 2];
        const uint32_t *std_w = k < 2 ? S.dev.dc[k] : S.dev.ac[k - 2];
        const uint32_t *own_w = k < 2 ? t.words : t.words + 12;
        for (int i = lane; i < (k < 2 ? 12 : AC_WORDS); i += 32) o[i] = own ? own_w[i] : std_w[i];
    }
}

}  // namespace

// Scratch of the entropy stage for n images: k_huff's status words, appended to L
struct EntropyPlan {
    size_t nunits;                 // k_huff work units per image
    unsigned long long *st1, *st2;
    uint32_t *ticket, *ovf;
    size_t zero_bytes;             // the regions above, from st1 on: cleared per launch
    uint64_t *out_len;
    unsigned long long *tail;
};

static EntropyPlan plan_entropy(Layout &L, uint32_t n, uint64_t nblocks, uint64_t rst_blocks)
{
    EntropyPlan p;
    p.nunits = (size_t)((nblocks + UB - 1) / UB);
    if (rst_blocks && rst_blocks < nblocks) {  // every interval is cut into units on its own
        const uint64_t n_int = (nblocks + rst_blocks - 1) / rst_blocks, upi = (rst_blocks + UB - 1) / UB;
        const uint64_t last = nblocks - (n_int - 1) * rst_blocks;
        p.nunits = (size_t)((n_int - 1) * upi + (last + UB - 1) / UB);
    }
    const size_t start = L.size();
    p.st1 = L.take<unsigned long long>((size_t)n * p.nunits);
    p.st2 = L.take<unsigned long long>((size_t)n * p.nunits);
    p.ticket = L.take<uint32_t>(1);
    p.ovf = L.take<uint32_t>(n);
    p.zero_bytes = L.size() - start;
    p.out_len = L.take<uint64_t>(n);
    p.tail = L.take<unsigned long long>(n);
    return p;
}

size_t entropy_scratch_bytes(uint32_t n, const FrameGeometry &g, uint32_t restart_interval)
{
    const uint64_t bpm = g.y_per_mcu + (g.has_chroma ? 2 : 0);
    Layout L;
    plan_entropy(L, n, g.ny + 2 * g.nc, (uint64_t)restart_interval * bpm);
    return L.size();
}

// ---- splicing a raw bit string into the stream's scan bytes -------------------------------------
// T = tail_in (s bits, the stream bits that precede the string inside its first byte) ++ B (the raw
// string, nbits).  The string owns T's whole bytes; the stream's last string also owns the final
// partial byte, padded with 1s (BitWriterMsb::flush, src/bits.rs:261-272).  Every 0xFF is followed
// by 0x00 (flush_byte_with_stuffing, :245-259).
namespace {

constexpr int SPL_TILE = 4096;  // T bytes per tile
constexpr int SPL_THREADS = 256;

// Sixteen bytes of T at once.  T is the raw string shifted right by `phase` bits behind the inherited
// bits, so four big-endian words of T are four funnel shifts over the raw words (and the raw byte before
// them).  Only for a thread whose piece lies wholly inside the raw string, short of its last byte (no
// padding, no missing bytes), at a 16-byte aligned address; the ragged ends take the byte-wise path.
__device__ __forceinline__ bool t_words16(const uint8_t *raw, unsigned long long rb, uint32_t phase, uint32_t tail_in,
                                          unsigned long long m0, uint32_t (&O)[4])
{
    if (m0 + 16 >= rb || (reinterpret_cast<uintptr_t>(raw + m0) & 15)) return false;
    const uint4 L = *reinterpret_cast<const uint4 *>(raw + m0);
    const uint32_t pb = m0 ? raw[m0 - 1] : tail_in;
    const uint32_t A0 = __byte_perm(L.x, 0, 0x0123), A1 = __byte_perm(L.y, 0, 0x0123);
    const uint32_t A2 = __byte_perm(L.z, 0, 0x0123), A3 = __byte_perm(L.w, 0, 0x0123);
    O[0] = __funnelshift_r(A0, pb, phase);
    O[1] = __funnelshift_r(A1, A0, phase);
    O[2] = __funnelshift_r(A2, A1, phase);
    O[3] = __funnelshift_r(A3, A2, phase);
    return true;
}
__device__ __forceinline__ uint32_t ff_count16(const uint32_t (&O)[4])
{
    return __popc(ff_bytes(O[0])) + __popc(ff_bytes(O[1])) + __popc(ff_bytes(O[2])) + __popc(ff_bytes(O[3]));
}
// sixteen stuffing-free bytes (four big-endian words) -> sb[dst .. dst + 16) at any byte alignment:
// three aligned word stores plus at most three single bytes at either end
__device__ __forceinline__ void put16(uint8_t *sb, uint32_t dst, const uint32_t (&O)[4])
{
    uint32_t m[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) m[k] = __byte_perm(O[k], 0, 0x0123);   // memory order
    const uint32_t al = dst & 3u, sh8 = 8u * al;
    uint8_t *base = sb + (dst - al);
    uint32_t *wb = reinterpret_cast<uint32_t *>(base);
#pragma unroll
    for (int k = 1; k < 4; ++k) wb[k] = __funnelshift_l(m[k - 1], m[k], sh8);
    if (al == 0) {
        wb[0] = m[0];
    } else {
        base[3] = (uint8_t)(m[0] >> (24u - sh8));
        if (al < 3) base[2] = (uint8_t)(m[0] >> (16u - sh8));
        if (al < 2) base[1] = (uint8_t)m[0];
        base[16] = (uint8_t)(m[3] >> (32u - sh8));
        if (al > 1) base[17] = (uint8_t)(m[3] >> (40u - sh8));
        if (al > 2) base[18] = (uint8_t)(m[3] >> 24);
    }
}

// ---- segmented coding: many short chains instead of one long one ------------------------------------
// One image (or a handful) gives the single-pass kernel only one look-back chain per image: with
// ~3500 warps in flight on the same chain a chunk has to look back over thousands of predecessors
// (see segments_for for what that costs a 16 384^2 frame).  Instead the image is
// cut into S runs of whole MCUs, each coded by k_huff<RAW> as a bit string of its own - S independent,
// short chains advancing side by side - and four small kernels splice the strings: per-segment bit
// offsets (k_seg_prefix), 0xFF counts per 4 KB tile of the shifted stream (k_seg_count), their prefix
// (k_seg_scan), and the stuffed bytes (k_seg_emit).  No host round trip in between.  The same
// machinery codes and splices a band of a frame tiled over several GPUs, S >= 1 (base bit offset and
// inherited bits come from the other ranks).

struct SegRec {
    unsigned long long nbits, byte_off, nbytes;   // byte_off: T-bytes of the image's earlier segments
    uint32_t phase, tail_in, tile_off, last;
};

struct SegParams {
    const uint8_t *raw;             // [n * S][raw_cap]
    unsigned long long raw_cap;
    const unsigned long long *bits; // [n * S] from k_huff<RAW>
    const unsigned long long *tails;
    uint32_t S, max_tiles;
    unsigned long long base_bit;    // bits of the stream before segment 0 (a band of a tiled frame; 0 otherwise)
    uint32_t base_tail, last_band;  // the stream's last base_bit % 8 bits; 1: the last segment ends the stream (1-pad)
    const unsigned long long *base_dev;   // {base_bit, the previous band's last 7 bits, last_band} in device memory, or null
    SegRec *rec;                    // [n * S]
    uint32_t *ntiles;               // [n]
    uint32_t *cnt;                  // [n][max_tiles] 0xFF counts, then their exclusive prefix
    uint8_t *out;                   // [n][out_cap]
    unsigned long long out_cap;
    unsigned long long *out_len;    // [n]
    uint32_t *overflow;             // [n]
    const uint32_t *raw_overflow;   // [n * S] flags of the coding kernel
};

__device__ __forceinline__ uint32_t seg_byte(const uint8_t *raw, const SegRec &r, unsigned long long m)
{
    const unsigned long long rb = (r.nbits + 7) >> 3;
    const uint32_t cur = m < rb ? raw[m] : 0u;
    const uint32_t prev = m ? raw[m - 1] : r.tail_in;
    uint32_t v = (((prev << 8) | cur) >> r.phase) & 0xFFu;
    const unsigned long long tbits = r.phase + r.nbits;
    if (m == (tbits >> 3)) v |= 0xFFu >> (uint32_t)(tbits & 7);   // reached only by the padded last byte
    return v;
}

// a band's totals for the exchange with the other ranks: {bits, last 7 bits}, and its flags
__global__ void k_band_totals(const unsigned long long *bits, const unsigned long long *tails, const uint32_t *ovf,
                              uint32_t S, unsigned long long *out2, uint32_t *flags)
{
    if (threadIdx.x || blockIdx.x) return;
    unsigned long long total = 0, tail = 0;
    uint32_t f = 0;
    for (uint32_t q = 0; q < S; ++q) {
        total += bits[q];
        if (bits[q]) tail = tails[q];
        f |= ovf[q];
    }
    out2[0] = total;
    out2[1] = tail & 0x7Full;
    if (f) atomicOr(flags, f);
}

// exclusive prefix over the CTA's SPL_THREADS values (every thread calls; `sh` holds one word per warp)
template <typename T>
__device__ __forceinline__ T cta_exclusive_scan(T x, T *sh, T *total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T inc = x;
    for (int o = 1; o < 32; o <<= 1) {
        const T v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    __syncthreads();              // sh may still be read from a previous scan
    if (lane == 31) sh[warp] = inc;
    __syncthreads();
    T before = 0, all = 0;
    for (int w = 0; w < SPL_THREADS / 32; ++w) { const T v = sh[w]; if (w < warp) before += v; all += v; }
    *total = all;
    return before + inc - x;
}

// Per image: every segment's record (bit phase, inherited bits, byte and tile offsets) from the
// segments' bit counts.  One CTA per image, thread s = segment s (S <= SEG_MAX == SPL_THREADS): three
// prefix sums (bits, bytes, tiles) and a "nearest earlier non-empty segment" scan for the inherited bits.
__global__ void __launch_bounds__(SPL_THREADS) k_seg_prefix(const __grid_constant__ SegParams P)
{
    __shared__ unsigned long long sh64[SPL_THREADS / 32];
    __shared__ uint32_t sh32[SPL_THREADS / 32];
    __shared__ int shmax[SPL_THREADS / 32];
    __shared__ uint32_t shbad;   // the OR of the segments' flags
    const uint32_t i = blockIdx.x, s = threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (s == 0) shbad = 0;       // (the scans' barriers below order this before the atomicOr)
    unsigned long long base = P.base_bit;
    uint32_t base_tail = P.base_tail, last_band = P.last_band;
    if (P.base_dev) { base = P.base_dev[0]; base_tail = (uint32_t)P.base_dev[1]; last_band = (uint32_t)P.base_dev[2]; }
    const bool live = s < P.S;
    const uint32_t q = i * P.S + s;
    const unsigned long long nbits = live ? P.bits[q] : 0ull;
    const uint32_t bad_here = (live && P.raw_overflow) ? P.raw_overflow[q] : 0u;
    unsigned long long total_bits;
    const unsigned long long start = base + cta_exclusive_scan<unsigned long long>(nbits, sh64, &total_bits);
    SegRec r;
    r.nbits = nbits;
    r.phase = (uint32_t)(start & 7);
    r.last = (live && s == P.S - 1 && last_band) ? 1u : 0u;
    const unsigned long long tbits = r.phase + r.nbits;
    r.nbytes = live ? (tbits >> 3) + ((r.last && (tbits & 7)) ? 1 : 0) : 0ull;
    unsigned long long total_bytes;
    r.byte_off = cta_exclusive_scan<unsigned long long>(r.nbytes, sh64, &total_bytes);
    uint32_t total_tiles;
    r.tile_off = cta_exclusive_scan<uint32_t>((uint32_t)((r.nbytes + SPL_TILE - 1) / SPL_TILE), sh32, &total_tiles);
    // the bits inherited in the first byte: the last 7 bits of the nearest earlier segment that has any
    int near = (live && nbits) ? (int)s : -1;      // inclusive running maximum, then shifted by one
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, near, o);
        if (lane >= o) near = max(near, v);
    }
    if (lane == 31) shmax[warp] = near;
    __syncthreads();
    int prev = __shfl_up_sync(0xffffffffu, near, 1);
    if (lane == 0) prev = -1;
    for (int w = 0; w < warp; ++w) prev = max(prev, shmax[w]);
    const uint32_t tail_prev = prev >= 0 ? (uint32_t)P.tails[i * P.S + prev] : base_tail;
    r.tail_in = tail_prev & ((1u << r.phase) - 1u);
    if (live) P.rec[q] = r;
    const uint32_t wbad = __reduce_or_sync(0xffffffffu, bad_here);
    if (lane == 0 && wbad) atomicOr(&shbad, wbad);
    __syncthreads();
    const uint32_t bad = shbad;
    if (s == 0) {
        P.ntiles[i] = total_tiles;
        // a raw segment that did not fit (or a faulted chain): the caller codes the image again unsegmented;
        // a coefficient outside the baseline range (bit 3) is passed on, the caller does not retry it
        if (bad || total_tiles > P.max_tiles) { P.overflow[i] = kOvfSegment | (bad & (kOvfFault | kOvfRange)); P.ntiles[i] = 0; P.out_len[i] = 0; }
        else if (total_tiles == 0) P.out_len[i] = 0;
    }
}

// A CTA of the splice kernels works through SPL_TPC consecutive tiles of one image (one tile per CTA
// left the kernels latency-bound: 17 000 CTAs for a 70 MB scan, each behind a chain of dependent loads).
// The image's segment records are read once into shared memory.
constexpr int SPL_TPC = 8;
constexpr int SEG_MAX = 256;
static_assert(SEG_MAX == SPL_THREADS, "thread s of a splice CTA looks at segment record s");

__device__ __forceinline__ void load_seg_table(const SegParams &P, uint32_t i, SegRec *tab)
{
    if (threadIdx.x < P.S) tab[threadIdx.x] = P.rec[i * P.S + threadIdx.x];
    __syncthreads();
}
// the segment tile t belongs to: the last one whose first tile is <= t (tile_off is non-decreasing and
// tab[0].tile_off == 0).  Whole CTA, one barrier: thread s looks at record s.
__device__ __forceinline__ uint32_t seg_of_tile(const SegRec *tab, uint32_t S, uint32_t t)
{
    return (uint32_t)__syncthreads_count(threadIdx.x < S && tab[threadIdx.x].tile_off <= t) - 1u;
}

// nout staged bytes -> outp[g0 ..).  The stage was filled from index shb = (address of outp + g0) & 15 on,
// so stage and destination agree modulo 16: whole 16-byte pieces, single bytes at the two ragged ends.
__device__ __forceinline__ void copy_out16(uint8_t *outp, unsigned long long g0, const uint8_t *sb, uint32_t shb,
                                           uint32_t nout, int tid)
{
    uint8_t *gdst = outp + g0 - shb;   // 16-byte aligned
    const uint32_t end = shb + nout;
    const uint32_t full_lo = (shb + 15u) >> 4, full_hi = end >> 4;
    for (uint32_t c16 = full_lo + tid; c16 < full_hi; c16 += SPL_THREADS)
        *reinterpret_cast<uint4 *>(gdst + c16 * 16) = *reinterpret_cast<const uint4 *>(sb + c16 * 16);
    if (tid < 16) {                       // ragged head
        const uint32_t hb = shb + tid;
        if (hb < min(full_lo * 16u, end)) gdst[hb] = sb[hb];
    } else if (tid < 32) {                // ragged tail
        const uint32_t tb = max(full_hi, full_lo) * 16u + (tid - 16);
        if (full_hi >= full_lo && tb < end) gdst[tb] = sb[tb];
    }
}

__global__ void __launch_bounds__(SPL_THREADS) k_seg_count(const __grid_constant__ SegParams P)
{
    __shared__ uint32_t red[SPL_TPC][SPL_THREADS / 32];
    __shared__ SegRec tab[SEG_MAX];
    const uint32_t i = blockIdx.y, t0 = blockIdx.x * SPL_TPC, nt = P.ntiles[i];
    if (t0 >= nt) return;
    load_seg_table(P, i, tab);
    const uint32_t t1 = min(nt, t0 + SPL_TPC);
    for (uint32_t t = t0; t < t1; ++t) {
        const uint32_t s = seg_of_tile(tab, P.S, t);
        const SegRec &r = tab[s];
        const uint8_t *raw = P.raw + (size_t)(i * P.S + s) * P.raw_cap;
        const unsigned long long m0 = (unsigned long long)(t - r.tile_off) * SPL_TILE + threadIdx.x * 16;
        uint32_t c = 0, O[4];
        if (t_words16(raw, (r.nbits + 7) >> 3, r.phase, r.tail_in, m0, O)) {
            c = ff_count16(O);
        } else {
            for (int k = 0; k < 16; ++k)
                if (m0 + k < r.nbytes) c += seg_byte(raw, r, m0 + k) == 0xFFu;
        }
        c = __reduce_add_sync(0xffffffffu, c);
        if ((threadIdx.x & 31) == 0) red[t - t0][threadIdx.x >> 5] = c;
    }
    __syncthreads();
    if (threadIdx.x < t1 - t0) {
        uint32_t tot = 0;
        for (int k = 0; k < SPL_THREADS / 32; ++k) tot += red[threadIdx.x][k];
        P.cnt[(size_t)i * P.max_tiles + t0 + threadIdx.x] = tot;
    }
}

// exclusive prefix of an image's tile counts, in place (one CTA per image)
__global__ void __launch_bounds__(1024) k_seg_scan(const __grid_constant__ SegParams P)
{
    __shared__ uint32_t wtot[32];
    const uint32_t i = blockIdx.x, n = P.ntiles[i];
    uint32_t *c = P.cnt + (size_t)i * P.max_tiles;
    const uint32_t per = (n + 1023) / 1024, lo = threadIdx.x * per, hi = min(n, lo + per);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t sum = 0;
    for (uint32_t k = lo; k < hi; ++k) sum += c[k];
    uint32_t inc = sum;                        // inclusive scan of the 1024 partial sums: warp, then warp totals
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) wtot[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = wtot[lane];
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += v;
        }
        wtot[lane] = w;
    }
    __syncthreads();
    uint32_t run = inc - sum + (warp ? wtot[warp - 1] : 0u);
    for (uint32_t k = lo; k < hi; ++k) { const uint32_t v = c[k]; c[k] = run; run += v; }
}

__global__ void __launch_bounds__(SPL_THREADS) k_seg_emit(const __grid_constant__ SegParams P)
{
    __shared__ uint32_t wsum[SPL_THREADS / 32];
    __shared__ __align__(16) uint8_t sb[2 * SPL_TILE + 32];
    __shared__ SegRec tab[SEG_MAX];
    const uint32_t i = blockIdx.y, t0 = blockIdx.x * SPL_TPC, nt = P.ntiles[i];
    if (t0 >= nt) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    load_seg_table(P, i, tab);
    uint8_t *outp = P.out + (size_t)i * P.out_cap;
    const uint32_t t1 = min(nt, t0 + SPL_TPC);
    for (uint32_t t = t0; t < t1; ++t) {
        const uint32_t s = seg_of_tile(tab, P.S, t);
        const SegRec &r = tab[s];
        const uint8_t *raw = P.raw + (size_t)(i * P.S + s) * P.raw_cap;
        const unsigned long long tile_first = (unsigned long long)(t - r.tile_off) * SPL_TILE;
        const unsigned long long m0 = tile_first + tid * 16;
        const unsigned long long g0 = r.byte_off + tile_first + P.cnt[(size_t)i * P.max_tiles + t];
        const uint32_t shb = (uint32_t)((reinterpret_cast<uintptr_t>(outp) + g0) & 15u);
        uint32_t v[16], c = 0, O[4];
        const bool fast = t_words16(raw, (r.nbits + 7) >> 3, r.phase, r.tail_in, m0, O);
        if (fast) {
            c = ff_count16(O);
        } else {
            for (int k = 0; k < 16; ++k) {
                v[k] = m0 + k < r.nbytes ? seg_byte(raw, r, m0 + k) : 0x100u;
                c += v[k] == 0xFFu;
            }
        }
        uint32_t inc = c;
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t nb = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += nb;
        }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        uint32_t woff = 0, total = 0;
        for (int k = 0; k < SPL_THREADS / 32; ++k) { if (k < warp) woff += wsum[k]; total += wsum[k]; }
        uint32_t dst = shb + tid * 16 + woff + inc - c;
        if (fast && c == 0) {
            put16(sb, dst, O);
        } else {
            if (fast)
                for (int k = 0; k < 16; ++k) v[k] = (O[k >> 2] >> (24 - 8 * (k & 3))) & 0xFFu;
            for (int k = 0; k < 16; ++k) {
                if (v[k] > 0xFFu) break;
                sb[dst++] = (uint8_t)v[k];
                if (v[k] == 0xFFu) sb[dst++] = 0;
            }
        }
        __syncthreads();
        const unsigned long long tile_n = min((unsigned long long)SPL_TILE, r.nbytes - tile_first);
        const uint32_t nout = (uint32_t)tile_n + total;
        if (g0 + nout <= P.out_cap) copy_out16(outp, g0, sb, shb, nout, tid);
        else if (tid == 0) atomicOr(&P.overflow[i], kOvfNoFit);
        if (tid == 0 && t == nt - 1) P.out_len[i] = g0 + nout;   // the size needed, also when it did not fit
        __syncthreads();   // the stage and wsum are rewritten by the next tile
    }
}

// Whole strings (S == 1) only, one CTA per image, after k_seg_scan: the stuffed offset of every bound of the
// image's string (its byte offset + the 0xFF bytes before it: the prefix of its tile, and the tile's bytes up to
// it counted here), the stuffed length of each range between bounds, and the image's total.  An image whose total
// does not fit out_cap gets overflow bit 0 and no tiles, so that k_seg_emit writes nothing of it.
__global__ void __launch_bounds__(SPL_THREADS) k_seg_fit(const __grid_constant__ SegParams P,
                                                         const unsigned long long *bounds, uint32_t nr,
                                                         unsigned long long *range_len)
{
    __shared__ uint32_t wsum[SPL_THREADS / 32];
    const uint32_t i = blockIdx.x, nt = P.ntiles[i];
    if (nt == 0) return;
    const SegRec r = P.rec[i];
    const uint8_t *raw = P.raw + (size_t)i * P.raw_cap;
    const unsigned long long *b = bounds + (size_t)i * (nr + 1);
    // stuffed offset of byte m (0 <= m <= nbytes) of the string (whole CTA)
    auto stuffed = [&](unsigned long long m) {
        const uint32_t t = m == r.nbytes ? nt - 1 : (uint32_t)(m / SPL_TILE);
        uint32_t c = 0;
        for (unsigned long long j = (unsigned long long)t * SPL_TILE + threadIdx.x; j < m; j += SPL_THREADS)
            c += seg_byte(raw, r, j) == 0xFFu;
        c = __reduce_add_sync(0xffffffffu, c);
        __syncthreads();   // wsum may still be read from the previous bound
        if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
        __syncthreads();
        unsigned long long tot = m + P.cnt[(size_t)i * P.max_tiles + t];
        for (int w = 0; w < SPL_THREADS / 32; ++w) tot += wsum[w];
        return tot;
    };
    unsigned long long prev = stuffed(b[0] >> 3);
    for (uint32_t k = 0; k < nr; ++k) {
        const unsigned long long next = stuffed(b[k + 1] >> 3);
        if (threadIdx.x == 0) range_len[(size_t)i * nr + k] = next - prev;
        prev = next;
    }
    if (threadIdx.x == 0 && prev > P.out_cap) {
        atomicOr(&P.overflow[i], kOvfNoFit);
        P.ntiles[i] = 0;
        P.out_len[i] = prev;
    }
}

}  // namespace

static void make_huff_dev(const HuffTables &t, HuffDev *Tp)
{
    HuffDev &T = *Tp;
    memset(&T, 0, sizeof T);
    for (int k = 0; k < 2; ++k) {
        for (int cat = 0; cat < 12; ++cat)
            if (t.len[k][cat])
                T.dc[k][cat] = ((uint32_t)t.code[k][cat] << (32 - t.len[k][cat])) | (uint32_t)(t.len[k][cat] + cat);
        for (int rs = 0; rs < 256; ++rs) {
            const int cat = rs & 15, run = rs >> 4;
            if (!t.len[2 + k][rs] || cat > 10) continue;
            const uint32_t e = ((uint32_t)t.code[2 + k][rs] << (32 - t.len[2 + k][rs])) | (uint32_t)(t.len[2 + k][rs] + cat);
            if (rs == 0x00) T.ac[k][AC_EOB] = e;
            else if (rs == 0xF0) T.ac[k][AC_ZRL] = e;
            else if (cat >= 1) T.ac[k][run * AC_STRIDE + cat - 1] = e;
        }
    }
}

// How many segments per image: enough chains to keep a look-back short (~256 chains in flight), none
// shorter than 512 chunks.  1 = do not segment.
static uint32_t segments_for(uint32_t n, uint64_t total_mcus, uint64_t bpm)
{
    if (const char *e = getenv("PIXO_B200_SEGMENTS")) return (uint32_t)std::min(SEG_MAX, std::max(1, atoi(e)));   // test hook
    // Measured on an H100 SXM 80 GB (400 W limit), whole device path, q80 4:2:0: for 4K frames (6 075
    // chunks) the extra launches cost more than the shorter chains save (one frame: unsegmented
    // 0.108-0.110 ms, 4-256 segments 0.124-0.130 ms; tools/segment_sweep.py, profiles/h100_segment_sweep.json); a 16 384^2 frame (196 608 chunks on ONE chain) is
    // where the look-back distance hurts.  So: few images, each long.
    const uint64_t chunks = total_mcus * bpm / 32;   // (the thresholds below count 32-block chunks)
    if (n > 8 || chunks < 16384) return 1;
    // 16 384^2 frame on the same H100: unsegmented 2.53-2.67 ms, 16 segments 2.11, 32: 1.90, 64: 1.73,
    // 128: 1.62, 256: 1.53-1.59 (more chains in flight keep the nearest inclusive prefix inside one
    // 32-wide look-back step)
    uint32_t S = SEG_MAX / n;
    while (S > 1 && chunks / S < 512) S >>= 1;
    return S < 2 ? 1 : S;
}

// Segments of raw_cap string bytes each
static void set_raw_cap(SegPlan &p, size_t raw_cap)
{
    p.raw_cap = raw_cap;
    p.max_tiles = (uint32_t)(p.S * (raw_cap / SPL_TILE + 2));
}

// The segment scratch of a plan: the entropy stage's status words for its n * S pseudo images, then the
// splice's records
struct SegScratch {
    EntropyPlan ent;
    SegRec *rec;
    uint32_t *ntiles, *cnt;
    size_t total;
};

static SegScratch seg_scratch(const SegPlan &p, void *base)
{
    Layout L(base);
    SegScratch s;
    s.ent = plan_entropy(L, p.n * p.S, p.seg_mcus * p.bpm, 0);
    s.rec = L.take<SegRec>((size_t)p.n * p.S);
    s.ntiles = L.take<uint32_t>(p.n);
    s.cnt = L.take<uint32_t>((size_t)p.n * p.max_tiles);
    s.total = L.size();
    return s;
}

size_t seg_scratch_bytes(const SegPlan &p) { return seg_scratch(p, nullptr).total; }

SegRaw seg_raw(const SegPlan &p, void *base)
{
    Layout L(base);
    SegRaw r;
    const size_t strings = (size_t)p.n * p.S;
    r.strings = L.take(strings * p.raw_cap);
    const size_t strings_bytes = L.size();
    r.bits = L.take<unsigned long long>(strings);
    r.tails = L.take<unsigned long long>(strings);
    r.total = L.size();
    r.trailer = r.total - strings_bytes;
    return r;
}

static SegPlan plan_segments(uint32_t n, uint32_t S, uint64_t total_mcus, uint64_t bpm, uint64_t mcu_raw_bytes)
{
    SegPlan p;
    p.n = n;
    p.bpm = bpm;
    p.seg_mcus = (total_mcus + S - 1) / S;
    S = (uint32_t)((total_mcus + p.seg_mcus - 1) / p.seg_mcus);   // no empty last segment
    p.S = S;
    p.last_mcus = total_mcus - p.seg_mcus * (S - 1);
    // room for a segment's raw string: as many bytes as its pixels take (q=100 noise stays below 0.7 of
    // that), at most what its blocks can possibly need (64 x 26 bits + DC < 216 bytes per block).  It
    // does not depend on the caller's output capacity, so an output that is too small is still measured.
    const uint64_t fair = p.seg_mcus * mcu_raw_bytes + 4096, worst = p.seg_mcus * bpm * 216 + 64;
    set_raw_cap(p, Layout::round((size_t)std::min(fair, worst)));
    return p;
}

static uint64_t mcu_raw_bytes(const FrameGeometry &g) { return (uint64_t)g.y_per_mcu * 64 * (g.has_chroma ? 3 : 1); }

// k_huff<RAW> over the n * S segments of sp (P: the coefficient arrays and DC predictors).  The strings go
// to raw_area, each segment's bit count and tail after them (seg_raw: a band's travel with its strings to a
// later splice); the segments' flags stay in seg_scratch (its ent.ovf).  Arrays without extents are the
// caller's: checked, see code_block.
static int code_segments(pixo_b200_ctx *ctx, EntParams P, const HuffDev &T, const HuffDev *tabs,
                         const FrameGeometry &g, const SegPlan &sp, uint8_t *scratch, uint8_t *raw_area)
{
    const bool check = P.e.y == nullptr;
    cudaStream_t st = ctx->stream;
    const EntropyPlan ent = seg_scratch(sp, scratch).ent;
    const SegRaw raw = seg_raw(sp, raw_area);
    P.nimages = sp.n * sp.S;
    P.seg_per_img = sp.S;
    P.nblocks = (uint32_t)(sp.seg_mcus * sp.bpm);
    P.nblocks_last = (uint32_t)(sp.last_mcus * sp.bpm);
    P.nunits = (uint32_t)ent.nunits;
    P.seg_y_stride = (size_t)sp.seg_mcus * g.y_per_mcu * 64;
    P.seg_c_stride = (size_t)sp.seg_mcus * 64;
    P.rst_blocks = P.rst_mcus = P.upi = 0;
    P.st_bits = ent.st1;
    P.st_ff = ent.st2;
    P.ticket = ent.ticket;
    P.overflow = ent.ovf;
    P.out_len = ent.out_len;
    P.out_tail = ent.tail;
    P.out = raw.strings;
    P.out_cap = sp.raw_cap;
    PIXO_CUDA(ctx, cudaMemsetAsync(ent.st1, 0, ent.zero_bytes, st));
    const size_t want = ((size_t)P.nimages * P.nunits + HUFF_WARPS - 1) / HUFF_WARPS;
    const unsigned grid = (unsigned)std::min<size_t>(want, (size_t)ctx->sm_count * HUFF_CTAS_PER_SM);
    if (tabs)
        PIXO_TRY(launch(ctx, check ? k_huff<true, true, true> : k_huff<true, false, true>, grid, 32 * HUFF_WARPS, 0, P,
                        FrameTables{tabs}));
    else
        PIXO_TRY(launch(ctx, check ? k_huff<true, true, false> : k_huff<true, false, false>, grid, 32 * HUFF_WARPS, 0, P, T));
    PIXO_CUDA(ctx, cudaMemcpyAsync(raw.bits, P.out_len, (size_t)sp.n * sp.S * 8, cudaMemcpyDeviceToDevice, st));
    PIXO_CUDA(ctx, cudaMemcpyAsync(raw.tails, P.out_tail, (size_t)sp.n * sp.S * 8, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// The splice kernels' parameters (see splice_segments)
static SegParams splice_params(const SegPlan &sp, uint8_t *scratch, const uint8_t *raw_area, const uint32_t *raw_overflow,
                               uint64_t base_bit, uint32_t base_tail, bool last, const uint64_t *base_dev, uint8_t *d_out,
                               uint64_t out_cap, uint64_t *d_out_len, uint32_t *d_overflow)
{
    const SegScratch s = seg_scratch(sp, scratch);
    const SegRaw raw = seg_raw(sp, const_cast<uint8_t *>(raw_area));
    SegParams Q;
    Q.raw = raw_area; Q.raw_cap = sp.raw_cap;
    Q.bits = raw.bits;
    Q.tails = raw.tails;
    Q.S = sp.S; Q.max_tiles = sp.max_tiles;
    Q.base_bit = base_bit; Q.base_tail = base_tail; Q.last_band = last ? 1u : 0u;
    Q.base_dev = reinterpret_cast<const unsigned long long *>(base_dev);
    Q.rec = s.rec;
    Q.ntiles = s.ntiles;
    Q.cnt = s.cnt;
    Q.out = d_out; Q.out_cap = out_cap;
    Q.out_len = reinterpret_cast<unsigned long long *>(d_out_len);
    Q.overflow = d_overflow;
    Q.raw_overflow = raw_overflow;
    return Q;
}

// The four splice kernels over the n images of sp whose segment strings, bit counts and tails are in
// raw_area: final bytes in d_out (out_cap per image), byte counts and flags in d_out_len / d_overflow.
// raw_overflow: the coding kernel's flags per segment, or null.  base_bit / base_tail / last / base_dev:
// see SegParams (a band of a tiled frame passes its place in the stream; a whole image passes 0, 0, true).
static int splice_segments(pixo_b200_ctx *ctx, const SegPlan &sp, uint8_t *scratch, const uint8_t *raw_area,
                           const uint32_t *raw_overflow, uint64_t base_bit, uint32_t base_tail, bool last,
                           const uint64_t *base_dev, uint8_t *d_out, uint64_t out_cap, uint64_t *d_out_len,
                           uint32_t *d_overflow)
{
    const SegParams Q = splice_params(sp, scratch, raw_area, raw_overflow, base_bit, base_tail, last, base_dev, d_out,
                                      out_cap, d_out_len, d_overflow);
    const dim3 tiles((sp.max_tiles + SPL_TPC - 1) / SPL_TPC, sp.n);
    PIXO_TRY(launch(ctx, k_seg_prefix, sp.n, SPL_THREADS, 0, Q));
    PIXO_TRY(launch(ctx, k_seg_count, tiles, SPL_THREADS, 0, Q));
    PIXO_TRY(launch(ctx, k_seg_scan, sp.n, 1024, 0, Q));
    return launch(ctx, k_seg_emit, tiles, SPL_THREADS, 0, Q);
}

// k_huff_tables over n frames: their statistics (K3, kHistWords each) at d_hist, or null for the standard tables.
// Each frame's tables go to d_dht as DHT data (kDhtBytes each) and to d_tabs as k_huff reads them (kHuffDevBytes
// each); either may be null.
int launch_huff_tables(pixo_b200_ctx *ctx, const uint64_t *d_hist, uint32_t n, bool has_chroma, uint8_t *d_dht,
                       void *d_tabs)
{
    HuffStd S;
    memcpy(S.dht, dht_standard(), kDhtBytes);
    HuffTables t;
    huff_standard(t);
    make_huff_dev(t, &S.dev);
    return launch(ctx, k_huff_tables, n, 128, 0, reinterpret_cast<const unsigned long long *>(d_hist),
                  has_chroma ? 1u : 0u, S, d_dht, static_cast<HuffDev *>(d_tabs));
}

// Enqueue the entropy stage for n whole images on ctx->stream.  d_scratch: entropy_scratch_bytes.
// d_out: n * out_cap bytes of scan data; *d_out_len / *d_overflow point into the scratch.
// allow_segments: few long images may be cut into segments.  ext: the arrays are the transform's
// coefficient records; null: they are the caller's natural-order arrays, and coefficients outside the
// baseline range are rejected (overflow bit 3, see code_block).  d_tabs: every frame's own tables
// (launch_huff_tables), t is then unused; null: t for every frame.
int launch_jpeg_entropy(pixo_b200_ctx *ctx, const int16_t *d_y, size_t y_stride, const int16_t *d_cb,
                        const int16_t *d_cr, size_t c_stride, uint32_t n, const FrameGeometry &g,
                        const HuffTables &t, uint32_t restart_interval, bool allow_segments,
                        const CoefExtents *ext, uint8_t *d_scratch, uint8_t *d_out, uint64_t out_cap,
                        uint64_t **d_out_len, uint32_t **d_overflow, const void *d_tabs)
{
    const bool check = ext == nullptr;
    const auto *tabs = static_cast<const HuffDev *>(d_tabs);
    const uint64_t nblocks = g.ny + 2 * g.nc;
    const uint64_t bpm_ = g.y_per_mcu + (g.has_chroma ? 2 : 0);
    uint64_t rst_blocks = (uint64_t)restart_interval * bpm_;
    if (rst_blocks >= nblocks) rst_blocks = 0;  // a single interval: no marker is ever written
    Layout L(d_scratch);
    const EntropyPlan pl = plan_entropy(L, n, nblocks, rst_blocks);
    if (nblocks > 0xFFFFFFFFull || (uint64_t)n * pl.nunits > 0x7FFFFFFFull)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "entropy stage: too many blocks per call");
    EntParams P;
    P.y = d_y; P.cb = d_cb; P.cr = d_cr; P.y_stride = y_stride; P.c_stride = c_stride;
    P.e = ext ? *ext : CoefExtents{nullptr, nullptr, nullptr, 0};
    P.bpm = g.y_per_mcu + (g.has_chroma ? 2 : 0);
    P.y_per_mcu = g.y_per_mcu;
    P.nblocks = (uint32_t)nblocks;
    P.nunits = (uint32_t)pl.nunits;
    P.rst_blocks = (uint32_t)rst_blocks;
    P.rst_mcus = rst_blocks ? restart_interval : 0u;
    P.upi = rst_blocks ? (uint32_t)((rst_blocks + UB - 1) / UB) : 0u;
    P.nimages = n;
    P.st_bits = pl.st1;
    P.st_ff = pl.st2;
    P.ticket = pl.ticket;
    P.overflow = pl.ovf;
    P.out_len = pl.out_len;
    P.out = d_out; P.out_cap = out_cap;
    P.out_tail = pl.tail;
    P.dc_seed[0] = P.dc_seed[1] = P.dc_seed[2] = 0;
    P.dc_seed_dev = nullptr;
    P.win = nullptr;   // set below; k_huff<RAW> has no phase B
    *d_out_len = P.out_len;
    *d_overflow = P.overflow;

    HuffDev T;
    make_huff_dev(t, &T);
    cudaStream_t st = ctx->stream;
    PIXO_CUDA(ctx, cudaMemsetAsync(pl.st1, 0, pl.zero_bytes, st));
    P.seg_per_img = 1; P.nblocks_last = P.nblocks; P.seg_y_stride = P.seg_c_stride = 0;
    // few images: cut each into segments (short look-back chains) and splice - see k_seg_*
    const uint32_t S = (rst_blocks == 0 && allow_segments) ? segments_for(n, g.total_mcus(), bpm_) : 1;
    const SegPlan sp = plan_segments(n, S, g.total_mcus(), bpm_, mcu_raw_bytes(g));
    if (sp.S > 1) {   // d_raw: the segment scratch, then the raw area
        uint8_t *scratch, *raw_area;
        PIXO_TRY(bind(ctx, ctx->d_raw, [&](Layout &R) {
            scratch = R.take(seg_scratch_bytes(sp)), raw_area = R.take(seg_raw(sp, nullptr).total);
        }));
        PIXO_TRY(code_segments(ctx, P, T, tabs, g, sp, scratch, raw_area));
        return splice_segments(ctx, sp, scratch, raw_area, seg_scratch(sp, scratch).ent.ovf, 0, 0, true, nullptr, d_out,
                               out_cap, P.out_len, P.overflow);
    }
    const size_t want = ((size_t)n * pl.nunits + HUFF_WARPS - 1) / HUFF_WARPS;
    const unsigned grid = (unsigned)std::min<size_t>(want, (size_t)ctx->sm_count * HUFF_CTAS_PER_SM);
    PIXO_TRY(ctx->d_hwin.ensure(ctx, (size_t)grid * HUFF_WARPS * GWIN_B));
    P.win = reinterpret_cast<uint8_t *>(ctx->d_hwin.ptr);
    if (tabs)
        return launch(ctx, check ? k_huff<false, true, true> : k_huff<false, false, true>, grid, 32 * HUFF_WARPS, 0, P,
                      FrameTables{tabs});
    return launch(ctx, check ? k_huff<false, true, false> : k_huff<false, false, false>, grid, 32 * HUFF_WARPS, 0, P, T);
}

size_t band_raw_bytes(const FrameGeometry &g)
{
    return seg_raw(plan_segments(1, 1, g.total_mcus(), g.y_per_mcu + (g.has_chroma ? 2 : 0), mcu_raw_bytes(g)), nullptr)
        .total;
}

// Code one band of a frame tiled over several GPUs into the caller's buffer d_raw (k_huff<RAW> over S >= 1
// segments, see code_segments), then k_band_totals: the band's {bit count, last 7 bits} to d_bits_tail, its
// flags OR-ed into *d_flags.  DC predictors: d_dc_seed (device memory) when it is not null, else dc_seed.
// A long band is cut into segments when allow_segments is set and their strings fit raw_cap; otherwise the
// band is one string, in whatever raw_cap leaves after the trailer of bit count and tail.  A segment's
// share is its pixel bytes + 4 KiB, so a dense band (large coefficients) can outgrow it (bit 0) although
// the band as one string fits raw_cap: the caller then codes it again without segments.
int launch_band_entropy(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb, const int16_t *d_cr,
                        const FrameGeometry &g, const HuffTables &t, const int dc_seed[3], const int *d_dc_seed,
                        bool allow_segments, uint8_t *d_raw, uint64_t raw_cap, uint64_t *d_bits_tail,
                        uint32_t *d_flags)
{
    if ((g.ny + 2 * g.nc) > 0xFFFFFFFFull)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "entropy stage: too many blocks per call");
    const uint64_t bpm = g.y_per_mcu + (g.has_chroma ? 2 : 0);
    SegPlan sp = plan_segments(1, allow_segments ? segments_for(1, g.total_mcus(), bpm) : 1, g.total_mcus(), bpm,
                               mcu_raw_bytes(g));
    if (sp.S == 1 || seg_raw(sp, nullptr).total > raw_cap) {
        sp = plan_segments(1, 1, g.total_mcus(), bpm, mcu_raw_bytes(g));
        const SegRaw need = seg_raw(sp, nullptr);
        if (raw_cap < need.trailer)
            return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "raw capacity %llu too small (need %zu)",
                             (unsigned long long)raw_cap, need.total);
        set_raw_cap(sp, Layout::floor((size_t)(raw_cap - need.trailer)));
    }
    PIXO_TRY(ctx->d_raw.ensure(ctx, seg_scratch_bytes(sp)));
    auto *scratch = static_cast<uint8_t *>(ctx->d_raw.ptr);
    EntParams P;
    memset(&P, 0, sizeof P);
    P.y = d_y; P.cb = d_cb; P.cr = d_cr;
    P.bpm = (uint32_t)bpm; P.y_per_mcu = g.y_per_mcu;
    for (int k = 0; k < 3; ++k) P.dc_seed[k] = dc_seed ? dc_seed[k] : 0;
    P.dc_seed_dev = d_dc_seed;
    HuffDev T;
    make_huff_dev(t, &T);
    ctx->bands[d_raw] = sp;
    PIXO_TRY(code_segments(ctx, P, T, nullptr, g, sp, scratch, d_raw));   // a band's arrays are the caller's (no extents)
    const SegRaw raw = seg_raw(sp, d_raw);
    return launch(ctx, k_band_totals, 1, 32, 0, raw.bits, raw.tails, seg_scratch(sp, scratch).ent.ovf, sp.S,
                  reinterpret_cast<unsigned long long *>(d_bits_tail), d_flags);
}

// Splice the strings launch_band_entropy left in the caller's buffer d_raw into the band's scan bytes.  The
// band's place in the frame's stream: {start bit, the stream's last 7 bits before it, last band} in device
// memory at d_base when it is not null, else base_bit / base_tail / last.
int launch_band_splice(pixo_b200_ctx *ctx, const uint8_t *d_raw, uint64_t base_bit, uint32_t base_tail, bool last,
                       const uint64_t *d_base, uint8_t *d_out, uint64_t out_cap, uint64_t *d_out_len,
                       uint32_t *d_flags)
{
    const auto it = ctx->bands.find(d_raw);
    if (it == ctx->bands.end())
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "this raw buffer was not coded by pixo_b200_jpeg_band_entropy_dev");
    const SegPlan sp = it->second;
    PIXO_TRY(ctx->d_raw.ensure(ctx, seg_scratch_bytes(sp)));
    return splice_segments(ctx, sp, static_cast<uint8_t *>(ctx->d_raw.ptr), d_raw, nullptr, base_bit, base_tail, last,
                           d_base, d_out, out_cap, d_out_len, d_flags);
}

SegPlan splice_plan(uint32_t n, size_t raw_cap)
{
    SegPlan p;
    p.n = n;
    p.S = 1;
    p.seg_mcus = p.last_mcus = 0;
    p.bpm = 1;
    set_raw_cap(p, raw_cap);
    return p;
}

// The progressive scans of whole frames: every frame one string, its scans byte-aligned in it.
// k_seg_fit runs between the prefix of the tiles' 0xFF counts and the emission, so that a frame is written whole or
// not at all.  d_overflow must be set before (k_seg_emit only ORs into it).
int launch_splice_bounded(pixo_b200_ctx *ctx, const SegPlan &sp, uint8_t *seg_scratch, const uint8_t *raw_area,
                          uint8_t *d_out, uint64_t out_cap, uint64_t *d_out_len, uint32_t *d_overflow,
                          const unsigned long long *bounds, uint32_t nr, uint64_t *range_len)
{
    const SegParams Q = splice_params(sp, seg_scratch, raw_area, nullptr, 0, 0, true, nullptr, d_out, out_cap,
                                      d_out_len, d_overflow);
    const dim3 tiles((sp.max_tiles + SPL_TPC - 1) / SPL_TPC, sp.n);
    PIXO_TRY(launch(ctx, k_seg_prefix, sp.n, SPL_THREADS, 0, Q));
    PIXO_TRY(launch(ctx, k_seg_count, tiles, SPL_THREADS, 0, Q));
    PIXO_TRY(launch(ctx, k_seg_scan, sp.n, 1024, 0, Q));
    PIXO_TRY(launch(ctx, k_seg_fit, sp.n, SPL_THREADS, 0, Q, bounds, nr,
                    reinterpret_cast<unsigned long long *>(range_len)));
    return launch(ctx, k_seg_emit, tiles, SPL_THREADS, 0, Q);
}

}  // namespace pixo
