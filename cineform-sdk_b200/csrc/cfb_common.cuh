// cfb_common.cuh -- shared device/host definitions for the sm_90a wavelet kernels.
//
// Arithmetic convention ("fast path"): every kernel computes the reference's 2-6
// lifting in exact 32-bit integer arithmetic.  The reference (SSE2) computes the
// same expressions with saturating 16-bit chains in its vector loops and int32 +
// clamp in its scalar tails; the two agree with exact arithmetic whenever no
// intermediate leaves int16, which holds for every coefficient produced from
// sources within their declared precision (10-bit 4:2:2, 12-bit RGB/Bayer) except
// the few positions handled explicitly (6-tap border filters are clamped exactly
// as the reference clamps them).  See DESIGN.md "Overflow semantics".
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace cfb {

constexpr int kMaxBatch = 16;     // == CFB_MAX_BATCH
constexpr int kMaxChannels = 4;
constexpr int kStripIn = 256;     // input samples per warp-row (8 per lane)
constexpr int kStripOut = 128;    // output coefficients per warp-row per band

// q = (x*m + (x < 0 ? cneg : cpos)) >> 16  ==  sign(x) * (((|x| + mid) * m) >> 16)
// with m = 65536/divisor, cpos = mid*m, cneg = 65535 - mid*m   (Codec/quantize.c:1395-1516)
struct QuantParam {
    int m;
    int cpos;
    int cneg;
    int pad;
};

struct PlaneGeom {
    int width;          // input samples per row of this channel
    int height;         // input rows
    int in_pitch;       // bytes
    int out_pitch;      // bytes
    long long in_off;   // byte offset of the plane from the frame's input base
    long long band_off[4];  // byte offsets of LL,LH,HL,HH from the frame's output base
    QuantParam q[4];
    int quant_ll;       // != 0: LL is quantised with q[0] (plain variant with divisor > 1)
};

struct FwdParams {
    int nchan;
    int nframes;
    int th;             // output rows per warp
    int shift;          // level 1: precision - 8 (8-bit 4:2:2), precision - 10 (10-bit RGB words), 16 - precision (16-bit, V210)
    int uyvy;           // packed 8-bit 4:2:2: 1 = UYVY byte order
    PlaneGeom ch[kMaxChannels];
    const unsigned char *in_base[kMaxBatch];
    unsigned char *out_base[kMaxBatch];
    const unsigned short *lut;      // Bayer only: encode curve, 1 << 14 entries (frame.c:5208), null = samples >> shift
    int byteswap;       // 10-bit RGB words: 1 = the word is stored byte-swapped (R210, DPX0)
    int field_pos;      // 10-bit RGB words: bit position of the field of the launch's one channel
    int bayer_phase;    // Bayer only: BAYER_FORMAT_* (0 RED_GRN, 1 GRN_RED, 2 GRN_BLU, 3 BLU_GRN)
};
// ch[] at byte 24 and the 64-byte-aligned FwdTmaMaps after FwdParams in the parameters of k_fwd_422_tma, k_fwd_422_l12_tma
// and k_fwd_tma at byte 832: the kernels that read none of the fields after lut keep their parameter offsets
static_assert(offsetof(FwdParams, ch) == 24 && sizeof(FwdParams) == 816, "FwdParams layout");
static_assert((sizeof(FwdParams) + 63) / 64 * 64 == 832, "FwdTmaMaps offset in the level-1 TMA kernels' parameters");

constexpr int kInvStrip = 120;    // band columns written per warp-row by the inverse kernels (30 lanes x 4)

struct InvGeom {
    int width;          // band width (coefficients)
    int height;         // band rows
    int pitch;          // band pitch in bytes
    int out_pitch;      // bytes
    long long band_off[4];
    long long out_off;
    int dq[4];          // dequantisation factors (divisors); LL normally 1
};

struct InvParams {
    int nchan;
    int nframes;
    int th;             // band rows per warp
    int shift;          // 8-bit 4:2:2 output: precision - 8
    int uyvy;           // 8-bit 4:2:2 output: 1 = UYVY byte order
    int ll_unsigned;    // reduced-resolution 8-bit output: LL is shifted as unsigned (quarter resolution)
    InvGeom ch[kMaxChannels];
    const unsigned char *in_base[kMaxBatch];
    unsigned char *out_base[kMaxBatch];
    // 16-bit unsigned outputs (YU64, RG48, B64A): v = max(t >> 1, 0) << up_shift, limited to hi_simd in the columns the
    // reference's 8-column SSE2 loop produces and to 65535 from band column tail_col[c] on (scalar tail + right border:
    // InvertHorizontalStrip16s.c:16571 InvertHorizontalStrip16sToRow16u, `protection` clamp vs SATURATE_16U)
    int up_shift;       // 16 - precision
    int hi_simd;        // ((1 << precision) - 1) << up_shift
    int tail_col[kMaxChannels];
    union {
        // 10-bit RGB outputs: bit positions of R, G, B in the 32-bit word, and whether the word is stored byte-swapped
        struct { int pos[3]; int byteswap; } rgb10;
        // BYR4 output: the linear-restore table (1 << 14 entries, null = the `& 0xfffe` rule) and the Bayer phase
        // (BAYER_FORMAT_*, as FwdParams::bayer_phase)
        struct { const unsigned short *restore; int phase; } bayer;
    };
};
// the kernels that take a second parameter after InvParams (k_inv_422_tma, k_inv_fields, k_fields_carry) keep its offset
static_assert(sizeof(InvParams) == 608, "InvParams layout");

// inverse levels 3 and 2 in one pass (k_inv_l32): the level-3 bands and the level-2 bands of every channel.  The output is
// LL1 at l2[c].out_off / out_pitch; LL2 stays in registers, so l3[c].out_off / out_pitch and l2[c].band_off[0] are not read.
struct InvL32Params {
    int nchan;
    int nframes;
    int th;             // level-2 band rows per warp
    int pad;
    InvGeom l3[kMaxChannels];
    InvGeom l2[kMaxChannels];
    const unsigned char *in_base[kMaxBatch];
    unsigned char *out_base[kMaxBatch];
};
static_assert(sizeof(InvGeom) == 72 && sizeof(InvL32Params) == 848, "InvL32Params layout");

// what the final inverse level writes: 8-bit YUYV / UYVY, YU64 and V210 of a 4:2:2 codec (k_inv_422_tma); RG48, B64A,
// B64A with the alpha of channel 3, and the 10-bit RGB words (RG30 / AB10 / AR10 / R210 / DPX0) of a 4:4:4 codec (k_inv_444);
// the int16 planes of any codec (k_inv_plane, interlaced: k_inv_fields<true>); the BYR4 mosaic of a Bayer codec (k_inv_444)
enum InvOut { kInvOut8, kInvOutYU64, kInvOutV210, kInvOutRG48, kInvOutB64A, kInvOutB64AAlpha, kInvOutRGB10, kInvOutPlanes, kInvOutBYR4 };
// what forward level 1 reads: 4:2:2 as 8-bit YUYV / UYVY (k_fwd_422_tma, k_fwd_422_l12_tma), 16-bit YU64 or 10-bit V210
// (k_fwd_422_src; interlaced: k_fwd_422_fields), int16 planes (k_fwd_plane), 4:4:4 as RG48, B64A or RG64 (k_fwd_tma),
// the 10-bit RGB words (k_fwd_rgb30), 16-bit or 12-bit packed Bayer (k_fwd_tma)
enum FwdSrc { kFwdPacked8, kFwdYU64, kFwdV210, kFwdPlanes, kFwdRG48, kFwdB64A, kFwdRG64, kFwdRGB10, kFwdBYR4, kFwdBYR5 };

// BYR5 (12-bit packed Bayer): segment s of a packed row -- s = 0..3 the high bytes of component s (`pw` bytes each, from
// byte s * pw), s = 4..7 the low nibbles of component s - 4 (pw / 2 bytes each, from byte 4 pw + (s - 4) pw / 2).  box =
// the first byte of the TMA box of a strip's columns in that segment: the strip's first byte rounded down to 16 bytes,
// minus 16 for the left halo; skew = the strip's first byte - box, in [16, 32).  The host checks box % 16 == 0 before
// every launch (a box that starts off a 16-byte boundary faults); the kernel adds the skew.
struct Byr5Seg { int box; int skew; };
__host__ __device__ __forceinline__ Byr5Seg byr5_seg(int s, int pw, int strip)
{
    const int first = (s < 4) ? s * pw + strip * kStripIn : 4 * pw + (s - 4) * (pw / 2) + strip * (kStripIn / 2);
    Byr5Seg g;
    g.box = (first & ~15) - 16;
    g.skew = first - g.box;
    return g;
}

// interlaced (field) inverse: per (frame, channel, band row, strip) carry-in of the difference-coded HL band
struct FieldsAux {
    int *carry;         // [(frame * nchan + c) * maxh + row] * nstrips + strip
    int nstrips;        // strips of the luma band
    int maxh;           // band rows
    int hl_integrated;  // != 0: the HL band arrives integrated (the reference decoder's bands), no carries needed
};

// fire-and-forget prefetch into L2 (no destination register, no scoreboard): hides DRAM latency for rows that
// will be loaded a few iterations later
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }

__device__ __forceinline__ int clamp16(int v) { return max(-32768, min(32767, v)); }

__device__ __forceinline__ int quant1(int x, const QuantParam &q) {
    return x * q.m + (x < 0 ? q.cneg : q.cpos);     // result in the upper halfword
}

// pack the upper halfwords of two products / the lower halfwords of two values
__device__ __forceinline__ unsigned pack_hi(int a, int b) { return __byte_perm((unsigned)a, (unsigned)b, 0x7632); }
__device__ __forceinline__ unsigned pack_lo(int a, int b) { return __byte_perm((unsigned)a, (unsigned)b, 0x5410); }

__device__ __forceinline__ int lo16(unsigned w) { return (int)(short)(w & 0xffffu); }
__device__ __forceinline__ int hi16(unsigned w) { return ((int)w) >> 16; }

// dp4a with unsigned data bytes and signed coefficient bytes
__device__ __forceinline__ int dp4a_us(unsigned a, int b, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

}  // namespace cfb
