// cfb_forward.cu -- forward 2-6 wavelet level + fused quantisation, sm_90a.
//
// Replaces (reference, per level and channel):
//   Codec/spatial.c:10026 FilterSpatialQuant16s      -> k_fwd_plane<0>
//   Codec/spatial.c:12942 FilterSpatialV210Quant16s  -> k_fwd_plane<2>
//   Codec/spatial.c:14726 FilterSpatialYUVQuant16s   -> k_fwd_422_tma (+ Codec/convert.c:4667 unpack)
//   Codec/quantize.c:1395 QuantizeRow16sTo16s         -> fused into the band stores
//
// Design (see DESIGN.md): one WARP owns a strip of 128 output columns x TH output
// rows.  Each lane takes 16 bytes of an input row into registers -- straight from
// global memory (coalesced 128-bit loads) in the plane and 16-bit / 10-bit packed
// kernels of this file, from a ring in shared memory that TMA keeps full in the
// level-1 kernels of packed 8-bit 4:2:2, RG48 and BYR4 (cfb_forward_tma.inl) --
// does the horizontal lifting for its 4 output columns exchanging one value with
// each neighbour lane by warp shuffle, and keeps two or three values per column of
// vertical state in registers.  With S_j = row(2j)+row(2j+1) and D_j = row(2j)-row(2j+1)
// the vertical 2-6 filter is   low_j = S_j,  high_j = ((S_{j+1} - S_{j-1} + 4) >> 3) + D_j,
// the top/bottom 6-tap border filters are (-3 S0 + 8 D0 + 4 S1 - S2 + 4) >> 3 and
// (3 S_n + 8 D_n - 4 S_{n-1} + S_{n-2} + 4) >> 3 (same identities horizontally).
// Every input sample is read from global memory once (+ 1 halo row pair per strip
// block, served by L2) and every coefficient is written once with 64-bit stores.
//
// Work split inside one launch: "main" warps run a compact loop that emits every
// LL/LH row and the interior HL/HH rows; the two border rows of HL/HH (first and
// last output row, which use the 6-tap border filters) are produced by dedicated
// border warps in an extra CTA row, so the hot loop carries no border code.
#include "cfb_host.h"
#include "cfb_tma.cuh"
#include <type_traits>

namespace cfb {

// ----------------------------------------------------------------------------
struct LaneInfo {
    unsigned amask;         // lanes of this warp that hold image columns
    bool left_border;       // lane owns output column 0
    bool right_border;      // lane owns the last output column
    bool has_border;        // warp-uniform: this strip touches the left or right image border
    bool use_lh, use_rh;    // lane 0 / last lane need a halo word from the neighbouring strip
    int col0;               // the lane's first input column
};

template <int NC> struct VecStore;
template <> struct VecStore<4> {
    static __device__ __forceinline__ void st(unsigned char *p, unsigned a, unsigned b) {
        *reinterpret_cast<uint2 *>(p) = make_uint2(a, b);
    }
};
template <> struct VecStore<2> {
    static __device__ __forceinline__ void st(unsigned char *p, unsigned a, unsigned) {
        *reinterpret_cast<unsigned *>(p) = a;
    }
};
template <int NC>
__device__ __forceinline__ void store_raw(unsigned char *p, const int *v) {
    if (NC == 4) VecStore<4>::st(p, pack_lo(v[0], v[1]), pack_lo(v[2], v[3]));
    else VecStore<2>::st(p, pack_lo(v[0], v[1]), 0u);
}
template <int NC>
__device__ __forceinline__ void store_quant(unsigned char *p, const int *v, const QuantParam &q) {
    if (NC == 4)
        VecStore<4>::st(p, pack_hi(quant1(v[0], q), quant1(v[1], q)), pack_hi(quant1(v[2], q), quant1(v[3], q)));
    else if (NC == 2)
        VecStore<2>::st(p, pack_hi(quant1(v[0], q), quant1(v[1], q)), 0u);
    else
        *reinterpret_cast<short *>(p) = (short)(quant1(v[0], q) >> 16);
}

// predicated 64/32/16-bit global stores: the address and the value are computed unconditionally and only the store is
// guarded, so the hot loop carries no divergence-safe branch (BSSY/BSYNC/BRA) around its band stores
__device__ __forceinline__ void st_pred(unsigned char *p, unsigned a, unsigned b, bool on) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %3, 0;\n\t@p st.global.v2.u32 [%0], {%1, %2};\n\t}"
                 :: "l"(p), "r"(a), "r"(b), "r"((int)on) : "memory");
}
__device__ __forceinline__ void st_pred(unsigned char *p, unsigned a, bool on) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %2, 0;\n\t@p st.global.u32 [%0], %1;\n\t}"
                 :: "l"(p), "r"(a), "r"((int)on) : "memory");
}
__device__ __forceinline__ void st_pred16(unsigned char *p, unsigned a, bool on) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %2, 0;\n\t@p st.global.u16 [%0], %1;\n\t}"
                 :: "l"(p), "h"((unsigned short)a), "r"((int)on) : "memory");
}
template <int NC>
__device__ __forceinline__ void store_raw_if(unsigned char *p, const int *v, bool on) {
    if (NC == 4) st_pred(p, pack_lo(v[0], v[1]), pack_lo(v[2], v[3]), on);
    else if (NC == 2) st_pred(p, pack_lo(v[0], v[1]), on);
    else st_pred16(p, (unsigned)v[0], on);
}
template <int NC>
__device__ __forceinline__ void store_quant_if(unsigned char *p, const int *v, const QuantParam &q, bool on) {
    if (NC == 4)
        st_pred(p, pack_hi(quant1(v[0], q), quant1(v[1], q)), pack_hi(quant1(v[2], q), quant1(v[3], q)), on);
    else if (NC == 2)
        st_pred(p, pack_hi(quant1(v[0], q), quant1(v[1], q)), on);
    else
        st_pred16(p, (unsigned)quant1(v[0], q) >> 16, on);
}

// Vertical state per column: two values.  With t_j = 8 D_j - S_{j-1} the interior highpass row is
//   high_{j-1} = ((S_j - S_{j-2} + 4) >> 3) + D_{j-1} = (S_j + t_{j-1} + 4) >> 3      (8 D is a multiple of 8: exact)
// so a step needs t_{j-1} and S_{j-1} only (to form t_j); S_{j-2} and D_{j-1} are never kept separately, which saves
// the register moves of a three-value state.  A warp starts at pair max(y0 - 1, 0) with zeroed state.
template <int NC> struct RotState {
    int t[2 * NC];      // t_{j-1} = 8 D_{j-1} - S_{j-2}
    int s[2 * NC];      // S_{j-1}; after a step, s[0..NC) = the lowpass (LL) sums of row j
};

// What vstep_rot does with the LL band: store it as is (the 4:2:2 level-1 filter, spatial.c:14726), store it quantised
// when g.quant_ll is set (planar filter with an LL divisor > 1, spatial.c:10480), or leave it in RotState::s for the
// caller (the fused levels 1 + 2 of cfb_forward_l12.inl).
enum LLStore { kLLRaw, kLLQuantIf, kLLNone };

// One vertical step on the horizontal outputs of rows 2j (a) and 2j+1 (b); [0,NC) = low, [NC,2NC) = high.
// emit_low : store LL/LH of output row j        at byte offset off
// emit_high: store HL/HH of output row j-1      at byte offset off - pitch   (interior formula)
// Both flags are warp-uniform.
template <int NC, LLStore LL>
__device__ __forceinline__ void vstep_rot(RotState<NC> &st, const int *a, const int *b, const PlaneGeom &g, unsigned char *out,
                                          unsigned off, bool emit_low, bool emit_high)
{
    int v[2 * NC], h[2 * NC];
#pragma unroll
    for (int i = 0; i < 2 * NC; i++) {
        v[i] = a[i] + b[i];
        h[i] = (v[i] + st.t[i] + 4) >> 3;
        st.t[i] = ((a[i] - b[i]) << 3) - st.s[i];
        st.s[i] = v[i];
    }
    if (LL == kLLQuantIf && g.quant_ll) store_quant_if<NC>(out + (g.band_off[0] + off), v, g.q[0], emit_low);
    else if (LL != kLLNone) store_raw_if<NC>(out + (g.band_off[0] + off), v, emit_low);
    store_quant_if<NC>(out + (g.band_off[1] + off), v + NC, g.q[1], emit_low);
    const unsigned offh = off - (unsigned)g.out_pitch;
    store_quant_if<NC>(out + (g.band_off[2] + offh), h, g.q[2], emit_high);
    store_quant_if<NC>(out + (g.band_off[3] + offh), h + NC, g.q[3], emit_high);
}

// Border rows of HL/HH from three consecutive pairs (S,D of each): spatial.c:10166-10208 / :10516-10558.
//   top   : pairs 0,1,2      -> row 0     = clamp((-3 S0 + 8 D0 + 4 S1 - S2 + 4) >> 3)
//   bottom: pairs n-2,n-1,n  -> row n     = clamp(( 3 Sn + 8 Dn - 4 S(n-1) + S(n-2) + 4) >> 3)
template <int NC>
__device__ __forceinline__ void border_emit(const int *s0, const int *s1, const int *s2, const int *dsel, bool bottom,
                                            const PlaneGeom &g, unsigned char *out, unsigned off)
{
    int h[2 * NC];
#pragma unroll
    for (int i = 0; i < 2 * NC; i++)
        h[i] = bottom ? clamp16((3 * s2[i] + 8 * dsel[i] - 4 * s1[i] + s0[i] + 4) >> 3)
                      : clamp16((-3 * s0[i] + 8 * dsel[i] + 4 * s1[i] - s2[i] + 4) >> 3);
    store_quant<NC>(out + (g.band_off[2] + off), h, g.q[2]);
    store_quant<NC>(out + (g.band_off[3] + off), h + NC, g.q[3]);
}

// S of three consecutive pairs and D of the outer pair (first pair for the top row, last pair for the bottom row)
template <int NC> struct BorderAcc {
    int s[3][2 * NC], d[2 * NC];
    __device__ __forceinline__ void add(int k, bool keep, const int *a, const int *b) {
#pragma unroll
        for (int i = 0; i < 2 * NC; i++) {
            s[k][i] = a[i] + b[i];
            if (keep) d[i] = a[i] - b[i];
        }
    }
    __device__ __forceinline__ void emit(bool bottom, const PlaneGeom &g, unsigned char *out, int row, unsigned colbyte) {
        border_emit<NC>(s[0], s[1], s[2], d, bottom, g, out, (unsigned)(row * g.out_pitch) + colbyte);
    }
};

// First (bottom = false) or last HL/HH row of a level, for a plane (NC1 = 0: NY columns per lane) or for the luma and the
// two chroma channels of a 4:2:2 source (NY luma and NC1 columns of each chroma channel per lane).  row(r, y, c1, c2)
// writes the horizontal outputs (low, then high) of input row r of the level; c1 goes to channel g1, c2 to g2.
template <int NY, int NC1, class ROW>
__device__ __forceinline__ void border_rows(const ROW &row, int oh, bool bottom, unsigned char *out,
                                            const PlaneGeom &gy, unsigned colbyte_y,
                                            const PlaneGeom &g1, const PlaneGeom &g2, unsigned colbyte_c)
{
    constexpr int NC = NC1 ? NC1 : 1;
    const int j0 = bottom ? oh - 3 : 0;
    BorderAcc<NY> ay;
    BorderAcc<NC> a1, a2;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        int y0[2 * NY], y1[2 * NY], c10[2 * NC], c11[2 * NC], c20[2 * NC], c21[2 * NC];
        row(2 * (j0 + k), y0, c10, c20);
        row(2 * (j0 + k) + 1, y1, c11, c21);
        const bool keep = (k == (bottom ? 2 : 0));
        ay.add(k, keep, y0, y1);
        if (NC1) { a1.add(k, keep, c10, c11); a2.add(k, keep, c20, c21); }
    }
    const int r = bottom ? oh - 1 : 0;
    ay.emit(bottom, gy, out, r, colbyte_y);
    if (NC1) { a1.emit(bottom, g1, out, r, colbyte_c); a2.emit(bottom, g2, out, r, colbyte_c); }
}

// ----------------------------------------------------------------------------
// int16 plane input
struct RawPlaneRow {
    uint4 v;            // 8 samples of this lane
    unsigned halo;      // lane 0: samples [-2,-1] of the strip; last lane: samples [+256,+257]
};

__device__ __forceinline__ void load_plane_row(const unsigned char *p, const LaneInfo &L, RawPlaneRow &r)
{
    r.v = __ldg(reinterpret_cast<const uint4 *>(p));
    // ONE predicated halo load per row (two loads into the same register would serialise on its scoreboard)
    r.halo = 0u;
    if (L.use_lh | L.use_rh) r.halo = __ldg(reinterpret_cast<const unsigned *>(p + (L.use_lh ? -4 : 16)));
}

// ---- packed 16-bit RGB (RG48) input: a lane's 8 pixels are 48 contiguous bytes; one channel (word SEL of each
// pixel: 0 = R, 1 = G, 2 = B) is extracted and reduced to the codec precision (>> shift), as
// Codec/frame.c:5968 ConvertRGB48ToFrame16s (default branch :6130-6164) does on the host.
struct RawRG48Row {
    uint4 a, b, c;      // 24 words = 8 pixels x 3
    unsigned halo;      // channel samples of pixels [-2,-1] (lane 0) or [+8,+9] (last lane), already packed
};

// word index w (0..23) of the 48-byte group as a (register, half) pair -> PRMT selector nibble pair
template <int SEL>
__device__ __forceinline__ void rg48_extract(const RawRG48Row &r, int shift, RawPlaneRow &o)
{
    const unsigned w[12] = {r.a.x, r.a.y, r.a.z, r.a.w, r.b.x, r.b.y, r.b.z, r.b.w, r.c.x, r.c.y, r.c.z, r.c.w};
    unsigned out[4];
#pragma unroll
    for (int m = 0; m < 4; m++) {
        const int w0 = 3 * (2 * m) + SEL, w1 = 3 * (2 * m + 1) + SEL;      // word indices of samples 2m, 2m+1
        const unsigned lo = (w0 & 1) ? (w[w0 >> 1] >> 16) : (w[w0 >> 1] & 0xffffu);
        const unsigned hi = (w1 & 1) ? (w[w1 >> 1] & 0xffff0000u) : (w[w1 >> 1] << 16);
        out[m] = lo | hi;
    }
    const unsigned mask = (0xffffu >> shift) * 0x00010001u;
    o.v = make_uint4((out[0] >> shift) & mask, (out[1] >> shift) & mask, (out[2] >> shift) & mask, (out[3] >> shift) & mask);
    o.halo = (r.halo >> shift) & mask;
}

template <int PRESCALE>
__device__ __forceinline__ int tap(int x) { return PRESCALE ? ((x + 3) >> 2) : x; }

// horizontal 2-6 for the lane's 4 output columns: o[0..3] = low, o[4..7] = high
// (Codec/spatial.c:253 FilterHorizontalRow16s / :3669 FilterHorizontalRow10bit16s)
// dp2a with unsigned 16-bit halves (a) and signed byte coefficients (b): lo16(a) * b0 + hi16(a) * b1 + c
__device__ __forceinline__ int dp2a_lo_us(unsigned a, unsigned b, int c) {
    int d;
    asm("dp2a.lo.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
// PRESCALE = 3: the prescaled filter (PRESCALE = 2 arithmetic) for planes known to be NON-NEGATIVE, which every level-2 / 3
// input of the codec pyramid is (an LL band of an unsigned source).  Both taps of a packed pair are then prescaled in the
// packed word -- (w + 0x00030003) >> 2, masked -- and tap sum, tap difference and the lowpass (x0 + x1 + 3) >> 2 are one
// dp2a each: 7 instructions per pair against 10 (the prescaled level is issue-bound)
constexpr unsigned kOnes2 = 0x0101u, kPlusMinus2 = 0xff01u;       // dp2a byte coefficients (+1, +1) and (+1, -1)
__device__ __forceinline__ unsigned prescale_pair_nonneg(unsigned w) { return ((w + 0x00030003u) >> 2) & 0x3fff3fffu; }

template <int PRESCALE>
__device__ __forceinline__ void hfilter_plane(const RawPlaneRow &r, const LaneInfo &L, int *o)
{
    const unsigned w[4] = {r.v.x, r.v.y, r.v.z, r.v.w};
    int S[4], d[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (PRESCALE == 3) {
            const unsigned t = prescale_pair_nonneg(w[k]);
            S[k] = dp2a_lo_us(t, kOnes2, 0);
            d[k] = dp2a_lo_us(t, kPlusMinus2, 0);
            o[k] = dp2a_lo_us(w[k], kOnes2, 3) >> 2;
        } else {
            const int x0 = lo16(w[k]), x1 = hi16(w[k]);
            const int t0 = tap<PRESCALE>(x0), t1 = tap<PRESCALE>(x1);
            S[k] = t0 + t1;
            d[k] = t0 - t1;
            o[k] = PRESCALE ? ((x0 + x1 + 3) >> 2) : S[k];
        }
    }
    int Sp = __shfl_up_sync(L.amask, S[3], 1);
    int Sn = __shfl_down_sync(L.amask, S[0], 1);
    const int hs = (PRESCALE == 3) ? dp2a_lo_us(prescale_pair_nonneg(r.halo), kOnes2, 0)
                                   : tap<PRESCALE>(lo16(r.halo)) + tap<PRESCALE>(hi16(r.halo));
    Sp = L.use_lh ? hs : Sp;
    Sn = L.use_rh ? hs : Sn;
    o[4] = ((S[1] - Sp + 4) >> 3) + d[0];
    o[5] = ((S[2] - S[0] + 4) >> 3) + d[1];
    o[6] = ((S[3] - S[1] + 4) >> 3) + d[2];
    o[7] = ((Sn - S[2] + 4) >> 3) + d[3];
    if (L.has_border) {     // warp-uniform: only the first and last strip of a row carry a border lane
        if (L.left_border) o[4] = clamp16((-3 * S[0] + 8 * d[0] + 4 * S[1] - S[2] + 4) >> 3);
        if (L.right_border) o[7] = clamp16((3 * S[3] + 8 * d[3] - 4 * S[2] + S[1] + 4) >> 3);
    }
}

__device__ __forceinline__ bool lane_setup(int strip, int width, int lane, LaneInfo &L)
{
    // A lane is active only when all of its 8 input columns exist.  When the width is not a multiple of 8 the last
    // 2-6 columns (1-3 output columns, the right border among them) are produced by k_fwd_plane_edge; the last full
    // lane then takes its right neighbour value from a halo word like the last lane of an interior strip does.
    const int col0 = strip * kStripIn + lane * 8;
    const bool active = col0 + 8 <= width;
    L.col0 = col0;
    L.amask = __ballot_sync(0xffffffffu, active);
    if (!active) return false;
    L.left_border = (col0 == 0);
    L.right_border = (col0 + 8 == width);
    L.has_border = (strip == 0) || ((strip + 1) * kStripIn >= width);
    L.use_lh = (lane == 0) && (strip > 0);
    L.use_rh = (col0 + 8 < width) && (lane == 31 || col0 + 16 > width);
    return true;
}

template <int PRESCALE>
__global__ void __launch_bounds__(128) k_fwd_plane(const __grid_constant__ FwdParams p)
{
    const int lane = threadIdx.x;
    const int f = blockIdx.z / p.nchan, c = blockIdx.z - f * p.nchan;
    const PlaneGeom &g = p.ch[c];
    const int strip = blockIdx.x;
    if (strip * kStripIn >= g.width) return;
    const int oh = g.height >> 1;
    LaneInfo L;
    if (!lane_setup(strip, g.width, lane, L)) return;
    const unsigned colbyte = (unsigned)((strip * kStripOut + lane * 4) * 2);
    const unsigned char *in = p.in_base[f] + g.in_off + (strip * kStripIn + lane * 8) * 2;
    unsigned char *out = p.out_base[f];

    if (blockIdx.y == gridDim.y - 1) {
        // ---- border warps: warp 0 -> first HL/HH row, warp 1 -> last HL/HH row ----
        if (threadIdx.y > 1) return;
        border_rows<4, 0>([&](int r, int *o, int *, int *) {
            RawPlaneRow raw;
            load_plane_row(in + (long long)r * g.in_pitch, L, raw);
            hfilter_plane<PRESCALE>(raw, L, o);
        }, oh, threadIdx.y == 1, out, g, colbyte, g, g, 0u);
        return;
    }

    const int y0 = (blockIdx.y * blockDim.y + threadIdx.y) * p.th;
    if (y0 >= oh) return;
    const int y1 = min(y0 + p.th, oh);
    const int jfirst = max(y0 - 1, 0), jlast = min(y1, oh - 1);
    const int hlo = max(y0, 1);     // first HL/HH row this warp emits (row 0 belongs to the border warp)

    RotState<4> st;
#pragma unroll
    for (int i = 0; i < 8; i++) { st.t[i] = st.s[i] = 0; }

    const unsigned char *rp = in + (long long)(2 * jfirst) * g.in_pitch;
    RawPlaneRow c0, c1, n0, n1;
    load_plane_row(rp, L, c0);
    load_plane_row(rp + g.in_pitch, L, c1);
    n0 = c0; n1 = c1;
    unsigned off = (unsigned)(jfirst * g.out_pitch) + colbyte;
    for (int j = jfirst; j <= jlast; j++) {
        rp += 2 * g.in_pitch;
        if (j < jlast) {
            load_plane_row(rp, L, n0);
            load_plane_row(rp + g.in_pitch, L, n1);
        }
        if (j + 2 < jlast) { prefetch_l2(rp + 4 * g.in_pitch); prefetch_l2(rp + 5 * g.in_pitch); }
        int a[8], b[8];
        hfilter_plane<PRESCALE>(c0, L, a);
        hfilter_plane<PRESCALE>(c1, L, b);
        vstep_rot<4, kLLQuantIf>(st, a, b, g, out, off, j >= y0 && j < y1, j - 1 >= hlo);
        off += (unsigned)g.out_pitch;
        c0 = n0; c1 = n1;
    }
}

// ----------------------------------------------------------------------------
// Ragged widths: output columns [4 * (width / 8), width / 2) of a plane level, one thread per coefficient position,
// written exactly as the formulas read (spatial.c:253-570 rows, :10166-10558 columns).  At most 3 columns per row, so
// the cost is nil; it keeps the lane-granular main kernel free of partial-lane cases.
template <int PRESCALE>
__global__ void __launch_bounds__(128) k_fwd_plane_edge(const __grid_constant__ FwdParams p)
{
    const int f = blockIdx.z / p.nchan, c = blockIdx.z - f * p.nchan;
    const PlaneGeom &g = p.ch[c];
    const int w = g.width, ow = w >> 1, oh = g.height >> 1;
    const int col = (w >> 3) * 4 + blockIdx.y;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= ow || j >= oh) return;
    const unsigned char *in = p.in_base[f] + g.in_off;
    auto px = [&](int r, int i) { return (int)*reinterpret_cast<const short *>(in + (long long)r * g.in_pitch + 2 * i); };
    auto hrow = [&](int r, int &lo, int &hi) {
        auto t = [&](int i) { return tap<PRESCALE>(px(r, i)); };
        const int i0 = 2 * col;
        lo = PRESCALE ? ((px(r, i0) + px(r, i0 + 1) + 3) >> 2) : (px(r, i0) + px(r, i0 + 1));
        if (col == ow - 1)
            hi = clamp16((11 * t(w - 2) - 5 * t(w - 1) - 4 * t(w - 3) - 4 * t(w - 4) + t(w - 5) + t(w - 6) + 4) >> 3);
        else
            hi = ((-t(i0 - 2) - t(i0 - 1) + t(i0 + 2) + t(i0 + 3) + 4) >> 3) + t(i0) - t(i0 + 1);
    };
    int l[6], h[6];
    const int r0 = (j == 0) ? 0 : ((j == oh - 1) ? g.height - 6 : 2 * j - 2);
#pragma unroll
    for (int k = 0; k < 6; k++) hrow(r0 + k, l[k], h[k]);
    int ll, lh, hl, hh;
    if (j == 0) {
        ll = l[0] + l[1]; lh = h[0] + h[1];
        hl = clamp16((5 * l[0] - 11 * l[1] + 4 * l[2] + 4 * l[3] - l[4] - l[5] + 4) >> 3);
        hh = clamp16((5 * h[0] - 11 * h[1] + 4 * h[2] + 4 * h[3] - h[4] - h[5] + 4) >> 3);
    } else if (j == oh - 1) {
        ll = l[4] + l[5]; lh = h[4] + h[5];
        hl = clamp16((11 * l[4] - 5 * l[5] - 4 * l[3] - 4 * l[2] + l[1] + l[0] + 4) >> 3);
        hh = clamp16((11 * h[4] - 5 * h[5] - 4 * h[3] - 4 * h[2] + h[1] + h[0] + 4) >> 3);
    } else {
        ll = l[2] + l[3]; lh = h[2] + h[3];
        hl = ((-l[0] - l[1] + l[4] + l[5] + 4) >> 3) + l[2] - l[3];
        hh = ((-h[0] - h[1] + h[4] + h[5] + 4) >> 3) + h[2] - h[3];
    }
    unsigned char *out = p.out_base[f] + (long long)j * g.out_pitch + 2 * col;
    *reinterpret_cast<short *>(out + g.band_off[0]) = (short)(g.quant_ll ? (quant1(ll, g.q[0]) >> 16) : ll);
    *reinterpret_cast<short *>(out + g.band_off[1]) = (short)(quant1(lh, g.q[1]) >> 16);
    *reinterpret_cast<short *>(out + g.band_off[2]) = (short)(quant1(hl, g.q[2]) >> 16);
    *reinterpret_cast<short *>(out + g.band_off[3]) = (short)(quant1(hh, g.q[3]) >> 16);
}

// ----------------------------------------------------------------------------
// 16-bit Bayer frames (BYR4, curve already applied): the four half-resolution planes
// G = (g1+g2)>>1, RG = (r-G+4096)>>1, BG = (b-G+4096)>>1, DG = (g1-g2+4096)>>1 at 12 bits
// (Codec/frame.c:4993 ConvertBYR4ToFrame16s, encode_curve_preset branch :5040-5200) are formed on the fly from the
// two Bayer lines of each plane row.
struct RawBYR4Row {
    uint4 a0, a1;       // Bayer line 2r   : 16 pixels of this lane
    uint4 b0, b1;       // Bayer line 2r+1
    uint2 ha, hb;       // 4 pixels of each line just outside the strip (lane 0: left, last lane: right)
};

// One plane sample is formed from a quad (w1 = two pixels of the first line, w2 = of the second line) with the channel
// known at compile time and the Bayer phase folded into byte-permute selectors (warp-uniform registers): g1 always sits
// on the first line of a quad and g2 on the second, red / blue on either.
//   selg1 / selg2: halfword of the line word holding g1 / g2;  selx: halfword holding the channel's colour sample,
//   xline: 0 = first line, 1 = second line
// LUT: the encode curve of Codec/frame.c:5208-5330 (default: log base 90), indexed by the 14 most significant bits
// (MAX_INPUT_PRECISION, frame.c:4843); without it the frame is taken as already curved (`>> shift`, encode_curve_preset).
struct BayerSel { unsigned selg1, selg2, selx; int xline; };

__device__ __forceinline__ BayerSel bayer_sel(int fmt, int chan)
{
    // quad layout (line 1: q0 q1, line 2: q2 q3): 0 RED_GRN r g / g b, 1 GRN_RED g r / b g, 2 GRN_BLU g b / r g, 3 BLU_GRN b g / g r
    const unsigned lo = 0x4410u, hi = 0x4432u;      // PRMT selectors: low / high halfword, upper half zero (second operand = 0)
    BayerSel s;
    const bool g_second = (fmt == 0) || (fmt == 3);
    s.selg1 = g_second ? hi : lo;
    s.selg2 = g_second ? lo : hi;
    const int rpos = (fmt == 0) ? 0 : (fmt == 1) ? 1 : (fmt == 2) ? 2 : 3;
    const int bpos = 3 - rpos;
    const int xpos = (chan == 1) ? rpos : bpos;
    s.selx = (xpos & 1) ? hi : lo;
    s.xline = xpos >> 1;
    return s;
}

template <bool LUT, int CHAN>
__device__ __forceinline__ int byr4_sample_c(unsigned w1, unsigned w2, int shift, const BayerSel &s, const unsigned short *lut)
{
    unsigned g1 = __byte_perm(w1, 0u, s.selg1), g2 = __byte_perm(w2, 0u, s.selg2);
    if (LUT) { g1 = __ldg(lut + (g1 >> 2)); g2 = __ldg(lut + (g2 >> 2)); } else { g1 >>= shift; g2 >>= shift; }
    if (CHAN == 3) return (int)(g1 - g2 + 4096u) >> 1;
    const unsigned gg = (g1 + g2) >> 1;
    if (CHAN == 0) return (int)gg;
    unsigned x = __byte_perm(s.xline ? w2 : w1, 0u, s.selx);
    if (LUT) x = __ldg(lut + (x >> 2)); else x >>= shift;
    return (int)(x - gg + 4096u) >> 1;
}

template <bool LUT, int CHAN>
__device__ __forceinline__ void byr4_extract_c(const RawBYR4Row &r, int shift, const BayerSel &s, const unsigned short *lut, RawPlaneRow &o)
{
    const unsigned l1[8] = {r.a0.x, r.a0.y, r.a0.z, r.a0.w, r.a1.x, r.a1.y, r.a1.z, r.a1.w};
    const unsigned l2[8] = {r.b0.x, r.b0.y, r.b0.z, r.b0.w, r.b1.x, r.b1.y, r.b1.z, r.b1.w};
    unsigned out[4];
#pragma unroll
    for (int m = 0; m < 4; m++)
        out[m] = pack_lo(byr4_sample_c<LUT, CHAN>(l1[2 * m], l2[2 * m], shift, s, lut),
                         byr4_sample_c<LUT, CHAN>(l1[2 * m + 1], l2[2 * m + 1], shift, s, lut));
    o.v = make_uint4(out[0], out[1], out[2], out[3]);
    o.halo = pack_lo(byr4_sample_c<LUT, CHAN>(r.ha.x, r.hb.x, shift, s, lut), byr4_sample_c<LUT, CHAN>(r.ha.y, r.hb.y, shift, s, lut));
}

// ----------------------------------------------------------------------------
// 10-bit packed RGB (RG30 / AB10 / AR10 / R210 / DPX0: one 32-bit word per pixel).  The reference transforms these
// frames directly (Codec/encoder.c:3158-3176 -> wavelet.c:3597 TransformForwardSpatialRGB30 ->
// spatial.c:2080 FilterHorizontalRowRGB30_16s): the 10-bit fields are filtered after `<< (precision - 10)`, planes in
// the order G, R, B like RG48.  One launch per channel: p.field_pos = bit position of the channel's field, p.byteswap != 0
// when the word is stored byte-swapped (R210, DPX0), p.shift = precision - 10.
struct RawRGB30Row {
    uint4 a, b;         // 8 pixels
    uint2 halo;         // pixels [-2,-1] (lane 0) or [+8,+9] (last lane)
};

__device__ __forceinline__ void load_rgb30_row(const unsigned char *p, const LaneInfo &L, RawRGB30Row &r)
{
    r.a = __ldg(reinterpret_cast<const uint4 *>(p));
    r.b = __ldg(reinterpret_cast<const uint4 *>(p + 16));
    r.halo = make_uint2(0u, 0u);
    if (L.use_lh | L.use_rh) r.halo = __ldg(reinterpret_cast<const uint2 *>(p + (L.use_lh ? -8 : 32)));
}

__device__ __forceinline__ unsigned rgb30_field(unsigned w, int swap, int pos, int shift)
{
    if (swap) w = __byte_perm(w, 0u, 0x0123);
    return ((w >> pos) & 0x3ffu) << shift;
}

__device__ __forceinline__ void rgb30_extract(const RawRGB30Row &r, int swap, int pos, int shift, RawPlaneRow &o)
{
    const unsigned w[8] = {r.a.x, r.a.y, r.a.z, r.a.w, r.b.x, r.b.y, r.b.z, r.b.w};
    unsigned out[4];
#pragma unroll
    for (int m = 0; m < 4; m++)
        out[m] = rgb30_field(w[2 * m], swap, pos, shift) | (rgb30_field(w[2 * m + 1], swap, pos, shift) << 16);
    o.v = make_uint4(out[0], out[1], out[2], out[3]);
    o.halo = rgb30_field(r.halo.x, swap, pos, shift) | (rgb30_field(r.halo.y, swap, pos, shift) << 16);
}

// k_fwd_rgb30 keeps the three-value vertical state (S_{j-2}, S_{j-1}, D_{j-1}): with RotState / vstep_rot the kernel
// took 911 us per 16 4K frames against 904 us with this step (H100 SXM, 400 W power limit, two alternating rounds).  As
// k_fwd_plane with a row source for these words (vstep_rot, border_rows, the plane kernel's L2 row prefetch; 80 registers
// against 94) level 1 of 16 4K RG30 or DPX0 frames took 1025.3 - 1026.5 us against 878.1 - 881.5 us for this kernel
// (H100 80GB HBM3, 700 W power limit, three alternating rounds).
template <int NC> struct VState {
    int llp[2 * NC];    // S_{j-2}
    int llc[2 * NC];    // S_{j-1}
    int dc[2 * NC];     // D_{j-1}
};

// vstep_rot<NC, kLLQuantIf> on a VState
template <int NC>
__device__ __forceinline__ void vstep(VState<NC> &s, const int *a, const int *b, const PlaneGeom &g, unsigned char *out,
                                      unsigned off, bool emit_low, bool emit_high)
{
    int v[2 * NC], dn[2 * NC];
#pragma unroll
    for (int i = 0; i < 2 * NC; i++) { v[i] = a[i] + b[i]; dn[i] = a[i] - b[i]; }
    if (g.quant_ll) store_quant_if<NC>(out + (g.band_off[0] + off), v, g.q[0], emit_low);
    else store_raw_if<NC>(out + (g.band_off[0] + off), v, emit_low);
    store_quant_if<NC>(out + (g.band_off[1] + off), v + NC, g.q[1], emit_low);
    {
        int h[2 * NC];
#pragma unroll
        for (int i = 0; i < 2 * NC; i++) h[i] = ((v[i] - s.llp[i] + 4) >> 3) + s.dc[i];
        const unsigned offh = off - (unsigned)g.out_pitch;
        store_quant_if<NC>(out + (g.band_off[2] + offh), h, g.q[2], emit_high);
        store_quant_if<NC>(out + (g.band_off[3] + offh), h + NC, g.q[3], emit_high);
    }
#pragma unroll
    for (int i = 0; i < 2 * NC; i++) { s.llp[i] = s.llc[i]; s.llc[i] = v[i]; s.dc[i] = dn[i]; }
}

__global__ void __launch_bounds__(128) k_fwd_rgb30(const __grid_constant__ FwdParams p)
{
    const int lane = threadIdx.x;
    const int f = blockIdx.z;
    const PlaneGeom &g = p.ch[0];
    const int strip = blockIdx.x;
    if (strip * kStripIn >= g.width) return;
    const int oh = g.height >> 1;
    LaneInfo L;
    if (!lane_setup(strip, g.width, lane, L)) return;
    const unsigned colbyte = (unsigned)((strip * kStripOut + lane * 4) * 2);
    const unsigned char *in = p.in_base[f] + g.in_off + (long long)(strip * kStripIn + lane * 8) * 4;
    unsigned char *out = p.out_base[f];
    const int shift = p.shift, swap = p.byteswap, pos = p.field_pos;

    if (blockIdx.y == gridDim.y - 1) {
        if (threadIdx.y > 1) return;
        border_rows<4, 0>([&](int r, int *o, int *, int *) {
            RawRGB30Row q;
            RawPlaneRow raw;
            load_rgb30_row(in + (long long)r * g.in_pitch, L, q);
            rgb30_extract(q, swap, pos, shift, raw);
            hfilter_plane<0>(raw, L, o);
        }, oh, threadIdx.y == 1, out, g, colbyte, g, g, 0u);
        return;
    }

    const int y0 = (blockIdx.y * blockDim.y + threadIdx.y) * p.th;
    if (y0 >= oh) return;
    const int y1 = min(y0 + p.th, oh);
    const int jfirst = max(y0 - 1, 0), jlast = min(y1, oh - 1);
    const int hlo = max(y0, 1);
    VState<4> st;
#pragma unroll
    for (int i = 0; i < 8; i++) { st.llp[i] = st.llc[i] = st.dc[i] = 0; }
    const unsigned char *rp = in + (long long)(2 * jfirst) * g.in_pitch;
    RawRGB30Row c0, c1, n0, n1;
    load_rgb30_row(rp, L, c0);
    load_rgb30_row(rp + g.in_pitch, L, c1);
    n0 = c0; n1 = c1;
    unsigned off = (unsigned)(jfirst * g.out_pitch) + colbyte;
    for (int j = jfirst; j <= jlast; j++) {
        rp += 2 * g.in_pitch;
        if (j < jlast) {
            load_rgb30_row(rp, L, n0);
            load_rgb30_row(rp + g.in_pitch, L, n1);
        }
        RawPlaneRow r0, r1;
        int a[8], b[8];
        rgb30_extract(c0, swap, pos, shift, r0);
        rgb30_extract(c1, swap, pos, shift, r1);
        hfilter_plane<0>(r0, L, a);
        hfilter_plane<0>(r1, L, b);
        vstep<4>(st, a, b, g, out, off, j >= y0 && j < y1, j - 1 >= hlo);
        off += (unsigned)g.out_pitch;
        c0 = n0; c1 = n1;
    }
}

// ----------------------------------------------------------------------------
// Packed 4:2:2 sources: one warp produces the Y strip (128 columns) and the matching U and V strips (64 columns each)
// from a single read of the packed rows.  A source (Src422, SrcYU64, SrcV210) supplies
//   Row, offset(lg)            the lane's registers of one input row and the byte offset of global lane lg in a row
//   param(p), load, linear     the row load and the linear (pre-rounding) sums of the row, which hfinish_422 turns into
//                              the horizontal 2-6 outputs
//   kPlanarLH                  LH rounding of the field transform (k_fwd_422_fields)
// Channels as the reference numbers them: p.ch[0] = Y, p.ch[1] = V (Cr), p.ch[2] = U (Cb) (Codec/convert.c:4793).
struct Lin422 {
    int S[4], d[4];     // luma pair sums / differences
    int cu[4], cv[4];   // chroma samples of channel 2 (U) / channel 1 (V)
    int hy, hu, hv;     // halo sums (lane 0 / last lane of strips with a neighbour strip)
};

// horizontal 2-6 on the linear sums.  Y: oy[0..3] low, oy[4..7] high; U/V: o[0..1], o[2..3].  BORDER: the strip may
// touch the image's left or right column (decided at run time by L.has_border).
template <bool BORDER>
__device__ __forceinline__ void hfinish_422(const Lin422 &t, const LaneInfo &L, int *oy, int *ou, int *ov)
{
    const int *S = t.S, *d = t.d;
    const int Su[2] = {t.cu[0] + t.cu[1], t.cu[2] + t.cu[3]}, du[2] = {t.cu[0] - t.cu[1], t.cu[2] - t.cu[3]};
    const int Sv[2] = {t.cv[0] + t.cv[1], t.cv[2] + t.cv[3]}, dv[2] = {t.cv[0] - t.cv[1], t.cv[2] - t.cv[3]};
    int Sp = __shfl_up_sync(L.amask, S[3], 1), Sn = __shfl_down_sync(L.amask, S[0], 1);
    int Sup = __shfl_up_sync(L.amask, Su[1], 1), Sun = __shfl_down_sync(L.amask, Su[0], 1);
    int Svp = __shfl_up_sync(L.amask, Sv[1], 1), Svn = __shfl_down_sync(L.amask, Sv[0], 1);
    // lane 0 / 31 of strips with a neighbour strip (divergent but tiny; never both: 4:2:2 widths are multiples of 16)
    if (L.use_lh | L.use_rh) {
        if (L.use_lh) { Sp = t.hy; Sup = t.hu; Svp = t.hv; } else { Sn = t.hy; Sun = t.hu; Svn = t.hv; }
    }
#pragma unroll
    for (int k = 0; k < 4; k++) oy[k] = S[k];
    oy[4] = ((S[1] - Sp + 4) >> 3) + d[0];
    oy[5] = ((S[2] - S[0] + 4) >> 3) + d[1];
    oy[6] = ((S[3] - S[1] + 4) >> 3) + d[2];
    oy[7] = ((Sn - S[2] + 4) >> 3) + d[3];
    ou[0] = Su[0]; ou[1] = Su[1];
    ou[2] = ((Su[1] - Sup + 4) >> 3) + du[0];
    ou[3] = ((Sun - Su[0] + 4) >> 3) + du[1];
    ov[0] = Sv[0]; ov[1] = Sv[1];
    ov[2] = ((Sv[1] - Svp + 4) >> 3) + dv[0];
    ov[3] = ((Svn - Sv[0] + 4) >> 3) + dv[1];
    if (BORDER) {
        if (L.left_border) {
            oy[4] = clamp16((-3 * S[0] + 8 * d[0] + 4 * S[1] - S[2] + 4) >> 3);
            ou[2] = clamp16((-3 * Su[0] + 8 * du[0] + 4 * Su[1] - Sun + 4) >> 3);
            ov[2] = clamp16((-3 * Sv[0] + 8 * dv[0] + 4 * Sv[1] - Svn + 4) >> 3);
        }
        if (L.right_border) {
            oy[7] = clamp16((3 * S[3] + 8 * d[3] - 4 * S[2] + S[1] + 4) >> 3);
            ou[3] = clamp16((3 * Su[1] + 8 * du[1] - 4 * Su[0] + Sup + 4) >> 3);
            ov[3] = clamp16((3 * Sv[1] + 8 * dv[1] - 4 * Sv[0] + Svp + 4) >> 3);
        }
    }
}

// packed 8-bit 4:2:2 (YUYV / UYVY): a lane's 8 pixels are 16 bytes, 8 luma + 4 U + 4 V
struct Raw422Row {
    uint4 v;        // 8 luma + 4 U + 4 V of this lane
    uint2 halo;     // lane 0: previous 8 bytes; last lane: next 8 bytes
};

struct Sel422 {     // dp4a coefficient words (already scaled by 1 << shift)
    int ysum, ydif, u, v;
};

// dp4a coefficient words of packed 8-bit 4:2:2 (YUYV or UYVY byte order), scaled by 1 << shift
__device__ __forceinline__ Sel422 sel_422(int shift, int uyvy)
{
    Sel422 sel;
    const int m = 1 << shift;
    const int neg = (-m) & 0xff;
    if (!uyvy) { sel.ysum = m | (m << 16); sel.ydif = m | (neg << 16); sel.u = m << 8; sel.v = m << 24; }
    else { sel.ysum = (m << 8) | (m << 24); sel.ydif = (m << 8) | (neg << 24); sel.u = m; sel.v = m << 16; }
    return sel;
}

struct Src422 {
    typedef Raw422Row Row;
    typedef Sel422 Param;
    static constexpr bool kPlanarLH = false;
    static __device__ __forceinline__ Param param(const FwdParams &p) { return sel_422(p.shift, p.uyvy); }
    static __device__ __forceinline__ long long offset(int lg) { return (long long)lg * 16; }
    static __device__ __forceinline__ void load(const unsigned char *p, int, const LaneInfo &L, Row &r) {
        r.v = __ldg(reinterpret_cast<const uint4 *>(p));
        // ONE predicated halo load per row (two loads into the same register would serialise on its scoreboard)
        r.halo = make_uint2(0u, 0u);
        if (L.use_lh | L.use_rh) r.halo = __ldg(reinterpret_cast<const uint2 *>(p + (L.use_lh ? -8 : 16)));
    }
    static __device__ __forceinline__ void linear(const Row &r, const Sel422 &sel, const LaneInfo &L, Lin422 &o) {
        const unsigned w[4] = {r.v.x, r.v.y, r.v.z, r.v.w};
#pragma unroll
        for (int k = 0; k < 4; k++) {
            o.S[k] = dp4a_us(w[k], sel.ysum, 0);
            o.d[k] = dp4a_us(w[k], sel.ydif, 0);
            o.cu[k] = dp4a_us(w[k], sel.u, 0);
            o.cv[k] = dp4a_us(w[k], sel.v, 0);
        }
        // left halo: luma pair of the later word (.y), chroma pair = both words; right halo: luma pair of word .x
        o.hy = o.hu = o.hv = 0;
        if (L.use_lh | L.use_rh) {
            o.hy = dp4a_us(L.use_lh ? r.halo.y : r.halo.x, sel.ysum, 0);
            o.hu = dp4a_us(r.halo.y, sel.u, dp4a_us(r.halo.x, sel.u, 0));
            o.hv = dp4a_us(r.halo.y, sel.v, dp4a_us(r.halo.x, sel.v, 0));
        }
    }
};

// ----------------------------------------------------------------------------
// 16-bit packed 4:2:2 sources (YU64: Y0 C1 Y1 C3, 16 bits each).  The reference converts them to 10-bit planes on the
// host first (Codec/frame.c:1556 ConvertYU64ToFrame16s: `(word >> 6) & 0x03ff03ff`, convert.c:3345, then
// convert.c:14370 de-interleave: position 1 -> channel 1, position 3 -> channel 2) and runs the planar level-1 filter on
// each plane (Codec/encoder.c:3180-3193 TransformForwardSpatial -> spatial.c:10026 FilterSpatialQuant16s).  Here the
// conversion is fused into the load of a one-pass register-fed kernel (k_fwd_422_src) that produces the three channels
// of a strip in one warp.
struct RawYU64Row {
    uint4 a, b;         // 8 luma + 4 + 4 chroma samples of this lane (32 bytes)
    uint4 halo;         // lane 0: previous 16 bytes; last lane: next 16 bytes
};

struct SrcYU64 {
    typedef RawYU64Row Row;
    typedef int Param;                  // 16 - precision
    static constexpr bool kPlanarLH = true;
    static __device__ __forceinline__ Param param(const FwdParams &p) { return p.shift; }
    // byte offset of global lane lg (8 luma pixels = 4 groups of Y0 C1 Y1 C3, 8 bytes each) inside a row
    static __device__ __forceinline__ long long offset(int lg) { return (long long)lg * 32; }
    static __device__ __forceinline__ void load(const unsigned char *p, int, const LaneInfo &L, Row &r) {
        r.a = __ldg(reinterpret_cast<const uint4 *>(p));
        r.b = __ldg(reinterpret_cast<const uint4 *>(p + 16));
        r.halo = make_uint4(0u, 0u, 0u, 0u);
        if (L.use_lh | L.use_rh) r.halo = __ldg(reinterpret_cast<const uint4 *>(p + (L.use_lh ? -16 : 32)));
    }
    // cv = the position-1 chroma sample (channel 1), cu = the position-3 sample (channel 2) of every 4-sample group
    static __device__ __forceinline__ void linear(const Row &r, int shift, const LaneInfo &L, Lin422 &o) {
        const unsigned M = (0xffffu >> shift) * 0x00010001u;
        const unsigned w[8] = {r.a.x, r.a.y, r.a.z, r.a.w, r.b.x, r.b.y, r.b.z, r.b.w};
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const unsigned t0 = (w[2 * k] >> shift) & M, t1 = (w[2 * k + 1] >> shift) & M;
            const int y0 = (int)(t0 & 0xffffu), y1 = (int)(t1 & 0xffffu);
            o.S[k] = y0 + y1; o.d[k] = y0 - y1;
            o.cv[k] = (int)(t0 >> 16); o.cu[k] = (int)(t1 >> 16);
        }
        const unsigned h0 = (r.halo.x >> shift) & M, h1 = (r.halo.y >> shift) & M, h2 = (r.halo.z >> shift) & M, h3 = (r.halo.w >> shift) & M;
        o.hy = L.use_lh ? (int)((h2 & 0xffffu) + (h3 & 0xffffu)) : (int)((h0 & 0xffffu) + (h1 & 0xffffu));
        o.hv = (int)((h0 >> 16) + (h2 >> 16));
        o.hu = (int)((h1 >> 16) + (h3 >> 16));
    }
};

// 10-bit packed 4:2:2 (V210): the row is a stream of 10-bit components Cb Y Cr Y Cb Y ... packed three per 32-bit
// word at bits 0, 10, 20 (Codec/convert.c:3365 ConvertYUVRowToV210 shows the layout; rows are padded to 128 bytes).  The
// reference unpacks it on the host into 10-bit planes (Codec/encoder.c:2518-2534 ConvertV210ToFrame16s: first chroma ->
// channel 2, second chroma -> channel 1, values unshifted) and runs the planar filter per plane (encoder.c:3180-3193).
// A lane's 8 pixels are 16 consecutive components starting at component 16 * lg, i.e. at word (16 * lg) / 3 with a
// phase of lg % 3 components into that word: six words always cover them.
struct RawV210Row {
    unsigned w[6];      // words (16 * lg) / 3 ... + 5
    unsigned hw[4];     // halo: the words holding the 8 components before (lane 0) / after (last lane) this lane's
    int phase;          // (16 * lg) % 3
};

// 60 useful bits of two consecutive words
__device__ __forceinline__ unsigned long long v210_pair(unsigned a, unsigned b) {
    return (unsigned long long)(a & 0x3fffffffu) | ((unsigned long long)(b & 0x3fffffffu) << 30);
}
// drop `sh` (0, 10 or 20) bits from the front of the 60-bit pair lo, refilling from the next pair hi
__device__ __forceinline__ unsigned long long v210_shift(unsigned long long lo, unsigned long long hi, int sh) {
    const unsigned long long m60 = (1ull << 60) - 1;
    return sh ? (((lo >> sh) | (hi << (60 - sh))) & m60) : lo;
}
__device__ __forceinline__ int v210_field(unsigned long long x, int i) { return (int)((x >> (10 * i)) & 0x3ffu); }

struct SrcV210 {
    typedef RawV210Row Row;
    typedef int Param;                  // unused: the components are 10-bit as stored
    static constexpr bool kPlanarLH = true;
    static __device__ __forceinline__ Param param(const FwdParams &) { return 0; }
    static __device__ __forceinline__ long long offset(int lg) { return (long long)((16 * lg) / 3) * 4; }
    static __device__ __forceinline__ void load(const unsigned char *p, int lg, const LaneInfo &L, Row &r) {
        const unsigned *wp = reinterpret_cast<const unsigned *>(p);
#pragma unroll
        for (int i = 0; i < 6; i++) r.w[i] = __ldg(wp + i);
        r.phase = (16 * lg) % 3;
#pragma unroll
        for (int i = 0; i < 4; i++) r.hw[i] = 0u;
        if (L.use_lh | L.use_rh) {
            // the 8 components before this lane start at component 16 lg - 8, the 8 after it at 16 lg + 16
            const int c0 = 16 * lg + (L.use_lh ? -8 : 16);
            const unsigned *hp = wp + (c0 / 3 - (16 * lg) / 3);
#pragma unroll
            for (int i = 0; i < 4; i++) r.hw[i] = __ldg(hp + i);
        }
    }
    // cv = the chroma that goes to channel 1 (the SECOND chroma component, Cr), cu = the one for channel 2 (Cb)
    static __device__ __forceinline__ void linear(const Row &r, int, const LaneInfo &L, Lin422 &o) {
        const int sh = 10 * r.phase;
        const unsigned long long A = v210_pair(r.w[0], r.w[1]), B = v210_pair(r.w[2], r.w[3]), C = v210_pair(r.w[4], r.w[5]);
        const unsigned long long a = v210_shift(A, B, sh), b = v210_shift(B, C, sh), c = v210_shift(C, 0ull, sh);
        int comp[16];
#pragma unroll
        for (int i = 0; i < 6; i++) { comp[i] = v210_field(a, i); comp[6 + i] = v210_field(b, i); }
#pragma unroll
        for (int i = 0; i < 4; i++) comp[12 + i] = v210_field(c, i);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int y0 = comp[4 * k + 1], y1 = comp[4 * k + 3];
            o.S[k] = y0 + y1; o.d[k] = y0 - y1;
            o.cu[k] = comp[4 * k]; o.cv[k] = comp[4 * k + 2];
        }
        // halo: 8 components starting at phase (phase + 1) % 3 of hw[0] (16 lg - 8 and 16 lg + 16 are both = 16 lg + 1 mod 3)
        const int hsh = 10 * ((r.phase + 1) % 3);
        const unsigned long long HA = v210_pair(r.hw[0], r.hw[1]), HB = v210_pair(r.hw[2], r.hw[3]);
        const unsigned long long ha = v210_shift(HA, HB, hsh), hb = v210_shift(HB, 0ull, hsh);
        int hc[8];
#pragma unroll
        for (int i = 0; i < 6; i++) hc[i] = v210_field(ha, i);
        hc[6] = v210_field(hb, 0); hc[7] = v210_field(hb, 1);
        // components: Cb Y Cr Y | Cb Y Cr Y ; the luma pair adjacent to this lane is the second group on the left
        // side and the first group on the right side
        o.hy = L.use_lh ? (hc[5] + hc[7]) : (hc[1] + hc[3]);
        o.hu = hc[0] + hc[4];
        o.hv = hc[2] + hc[6];
    }
};

__device__ __forceinline__ unsigned colbyte_luma(int strip, int lane) { return (unsigned)((strip * kStripOut + lane * 4) * 2); }
__device__ __forceinline__ unsigned colbyte_chroma(int strip, int lane) { return (unsigned)((strip * (kStripOut / 2) + lane * 2) * 2); }

// First (bottom = false) or last HL/HH row of the three channels of a packed 4:2:2 source, from six input rows read
// straight from global memory
template <class SRC>
__device__ __forceinline__ void border_422(const FwdParams &p, int f, int strip, int lane, const LaneInfo &L, bool bottom)
{
    const PlaneGeom &gy = p.ch[0];
    const int lg = strip * 32 + lane;           // global lane index: 8 luma pixels each
    const unsigned char *in = p.in_base[f] + gy.in_off + SRC::offset(lg);
    const typename SRC::Param sp = SRC::param(p);
    border_rows<4, 2>([&](int r, int *y, int *u, int *v) {
        typename SRC::Row raw;
        Lin422 t;
        SRC::load(in + (long long)r * gy.in_pitch, lg, L, raw);
        SRC::linear(raw, sp, L, t);
        hfinish_422<true>(t, L, y, u, v);
    }, gy.height >> 1, bottom, p.out_base[f], gy, colbyte_luma(strip, lane), p.ch[2], p.ch[1], colbyte_chroma(strip, lane));
}

// One-pass register-fed level 1 of a packed 4:2:2 source (YU64 and V210; packed 8-bit runs the TMA-fed k_fwd_422_tma)
template <class SRC>
__global__ void __launch_bounds__(128) k_fwd_422_src(const __grid_constant__ FwdParams p)
{
    const int lane = threadIdx.x;
    const int f = blockIdx.z;
    const PlaneGeom &gy = p.ch[0];
    const PlaneGeom &gv = p.ch[1];
    const PlaneGeom &gu = p.ch[2];
    const int strip = blockIdx.x;
    if (strip * kStripIn >= gy.width) return;
    const int oh = gy.height >> 1;
    LaneInfo L;
    if (!lane_setup(strip, gy.width, lane, L)) return;

    if (blockIdx.y == gridDim.y - 1) {      // border warps: first / last HL,HH row of all three channels
        if (threadIdx.y > 1) return;
        border_422<SRC>(p, f, strip, lane, L, threadIdx.y == 1);
        return;
    }

    const unsigned colbyte_y = colbyte_luma(strip, lane), colbyte_c = colbyte_chroma(strip, lane);
    const int lg = strip * 32 + lane;
    const unsigned char *in = p.in_base[f] + gy.in_off + SRC::offset(lg);
    unsigned char *out = p.out_base[f];
    const typename SRC::Param sp = SRC::param(p);
    const int y0 = (blockIdx.y * blockDim.y + threadIdx.y) * p.th;
    if (y0 >= oh) return;
    const int y1 = min(y0 + p.th, oh);
    const int jfirst = max(y0 - 1, 0), jlast = min(y1, oh - 1);
    const int hlo = max(y0, 1);
    RotState<4> sy;
    RotState<2> su, sv;
#pragma unroll
    for (int i = 0; i < 8; i++) { sy.t[i] = sy.s[i] = 0; }
#pragma unroll
    for (int i = 0; i < 4; i++) { su.t[i] = su.s[i] = 0; sv.t[i] = sv.s[i] = 0; }
    const unsigned char *rp = in + (long long)(2 * jfirst) * gy.in_pitch;
    typename SRC::Row c0, c1, n0, n1;
    SRC::load(rp, lg, L, c0);
    SRC::load(rp + gy.in_pitch, lg, L, c1);
    n0 = c0; n1 = c1;
    unsigned offy = (unsigned)(jfirst * gy.out_pitch) + colbyte_y;
    unsigned offc = (unsigned)(jfirst * gu.out_pitch) + colbyte_c;
    for (int j = jfirst; j <= jlast; j++) {
        rp += 2 * gy.in_pitch;
        if (j < jlast) {
            SRC::load(rp, lg, L, n0);
            SRC::load(rp + gy.in_pitch, lg, L, n1);
        }
        Lin422 t;
        int ay[8], by[8], au[4], bu[4], av[4], bv[4];
        SRC::linear(c0, sp, L, t); hfinish_422<true>(t, L, ay, au, av);
        SRC::linear(c1, sp, L, t); hfinish_422<true>(t, L, by, bu, bv);
        const bool emit_low = (j >= y0) && (j < y1), emit_high = (j - 1 >= hlo);
        vstep_rot<4, kLLQuantIf>(sy, ay, by, gy, out, offy, emit_low, emit_high);
        vstep_rot<2, kLLQuantIf>(sv, av, bv, gv, out, offc, emit_low, emit_high);
        vstep_rot<2, kLLQuantIf>(su, au, bu, gu, out, offc, emit_low, emit_high);
        offy += (unsigned)gy.out_pitch;
        offc += (unsigned)gu.out_pitch;
        c0 = n0; c1 = n1;
    }
}

// ----------------------------------------------------------------------------
// Interlaced sources: level 1 is the frame (field) transform, Codec/wavelet.c:6076 TransformForwardFrameYUV
// (Codec/filter.c:273 FilterFrameQuant16s is the planar form of the same transform):
//   t_low = even + odd, t_high = odd - even (Codec/temporal.c:1568), then the horizontal 2-6 filter on both;
//   LL = low(t_low), LH = Q(high(t_low)), HH = Q(high(t_high)) and HL = Q'(low(t_high)) difference coded along the
//   row (Codec/spatial.c:5327: Q' uses the midpoint divisor/g without the "-1", out[i] = q[i] - q[i-1]).
// The temporal step is linear in the samples, so it is applied to the linear sums of the two rows before the
// (non-linear) rounding of the highpass filter.  No vertical neighbourhood: no border warps, no carried state.
// The 16-bit / 10-bit sources (kPlanarLH) follow the planar routine: the reference converts them to planes and runs
//   Codec/filter.c:273 FilterFrameQuant16s: temporal.c FilterTemporalRow16s (even + odd, odd - even), then
//   spatial.c:5826 FilterHorizontalRowQuant16s on the temporal lowpass -- LL (quantised only when its divisor > 1) and LH,
//   both with the midpoint divisor / 2 (filter.c:352 / spatial.c:5856; the packed 8-bit path rounds LH with
//   divisor / 2 - 1) in the columns its 16-sample SSE2 loop produces and WITHOUT a midpoint in the columns of its scalar
//   tail and in the last column, which it redoes with the border filter (spatial.c:6192-6266) -- and spatial.c:5327
//   ...DifferenceFiltered + QuantizeRow16sTo16s on the temporal highpass, as the packed path.  (LL is quantised by the
//   same routine when its divisor exceeds 1, which no schedule of the reference produces at level 1: the host side
//   rejects such a table.)

// a + sgn * b on every member
__device__ __forceinline__ void lin_combine(const Lin422 &a, const Lin422 &b, int sgn, Lin422 &o)
{
#pragma unroll
    for (int k = 0; k < 4; k++) {
        o.S[k] = b.S[k] + sgn * a.S[k]; o.d[k] = b.d[k] + sgn * a.d[k];
        o.cu[k] = b.cu[k] + sgn * a.cu[k]; o.cv[k] = b.cv[k] + sgn * a.cv[k];
    }
    o.hy = b.hy + sgn * a.hy; o.hu = b.hu + sgn * a.hu; o.hv = b.hv + sgn * a.hv;
}

// quantise NC lowpass values of t_high and difference-code them along the row; prev_raw = the lowpass value of the
// column left of the strip (halo), used by lane 0 of strips > 0
template <int NC>
__device__ __forceinline__ void store_diffq(unsigned char *p, const int *v, int prev_raw, const QuantParam &q, const LaneInfo &L)
{
    int Q[NC];
#pragma unroll
    for (int i = 0; i < NC; i++) Q[i] = quant1(v[i], q) >> 16;
    int prev = __shfl_up_sync(L.amask, Q[NC - 1], 1);
    if (L.use_lh) prev = quant1(prev_raw, q) >> 16;
    if (L.left_border) prev = 0;
    int o[NC];
#pragma unroll
    for (int i = 0; i < NC; i++) { o[i] = Q[i] - prev; prev = Q[i]; }
    store_raw<NC>(p, o);
}

// LH of the field transform: the ordinary quantiser for packed 8-bit sources; for the planar routine of the 16-bit /
// 10-bit sources the midpoint divisor / 2 or none, per column
template <class SRC, int NC>
__device__ __forceinline__ void store_quant_lh(unsigned char *ptr, const int *v, const QuantParam &q, int col0, int width_out)
{
    if (!SRC::kPlanarLH) { store_quant<NC>(ptr, v, q); return; }
    // columns >= tail belong to the scalar tail of a (2 * width_out)-sample row; the last column is the border column
    const int tail = (2 * width_out - (2 * width_out) % 16) / 2;
    int o[NC];
#pragma unroll
    for (int i = 0; i < NC; i++) {
        const int col = col0 + i;
        const bool nomid = (col >= tail) || (col == width_out - 1);
        o[i] = (v[i] * q.m + (v[i] < 0 ? (nomid ? 65535 : q.cneg) : (nomid ? 0 : q.cpos))) >> 16;
    }
    store_raw<NC>(ptr, o);
}

template <class SRC>
__global__ void __launch_bounds__(128) k_fwd_422_fields(const __grid_constant__ FwdParams p)
{
    const int lane = threadIdx.x;
    const int f = blockIdx.z;
    const PlaneGeom &gy = p.ch[0];
    const PlaneGeom &gv = p.ch[1];
    const PlaneGeom &gu = p.ch[2];
    const int strip = blockIdx.x;
    if (strip * kStripIn >= gy.width) return;
    const int oh = gy.height >> 1;
    LaneInfo L;
    if (!lane_setup(strip, gy.width, lane, L)) return;
    const unsigned colbyte_y = colbyte_luma(strip, lane), colbyte_c = colbyte_chroma(strip, lane);
    const int col_y = strip * kStripOut + lane * 4, col_c = strip * (kStripOut / 2) + lane * 2;
    const int lg = strip * 32 + lane;
    const unsigned char *in = p.in_base[f] + gy.in_off + SRC::offset(lg);
    unsigned char *out = p.out_base[f];
    const typename SRC::Param sp = SRC::param(p);
    const int y0 = (blockIdx.y * blockDim.y + threadIdx.y) * p.th;
    if (y0 >= oh) return;
    const int y1 = min(y0 + p.th, oh);
    const unsigned char *rp = in + (long long)(2 * y0) * gy.in_pitch;
    typename SRC::Row c0, c1, n0, n1;
    SRC::load(rp, lg, L, c0);
    SRC::load(rp + gy.in_pitch, lg, L, c1);
    n0 = c0; n1 = c1;
    unsigned offy = (unsigned)(y0 * gy.out_pitch) + colbyte_y;
    unsigned offc = (unsigned)(y0 * gu.out_pitch) + colbyte_c;
    for (int j = y0; j < y1; j++) {
        rp += 2 * gy.in_pitch;
        if (j + 1 < y1) {
            SRC::load(rp, lg, L, n0);
            SRC::load(rp + gy.in_pitch, lg, L, n1);
        }
        if (j + 3 < y1) { prefetch_l2(rp + 4 * gy.in_pitch); prefetch_l2(rp + 5 * gy.in_pitch); }
        Lin422 e, o, t;
        SRC::linear(c0, sp, L, e);
        SRC::linear(c1, sp, L, o);
        int ay[8], au[4], av[4];
        lin_combine(e, o, +1, t);               // temporal lowpass: even + odd
        hfinish_422<true>(t, L, ay, au, av);
        store_raw<4>(out + (gy.band_off[0] + offy), ay);
        store_quant_lh<SRC, 4>(out + (gy.band_off[1] + offy), ay + 4, gy.q[1], col_y, gy.width >> 1);
        store_raw<2>(out + (gu.band_off[0] + offc), au);
        store_quant_lh<SRC, 2>(out + (gu.band_off[1] + offc), au + 2, gu.q[1], col_c, gu.width >> 1);
        store_raw<2>(out + (gv.band_off[0] + offc), av);
        store_quant_lh<SRC, 2>(out + (gv.band_off[1] + offc), av + 2, gv.q[1], col_c, gv.width >> 1);
        lin_combine(e, o, -1, t);               // temporal highpass: odd - even
        hfinish_422<true>(t, L, ay, au, av);
        store_diffq<4>(out + (gy.band_off[2] + offy), ay, t.hy, gy.q[2], L);
        store_quant<4>(out + (gy.band_off[3] + offy), ay + 4, gy.q[3]);
        store_diffq<2>(out + (gu.band_off[2] + offc), au, t.hu, gu.q[2], L);
        store_quant<2>(out + (gu.band_off[3] + offc), au + 2, gu.q[3]);
        store_diffq<2>(out + (gv.band_off[2] + offc), av, t.hv, gv.q[2], L);
        store_quant<2>(out + (gv.band_off[3] + offc), av + 2, gv.q[3]);
        offy += (unsigned)gy.out_pitch;
        offc += (unsigned)gu.out_pitch;
        c0 = n0; c1 = n1;
    }
}

#include "cfb_forward_tma.inl"
#include "cfb_forward_l12.inl"


// ----------------------------------------------------------------------------
// host-side launchers (called from cfb_api.cu)
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// (strips, row blocks of `warps` warps of th rows each [+ 1 border CTA row], frames)
static dim3 fwd_grid(int width, int rows, int th, int warps, bool border_row, int frames)
{
    return dim3(ceil_div(width, kStripIn), ceil_div(ceil_div(rows, th), warps) + (border_row ? 1 : 0), frames);
}

// Single planes (levels 2 and 3 of every format, PLANAR16 level 1, cfb_level_*) run the register-fed k_fwd_plane: a ring
// in shared memory does not pay off over the 8-16 row pairs a warp streams.  On an H100 SXM (400 W power limit, two
// alternating rounds) levels 2 and 3 of 16 4K 4:2:2 frames took 110 / 32 us with it, against 126 / 39 us through a
// TMA-fed ring of one warp per plane.
cudaError_t launch_fwd_plane(cfb_context *ctx, FwdParams &p, int prescale, bool nonneg)
{
    int maxw = 0, maxoh = 0;
    bool ragged = false;
    for (int c = 0; c < p.nchan; c++) {
        maxw = max(maxw, p.ch[c].width); maxoh = max(maxoh, p.ch[c].height / 2);
        ragged = ragged || (p.ch[c].width & 7);
    }
    p.th = pick_th(ceil_div(maxw, kStripIn), maxoh, p.nframes * p.nchan, ctx->sm_count);
    if (ragged) {       // the 1-3 output columns right of the last full lane (they include the right border)
        const dim3 eblock(128), egrid(ceil_div(maxoh, 128), 3, p.nframes * p.nchan);
        const cudaError_t e = launch_kernel(ctx, prescale ? k_fwd_plane_edge<2> : k_fwd_plane_edge<0>, egrid, eblock, 0, p);
        if (e != cudaSuccess) return e;
    }
    dim3 block(32, 4);
    dim3 grid = fwd_grid(maxw, maxoh, p.th, block.y, true, p.nframes * p.nchan);
    // nonneg: the caller vouches that the planes are non-negative (LL bands of an unsigned source)
    return launch_kernel(ctx, (prescale && nonneg) ? k_fwd_plane<3> : prescale ? k_fwd_plane<2> : k_fwd_plane<0>, grid, block, 0, p);
}

// k_fwd_tma<SRC> over the rows of every channel (one warp per channel and strip), then k_fwd_tma_border<SRC> for the
// first and last HL/HH row of each
template <class SRC, int MINB>
static cudaError_t launch_fwd_tma(cfb_context *ctx, FwdParams &p, uint64_t row_bytes, uint64_t rows, int elem_bytes)
{
    const PlaneGeom &g = p.ch[0];
    FwdTmaMaps tm;
    for (int i = 0; i < p.nframes; i++) {
        cudaError_t e = tmap_encode_2d(&tm.in_map[i], p.in_base[i] + g.in_off, row_bytes, rows, (uint64_t)g.in_pitch,
                                       SRC::kRowBytes, elem_bytes, 8);
        if (e != cudaSuccess) return e;
    }
    p.th = pick_th(ceil_div(g.width, kStripIn), g.height / 2, p.nframes * p.nchan, ctx->sm_count);
    const dim3 tgrid = fwd_grid(g.width, g.height / 2, p.th, 1, false, p.nframes);
    const cudaError_t e = launch_kernel(ctx, k_fwd_tma<SRC, MINB>, tgrid, dim3(32, SRC::kWarps),
                                        kTmaStages * SRC::kStageBytes + 2 * kTmaStages * 8, p, tm);
    if (e != cudaSuccess) return e;
    return launch_kernel(ctx, k_fwd_tma_border<SRC>, dim3(tgrid.x * SRC::kWarps, 1, p.nframes), dim3(32, 2), 0, p);
}

// All three channels of packed RG48 frames, p.ch[0..2] = G, R, B, from ONE read of the pixel groups, plus the border rows
// of each channel.  On an H100 SXM (400 W power limit, two alternating rounds) 8 4K frames took 336 us, against 615 us
// with one register-fed launch per channel.
cudaError_t launch_fwd_rg48(cfb_context *ctx, FwdParams &p)
{
    return launch_fwd_tma<SrcRG48, 5>(ctx, p, (uint64_t)p.ch[0].width * 6, (uint64_t)p.ch[0].height, 2);
}

// Every channel of packed 16-bit RGBA frames (B64A: rg64 = false, RG64: true), p.ch[0..p.nchan) = G, R, B (+ A), plus the
// border rows of each channel.  On an H100 SXM (400 W power limit, 16 4K frames per launch, two alternating rounds) level 1
// took 1022 - 1055 us with alpha (16 bytes per pixel: 2012 - 2077 GB/s) and 781 - 805 us without (14 bytes: 2308 - 2378 GB/s),
// against 628 - 637 us for RG48 (12 bytes: 2499 - 2538 GB/s); 76 registers, no spills (border kernel 60 / 64).  Of the ~18 %
// per byte that RGBA loses to RG48, the alpha curve is about 8 points: the same kernel with `>> 4` in its place took 952 - 953
// us (2227 - 2231 GB/s) in the same call -- the alpha warp unpacks, multiplies and selects per sample, and every warp of the
// CTA waits for the slowest before its stage is refilled.  The rest is common to the 64-bit sources: every channel warp reads
// all 64 bytes of its lane from the stage (4 LDS.128 per row, three of four words dropped) and each stage row takes two TMA
// boxes.
cudaError_t launch_fwd_rgba64(cfb_context *ctx, FwdParams &p, bool rg64)
{
    const uint64_t row_bytes = (uint64_t)p.ch[0].width * 8, rows = (uint64_t)p.ch[0].height;
    if (p.nchan == 4) {
        if (rg64) return launch_fwd_tma<SrcRGBA64<1, 4>, 4>(ctx, p, row_bytes, rows, 2);
        return launch_fwd_tma<SrcRGBA64<0, 4>, 4>(ctx, p, row_bytes, rows, 2);
    }
    if (rg64) return launch_fwd_tma<SrcRGBA64<1, 3>, 5>(ctx, p, row_bytes, rows, 2);
    return launch_fwd_tma<SrcRGBA64<0, 3>, 5>(ctx, p, row_bytes, rows, 2);
}

// One channel (p.ch[0], p.nchan = 1) of 10-bit RGB frames: one launch per channel
cudaError_t launch_fwd_rgb30(cfb_context *ctx, FwdParams &p)
{
    dim3 block(32, 4);
    p.th = pick_th(ceil_div(p.ch[0].width, kStripIn), p.ch[0].height / 2, p.nframes, ctx->sm_count);
    return launch_kernel(ctx, k_fwd_rgb30, fwd_grid(p.ch[0].width, p.ch[0].height / 2, p.th, block.y, true, p.nframes), block, 0, p);
}

// All four Bayer-derived channels, plus their border rows, in the Bayer phase p.bayer_phase.  One read of the Bayer lines
// feeds the four channel warps of a CTA (plane width = half the Bayer width).  On an H100 SXM (400 W power limit, two
// alternating rounds) 4 8K frames took 250 us, against 392 us with one register-fed warp per channel.
cudaError_t launch_fwd_byr4(cfb_context *ctx, FwdParams &p)
{
    const uint64_t row_bytes = (uint64_t)p.ch[0].width * 4, rows = (uint64_t)p.ch[0].height * 2;
    if (p.lut) return launch_fwd_tma<SrcBYR4<true>, 3>(ctx, p, row_bytes, rows, 4);
    return launch_fwd_tma<SrcBYR4<false>, 3>(ctx, p, row_bytes, rows, 4);
}

// The same four channels from 12-bit packed Bayer frames (one packed row of 6 * pw bytes per plane row).  Every TMA box
// start is checked here, on the host: a box that starts off a 16-byte boundary faults on the device.
cudaError_t launch_fwd_byr5(cfb_context *ctx, FwdParams &p)
{
    const PlaneGeom &g = p.ch[0];
    const int pw = g.width;
    if (g.in_pitch % 16) return cudaErrorMisalignedAddress;
    for (int i = 0; i < p.nframes; i++)
        if ((uintptr_t)(p.in_base[i] + g.in_off) % 16) return cudaErrorMisalignedAddress;
    for (int strip = 0; strip * kStripIn < pw; strip++)
        for (int s = 0; s < 8; s++)
            if (byr5_seg(s, pw, strip).box % 16) return cudaErrorMisalignedAddress;
    return launch_fwd_tma<SrcBYR5, 3>(ctx, p, (uint64_t)pw * 6, (uint64_t)g.height, SrcBYR5::kBoxRows);
}

// One tensor map per frame of a packed 4:2:2 batch: rows of 2 * width bytes, `height` rows, the caller's pitch
static cudaError_t encode_422_maps(const FwdParams &p, FwdTmaMaps &tm)
{
    const PlaneGeom &g = p.ch[0];
    for (int i = 0; i < p.nframes; i++) {
        cudaError_t e = tmap_encode_2d(&tm.in_map[i], p.in_base[i] + g.in_off, (uint64_t)g.width * 2, (uint64_t)g.height,
                                       (uint64_t)g.in_pitch, kTmaRowBytes, 2);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// On an H100 SXM (700 W power limit, 16 4K frames per launch) k_fwd_422_tma took 315 us; a register-fed kernel of the same
// arithmetic took 312 us, within the run-to-run spread.
cudaError_t launch_fwd_422(cfb_context *ctx, FwdParams &p)
{
    dim3 block(32, 4);
    p.th = pick_th(ceil_div(p.ch[0].width, kStripIn), p.ch[0].height / 2, p.nframes, ctx->sm_count);
    dim3 grid = fwd_grid(p.ch[0].width, p.ch[0].height / 2, p.th, block.y, true, p.nframes);
    FwdTmaMaps tm;
    cudaError_t e = encode_422_maps(p, tm);
    if (e != cudaSuccess) return e;
    return launch_kernel(ctx, k_fwd_422_tma, grid, block, 4 * kTmaWarpBytes + 4 * kTmaStages * 8, p, tm);
}

// Levels 1 and 2 in one pass (cfb_forward_l12.inl), plus the border rows of both levels in a second launch:
// p.th = level-2 rows per warp.  The caller guarantees a width that is a
// multiple of 32 (every level-2 lane whole) and a level-2 band of exactly half the level-1 height.  On an H100 SXM (700 W
// power limit, 16 4K frames per launch, th = 4) the two launches took 333 - 335 us, against 316 + 113 us for k_fwd_422_tma +
// k_fwd_plane<3>; the main kernel has 168 registers, no spills, 3 CTAs (12 warps) per SM.  (With the border rows in an
// extra CTA row of the main kernel instead, the pass took 325 us.)
cudaError_t launch_fwd_422_l12(cfb_context *ctx, FwdParams &p, const PlaneGeom *l2)
{
    FwdL2Geom q;
    for (int c = 0; c < 3; c++) q.ch[c] = l2[c];
    dim3 block(32, 4);
    // At most 4 level-2 rows per warp.  On an H100 SXM (700 W power limit, 16 4K frames, two rounds, border rows then still
    // inside the kernel) the pass took 325 - 326 / 326 - 384 / 332 / 337 / 344 / 357 - 358 / 367 - 368 us at th = 4 / 6 / 8 /
    // 12 / 16 / 24 / 32, although a warp streams 4 row pairs beyond its own 2 th.
    p.th = pick_th(ceil_div(p.ch[0].width, kStripIn), q.ch[0].height / 2, p.nframes, ctx->sm_count, 4);
    dim3 grid = fwd_grid(p.ch[0].width, q.ch[0].height / 2, p.th, block.y, false, p.nframes);
    FwdTmaMaps tm;
    cudaError_t e = encode_422_maps(p, tm);
    if (e != cudaSuccess) return e;
    e = launch_kernel(ctx, k_fwd_422_l12_tma, grid, block, 4 * kTmaWarpBytes + 4 * kTmaStages * 8, p, tm, q);
    if (e != cudaSuccess) return e;
    // first / last HL,HH row of both levels
    return launch_kernel(ctx, k_fwd_422_l12_border, dim3(grid.x, 1, p.nframes), block, 0, p, q);
}

// YU64 / V210 sources, progressive
cudaError_t launch_fwd_422_src(cfb_context *ctx, FwdParams &p, FwdSrc src)
{
    dim3 block(32, 4);
    p.th = pick_th(ceil_div(p.ch[0].width, kStripIn), p.ch[0].height / 2, p.nframes, ctx->sm_count);
    dim3 grid = fwd_grid(p.ch[0].width, p.ch[0].height / 2, p.th, block.y, true, p.nframes);
    return launch_kernel(ctx, src == kFwdV210 ? k_fwd_422_src<SrcV210> : k_fwd_422_src<SrcYU64>, grid, block, 0, p);
}

// Interlaced level 1 of every packed 4:2:2 source
cudaError_t launch_fwd_422_fields(cfb_context *ctx, FwdParams &p, FwdSrc src)
{
    dim3 block(32, 4);
    p.th = pick_th(ceil_div(p.ch[0].width, kStripIn), p.ch[0].height / 2, p.nframes, ctx->sm_count);
    dim3 grid = fwd_grid(p.ch[0].width, p.ch[0].height / 2, p.th, block.y, false, p.nframes);
    return launch_kernel(ctx, src == kFwdV210 ? k_fwd_422_fields<SrcV210> : src == kFwdYU64 ? k_fwd_422_fields<SrcYU64>
                                                                                            : k_fwd_422_fields<Src422>,
                         grid, block, 0, p);
}

}  // namespace cfb
