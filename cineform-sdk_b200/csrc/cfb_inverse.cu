// cfb_inverse.cu -- inverse 2-6 wavelet level with fused dequantisation, sm_90a.
//
// Replaces (reference):
//   Codec/spatial.c:21877 InvertSpatialQuant16s + Codec/InvertHorizontalStrip16s.c:459   -> k_inv_plane<0>
//   Codec/spatial.c:22414 InvertSpatialQuantDescale16s + InvertHorizontalStrip16s.c:1700 -> k_inv_plane<2>
//   Codec/spatial.c:31341/:31511/:31975 InvertSpatial{Top,Middle,Bottom}Row16sToOutput +
//   Codec/InvertHorizontalStrip16s.c:3770/:5025 InvertHorizontalStrip16sToYUYV/ToUYVY   -> k_inv_422_tma
//   Codec/decoder.c:20551 DeQuantFSM (coefficient * quant)                               -> fused into the loads
//
// Same structure as the forward kernels: one warp per strip.  The final 4:2:2 level stages its band rows in shared
// memory through a TMA ring (cfb_inverse_tma.inl); the other kernels load them straight into registers.
// A lane owns 4 band columns; per band row it loads 8 bytes from each of the four bands, keeps a
// three-row window of the two vertically-lowpass bands (LL, LH) in registers, produces the even/odd
// intermediate rows, exchanges one value with each neighbour lane by shuffle for the horizontal
// stage and writes 8 output samples per row with one 128-bit store.  Lanes 0 and 31 of a warp are
// halo lanes (their columns belong to the neighbouring strips), so a strip covers 120 band columns.
#include "cfb_host.h"
#include "cfb_tma.cuh"

#include <type_traits>

namespace cfb {

constexpr unsigned kFullMask = 0xffffffffu;

// raw (still packed, still quantised) coefficients of NC columns of one band row
template <int NC> struct RawCols;
template <> struct RawCols<4> { uint2 w; };
template <> struct RawCols<2> { unsigned w; };

template <int NC>
__device__ __forceinline__ void load_raw(const unsigned char *in, long long band_off, unsigned off, bool active, RawCols<NC> &r);
template <>
__device__ __forceinline__ void load_raw<4>(const unsigned char *in, long long band_off, unsigned off, bool active, RawCols<4> &r) {
    r.w = active ? __ldg(reinterpret_cast<const uint2 *>(in + band_off + off)) : make_uint2(0, 0);
}
template <>
__device__ __forceinline__ void load_raw<2>(const unsigned char *in, long long band_off, unsigned off, bool active, RawCols<2> &r) {
    r.w = active ? __ldg(reinterpret_cast<const unsigned *>(in + band_off + off)) : 0u;
}

// dp2a with signed 16-bit halves (a) and unsigned byte coefficients (b): lo16(a)*b0 + hi16(a)*b1 (+ c)
__device__ __forceinline__ int dp2a_lo_su(unsigned a, unsigned b, int c) {
    int d;
    asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// unpack + dequantise one packed pair.  SMALLDQ: divisor <= 255 -> one dp2a per coefficient.
template <bool SMALLDQ>
__device__ __forceinline__ void deq_pair(unsigned w, int dq, int &lo, int &hi) {
    if (SMALLDQ) {
        lo = dp2a_lo_su(w, (unsigned)dq, 0);
        hi = dp2a_lo_su(w, (unsigned)dq << 8, 0);
    } else {
        lo = lo16(w) * dq;
        hi = hi16(w) * dq;
    }
}
__device__ __forceinline__ void unpack_pair(unsigned w, int &lo, int &hi) { lo = lo16(w); hi = hi16(w); }

template <bool SMALLDQ, int NC>
struct Expand;
template <bool SMALLDQ>
struct Expand<SMALLDQ, 4> {
    static __device__ __forceinline__ void ll(const RawCols<4> &r, int *v) { unpack_pair(r.w.x, v[0], v[1]); unpack_pair(r.w.y, v[2], v[3]); }
    static __device__ __forceinline__ void hp(const RawCols<4> &r, int dq, int *v) {
        deq_pair<SMALLDQ>(r.w.x, dq, v[0], v[1]); deq_pair<SMALLDQ>(r.w.y, dq, v[2], v[3]);
    }
};
template <bool SMALLDQ>
struct Expand<SMALLDQ, 2> {
    static __device__ __forceinline__ void ll(const RawCols<2> &r, int *v) { unpack_pair(r.w, v[0], v[1]); }
    static __device__ __forceinline__ void hp(const RawCols<2> &r, int dq, int *v) { deq_pair<SMALLDQ>(r.w, dq, v[0], v[1]); }
};

// What a lane of a strip owns: band columns col0 .. col0 + 3 (luma columns in the 4:2:2 kernels, whose chroma lane owns
// col0 / 2 and col0 / 2 + 1).  Lanes 0 and 31 are halo lanes: they load, their columns are the neighbouring strips'.
struct InvLane {
    int col0;               // first band column
    bool active;            // the lane's first column is inside the band: it loads
    bool writer;            // it writes output
    bool left_border;       // it owns band column 0
    bool right_border;      // it owns the last band column
    bool has_border;        // warp-uniform: the strip touches the left or right band border
};

// ragged: the band width need not be a multiple of 4 (k_inv_plane).  A lane whose 4 columns are not all inside the band
// then still loads (its first column is its left neighbour's right tap) but does not write: those 1-3 columns, the right
// border among them, are k_inv_plane_edge's.  Level-1 bands of 4:2:2 and 4:4:4 frames are whole lanes wide.
__device__ __forceinline__ InvLane inv_lane(int strip, int width, int lane, bool ragged)
{
    InvLane L;
    L.col0 = strip * kInvStrip - 4 + lane * 4;
    L.active = (L.col0 >= 0) && (L.col0 < width);
    L.writer = L.active && lane >= 1 && lane <= 30 && (!ragged || L.col0 + 4 <= width);
    L.left_border = (L.col0 == 0);
    L.right_border = (L.col0 + 4 == width);
    L.has_border = (strip == 0) || ((strip + 1) * kInvStrip + 4 >= width);
    return L;
}

// vertical inverse for NC columns: rows (p, c, n) of the low band and row c of the high band
template <int NC>
__device__ __forceinline__ void vinv_mid(const int *p, const int *c, const int *n, const int *h, int *e, int *o)
{
#pragma unroll
    for (int i = 0; i < NC; i++) {
        e[i] = (((p[i] - n[i] + 4) >> 3) + c[i] + h[i]) >> 1;
        o[i] = (((n[i] - p[i] + 4) >> 3) + c[i] - h[i]) >> 1;
    }
}
// top border: a0,a1,a2 = rows 0,1,2 ; bottom border: call with a0,a1,a2 = rows H-1,H-2,H-3 and bottom=true
template <int NC>
__device__ __forceinline__ void vinv_border(const int *a0, const int *a1, const int *a2, const int *h, bool bottom, int *e, int *o)
{
#pragma unroll
    for (int i = 0; i < NC; i++) {
        const int x = (11 * a0[i] - 4 * a1[i] + a2[i] + 4) >> 3;
        const int y = (5 * a0[i] + 4 * a1[i] - a2[i] + 4) >> 3;
        e[i] = ((bottom ? y : x) + h[i]) >> 1;
        o[i] = ((bottom ? x : y) - h[i]) >> 1;
    }
}

// horizontal inverse for NC columns -> 2*NC samples t (BEFORE the final >>1 / <<1):
//   t[2i] = ((l[i-1] - l[i+1] + 4) >> 3) + l[i] + h[i],  t[2i+1] = ((l[i+1] - l[i-1] + 4) >> 3) + l[i] - h[i]
template <int NC>
__device__ __forceinline__ void hinv(const int *l, const int *h, const InvLane &L, int *t)
{
    const int lp = __shfl_up_sync(kFullMask, l[NC - 1], 1);
    const int ln = __shfl_down_sync(kFullMask, l[0], 1);
#pragma unroll
    for (int i = 0; i < NC; i++) {
        const int a = (i == 0) ? lp : l[i - 1];
        const int b = (i == NC - 1) ? ln : l[i + 1];
        t[2 * i] = ((a - b + 4) >> 3) + l[i] + h[i];
        t[2 * i + 1] = ((b - a + 4) >> 3) + l[i] - h[i];
    }
    if (L.has_border) {
    if (L.left_border) {
        const int l2 = (NC > 2) ? l[2] : ln;
        t[0] = ((11 * l[0] - 4 * l[1] + l2 + 4) >> 3) + h[0];
        t[1] = ((5 * l[0] + 4 * l[1] - l2 + 4) >> 3) - h[0];
    }
    if (L.right_border) {
        const int k = NC - 1;
        const int l2 = (NC > 2) ? l[k - 2] : lp;
        t[2 * k] = ((5 * l[k] + 4 * l[k - 1] - l2 + 4) >> 3) + h[k];
        t[2 * k + 1] = ((11 * l[k] - 4 * l[k - 1] + l2 + 4) >> 3) - h[k];
    }
    }
}

__device__ __forceinline__ unsigned pack_sat16(int lo, int hi) {
    unsigned d;
    asm("cvt.pack.sat.s16.s32 %0, %1, %2;" : "=r"(d) : "r"(hi), "r"(lo));
    return d;
}

// ----------------------------------------------------------------------------
// Lane-distributed L2 prefetch.  A future band row of one strip touches <= 3 cache lines per luma band and <= 2 per
// chroma band; instead of every lane prefetching its own 8 bytes of each of the 12 bands (12 address computations
// per warp and row), each lane owns ONE (channel, band, 128-byte line) and the whole set costs one prefetch
// instruction per row.  LL/LH are fetched 4 rows ahead (the vertical window reads row r+1), HL/HH 3 rows ahead.
struct LanePrefetch {
    const unsigned char *base;      // in + band offset + line start (row 0)
    int pitch;
    int ahead;
    bool valid;
    __device__ __forceinline__ void issue(int r, int y1, int H) const {
        if (valid && r + 3 < y1) prefetch_l2(base + (long long)min(r + ahead, H - 1) * pitch);
    }
};

// chan_of_lane < 0: lane idle.  bytes_per_col = 2 for a full-width band, 1 for the half-width chroma bands of 4:2:2
// (their columns are addressed as luma_column / 2).
__device__ __forceinline__ LanePrefetch make_prefetch(const InvGeom &g, const unsigned char *in, int strip, int band, int line,
                                                      int bytes_per_col, bool on)
{
    LanePrefetch pf;
    const int col = ((max(strip * kInvStrip - 4, 0) * bytes_per_col) & ~127) + line * 128;
    pf.valid = on && col < g.pitch;
    pf.base = in + g.band_off[band] + col;
    pf.pitch = g.pitch;
    pf.ahead = (band < 2) ? 4 : 3;
    return pf;
}

// ----------------------------------------------------------------------------
// The vertical step of every inverse kernel.  A window holds the expanded LL / LH rows r - 1 and r of one channel; a step
// takes the columns of LL / LH row r + 1 and HL / HH row r (inv_expand of the raw ones) and produces the t values (before
// the filter's final shift) of output rows 2r (te) and 2r + 1 (to).  Where the raw columns come from (global memory one
// iteration ahead, expanded before the next loads are issued, or a TMA ring) is the kernel's business.
template <int NC> struct InvWin { int lp[NC], lc[NC], hp[NC], hc[NC]; };
template <int NC> struct InvRaw { RawCols<NC> ll, lh, hl, hh; };

// window <- LL / LH of the next band row
template <int NC, bool SMALLDQ>
__device__ __forceinline__ void inv_fill(InvWin<NC> &w, const InvGeom &g, const RawCols<NC> &ll, const RawCols<NC> &lh)
{
#pragma unroll
    for (int i = 0; i < NC; i++) { w.lp[i] = w.lc[i]; w.hp[i] = w.hc[i]; }
    Expand<SMALLDQ, NC>::ll(ll, w.lc);
    Expand<SMALLDQ, NC>::hp(lh, g.dq[1], w.hc);
}

// the raw columns of a step expanded / dequantised
template <int NC> struct InvCols { int ll[NC], lh[NC], hl[NC], hh[NC]; };
template <int NC, bool SMALLDQ>
__device__ __forceinline__ InvCols<NC> inv_expand(const InvGeom &g, const InvRaw<NC> &x)
{
    InvCols<NC> v;
    Expand<SMALLDQ, NC>::ll(x.ll, v.ll);
    Expand<SMALLDQ, NC>::hp(x.lh, g.dq[1], v.lh);
    Expand<SMALLDQ, NC>::hp(x.hl, g.dq[2], v.hl);
    Expand<SMALLDQ, NC>::hp(x.hh, g.dq[3], v.hh);
    return v;
}

template <int NC>
__device__ __forceinline__ void inv_step(InvWin<NC> &w, const InvCols<NC> &x, const InvLane &L, int *te, int *to)
{
    int el[NC], ol[NC], eh[NC], oh[NC];
    vinv_mid<NC>(w.lp, w.lc, x.ll, x.hl, el, ol);
    vinv_mid<NC>(w.hp, w.hc, x.lh, x.hh, eh, oh);
    hinv<NC>(el, eh, L, te);
    hinv<NC>(ol, oh, L, to);
#pragma unroll
    for (int i = 0; i < NC; i++) { w.lp[i] = w.lc[i]; w.lc[i] = x.ll[i]; w.hp[i] = w.hc[i]; w.hc[i] = x.lh[i]; }
}

// Register-fed kernels: the raw columns of one step (LL / LH of band row r + 1, HL / HH of row r) from global memory
template <int NC>
__device__ __forceinline__ void load_step(const InvGeom &g, const unsigned char *in, int r, int H, unsigned colbyte, bool active,
                                          InvRaw<NC> &x)
{
    const unsigned rn = (unsigned)min(r + 1, H - 1) * g.pitch + colbyte, rc = (unsigned)r * g.pitch + colbyte;
    load_raw<NC>(in, g.band_off[0], rn, active, x.ll);
    load_raw<NC>(in, g.band_off[1], rn, active, x.lh);
    load_raw<NC>(in, g.band_off[2], rc, active, x.hl);
    load_raw<NC>(in, g.band_off[3], rc, active, x.hh);
}

// Register-fed kernels: window rows y0 - 1 and y0, and the raw columns of the first step
template <int NC, bool SMALLDQ>
__device__ __forceinline__ void inv_begin(InvWin<NC> &w, InvRaw<NC> &x, const InvGeom &g, const unsigned char *in, int y0, int H,
                                          unsigned colbyte, bool active)
{
    RawCols<NC> ll, lh;
    const unsigned rp = (unsigned)max(y0 - 1, 0) * g.pitch + colbyte, rc = (unsigned)y0 * g.pitch + colbyte;
    load_raw<NC>(in, g.band_off[0], rp, active, ll);
    load_raw<NC>(in, g.band_off[1], rp, active, lh);
    inv_fill<NC, SMALLDQ>(w, g, ll, lh);
    load_raw<NC>(in, g.band_off[0], rc, active, ll);
    load_raw<NC>(in, g.band_off[1], rc, active, lh);
    inv_fill<NC, SMALLDQ>(w, g, ll, lh);
    load_step<NC>(g, in, y0, H, colbyte, active, x);
}

// Border band rows (r = 0 or r = H-1), computed from scratch by the border warps with the full multiply
// (spatial.c:21980-22060 top, :22320-22400 bottom).
template <int NC>
__device__ __forceinline__ void inv_border_row(const InvGeom &g, const unsigned char *in, bool bottom, int H, unsigned colbyte,
                                               const InvLane &L, int *te, int *to)
{
    const int rows[3] = {bottom ? H - 1 : 0, bottom ? H - 2 : 1, bottom ? H - 3 : 2};
    int a[3][NC], b[3][NC], vhl[NC], vhh[NC];
    RawCols<NC> r;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const unsigned off = (unsigned)rows[k] * g.pitch + colbyte;
        load_raw<NC>(in, g.band_off[0], off, L.active, r); Expand<false, NC>::ll(r, a[k]);
        load_raw<NC>(in, g.band_off[1], off, L.active, r); Expand<false, NC>::hp(r, g.dq[1], b[k]);
    }
    const unsigned off = (unsigned)rows[0] * g.pitch + colbyte;
    load_raw<NC>(in, g.band_off[2], off, L.active, r); Expand<false, NC>::hp(r, g.dq[2], vhl);
    load_raw<NC>(in, g.band_off[3], off, L.active, r); Expand<false, NC>::hp(r, g.dq[3], vhh);
    int el[NC], ol[NC], eh[NC], oh[NC];
    vinv_border<NC>(a[0], a[1], a[2], vhl, bottom, el, ol);
    vinv_border<NC>(b[0], b[1], b[2], vhh, bottom, eh, oh);
    hinv<NC>(el, eh, L, te);
    hinv<NC>(ol, oh, L, to);
}

// ----------------------------------------------------------------------------
// generic level: 4 bands -> int16 plane (2W x 2H)
template <int DESCALE, bool SMALLDQ>
__global__ void __launch_bounds__(128) k_inv_plane(const __grid_constant__ InvParams p)
{
    const int lane = threadIdx.x;
    const int f = blockIdx.z / p.nchan, c = blockIdx.z - f * p.nchan;
    const InvGeom &g = p.ch[c];
    const int strip = blockIdx.x;
    if (strip * kInvStrip >= g.width) return;
    const int H = g.height;
    const InvLane L = inv_lane(strip, g.width, lane, true);
    const unsigned colbyte = (unsigned)(L.col0 * 2);
    const unsigned char *in = p.in_base[f];
    unsigned char *out = p.out_base[f] + g.out_off + (long long)L.col0 * 4;

    auto emit = [&](int r, const int *te, const int *to) {
        uint4 a, b;
        if (DESCALE) {
            a = make_uint4(pack_sat16(te[0] << 1, te[1] << 1), pack_sat16(te[2] << 1, te[3] << 1),
                           pack_sat16(te[4] << 1, te[5] << 1), pack_sat16(te[6] << 1, te[7] << 1));
            b = make_uint4(pack_sat16(to[0] << 1, to[1] << 1), pack_sat16(to[2] << 1, to[3] << 1),
                           pack_sat16(to[4] << 1, to[5] << 1), pack_sat16(to[6] << 1, to[7] << 1));
        } else {
            a = make_uint4(pack_sat16(te[0] >> 1, te[1] >> 1), pack_sat16(te[2] >> 1, te[3] >> 1),
                           pack_sat16(te[4] >> 1, te[5] >> 1), pack_sat16(te[6] >> 1, te[7] >> 1));
            b = make_uint4(pack_sat16(to[0] >> 1, to[1] >> 1), pack_sat16(to[2] >> 1, to[3] >> 1),
                           pack_sat16(to[4] >> 1, to[5] >> 1), pack_sat16(to[6] >> 1, to[7] >> 1));
        }
        unsigned char *o = out + (long long)(2 * r) * g.out_pitch;
        *reinterpret_cast<uint4 *>(o) = a;
        *reinterpret_cast<uint4 *>(o + g.out_pitch) = b;
    };

    if (blockIdx.y == gridDim.y - 1) {          // border warps: band rows 0 and H-1
        if (threadIdx.y > 1) return;
        const bool bottom = (threadIdx.y == 1);
        int te[8], to[8];
        inv_border_row<4>(g, in, bottom, H, colbyte, L, te, to);
        if (L.writer) emit(bottom ? H - 1 : 0, te, to);
        return;
    }
    const int y0 = max((int)(blockIdx.y * blockDim.y + threadIdx.y) * p.th, 1);
    const int y1 = min((int)(blockIdx.y * blockDim.y + threadIdx.y + 1) * p.th, H - 1);
    if (y0 >= y1) return;

    const LanePrefetch pf = make_prefetch(g, in, strip, lane / 3, lane % 3, 2, lane < 12);
    InvWin<4> w{};
    InvRaw<4> nx;
    inv_begin<4, SMALLDQ>(w, nx, g, in, y0, H, colbyte, L.active);
    for (int r = y0; r < y1; r++) {
        pf.issue(r, y1, H);
        const InvCols<4> x = inv_expand<4, SMALLDQ>(g, nx);
        if (r + 1 < y1) load_step<4>(g, in, r + 1, H, colbyte, L.active, nx);       // the next iteration's rows
        int te[8], to[8];
        inv_step<4>(w, x, L, te, to);
        if (L.writer) emit(r, te, to);
    }
}

// ----------------------------------------------------------------------------
// Ragged widths: band columns [4 * (width / 4), width) of an inverse level, one thread per band coefficient position
// (-> a 2x2 block of output samples), written as the formulas read (spatial.c:21980-22400 vertical,
// InvertHorizontalStrip16s.c:459-896 / :1700-2166 horizontal).
template <int DESCALE>
__global__ void __launch_bounds__(128) k_inv_plane_edge(const __grid_constant__ InvParams p)
{
    const int f = blockIdx.z / p.nchan, c = blockIdx.z - f * p.nchan;
    const InvGeom &g = p.ch[c];
    const int W = g.width, H = g.height;
    const int col = (W >> 2) * 4 + blockIdx.y;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= W || r >= H) return;
    const unsigned char *in = p.in_base[f];
    auto coef = [&](int b, int row, int cc) {
        return (int)*reinterpret_cast<const short *>(in + g.band_off[b] + (long long)row * g.pitch + 2 * cc) * (b ? g.dq[b] : 1);
    };
    // vertical inverse of (low band lb, high band hb) at band column cc -> even / odd intermediate rows
    auto vinv = [&](int lb, int hb, int cc, int &e, int &o) {
        const int hv = coef(hb, r, cc);
        if (r == 0 || r == H - 1) {
            const bool bottom = (r != 0);
            const int a0 = coef(lb, bottom ? H - 1 : 0, cc), a1 = coef(lb, bottom ? H - 2 : 1, cc), a2 = coef(lb, bottom ? H - 3 : 2, cc);
            const int x = (11 * a0 - 4 * a1 + a2 + 4) >> 3, y = (5 * a0 + 4 * a1 - a2 + 4) >> 3;
            e = ((bottom ? y : x) + hv) >> 1;
            o = ((bottom ? x : y) - hv) >> 1;
        } else {
            const int pv = coef(lb, r - 1, cc), cv = coef(lb, r, cc), nv = coef(lb, r + 1, cc);
            e = (((pv - nv + 4) >> 3) + cv + hv) >> 1;
            o = (((nv - pv + 4) >> 3) + cv - hv) >> 1;
        }
    };
    // columns col-2 .. col+1 of the vertically inverted lowpass (LL/HL) and column col of the highpass (LH/HH)
    int le[4], lo[4], he, ho;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int cc = min(max(col - 2 + k, 0), W - 1);
        vinv(0, 2, cc, le[k], lo[k]);
    }
    vinv(1, 3, col, he, ho);
    auto hpair = [&](const int *l, int hv, int &t0, int &t1) {      // l[0..3] = columns col-2 .. col+1
        if (col == W - 1) {
            t0 = ((5 * l[2] + 4 * l[1] - l[0] + 4) >> 3) + hv;
            t1 = ((11 * l[2] - 4 * l[1] + l[0] + 4) >> 3) - hv;
        } else {
            t0 = ((l[1] - l[3] + 4) >> 3) + l[2] + hv;
            t1 = ((l[3] - l[1] + 4) >> 3) + l[2] - hv;
        }
    };
    int e0, e1, o0, o1;
    hpair(le, he, e0, e1);
    hpair(lo, ho, o0, o1);
    unsigned char *out = p.out_base[f] + g.out_off + (long long)(2 * r) * g.out_pitch + (long long)col * 4;
    if (DESCALE) {
        *reinterpret_cast<unsigned *>(out) = pack_sat16(e0 << 1, e1 << 1);
        *reinterpret_cast<unsigned *>(out + g.out_pitch) = pack_sat16(o0 << 1, o1 << 1);
    } else {
        *reinterpret_cast<unsigned *>(out) = pack_sat16(e0 >> 1, e1 >> 1);
        *reinterpret_cast<unsigned *>(out + g.out_pitch) = pack_sat16(o0 >> 1, o1 >> 1);
    }
}

// ----------------------------------------------------------------------------
// final level of a 4:2:2 frame: 12 bands -> packed 8-bit YUYV / UYVY.
// 8-bit reduction: the reference computes v = max(t, 0) >> 1 (10-bit) and out = sat_u8((v + d) >> 2) with
// d = rand() & 1 per position (InvertHorizontalStrip16s.c:3807-3892) - not reproducible.  We use the
// deterministic ordered dither d = (x ^ y) & 1, i.e. out = sat_u8((t + 2d) >> 3), which stays inside the
// reference's envelope {(v) >> 2, (v + 1) >> 2} at every pixel.
__device__ __forceinline__ unsigned pack_u8x4(int a, int b, int c, int d) {
    // bytes (LSB first): a, b, c, d, each saturated to [0,255].
    // cvt.pack.sat.u8.s32.b32 r, x, y, z  ->  r = (z << 16) | (sat(x) << 8) | sat(y)
    unsigned t, r;
    asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(t) : "r"(d), "r"(c), "r"(0));
    asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(b), "r"(a), "r"(t));
    return r;
}

// 16-bit unsigned output sample of the final level: see InvParams::up_shift (the reference's ...ToRow16u rule)
__device__ __forceinline__ unsigned row16u(int t, int up_shift, int hi) {
    return (unsigned)min(max(t >> 1, 0) << up_shift, hi);
}

// B64A alpha word of a four-channel sample: the channel-3 sample with the encoder's alpha curve removed (alphacompandDCoffset
// 256, alphacompandGain 9400, Codec/codec.h:164).  The reference decoder takes RGBA 4:4:4:4 samples with an alpha output
// through its active-metadata path (bayer.c:7144-7147): the ...ToRow16u sample >> 4, i.e. the 12-bit sample limited to
// [0, 4095] in every column, then ((a - 256) << 3) * 9400 >> 12 limited to [0, 65535] (bayer.c:16215-16224
// Convert4444LinesToOutput; its SSE2 loop never runs there, width8 is forced to 0).
__device__ __forceinline__ unsigned b64a_alpha(int t) {
    const int a = min(max(t >> 1, 0), 4095);
    return (unsigned)min(max(((a - 256) * (8 * 9400)) >> 12, 0), 65535);
}

// ...ToRow16u limit of band column `band_col` of channel c: hi_simd where the reference's SSE2 loop runs, 65535 beyond
__device__ __forceinline__ int limit16(const InvParams &p, int c, int band_col) { return band_col >= p.tail_col[c] ? 65535 : p.hi_simd; }

// One output row of a lane's 8 luma + 4 + 4 chroma samples as 8-bit YUYV / UYVY: sat_u8((t + d) >> sh), d the ordered
// dither (x ^ y) & 1 on the sample's own column index scaled to the shift (odd: the row is output row 2r + 1)
__device__ __forceinline__ uint4 pack_422_8(const int *yy, const int *uu, const int *vv, int sh, bool odd, bool uyvy)
{
    const int d0 = (odd ? 1 : 0) << (sh - 2), d1 = (odd ? 0 : 1) << (sh - 2);
    unsigned w[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int ya = (yy[2 * k] + d0) >> sh, yb = (yy[2 * k + 1] + d1) >> sh;
        const int cu = (uu[k] + ((k & 1) ? d1 : d0)) >> sh, cv = (vv[k] + ((k & 1) ? d1 : d0)) >> sh;
        w[k] = uyvy ? pack_u8x4(cu, ya, cv, yb) : pack_u8x4(ya, cu, yb, cv);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// One band row r of the final 4:2:2 level -> output rows 2r and 2r + 1 of the lane's 8 luma samples (+ 4 + 4 chroma) as
// 8-bit YUYV / UYVY or YU64.  `out` already points at the lane's first sample of row 0.  t values arrive BEFORE the
// filter's final >> 1.
template <InvOut OUT>
__device__ __forceinline__ void emit_422(const InvParams &p, unsigned char *out, int col0, int r, const int *ye, const int *yo,
                                         const int *ue, const int *uo, const int *ve, const int *vo)
{
    const InvGeom &gy = p.ch[0];
    unsigned char *o = out + (long long)(2 * r) * gy.out_pitch;
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
        const int *yy = rr ? yo : ye, *uu = rr ? uo : ue, *vv = rr ? vo : ve;
        unsigned char *q = o + (rr ? gy.out_pitch : 0);
        if constexpr (OUT == kInvOutYU64) {
            const int us = p.up_shift;
            unsigned w[8];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                // luma band column col0 + k -> samples 2k, 2k + 1; chroma band column col0 / 2 + (k >> 1) -> sample k
                const int hy = limit16(p, 0, col0 + k);
                const int hc1 = limit16(p, 1, (col0 >> 1) + (k >> 1)), hc2 = limit16(p, 2, (col0 >> 1) + (k >> 1));
                // pixel pair k: words (Y0, C1) (Y1, C3); C1 = channel 1 (the v arrays), C3 = channel 2 (the u arrays)
                w[2 * k] = row16u(yy[2 * k], us, hy) | (row16u(vv[k], us, hc1) << 16);
                w[2 * k + 1] = row16u(yy[2 * k + 1], us, hy) | (row16u(uu[k], us, hc2) << 16);
            }
            *reinterpret_cast<uint4 *>(q) = make_uint4(w[0], w[1], w[2], w[3]);
            *reinterpret_cast<uint4 *>(q + 16) = make_uint4(w[4], w[5], w[6], w[7]);
        } else {
            // final >> 1 of the filter merged with the >> (precision - 8) reduction
            *reinterpret_cast<uint4 *>(q) = pack_422_8(yy, uu, vv, p.shift + 1, rr, p.uyvy);
        }
    }
}

__device__ __forceinline__ unsigned v210_word(unsigned a, unsigned b, unsigned c) { return a | (b << 10) | (c << 20); }

// One band row r of the final 4:2:2 level -> output rows 2r and 2r + 1 as V210: groups of 6 pixels in 4 little-endian
// words, components at bits 0 / 10 / 20 in the order Cb0 Y0 Cr0 | Y1 Cb1 Y2 | Cr1 Y3 Cb2 | Y4 Cr2 Y5 (Cb = channel 2, the u
// arrays; Cr = channel 1).  Reference: decoder.c:26303 -> InvertHorizontalStrip16s.c:6490 InvertHorizontalYUVStrip16sToYUVOutput
// (the ...ToRow16u samples of YU64) -> convert.c:13526 ConvertPlanarYUVToV210 with upshift -6.  Both limits of ...ToRow16u
// (1023 << 6 in its SSE2 columns, 65535 in its scalar tail) are 1023 after the >> 6, so every component is
// min(max(t >> 1, 0), 1023) of the 10-bit 4:2:2 precision, in every column.
//
// A lane's 8 pixels are 16 components; lanes (1, 2, 3), (4, 5, 6) ... (28, 29, 30) form trios (a, b, c) of 24 pixels = 4
// groups = 64 bytes, and a strip's 240 pixels are 40 groups.  b's components straddle groups 1 and 2: it hands three words
// (two of them partial) to a and three to c by shuffle; a stores groups 0-1 and c groups 2-3, 32 contiguous bytes each.
// `out` points at the lane's 32 bytes (a: trio start, b and c: trio start + 32).  Every lane of the warp must call this.
//
// The image's last group (convert.c:13889-13965, the scalar loop for W % 6 != 0, which repeats stale components):
//   W % 24 == 8  (W % 6 == 2): lane a has no b; its group 1 is  Cb0 Y0 Cr0 | Y1 Cb0 Y0 | Cr0 Y1 Cb0 | Y1 Cr0 Y0;
//   W % 24 == 16 (W % 6 == 4): lane b has no c and writes group 2 itself: Cb0 Y0 Cr0 | Y1 Cb1 Y2 | Cr1 Y3 X | Y3 Cr1 Y2.
//   The reference reads X one element past its Cb row (the next row's first luma sample on most rows, not reproducible);
//   we write Cb1 there.
// role: 0 a, 1 b, 2 c; tail: the next lane is right of the image; store: this lane writes (b only at the tail).
__device__ __forceinline__ void emit_v210(const InvParams &p, unsigned char *out, int role, bool tail, bool store, int r,
                                          const int *ye, const int *yo, const int *ue, const int *uo, const int *ve, const int *vo)
{
    const InvGeom &gy = p.ch[0];
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
        const int *yy = rr ? yo : ye, *uu = rr ? uo : ue, *vv = rr ? vo : ve;
        unsigned s[16];         // component stream Cb Y Cr Y of the lane's 4 pixel pairs
#pragma unroll
        for (int k = 0; k < 4; k++) {
            s[4 * k] = row16u(uu[k], 0, 1023); s[4 * k + 1] = row16u(yy[2 * k], 0, 1023);
            s[4 * k + 2] = row16u(vv[k], 0, 1023); s[4 * k + 3] = row16u(yy[2 * k + 1], 0, 1023);
        }
        // b's stream starts at bit 10 of a's sixth word and ends at bit 10 of c's first word
        const unsigned d0 = __shfl_down_sync(kFullMask, (s[0] << 10) | (s[1] << 20), 1);
        const unsigned d1 = __shfl_down_sync(kFullMask, v210_word(s[2], s[3], s[4]), 1);
        const unsigned d2 = __shfl_down_sync(kFullMask, v210_word(s[5], s[6], s[7]), 1);
        const unsigned u0 = __shfl_up_sync(kFullMask, v210_word(s[8], s[9], s[10]), 1);
        const unsigned u1 = __shfl_up_sync(kFullMask, v210_word(s[11], s[12], s[13]), 1);
        const unsigned u2 = __shfl_up_sync(kFullMask, s[14] | (s[15] << 10), 1);
        const unsigned last = v210_word(s[15], s[14], s[13]);       // word 3 of either tail group
        uint4 v0, v1;
        if (role == 0) {
            v0 = make_uint4(v210_word(s[0], s[1], s[2]), v210_word(s[3], s[4], s[5]), v210_word(s[6], s[7], s[8]), v210_word(s[9], s[10], s[11]));
            v1 = tail ? make_uint4(v210_word(s[12], s[13], s[14]), v210_word(s[15], s[12], s[13]), v210_word(s[14], s[15], s[12]), last)
                      : make_uint4(v210_word(s[12], s[13], s[14]), s[15] | d0, d1, d2);
        } else if (role == 1) {
            v0 = make_uint4(v210_word(s[8], s[9], s[10]), v210_word(s[11], s[12], s[13]), v210_word(s[14], s[15], s[12]), last);
            v1 = v0;
        } else {
            v0 = make_uint4(u0, u1, u2 | (s[0] << 20), v210_word(s[1], s[2], s[3]));
            v1 = make_uint4(v210_word(s[4], s[5], s[6]), v210_word(s[7], s[8], s[9]), v210_word(s[10], s[11], s[12]), v210_word(s[13], s[14], s[15]));
        }
        unsigned char *q = out + (long long)(2 * r + rr) * gy.out_pitch;
        if (store) {
            *reinterpret_cast<uint4 *>(q) = v0;
            if (role != 1) *reinterpret_cast<uint4 *>(q + 16) = v1;
        }
    }
}

#include "cfb_inverse_tma.inl"

// ----------------------------------------------------------------------------
// final level of a 4:4:4 frame (channels G, R, B [, A]): 12 (16) bands -> packed RGB.  One warp reconstructs every channel
// of its strip, so every lane owns 8 whole pixels.
// RG48: 16-bit R,G,B, 48 contiguous bytes per lane.  Reference: Codec/decoder.c:26886 -> wavelet.c:4947
// TransformInverseRGB444ToRGB48: InvertSpatial{Top,Middle,Bottom}Row16sToYUV16 per channel (horizontal stage
// InvertHorizontalStrip16s.c:16571 ...ToRow16u: max(t >> 1, 0) << (16 - precision), limited as InvParams::hi_simd /
// tail_col describe), then ConvertPlanarRGB16uToPackedRGB48 (plane 1 -> R, 0 -> G, 2 -> B).
// B64A: 16-bit A,R,G,B words instead (64 contiguous bytes per lane), decoder.c:26862 -> InvertHorizontalStrip16s.c:13298
// InvertHorizontalStrip16sRGB2B64A: alpha is the constant 0xfff << 4 (:13385 a_epi16); colour samples are limited to the
// 12-bit maximum where its SSE2 loop runs (:13387 limiterRGB) and to 65535 in its scalar tail and right border column
// (InvParams::tail_col, the same for the three channels); native (little-endian) words as the reference's decoder leaves them.
// B64A with alpha, of a four-channel (RGBA 4:4:4:4) sample (kInvOutB64AAlpha): the same warp reconstructs channel 3 as a
// fourth plane and writes it de-companded as alpha (b64a_alpha); the colour samples follow the RG48 rule (tail_col[c] per
// channel), because the reference decoder forms this frame from its ...ToRow16u rows (bayer.c:16691-16780 copies them into
// the A,R,G,B words).
// 10-bit RGB: one 32-bit word per pixel with 10-bit components (RG30 / AB10 / AR10 / R210 / DPX0; decoder.c:26893 ->
// InvertHorizontalStrip16s.c:14812 InvertHorizontalStrip16sRGB2RG30): the 12-bit sample limited to [0, 4095] in every column
// (:14892 limiterRGB; the scalar code clamps alike), >> 2 (:15552), components at bit positions rgb10.pos[0..2] = R, G, B,
// the word byte-swapped when p.rgb10.byteswap is set (R210, DPX0; :15577-15613).  32 contiguous bytes per lane.
// One band row r -> output rows 2r and 2r + 1 of the lane's 8 pixels; te / to[c] = t values of channel c (0 G, 1 R, 2 B, 3 A)
template <InvOut OUT>
__device__ __forceinline__ void emit_444(const InvParams &p, unsigned char *out, int col0, int r, const int (*te)[8], const int (*to)[8])
{
    const int us = p.up_shift;
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
        const int *G = rr ? to[0] : te[0], *R = rr ? to[1] : te[1], *B = rr ? to[2] : te[2];
        unsigned char *q = out + (long long)(2 * r + rr) * p.ch[0].out_pitch;
        if constexpr (OUT == kInvOutRGB10) {
            unsigned w[8];
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const unsigned word = ((row16u(R[i], 0, 4095) >> 2) << p.rgb10.pos[0]) | ((row16u(G[i], 0, 4095) >> 2) << p.rgb10.pos[1]) |
                                      ((row16u(B[i], 0, 4095) >> 2) << p.rgb10.pos[2]);
                w[i] = p.rgb10.byteswap ? __byte_perm(word, 0, 0x0123) : word;
            }
            *reinterpret_cast<uint4 *>(q) = make_uint4(w[0], w[1], w[2], w[3]);
            *reinterpret_cast<uint4 *>(q + 16) = make_uint4(w[4], w[5], w[6], w[7]);
        } else if constexpr (OUT == kInvOutRG48) {
            unsigned short v[24];
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int bc = col0 + (i >> 1);
                v[3 * i + 0] = (unsigned short)row16u(R[i], us, limit16(p, 1, bc));
                v[3 * i + 1] = (unsigned short)row16u(G[i], us, limit16(p, 0, bc));
                v[3 * i + 2] = (unsigned short)row16u(B[i], us, limit16(p, 2, bc));
            }
            unsigned w[12];
#pragma unroll
            for (int i = 0; i < 12; i++) w[i] = (unsigned)v[2 * i] | ((unsigned)v[2 * i + 1] << 16);
            *reinterpret_cast<uint4 *>(q) = make_uint4(w[0], w[1], w[2], w[3]);
            *reinterpret_cast<uint4 *>(q + 16) = make_uint4(w[4], w[5], w[6], w[7]);
            *reinterpret_cast<uint4 *>(q + 32) = make_uint4(w[8], w[9], w[10], w[11]);
        } else {        // B64A: the alpha word is channel 3 de-companded (kInvOutB64AAlpha) or the constant hi_simd
            auto alpha = [&](int i) -> unsigned {
                if constexpr (OUT == kInvOutB64AAlpha) return b64a_alpha((rr ? to[3] : te[3])[i]);
                else return (unsigned)p.hi_simd;
            };
#pragma unroll
            for (int i = 0; i < 8; i += 2) {        // pixels i and i + 1 belong to band column col0 + i / 2
                const int bc = col0 + (i >> 1);
                const int hr = limit16(p, 1, bc), hg = limit16(p, 0, bc), hb = limit16(p, 2, bc);
                uint4 w;
                w.x = alpha(i) | (row16u(R[i], us, hr) << 16);
                w.y = row16u(G[i], us, hg) | (row16u(B[i], us, hb) << 16);
                w.z = alpha(i + 1) | (row16u(R[i + 1], us, hr) << 16);
                w.w = row16u(G[i + 1], us, hg) | (row16u(B[i + 1], us, hb) << 16);
                *reinterpret_cast<uint4 *>(q + 8 * i) = w;
            }
        }
    }
}

// BYR4: the mosaic of a Bayer sample (channels G, R-G, B-G, G1-G2 of half the mosaic's size each way; a full-resolution decode
// to DECODED_FORMAT_BYR4 runs no demosaic, decoder.c:13662-13669, :14738-14767).  The reference writes the four channels'
// ...ToRow16u rows into RawBayer16 (decoder.c:14629 -> InvertHorizontalStrip16s.c:17462 ...ToRow16uPlanar -> :16571, the RG48
// rule with tail_col[c] per channel) and Codec/bayer.c:13237 GenerateBYR2 turns one row of them into two mosaic rows:
//   d = GD - 32768; r = ((RG - 32768) << 1) + G; b = ((BG - 32768) << 1) + G; g1 = G + d; g2 = G - d, limited to [0, 65535]
//   (:13288-13310), then restore[v >> 2] when the decoder holds a linear-restore table (encode_curve_preset == 0, :13313-13319)
//   or v & 0xfffe (:13320-13326), in the 2 x 2 cell R G1 / G2 B, G1 R / B G2, G1 B / R G2, B G1 / G2 R for phases 0-3 (:13329-13355).
// Here the rows never exist: one band row r -> plane rows 2r, 2r + 1 -> mosaic rows 4r .. 4r + 3 of the lane's 16 mosaic
// columns, 32 contiguous bytes per row.  te / to[c] = t values of channel c.  The table is read through the read-only path.
__device__ __forceinline__ unsigned bayer_sample(const InvParams &p, int v)
{
    const unsigned u = (unsigned)min(max(v, 0), 65535);
    return p.bayer.restore ? (unsigned)__ldg(p.bayer.restore + (u >> 2)) : (u & 0xfffeu);
}

__device__ __forceinline__ void emit_bayer(const InvParams &p, unsigned char *out, int col0, int r, const int (*te)[8], const int (*to)[8])
{
    const int us = p.up_shift;
    // phases 2 and 3 are phases 1 and 0 with red and blue exchanged; phases 1 and 2 start their lines with green
    const bool swap_rb = p.bayer.phase >= 2, green_first = (p.bayer.phase == 1 || p.bayer.phase == 2);
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
        unsigned a[8], b[8];        // the two mosaic rows of plane row 2r + rr, one word per plane pixel
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int bc = col0 + (i >> 1);
            const int g = (int)row16u((rr ? to[0] : te[0])[i], us, limit16(p, 0, bc));
            const int rg = (int)row16u((rr ? to[1] : te[1])[i], us, limit16(p, 1, bc));
            const int bg = (int)row16u((rr ? to[2] : te[2])[i], us, limit16(p, 2, bc));
            const int d = (int)row16u((rr ? to[3] : te[3])[i], us, limit16(p, 3, bc)) - 32768;
            const unsigned red = bayer_sample(p, ((rg - 32768) << 1) + g), blue = bayer_sample(p, ((bg - 32768) << 1) + g);
            const unsigned g1 = bayer_sample(p, g + d), g2 = bayer_sample(p, g - d);
            const unsigned x = swap_rb ? blue : red, y = swap_rb ? red : blue;
            a[i] = green_first ? (g1 | (x << 16)) : (x | (g1 << 16));
            b[i] = green_first ? (y | (g2 << 16)) : (g2 | (y << 16));
        }
        unsigned char *q = out + (long long)(4 * r + 2 * rr) * p.ch[0].out_pitch;
        *reinterpret_cast<uint4 *>(q) = make_uint4(a[0], a[1], a[2], a[3]);
        *reinterpret_cast<uint4 *>(q + 16) = make_uint4(a[4], a[5], a[6], a[7]);
        q += p.ch[0].out_pitch;
        *reinterpret_cast<uint4 *>(q) = make_uint4(b[0], b[1], b[2], b[3]);
        *reinterpret_cast<uint4 *>(q + 16) = make_uint4(b[4], b[5], b[6], b[7]);
    }
}

template <InvOut OUT>
__device__ __forceinline__ void emit_444_or_bayer(const InvParams &p, unsigned char *out, int col0, int r, const int (*te)[8], const int (*to)[8])
{
    if constexpr (OUT == kInvOutBYR4) emit_bayer(p, out, col0, r, te, to);
    else emit_444<OUT>(p, out, col0, r, te, to);
}

template <bool SMALLDQ, InvOut OUT>
__global__ void __launch_bounds__(128) k_inv_444(const __grid_constant__ InvParams p)
{
    static_assert(OUT == kInvOutRG48 || OUT == kInvOutB64A || OUT == kInvOutB64AAlpha || OUT == kInvOutRGB10 || OUT == kInvOutBYR4,
                  "k_inv_444 writes the RGB(A) outputs of a 4:4:4 (4:4:4:4) codec and the BYR4 mosaic of a Bayer codec");
    constexpr int NCH = (OUT == kInvOutB64AAlpha || OUT == kInvOutBYR4) ? 4 : 3;
    const int lane = threadIdx.x;
    const int f = blockIdx.z;
    const InvGeom &gg = p.ch[0];
    const int strip = blockIdx.x;
    if (strip * kInvStrip >= gg.width) return;
    const int H = gg.height;
    const InvLane L = inv_lane(strip, gg.width, lane, false);
    const unsigned cb = (unsigned)(L.col0 * 2);
    const unsigned char *in = p.in_base[f];
    // 2 pixels per band column (BYR4: 4 mosaic samples)
    constexpr int kColBytes = (OUT == kInvOutRGB10 || OUT == kInvOutBYR4) ? 8 : (OUT == kInvOutRG48) ? 12 : 16;
    unsigned char *out = p.out_base[f] + gg.out_off + (long long)L.col0 * kColBytes;
    int te[NCH][8], to[NCH][8];

    if (blockIdx.y == gridDim.y - 1) {          // border warps: band rows 0 and H-1
        if (threadIdx.y > 1) return;
        const bool bottom = (threadIdx.y == 1);
#pragma unroll
        for (int c = 0; c < NCH; c++) inv_border_row<4>(p.ch[c], in, bottom, H, cb, L, te[c], to[c]);
        if (L.writer) emit_444_or_bayer<OUT>(p, out, L.col0, bottom ? H - 1 : 0, te, to);
        return;
    }
    const int y0 = max((int)(blockIdx.y * blockDim.y + threadIdx.y) * p.th, 1);
    const int y1 = min((int)(blockIdx.y * blockDim.y + threadIdx.y + 1) * p.th, H - 1);
    if (y0 >= y1) return;
    InvWin<4> w[NCH] = {};
    InvRaw<4> nx[NCH];
#pragma unroll
    for (int c = 0; c < NCH; c++) inv_begin<4, SMALLDQ>(w[c], nx[c], p.ch[c], in, y0, H, cb, L.active);
    for (int r = y0; r < y1; r++) {
#pragma unroll
        for (int c = 0; c < NCH; c++) {
            const InvCols<4> x = inv_expand<4, SMALLDQ>(p.ch[c], nx[c]);
            if (r + 1 < y1) load_step<4>(p.ch[c], in, r + 1, H, cb, L.active, nx[c]);
            inv_step<4>(w[c], x, L, te[c], to[c]);
        }
        if (L.writer) emit_444_or_bayer<OUT>(p, out, L.col0, r, te, to);
    }
}

// ----------------------------------------------------------------------------
// Interlaced sources: inverse of the frame (field) transform at level 1
//   Codec/decoder.c:21493 TransformInverseFrameToYUV / :22027 TransformInverseFrameToRow16u:
//   t_low = hinv(LL, LH), t_high = hinv(HL, HH) (InvertHorizontalRow16s8sTo16sBuffered), then
//   even row = (t_low - t_high) >> 1, odd row = (t_low + t_high) >> 1 (Codec/temporal.c:3741 InvertInterlaced16s).
// The coded HL band is difference coded along each row; the reference integrates it on the host after the FSM
// decode (decoder.c:20822-20836 `line[x] += line[x-1]`, int16 wrap).  Here k_fields_carry computes, per band row
// and strip, the sum of all coefficients left of the strip, and the inverse kernel finishes the prefix sum with a
// warp scan, so the coded buffer keeps the exact format the forward path wrote.
template <int NC>
__device__ __forceinline__ int row_segment_sum(const unsigned char *row, int c0, int c1, int lane)
{
    const int col = c0 + NC * lane;
    int v = 0;
    if (col < c1) {
        if (NC == 4) { const uint2 w = __ldg(reinterpret_cast<const uint2 *>(row + col * 2)); v = lo16(w.x) + hi16(w.x) + lo16(w.y) + hi16(w.y); }
        else { const unsigned w = __ldg(reinterpret_cast<const unsigned *>(row + col * 2)); v = lo16(w) + hi16(w); }
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(kFullMask, v, d);
    return v;
}

__global__ void __launch_bounds__(128) k_fields_carry(const __grid_constant__ InvParams p, const FieldsAux a)
{
    const int lane = threadIdx.x;
    const int row = blockIdx.x * blockDim.y + threadIdx.y;
    const int c = blockIdx.y, f = blockIdx.z;
    const InvGeom &g = p.ch[c];
    if (row >= g.height) return;
    const unsigned char *hl = p.in_base[f] + g.band_off[2] + (long long)row * g.pitch;
    int *out = a.carry + ((long long)(f * p.nchan + c) * a.maxh + row) * a.nstrips;
    const int W = (c == 0) ? kInvStrip : kInvStrip / 2, halo = (c == 0) ? 4 : 2;
    int total = 0;
    for (int s = 0; s < a.nstrips; s++) {
        const int c0 = max(s * W - halo, 0), c1 = min((s + 1) * W - halo, g.width);
        if (lane == 0) out[s] = total;
        if (c0 >= g.width) continue;
        total += (c == 0) ? row_segment_sum<4>(hl, c0, c1, lane) : row_segment_sum<2>(hl, c0, c1, lane);
    }
}

// inclusive prefix of the lane's NC raw HL values across the warp (lane order = column order) + carry-in
template <int NC>
__device__ __forceinline__ void integrate_row(int *h, int carry)
{
#pragma unroll
    for (int i = 1; i < NC; i++) h[i] += h[i - 1];
    int t = h[NC - 1];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int u = __shfl_up_sync(kFullMask, t, d);
        if ((int)threadIdx.x >= d) t += u;
    }
    const int excl = t - h[NC - 1] + carry;
#pragma unroll
    for (int i = 0; i < NC; i++) h[i] += excl;
}

template <int NC>
__device__ __forceinline__ void fields_channel(const InvGeom &g, const unsigned char *in, int r, unsigned colbyte, const InvLane &L,
                                               int carry, bool integrate, int *even, int *odd)
{
    RawCols<NC> a, b, c, d;
    const unsigned off = (unsigned)r * g.pitch + colbyte;
    load_raw<NC>(in, g.band_off[0], off, L.active, a);
    load_raw<NC>(in, g.band_off[1], off, L.active, b);
    load_raw<NC>(in, g.band_off[2], off, L.active, c);
    load_raw<NC>(in, g.band_off[3], off, L.active, d);
    int ll[NC], lh[NC], hl[NC], hh[NC];
    Expand<false, NC>::ll(a, ll);
    Expand<false, NC>::hp(b, g.dq[1], lh);
    Expand<false, NC>::ll(c, hl);               // raw: integrate first, dequantise after (ring arithmetic, same result)
    Expand<false, NC>::hp(d, g.dq[3], hh);
    if (integrate) integrate_row<NC>(hl, carry);     // warp-uniform: off when the host already integrated the band
#pragma unroll
    for (int i = 0; i < NC; i++) hl[i] = (int)(short)(hl[i] * g.dq[2]);     // int16 wrap as `line[x] += line[x-1]` on PIXEL
    int tl[2 * NC], th[2 * NC];
    hinv<NC>(ll, lh, L, tl);
    hinv<NC>(hl, hh, L, th);
#pragma unroll
    for (int i = 0; i < 2 * NC; i++) {
        const int lo = tl[i] >> 1, hi = th[i] >> 1;
        even[i] = (lo - hi) >> 1;
        odd[i] = (lo + hi) >> 1;
    }
}

template <bool PLANAR>
__global__ void __launch_bounds__(128) k_inv_fields(const __grid_constant__ InvParams p, const FieldsAux a)
{
    const int lane = threadIdx.x;
    const int f = blockIdx.z;
    const InvGeom &gy = p.ch[0];
    const InvGeom &gv = p.ch[1];
    const InvGeom &gu = p.ch[2];
    const int strip = blockIdx.x;
    if (strip * kInvStrip >= gy.width) return;
    const int H = gy.height;
    const InvLane L = inv_lane(strip, gy.width, lane, false);      // luma band columns
    const int col0 = L.col0;
    const unsigned ycol = (unsigned)(col0 * 2), ccol = (unsigned)col0;
    const unsigned char *in = p.in_base[f];
    unsigned char *out = p.out_base[f];
    const int y0 = (blockIdx.y * blockDim.y + threadIdx.y) * p.th;
    const int y1 = min(y0 + p.th, H);
    const int *cy = a.carry + ((long long)(f * 3 + 0) * a.maxh) * a.nstrips + strip;
    const int *cv = a.carry + ((long long)(f * 3 + 1) * a.maxh) * a.nstrips + strip;
    const int *cu = a.carry + ((long long)(f * 3 + 2) * a.maxh) * a.nstrips + strip;
    for (int r = y0; r < y1; r++) {
        int ye[8], yo[8], ue[4], uo[4], ve[4], vo[4];
        const bool integ = !a.hl_integrated;
        fields_channel<4>(gy, in, r, ycol, L, integ ? __ldg(cy + (long long)r * a.nstrips) : 0, integ, ye, yo);
        fields_channel<2>(gu, in, r, ccol, L, integ ? __ldg(cu + (long long)r * a.nstrips) : 0, integ, ue, uo);
        fields_channel<2>(gv, in, r, ccol, L, integ ? __ldg(cv + (long long)r * a.nstrips) : 0, integ, ve, vo);
        if (!L.writer) continue;
        if (PLANAR) {
#pragma unroll
            for (int rr = 0; rr < 2; rr++) {
                const int *yy = rr ? yo : ye, *uu = rr ? uo : ue, *vv = rr ? vo : ve;
                const long long row = 2 * r + rr;
                *reinterpret_cast<uint4 *>(out + gy.out_off + row * gy.out_pitch + (long long)col0 * 4) =
                    make_uint4(pack_sat16(yy[0], yy[1]), pack_sat16(yy[2], yy[3]), pack_sat16(yy[4], yy[5]), pack_sat16(yy[6], yy[7]));
                *reinterpret_cast<uint2 *>(out + gu.out_off + row * gu.out_pitch + (long long)col0 * 2) =
                    make_uint2(pack_sat16(uu[0], uu[1]), pack_sat16(uu[2], uu[3]));
                *reinterpret_cast<uint2 *>(out + gv.out_off + row * gv.out_pitch + (long long)col0 * 2) =
                    make_uint2(pack_sat16(vv[0], vv[1]), pack_sat16(vv[2], vv[3]));
            }
        } else {
            // the 8-bit reduction of emit_422 on rows that arrive fully shifted
            unsigned char *o = out + gy.out_off + (long long)(2 * r) * gy.out_pitch + (long long)col0 * 4;
#pragma unroll
            for (int rr = 0; rr < 2; rr++)
                *reinterpret_cast<uint4 *>(o + (rr ? gy.out_pitch : 0)) = pack_422_8(rr ? yo : ye, rr ? uo : ue, rr ? vo : ve, p.shift, rr, p.uyvy);
        }
    }
}

// ----------------------------------------------------------------------------
// Reduced-resolution decode: pack the lowpass images of the three 4:2:2 channels (Y, channel 1, channel 2).  One thread =
// 8 luma + 4 + 4 chroma coefficients; purely streaming.
// 8-bit YUYV / UYVY:
//   half    (LL1): Codec/frame.c:11742 ConvertLowpass16s10bitToYUV   out = sat_u8(ll >> 4)        (signed shift)
//   quarter (LL2): Codec/temporal.c:11362 CopyQuarterRowToBuffer     out = packus((uint16)ll >> 4) (unsigned shift)
//   Byte order Y0 U Y1 V with U = channel 2, V = channel 1 (the reference's "u"/"v" names are swapped, the bytes are these).
// YU64, half only (decoder.c:22883 CopyLowpass16sToBuffer -> Codec/frame.c:11146 ConvertLowpass16sToYUV64, its scalar loop;
// the MMX block is compiled out): out = min(max(ll, 0), 0xffff >> up_shift) << up_shift, up_shift = 16 - precision - 2
// (4095 << 4 at 10 bits), words Y0 C1 Y1 C2 with C1 = channel 1, C2 = channel 2 as the full-resolution YU64.
template <InvOut OUT>
__global__ void __launch_bounds__(256) k_lowpass_422(const __grid_constant__ InvParams p)
{
    static_assert(OUT == kInvOut8 || OUT == kInvOutYU64, "k_lowpass_422 writes 8-bit 4:2:2 or YU64");
    const int frame = blockIdx.z;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int x8 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    const InvGeom &gy = p.ch[0], &gv = p.ch[1], &gu = p.ch[2];
    if (y >= gy.height || x8 >= gy.width) return;
    const unsigned char *in = p.in_base[frame];
    const uint4 yr = *reinterpret_cast<const uint4 *>(in + gy.band_off[0] + (long long)y * gy.pitch + x8 * 2);
    const uint2 ur = *reinterpret_cast<const uint2 *>(in + gu.band_off[0] + (long long)y * gu.pitch + x8);
    const uint2 vr = *reinterpret_cast<const uint2 *>(in + gv.band_off[0] + (long long)y * gv.pitch + x8);
    const unsigned yw[4] = {yr.x, yr.y, yr.z, yr.w}, uw[2] = {ur.x, ur.y}, vw[2] = {vr.x, vr.y};
    unsigned char *out = p.out_base[frame] + (long long)y * gy.out_pitch + x8 * (OUT == kInvOutYU64 ? 4 : 2);
    const int rem = gy.width - x8;          // widths are even; a ragged tail stores whole pixel pairs
    if constexpr (OUT == kInvOutYU64) {
        const int us = p.up_shift, hi = 0xffff >> us;
        auto cv = [&](int v) { return (unsigned)min(max(v, 0), hi) << us; };
        unsigned o[8];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const unsigned c1 = (k & 1) ? vw[k >> 1] >> 16 : vw[k >> 1], c2 = (k & 1) ? uw[k >> 1] >> 16 : uw[k >> 1];
            o[2 * k] = cv(lo16(yw[k])) | (cv((short)c1) << 16);
            o[2 * k + 1] = cv(hi16(yw[k])) | (cv((short)c2) << 16);
        }
        if (rem >= 8) {
            *reinterpret_cast<uint4 *>(out) = make_uint4(o[0], o[1], o[2], o[3]);
            *reinterpret_cast<uint4 *>(out + 16) = make_uint4(o[4], o[5], o[6], o[7]);
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++)
                if (2 * k < rem) reinterpret_cast<uint2 *>(out)[k] = make_uint2(o[2 * k], o[2 * k + 1]);
        }
    } else {
        const int sh = p.shift;
        const bool uns = p.ll_unsigned != 0;
        auto lo = [&](unsigned w) { return uns ? (int)(w & 0xffffu) >> sh : lo16(w) >> sh; };
        auto hi = [&](unsigned w) { return uns ? (int)(w >> 16) >> sh : hi16(w) >> sh; };
        unsigned o[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int ya = lo(yw[k]), yb = hi(yw[k]);
            const int cu = (k & 1) ? hi(uw[k >> 1]) : lo(uw[k >> 1]);
            const int cv = (k & 1) ? hi(vw[k >> 1]) : lo(vw[k >> 1]);
            o[k] = p.uyvy ? pack_u8x4(cu, ya, cv, yb) : pack_u8x4(ya, cu, yb, cv);
        }
        if (rem >= 8) *reinterpret_cast<uint4 *>(out) = make_uint4(o[0], o[1], o[2], o[3]);
        else for (int k = 0; k < rem / 2; k++) reinterpret_cast<unsigned *>(out)[k] = o[k];
    }
}

// Quarter-resolution decode of an RGB 4:4:4 codec to the 10-bit RGB words (channels G, R, B; the alpha channel of an RGBA
// sample does not enter): decoder.c:17000 ConvertQuarterFrameToBuffer, descale 2 -> Codec/convert.c:16869
// ConvertUnpacked16sRowToRGB30, up_shift = 16 - precision - 2.  Its SSE2 loop covers the columns below width - width % 8:
// v = subs_epu16(adds_epi16(ll, 0x4000), 0x4000), out = (uint16)(v << up_shift) >> 6 -- a value below -0x4000 is not
// sent to 0 there, because the saturating add does not saturate it.  The scalar tail: min(max(ll, 0) << up_shift, 65535)
// >> 6.  Components packed at rgb10.pos / rgb10.byteswap as the full-resolution words.  One thread = 8 columns of each
// channel (three 128-bit loads, two 128-bit stores); purely streaming.
__device__ __forceinline__ unsigned rgb10_simd(int v, int us)
{
    const unsigned a = (unsigned)clamp16(v + 0x4000) & 0xffffu;
    return (((unsigned)max((int)a - 0x4000, 0) << us) & 0xffffu) >> 6;
}

__global__ void __launch_bounds__(256) k_lowpass_444(const __grid_constant__ InvParams p)
{
    const int frame = blockIdx.z;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int x8 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    const InvGeom &g0 = p.ch[0];
    if (y >= g0.height || x8 >= g0.width) return;
    const unsigned char *in = p.in_base[frame];
    int v[3][8];            // G, R, B
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const InvGeom &g = p.ch[c];
        const uint4 r = *reinterpret_cast<const uint4 *>(in + g.band_off[0] + (long long)y * g.pitch + x8 * 2);
        const unsigned w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int k = 0; k < 4; k++) { v[c][2 * k] = lo16(w[k]); v[c][2 * k + 1] = hi16(w[k]); }
    }
    const int us = p.up_shift;
    const int rem = g0.width - x8;
    const bool simd = rem >= 8;             // the reference's SSE2 loop runs over whole groups of 8 columns
    unsigned w[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        unsigned comp[3];
#pragma unroll
        for (int c = 0; c < 3; c++)
            comp[c] = simd ? rgb10_simd(v[c][i], us) : (unsigned)min(max(v[c][i], 0) << us, 65535) >> 6;
        // comp[] is G, R, B; rgb10.pos[] is R, G, B
        const unsigned word = (comp[1] << p.rgb10.pos[0]) | (comp[0] << p.rgb10.pos[1]) | (comp[2] << p.rgb10.pos[2]);
        w[i] = p.rgb10.byteswap ? __byte_perm(word, 0, 0x0123) : word;
    }
    unsigned char *out = p.out_base[frame] + (long long)y * g0.out_pitch + x8 * 4;
    if (simd) {
        *reinterpret_cast<uint4 *>(out) = make_uint4(w[0], w[1], w[2], w[3]);
        *reinterpret_cast<uint4 *>(out + 16) = make_uint4(w[4], w[5], w[6], w[7]);
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++)
            if (i < rem) reinterpret_cast<unsigned *>(out)[i] = w[i];
    }
}

#include "cfb_inverse_l32.inl"

// ----------------------------------------------------------------------------
static inline int ceil_div_i(int a, int b) { return (a + b - 1) / b; }

// (strips, row blocks of `warps` warps of th band rows each [+ 1 CTA row of border warps], frames)
static dim3 inv_grid(int width, int rows, int th, int warps, bool border_row, int frames)
{
    return dim3(ceil_div_i(width, kInvStrip), ceil_div_i(ceil_div_i(rows, th), warps) + (border_row ? 1 : 0), frames);
}

// every highpass divisor of channels [0, nchan) fits a byte: the SMALLDQ (dp2a) instantiations apply
static bool dq_small(const InvGeom *ch, int nchan)
{
    for (int c = 0; c < nchan; c++)
        for (int b = 1; b < 4; b++)
            if (ch[c].dq[b] < 0 || ch[c].dq[b] > 255) return false;
    return true;
}
static bool dq_small(const InvParams &p, int nchan) { return dq_small(p.ch, nchan); }

// f(std::true_type / std::false_type): a runtime bool as a template argument
template <class F>
static cudaError_t with_bool(bool b, F &&f) { return b ? f(std::true_type{}) : f(std::false_type{}); }

cudaError_t launch_inv_plane(cfb_context *ctx, InvParams &p, int descale)
{
    int maxw = 0, maxh = 0;
    for (int c = 0; c < p.nchan; c++) { maxw = max(maxw, p.ch[c].width); maxh = max(maxh, p.ch[c].height); }
    p.th = pick_th(ceil_div_i(maxw, kInvStrip), maxh, p.nframes * p.nchan, ctx->sm_count);
    const dim3 block(32, 4), grid = inv_grid(maxw, maxh, p.th, block.y, true, p.nframes * p.nchan);
    const cudaError_t e = with_bool(dq_small(p, p.nchan), [&](auto small) {
        constexpr bool S = decltype(small)::value;
        return launch_kernel(ctx, descale ? k_inv_plane<2, S> : k_inv_plane<0, S>, grid, block, 0, p);
    });
    if (e != cudaSuccess) return e;
    bool ragged = false;
    for (int c = 0; c < p.nchan; c++) ragged = ragged || (p.ch[c].width & 3);
    if (!ragged) return cudaSuccess;
    // the 1-3 band columns right of the last full lane (they include the right border)
    const dim3 eblock(128), egrid(ceil_div_i(maxh, 128), 3, p.nframes * p.nchan);
    return launch_kernel(ctx, descale ? k_inv_plane_edge<2> : k_inv_plane_edge<0>, egrid, eblock, 0, p);
}

// Levels 3 and 2 in one pass (k_inv_l32 + k_inv_l32_border).  The caller checks what the kernels assume: level 2 is
// prescaled, every level-2 band is a multiple of 4 wide and exactly twice as wide and high as its level-3 band, and level
// 3 has at least 3 rows.  p.th counts level-2 rows.
cudaError_t launch_inv_l32(cfb_context *ctx, InvL32Params &p, int descale3)
{
    int maxw = 0, maxh = 0;
    for (int c = 0; c < p.nchan; c++) { maxw = max(maxw, p.l2[c].width); maxh = max(maxh, p.l2[c].height); }
    // At most 6 level-2 rows per warp.  On an H100 SXM (700 W power limit, 16 4K 4:2:2 frames) both launches took 144.5 /
    // 130.3 / 125.0 / 116.7 / 118.3 / 120.6 / 123.0 us at th = 2 / 3 / 4 / 6 / 8 / 12 / 16.
    p.th = pick_th(ceil_div_i(maxw, kInvStrip), maxh, p.nframes * p.nchan, ctx->sm_count, 6);
    const dim3 block(32, 4), grid = inv_grid(maxw, maxh, p.th, block.y, false, p.nframes * p.nchan);
    const cudaError_t e = with_bool(dq_small(p.l3, p.nchan), [&](auto small3) {
        return with_bool(dq_small(p.l2, p.nchan), [&](auto small2) {
            constexpr bool S3 = decltype(small3)::value, S2 = decltype(small2)::value;
            return launch_kernel(ctx, descale3 ? k_inv_l32<2, 2, S3, S2> : k_inv_l32<0, 2, S3, S2>, grid, block, 0, p);
        });
    });
    if (e != cudaSuccess) return e;
    return launch_kernel(ctx, descale3 ? k_inv_l32_border<2, 2> : k_inv_l32_border<0, 2>, dim3(grid.x, 1, grid.z), dim3(32, 2), 0, p);
}

// The final 4:2:2 level.  Its band rows are streamed through a TMA ring of kInvRows band rows per stage and kInvStages
// stages per warp: on an H100 SXM (700 W power limit, 16 4K frames per launch, three alternating rounds) it took 307 us,
// against 318 us for a register-fed kernel of the same arithmetic.  The ring's boxes need 16-byte aligned band starts and
// pitches, whole 32-bit elements per band row, and LH / HL / HH of a channel equally spaced.  cfb_layout_compute and
// cfb_gop2_layout_compute lay out every pyramid this way, so any other layout is rejected rather than decoded.
// The ring needs more than the default 48 KB of shared memory: every instantiation is opted in, on each device that runs it.
cudaError_t inv_opt_in_smem()
{
    for (const void *k : {(const void *)k_inv_422_tma<false, kInvOut8>, (const void *)k_inv_422_tma<true, kInvOut8>,
                          (const void *)k_inv_422_tma<false, kInvOutYU64>, (const void *)k_inv_422_tma<true, kInvOutYU64>,
                          (const void *)k_inv_422_tma<false, kInvOutV210>, (const void *)k_inv_422_tma<true, kInvOutV210>}) {
        const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kInvRingSmem);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_inv_422(cfb_context *ctx, InvParams &p, InvOut out)
{
    if (out != kInvOut8 && out != kInvOutYU64 && out != kInvOutV210) return cudaErrorInvalidValue;
    for (int c = 0; c < 3; c++) {
        const InvGeom &g = p.ch[c];
        const long long d1 = g.band_off[2] - g.band_off[1], d2 = g.band_off[3] - g.band_off[2];
        if ((g.width & 1) || (g.pitch & 15) || d1 != d2 || d1 <= 0 || (d1 & 15) || (g.band_off[0] & 15) || (g.band_off[1] & 15))
            return cudaErrorInvalidValue;
    }
    for (int i = 0; i < p.nframes; i++)
        if ((uintptr_t)p.in_base[i] & 15) return cudaErrorInvalidValue;
    InvTmaMaps tm;
    for (int i = 0; i < p.nframes; i++)
        for (int c = 0; c < 3; c++) {
            const InvGeom &g = p.ch[c];
            const uint32_t box = (c == 0) ? kInvBoxY : kInvBoxC;
            cudaError_t e = tmap_encode_2d(&tm.m[i][2 * c], p.in_base[i] + g.band_off[0], (uint64_t)g.width * 2, (uint64_t)g.height,
                                           (uint64_t)g.pitch, box, kInvRows);
            if (e == cudaSuccess)
                e = tmap_encode_3d(&tm.m[i][2 * c + 1], p.in_base[i] + g.band_off[1], (uint64_t)g.width * 2, (uint64_t)g.height,
                                   (uint64_t)g.pitch, 3, (uint64_t)(g.band_off[2] - g.band_off[1]), box, kInvRows, 3);
            if (e != cudaSuccess) return e;
        }
    p.th = pick_th(ceil_div_i(p.ch[0].width, kInvStrip), p.ch[0].height, p.nframes, ctx->sm_count);
    const dim3 block(32, 4), grid = inv_grid(p.ch[0].width, p.ch[0].height, p.th, block.y, true, p.nframes);
    return with_bool(dq_small(p, 3), [&](auto small) {
        constexpr bool S = decltype(small)::value;
        return launch_kernel(ctx, out == kInvOutV210 ? k_inv_422_tma<S, kInvOutV210> : out == kInvOutYU64 ? k_inv_422_tma<S, kInvOutYU64>
                                                                                                         : k_inv_422_tma<S, kInvOut8>,
                             grid, block, kInvRingSmem, p, tm);
    });
}

template <InvOut OUT>
static cudaError_t launch_inv_444_out(cfb_context *ctx, InvParams &p)
{
    p.th = pick_th(ceil_div_i(p.ch[0].width, kInvStrip), p.ch[0].height, p.nframes, ctx->sm_count);
    const dim3 block(32, 4), grid = inv_grid(p.ch[0].width, p.ch[0].height, p.th, block.y, true, p.nframes);
    return with_bool(dq_small(p, (OUT == kInvOutB64AAlpha || OUT == kInvOutBYR4) ? 4 : 3), [&](auto small) {
        return launch_kernel(ctx, k_inv_444<decltype(small)::value, OUT>, grid, block, 0, p);
    });
}

// B64A with alpha keeps a fourth channel's vertical state in the warp: 246 / 244 registers (SMALLDQ false / true, no
// spills) against 168, so 2 CTAs of 4 warps fit an SM instead of 3.  On an H100 80GB HBM3 (700 W power limit, 16 4K frames
// per launch, three alternating rounds) it took 825.1 - 826.0 us (8 bytes of bands in + 8 out per pixel: 2571 - 2573 GB/s),
// against 821.3 - 823.0 us for a separate kernel with its own copy of the window, step and border row.
// BYR4 (the mosaic of a Bayer codec) is the same kernel with four channels and emit_bayer: 254 / 252 registers, no spills,
// 2 CTAs per SM.  On an H100 80GB HBM3 (700 W power limit, 4 mosaics of 8192 x 4320 per launch = 566.2 MB of bands in + frame
// out, three alternating rounds, tools/byr4_out_ab.py): 237 - 238 us with the `& 0xfffe` rule (2378 - 2387 GB/s), 268 - 270 us
// through the restore table on smooth mosaics and 277 - 279 us on random ones (2032 - 2115 GB/s), against 229 - 230 us for
// the PLANAR16 output of the same codec (k_inv_plane, the same bytes).  A shared-memory copy of the table was not built.
cudaError_t launch_inv_444(cfb_context *ctx, InvParams &p, InvOut out)
{
    switch (out) {
    case kInvOutRG48: return launch_inv_444_out<kInvOutRG48>(ctx, p);
    case kInvOutB64A: return launch_inv_444_out<kInvOutB64A>(ctx, p);
    case kInvOutB64AAlpha: return launch_inv_444_out<kInvOutB64AAlpha>(ctx, p);
    case kInvOutRGB10: return launch_inv_444_out<kInvOutRGB10>(ctx, p);
    case kInvOutBYR4: return launch_inv_444_out<kInvOutBYR4>(ctx, p);
    default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_inv_fields(cfb_context *ctx, InvParams &p, const FieldsAux &a, bool planar)
{
    const dim3 block(32, 4);
    p.th = pick_th(ceil_div_i(p.ch[0].width, kInvStrip), p.ch[0].height, p.nframes, ctx->sm_count);
    if (!a.hl_integrated) {
        const cudaError_t e = launch_kernel(ctx, k_fields_carry, dim3(ceil_div_i(p.ch[0].height, (int)block.y), 3, p.nframes), block, 0, p, a);
        if (e != cudaSuccess) return e;
    }
    const dim3 grid = inv_grid(p.ch[0].width, p.ch[0].height, p.th, block.y, false, p.nframes);
    return launch_kernel(ctx, planar ? k_inv_fields<true> : k_inv_fields<false>, grid, block, 0, p, a);
}

// Reduced-resolution output: one launch of k_lowpass_422 (8-bit 4:2:2, YU64) or k_lowpass_444 (10-bit RGB)
cudaError_t launch_lowpass(cfb_context *ctx, const InvParams &p, InvOut out)
{
    dim3 block(32, 8);
    dim3 grid(ceil_div_i(ceil_div_i(p.ch[0].width, 8), 32), ceil_div_i(p.ch[0].height, 8), p.nframes);
    switch (out) {
    case kInvOut8: return launch_kernel(ctx, k_lowpass_422<kInvOut8>, grid, block, 0, p);
    case kInvOutYU64: return launch_kernel(ctx, k_lowpass_422<kInvOutYU64>, grid, block, 0, p);
    case kInvOutRGB10: return launch_kernel(ctx, k_lowpass_444, grid, block, 0, p);
    default: return cudaErrorInvalidValue;
    }
}

}  // namespace cfb
