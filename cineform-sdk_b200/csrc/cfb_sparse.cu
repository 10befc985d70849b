// cfb_sparse.cu -- lossless sparse transfer format for the coded region (SURVEY 8f rank 1), version 2 ('CFS2').
//
// After quantisation ~90 % of the highpass coefficients are zero and ~99 % of the rest fit a byte, and the dense int16
// bands (33 MB per 4K 4:2:2 frame) are what limits the host<->device path (PCIe), not the kernels.  The host entropy
// coder only ever needs (zero run, value) sequences (Codec/encoder.c:5386-5700 EncodeQuantLongRuns walks the band
// counting zeros, incl. the pitch gap :5653), so the wire format keeps exactly that information, in blocks that both
// the GPU and the host can address independently:
//
//   header   32 B : u32 'CFS2', u32 nwords, u32 total_bytes, u32 nblocks, 4 x u32 0
//   table    nblocks x 16 B : { u32 chunk offset (bytes from the buffer start), u32 groups, u32 values, u32 escapes }
//   chunks   one per block of 8192 int16 words of the flat coded region [0, coded_bytes) (pitch padding included, it
//            is zero), 16-byte aligned, EMPTY (0 bytes) when the whole block is zero:
//              l1     32 B  : bit g set <=> group g (32 consecutive words) of the block holds a non-zero word
//              masks  4 B per non-empty group, in order: bit i <=> word i of the group is non-zero
//              bytes  1 B per non-zero word, in raster order: the value if -127 <= v <= 127, else -128 (escape)
//              wide   2 B per escape, in order: the int16 value            (each array padded with zeros to 4 B)
//
// A 4K 4:2:2 frame at FILMSCAN1 (1.5 M non-zero words) is 2.3 MB instead of 33.2 MB dense (round 1's flat bitmap +
// int16 values: 5.1 MB).  Packing is ONE kernel that reads the dense region once: every CTA builds its chunk in shared
// memory, publishes the chunk size, obtains its byte offset by decoupled look-back over the preceding CTAs of the frame
// and copies the chunk out with 16-byte stores.  Unpacking is one kernel as well: the table gives every CTA its chunk.
// The host helpers cfb_sparse_expand / cfb_sparse_compact are pure format conversions (cfb_sparse_compact produces
// byte for byte what the GPU produces); cfb_vlc.cu walks the chunks to emit the run-length / VLC stream directly.
#include "cfb_host.h"
#include "cfb_sparse_format.h"

namespace cfb {

struct SparseParams {
    int nframes;
    unsigned nwords;                // int16 words in the coded region (a multiple of 32)
    unsigned nblocks;
    unsigned chunks_off;            // byte offset of the first chunk
    const unsigned char *dense[kMaxBatch];      // pyramids (coded region at offset 0)
    unsigned char *sparse[kMaxBatch];
    unsigned long long *status[kMaxBatch];      // look-back state: nblocks entries + 1 ticket counter per frame
};

__device__ __forceinline__ unsigned nonzero_mask8(const uint4 &w) {
    unsigned m = 0;
    m |= (w.x & 0xffffu) ? 1u : 0u;   m |= (w.x >> 16) ? 2u : 0u;
    m |= (w.y & 0xffffu) ? 4u : 0u;   m |= (w.y >> 16) ? 8u : 0u;
    m |= (w.z & 0xffffu) ? 16u : 0u;  m |= (w.z >> 16) ? 32u : 0u;
    m |= (w.w & 0xffffu) ? 64u : 0u;  m |= (w.w >> 16) ? 128u : 0u;
    return m;
}

__device__ __forceinline__ unsigned warp_incl_scan(unsigned v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
    return v;
}

// exclusive offset of this warp inside its CTA + the CTA total (all 32 warps call it; one barrier)
__device__ __forceinline__ unsigned block_exclusive(unsigned warp_total, int lane, int wid, unsigned *smem32, unsigned *cta_total) {
    if (lane == 0) smem32[wid] = warp_total;
    __syncthreads();
    const unsigned mine = smem32[lane];
    const unsigned incl = warp_incl_scan(mine, lane);
    if (cta_total) *cta_total = __shfl_sync(0xffffffffu, incl, 31);
    return __shfl_sync(0xffffffffu, incl - mine, wid);
}

constexpr unsigned long long kFlagAggregate = 1ull << 62, kFlagPrefix = 2ull << 62, kFlagMask = 3ull << 62;
constexpr int kSpThreads = 256, kSpWarps = kSpThreads / 32, kSpPieces = kSparseBlockWords / (8 * kSpThreads);     // 4 pieces of 8 words per thread

// ---------------------------------------------------------------------------------------------------------------
// dense -> sparse, one pass.  CTA = 256 threads = one block of 8192 words; thread t owns words 8 (256 j + t) ... + 7 for
// j = 0..3, so every load is a coalesced 16-byte access, all four are in flight together, and four consecutive lanes
// hold one 32-word group of piece j.  A 1024-thread CTA with one piece per thread (the first version) capped the SM at
// two resident CTAs = 32 KB in flight; eight resident CTAs of this shape keep 128 KB in flight.
// Blocks take their index from a per-frame ticket, so a CTA only ever waits for CTAs that already run.
__global__ void __launch_bounds__(kSpThreads, 4) k_sparse_pack(const __grid_constant__ SparseParams p)
{
    __shared__ __align__(16) unsigned char chunk[kSparseMaxChunk];
    __shared__ unsigned s_cnt[kSpPieces][kSpWarps], s_grp[kSpPieces][kSpWarps], s_ticket, s_base;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int f = blockIdx.y;
    unsigned long long *status = p.status[f];
    if (tid == 0) s_ticket = (unsigned)atomicAdd(&status[p.nblocks], 1ull);
    __syncthreads();
    const unsigned blk = s_ticket;
    const unsigned char *src = p.dense[f] + ((size_t)blk * kSparseBlockWords + (size_t)tid * 8) * 2;
    const unsigned wfirst = blk * kSparseBlockWords + tid * 8;
    // ---- phase 1: counts only (the words are read again in phase 2, from L2 / L1: keeping them would cost 16 registers
    //      and halve the resident CTAs) ----
    unsigned packed[kSpPieces], incl[kSpPieces], gb[kSpPieces];
    {
        uint4 w[kSpPieces];
#pragma unroll
        for (int j = 0; j < kSpPieces; j++)
            w[j] = (wfirst + j * kSpThreads * 8 < p.nwords) ? __ldg(reinterpret_cast<const uint4 *>(src + (size_t)j * kSpThreads * 16)) : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int j = 0; j < kSpPieces; j++) {
            // most 256-word warp pieces of a quantised frame are all zero: one OR + one ballot settles those
            const unsigned any = __ballot_sync(0xffffffffu, (w[j].x | w[j].y | w[j].z | w[j].w) != 0);
            packed[j] = 0; incl[j] = 0; gb[j] = 0;
            if (any) {
                const unsigned m8 = nonzero_mask8(w[j]);
                const unsigned ws[4] = {w[j].x, w[j].y, w[j].z, w[j].w};
                unsigned nesc = 0;
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const int v = (k & 1) ? ((int)ws[k >> 1] >> 16) : (int)(short)(ws[k >> 1] & 0xffffu);
                    nesc += ((unsigned)(v + 127) > 254u) ? 1u : 0u;
                }
                packed[j] = __popc(m8) | (nesc << 16);      // values | escapes in one scan (<= 256 each per warp)
                incl[j] = warp_incl_scan(packed[j], lane);
                // bit 4g of gb <=> group g of this (piece, warp) is non-empty: OR of its four lanes, kept at the leader's position
                gb[j] = (any | (any >> 1) | (any >> 2) | (any >> 3)) & 0x11111111u;
            }
            if (lane == 31) s_cnt[j][wid] = incl[j];
            if (lane == 0) s_grp[j][wid] = __popc(gb[j]);
        }
    }
    __syncthreads();
    // raster order = piece-major: offsets of (piece j, warp wid) and the block totals
    unsigned vbase[kSpPieces], gbase[kSpPieces], tot = 0, gtot = 0;
#pragma unroll
    for (int j = 0; j < kSpPieces; j++) {
#pragma unroll
        for (int q = 0; q < kSpWarps; q++) {
            if (q == wid) { vbase[j] = tot; gbase[j] = gtot; }
            tot += s_cnt[j][q]; gtot += s_grp[j][q];
        }
    }
    const unsigned V = tot & 0xffffu, E = tot >> 16, G = gtot;
    const unsigned bytes = sparse_chunk_bytes(G, V, E);
    // ---- publish the chunk size, look back for the offset (warp 0), meanwhile everyone fills the chunk ----
    if (wid == 0) {
        const unsigned units = bytes >> 4;
        unsigned excl = 0;
        if (blk == 0) {
            if (lane == 0) atomicExch(&status[0], kFlagPrefix | units);
        } else {
            if (lane == 0) atomicExch(&status[blk], kFlagAggregate | units);
            int look = (int)blk - 1;
            while (true) {
                const int idx = look - lane;
                unsigned long long st = kFlagPrefix;        // before block 0: an empty prefix
                if (idx >= 0) {
                    const volatile unsigned long long *sp = status + idx;
                    do { st = *sp; } while ((st & kFlagMask) == 0);
                }
                const unsigned pm = __ballot_sync(0xffffffffu, (st & kFlagMask) == kFlagPrefix);
                const int first = pm ? (__ffs(pm) - 1) : 31;
                unsigned c = (lane <= first) ? (unsigned)(st & 0xffffffffull) : 0u;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
                excl += c;
                if (pm) break;
                look -= 32;
            }
            if (lane == 0) atomicExch(&status[blk], kFlagPrefix | (unsigned long long)(excl + units));
        }
        if (lane == 0) {
            s_base = excl;
            const unsigned off = p.chunks_off + (excl << 4);
            reinterpret_cast<uint4 *>(p.sparse[f] + kSparseHeaderBytes)[blk] = make_uint4(off, G, V, E);
            if (blk == p.nblocks - 1) {
                uint4 *h = reinterpret_cast<uint4 *>(p.sparse[f]);
                h[0] = make_uint4(kSparseMagic, p.nwords, off + bytes, p.nblocks);
                h[1] = make_uint4(0, 0, 0, 0);
            }
        }
    }
    // ---- phase 2: fill the chunk ----
    if (G) {
        const unsigned masks_off = kSparseL1Bytes, bytes_off = masks_off + 4 * G, wide_off = bytes_off + ((V + 3) & ~3u);
#pragma unroll
        for (int j = 0; j < kSpPieces; j++) {
            if (lane == 0) {            // l1: the 8 groups of (piece j, warp wid) are groups 64 j + 8 wid ... + 7 of the block = one byte
                unsigned b = 0;
#pragma unroll
                for (int k = 0; k < 8; k++) b |= ((gb[j] >> (4 * k)) & 1u) << k;
                chunk[j * kSpWarps + wid] = (unsigned char)b;
            }
            if (!gb[j]) continue;       // nothing in this warp's 256 words (warp-uniform)
            const uint4 w = (wfirst + j * kSpThreads * 8 < p.nwords) ? __ldg(reinterpret_cast<const uint4 *>(src + (size_t)j * kSpThreads * 16)) : make_uint4(0, 0, 0, 0);
            const unsigned m8 = nonzero_mask8(w);
            unsigned mm = m8 << ((lane & 3) * 8);
            mm |= __shfl_xor_sync(0xffffffffu, mm, 1);
            mm |= __shfl_xor_sync(0xffffffffu, mm, 2);      // all four lanes of a group hold its 32-bit mask
            if (((lane & 3) == 0) && mm)
                *reinterpret_cast<unsigned *>(chunk + masks_off + 4 * (gbase[j] + __popc(gb[j] & ((1u << lane) - 1u)))) = mm;
            unsigned vpos = bytes_off + (vbase[j] & 0xffffu) + ((incl[j] - packed[j]) & 0xffffu);
            unsigned epos = wide_off + 2 * ((vbase[j] >> 16) + ((incl[j] - packed[j]) >> 16));
            const unsigned ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int k = 0; k < 8; k++) {
                if (m8 & (1u << k)) {
                    const int v = (k & 1) ? ((int)ws[k >> 1] >> 16) : (int)(short)(ws[k >> 1] & 0xffffu);
                    const bool esc = (v < -127 || v > 127);
                    chunk[vpos++] = (unsigned char)(esc ? 0x80 : (v & 0xff));
                    if (esc) { *reinterpret_cast<short *>(chunk + epos) = (short)v; epos += 2; }
                }
            }
        }
        // zero padding: bytes [V, align4(V)), wide [2E, align4(2E)) and the tail up to the 16-byte boundary
        if (tid < 3 && bytes_off + V + tid < wide_off) chunk[bytes_off + V + tid] = 0;
        if (tid >= 32 && tid < 48) { const unsigned q = wide_off + 2 * E + (tid - 32); if (q < bytes) chunk[q] = 0; }
    }
    __syncthreads();
    if (G) {
        unsigned char *dst = p.sparse[f] + p.chunks_off + ((size_t)s_base << 4);
        for (unsigned i = tid * 16; i < bytes; i += kSpThreads * 16)
            *reinterpret_cast<uint4 *>(dst + i) = *reinterpret_cast<const uint4 *>(chunk + i);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// sparse -> dense: one CTA per block (same thread-to-word mapping as the packer), the table entry gives the chunk
__global__ void __launch_bounds__(kSpThreads, 4) k_sparse_unpack(const __grid_constant__ SparseParams p)
{
    __shared__ __align__(16) unsigned char chunk[kSparseMaxChunk];
    __shared__ unsigned s_cnt[kSpPieces][kSpWarps];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int f = blockIdx.y;
    const unsigned blk = blockIdx.x;
    const uint4 ent = __ldg(reinterpret_cast<const uint4 *>(p.sparse[f] + kSparseHeaderBytes) + blk);
    const unsigned G = min(ent.y, (unsigned)kSparseBlockGroups), V = min(ent.z, (unsigned)kSparseBlockWords), E = min(ent.w, V);
    unsigned char *out = const_cast<unsigned char *>(p.dense[f]) + ((size_t)blk * kSparseBlockWords + (size_t)tid * 8) * 2;
    const unsigned wfirst = blk * kSparseBlockWords + tid * 8;
    if (G == 0) {
#pragma unroll
        for (int j = 0; j < kSpPieces; j++)
            if (wfirst + j * kSpThreads * 8 < p.nwords) *reinterpret_cast<uint4 *>(out + (size_t)j * kSpThreads * 16) = make_uint4(0, 0, 0, 0);
        return;
    }
    const unsigned bytes = sparse_chunk_bytes(G, V, E);
    const unsigned char *src = p.sparse[f] + ent.x;
    for (unsigned i = tid * 16; i < bytes; i += kSpThreads * 16)
        *reinterpret_cast<uint4 *>(chunk + i) = __ldg(reinterpret_cast<const uint4 *>(src + i));
    __syncthreads();
    const unsigned masks_off = kSparseL1Bytes, bytes_off = masks_off + 4 * G, wide_off = bytes_off + ((V + 3) & ~3u);
    // group rank: l1 byte (j * 8 + w) belongs to (piece j, warp w); every warp scans the 32 bytes itself
    const unsigned pc = __popc((unsigned)chunk[lane]);
    const unsigned gincl = warp_incl_scan(pc, lane);
    unsigned m8all = 0, vexcl[kSpPieces];
#pragma unroll
    for (int j = 0; j < kSpPieces; j++) {
        const unsigned gbase = __shfl_sync(0xffffffffu, gincl - pc, j * kSpWarps + wid);
        const unsigned l1b = chunk[j * kSpWarps + wid];
        const int gi = lane >> 2;
        unsigned m = 0;
        if ((l1b >> gi) & 1u) {
            const unsigned grank = min(gbase + __popc(l1b & ((1u << gi) - 1u)), G - 1);
            m = *reinterpret_cast<const unsigned *>(chunk + masks_off + 4 * grank);
        }
        const unsigned m8 = (m >> ((lane & 3) * 8)) & 0xffu;
        m8all |= m8 << (8 * j);
        const unsigned nval = __popc(m8);
        const unsigned incl = warp_incl_scan(nval, lane);
        if (lane == 31) s_cnt[j][wid] = incl;
        vexcl[j] = incl - nval;                             // exclusive inside the warp
    }
    __syncthreads();
    // value positions; escapes among this thread's values (the bytes are read again below: keeping them would cost 32 registers)
    unsigned vpos[kSpPieces], nesc[kSpPieces], eexcl[kSpPieces];
    {
        unsigned tot = 0;
#pragma unroll
        for (int j = 0; j < kSpPieces; j++) {
            unsigned vbase = 0;
#pragma unroll
            for (int q = 0; q < kSpWarps; q++) { if (q == wid) vbase = tot; tot += s_cnt[j][q]; }
            vpos[j] = vbase + vexcl[j];
            unsigned e = 0;
            if (E && chunk[j * kSpWarps + wid]) {           // warp-uniform: blocks without escapes / empty warp pieces skip the byte scan
                const unsigned n = __popc((m8all >> (8 * j)) & 0xffu);
                for (unsigned k = 0; k < n; k++) e += ((signed char)chunk[bytes_off + min(vpos[j] + k, V - 1)] == -128) ? 1u : 0u;
            }
            nesc[j] = e;
        }
    }
    __syncthreads();                    // s_cnt is reused for the escape counts
#pragma unroll
    for (int j = 0; j < kSpPieces; j++) {
        const unsigned incl = warp_incl_scan(nesc[j], lane);
        if (lane == 31) s_cnt[j][wid] = incl;
        eexcl[j] = incl - nesc[j];
    }
    __syncthreads();
    {
        unsigned tot = 0;
#pragma unroll
        for (int j = 0; j < kSpPieces; j++) {
            unsigned ebase = 0;
#pragma unroll
            for (int q = 0; q < kSpWarps; q++) { if (q == wid) ebase = tot; tot += s_cnt[j][q]; }
            unsigned epos = ebase + eexcl[j], vp = vpos[j];
            const unsigned m8 = (m8all >> (8 * j)) & 0xffu;
            if (!chunk[j * kSpWarps + wid]) {               // warp-uniform: the whole 256-word piece is zero
                if (wfirst + j * kSpThreads * 8 < p.nwords) *reinterpret_cast<uint4 *>(out + (size_t)j * kSpThreads * 16) = make_uint4(0, 0, 0, 0);
                continue;
            }
            int vals[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                vals[k] = 0;
                if (m8 & (1u << k)) {
                    int v = (int)(signed char)chunk[bytes_off + min(vp, V - 1)];
                    vp++;
                    if (v == -128) { v = *reinterpret_cast<const short *>(chunk + wide_off + 2 * min(epos, E ? E - 1 : 0)); epos++; }
                    vals[k] = v;
                }
            }
            if (wfirst + j * kSpThreads * 8 < p.nwords)
                *reinterpret_cast<uint4 *>(out + (size_t)j * kSpThreads * 16) = make_uint4(pack_lo(vals[0], vals[1]), pack_lo(vals[2], vals[3]),
                                                                                      pack_lo(vals[4], vals[5]), pack_lo(vals[6], vals[7]));
        }
    }
}

cudaError_t launch_sparse_compact(cfb_context *ctx, const SparseParams &p)
{
    for (int i = 0; i < p.nframes; i++) {
        cudaError_t e = cudaMemsetAsync(p.status[i], 0, sizeof(unsigned long long) * (p.nblocks + 1), ctx->stream);
        if (e != cudaSuccess) return e;
    }
    return launch_kernel(ctx, k_sparse_pack, dim3(p.nblocks, p.nframes), dim3(kSpThreads), 0, p);
}

cudaError_t launch_sparse_expand(cfb_context *ctx, const SparseParams &p)
{
    return launch_kernel(ctx, k_sparse_unpack, dim3(p.nblocks, p.nframes), dim3(kSpThreads), 0, p);
}

}  // namespace cfb

// ---------------------------------------------------------------------------
// C ABI
using namespace cfb;

static cfb_error sparse_prepare(cfb_codec *cd, SparseParams &p, int n)
{
    const cfb_layout &L = cd->layout;
    p.nframes = n;
    p.nwords = (unsigned)(L.coded_bytes / 2);
    p.nblocks = sparse_nblocks(p.nwords);
    p.chunks_off = sparse_chunks_off(p.nblocks);
    // each staging buffer under its own check: a failed allocation leaves the others usable for the retry
    cd->sparse_stride = (cfb_sparse_max_bytes(&L) + 255) & ~(size_t)255;
    if (!cd->d_sparse) CFB_CUDA(cudaMalloc((void **)&cd->d_sparse, cd->sparse_stride * cd->max_batch));
    if (!cd->d_status) CFB_CUDA(cudaMalloc((void **)&cd->d_status, sizeof(unsigned long long) * (size_t)(p.nblocks + 1) * cd->max_batch));
    if (!cd->h_headers) CFB_CUDA(cudaHostAlloc((void **)&cd->h_headers, 16 * (size_t)cd->max_batch, cudaHostAllocPortable));
    for (int i = 0; i < n; i++) {
        p.dense[i] = cd->d_pyramids + cd->pyramid_stride * i;
        p.sparse[i] = cd->d_sparse + cd->sparse_stride * i;
        p.status[i] = cd->d_status + (size_t)(p.nblocks + 1) * i;
    }
    return CFB_OK;
}

// what the fixed part (header + table) of a sparse buffer says about its size; 0 = not a sparse buffer of this layout
static size_t sparse_checked_bytes(const void *sparse, unsigned nwords)
{
    const unsigned *h = (const unsigned *)sparse;
    const unsigned nblocks = sparse_nblocks(nwords);
    const size_t lo = sparse_chunks_off(nblocks), hi = lo + (size_t)nblocks * kSparseMaxChunk;
    if (h[0] != kSparseMagic || h[1] != nwords || h[3] != nblocks || h[2] < lo || h[2] > hi || (h[2] & 15)) return 0;
    return h[2];
}

namespace cfb {

// sizes are in BYTES of the whole sparse buffer
unsigned sparse_initial_guess(const cfb_codec *cd)
{
    const unsigned nwords = (unsigned)(cd->layout.coded_bytes / 2);
    return sparse_chunks_off(sparse_nblocks(nwords)) + nwords / 4;         // 1/8 of the words non-zero
}

unsigned sparse_next_guess(const cfb_codec *cd, unsigned max_bytes)
{
    const size_t cap = cfb_sparse_max_bytes(&cd->layout);
    size_t g = ((size_t)max_bytes + max_bytes / 8 + 65536 + 255u) & ~(size_t)255;
    if (g > cap) g = cap;               // clamp AFTER the rounding: the copy must stay inside cfb_sparse_max_bytes
    return (unsigned)g;
}

cfb_error sparse_compact_device(cfb_codec *cd, int n)
{
    SparseParams sp;
    cfb_error err = sparse_prepare(cd, sp, n);
    if (err) return err;
    CFB_CUDA(launch_sparse_compact(cd->ctx, sp));
    return CFB_OK;
}

cfb_error sparse_expand_device(cfb_codec *cd, int n)
{
    SparseParams sp;
    cfb_error err = sparse_prepare(cd, sp, n);
    if (err) return err;
    CFB_CUDA(launch_sparse_expand(cd->ctx, sp));
    return CFB_OK;
}

cfb_error sparse_download(cfb_codec *cd, int n, void *const *h_sparse, unsigned guess, cudaStream_t s)
{
    SparseParams sp;
    cfb_error err = sparse_prepare(cd, sp, n);
    if (err) return err;
    const size_t cap = cfb_sparse_max_bytes(&cd->layout);
    size_t bytes = guess;
    if (bytes > cap) bytes = cap;       // never more than the caller's buffer holds (cfb_sparse_max_bytes)
    if (bytes < sp.chunks_off) bytes = sp.chunks_off;
    for (int i = 0; i < n; i++) {
        if (!h_sparse[i]) { set_error("null host buffer %d", i); return CFB_ERROR_INVALID_ARGUMENT; }
        CFB_CUDA(cudaMemcpyAsync(h_sparse[i], sp.sparse[i], bytes, cudaMemcpyDeviceToHost, s));
        cd->ctx->d2h_bytes += (uint64_t)bytes;
    }
    return CFB_OK;
}

cfb_error stage_fwd_tail(cfb_codec *cd, int n, void *const *h_sparse, unsigned guess, cudaStream_t s, size_t *sizes,
                         unsigned *max_bytes, bool *more)
{
    SparseParams sp;
    cfb_error err = sparse_prepare(cd, sp, n);
    if (err) return err;
    const size_t cap = cfb_sparse_max_bytes(&cd->layout);
    size_t have = guess;
    if (have > cap) have = cap;
    if (have < sp.chunks_off) have = sp.chunks_off;
    unsigned maxb = 0;
    *more = false;
    for (int i = 0; i < n; i++) {
        const size_t total = sparse_checked_bytes(h_sparse[i], sp.nwords);
        if (!total) { set_error("sparse header %d corrupt", i); return CFB_ERROR_UNEXPECTED; }
        if (total > maxb) maxb = (unsigned)total;
        if (total > have) {
            CFB_CUDA(cudaMemcpyAsync((unsigned char *)h_sparse[i] + have, sp.sparse[i] + have, total - have, cudaMemcpyDeviceToHost, s));
            cd->ctx->d2h_bytes += (uint64_t)(total - have);
            *more = true;
        }
        if (sizes) sizes[i] = total;
    }
    if (max_bytes) *max_bytes = maxb;
    return CFB_OK;
}

cfb_error sparse_upload(cfb_codec *cd, int n, const void *const *h_sparse, cudaStream_t s)
{
    SparseParams sp;
    cfb_error err = sparse_prepare(cd, sp, n);
    if (err) return err;
    for (int i = 0; i < n; i++) {
        if (!h_sparse[i]) { set_error("null host buffer %d", i); return CFB_ERROR_INVALID_ARGUMENT; }
        const size_t bytes = sparse_checked_bytes(h_sparse[i], sp.nwords);
        if (!bytes) { set_error("sparse buffer %d: bad header", i); return CFB_ERROR_BADFORMAT; }
        // the table is the only part the kernel trusts for addressing: every chunk must lie inside the buffer
        const unsigned *tab = (const unsigned *)((const unsigned char *)h_sparse[i] + kSparseHeaderBytes);
        for (unsigned b = 0; b < sp.nblocks; b++) {
            const unsigned off = tab[4 * b], G = tab[4 * b + 1], V = tab[4 * b + 2], E = tab[4 * b + 3];
            if (G > kSparseBlockGroups || V > kSparseBlockWords || E > V || (G == 0) != (V == 0) || (off & 15) || off < sp.chunks_off ||
                (size_t)off + sparse_chunk_bytes(G, V, E) > bytes) {
                set_error("sparse buffer %d: block %u out of bounds", i, b);
                return CFB_ERROR_BADFORMAT;
            }
        }
        CFB_CUDA(cudaMemcpyAsync(sp.sparse[i], h_sparse[i], bytes, cudaMemcpyHostToDevice, s));
        cd->ctx->h2d_bytes += (uint64_t)bytes;
    }
    return CFB_OK;
}

}  // namespace cfb

// fetch(b, buf): returns a pointer to the 8192 words of block b (its own storage, or buf after filling it)
template <class Fetch>
static size_t compact_all(unsigned nwords, void *sparse, Fetch &&fetch)
{
    const unsigned nblocks = sparse_nblocks(nwords);
    unsigned *h = (unsigned *)sparse;
    unsigned *tab = (unsigned *)((unsigned char *)sparse + kSparseHeaderBytes);
    size_t off = sparse_chunks_off(nblocks);
    memset((unsigned char *)sparse + kSparseHeaderBytes + (size_t)nblocks * kSparseTableEntry, 0, off - kSparseHeaderBytes - (size_t)nblocks * kSparseTableEntry);
    alignas(64) int16_t buf[kSparseBlockWords];
    for (unsigned b = 0; b < nblocks; b++) {
        const unsigned nvalid = nwords - b * kSparseBlockWords < kSparseBlockWords ? nwords - b * kSparseBlockWords : kSparseBlockWords;
        const int16_t *in = fetch(b, buf);
        unsigned G, V, E;
        const unsigned cb = sparse_compact_block(in, nvalid, (unsigned char *)sparse + off, &G, &V, &E);
        tab[4 * b] = (unsigned)off; tab[4 * b + 1] = G; tab[4 * b + 2] = V; tab[4 * b + 3] = E;
        off += cb;
    }
    h[0] = kSparseMagic; h[1] = nwords; h[2] = (unsigned)off; h[3] = nblocks; h[4] = h[5] = h[6] = h[7] = 0;
    return off;
}

extern "C" {

size_t cfb_sparse_max_bytes(const cfb_layout *L)
{
    if (!L) return 0;
    const unsigned nblocks = sparse_nblocks((unsigned)(L->coded_bytes / 2));
    return (size_t)sparse_chunks_off(nblocks) + (size_t)nblocks * kSparseMaxChunk;
}

size_t cfb_sparse_bytes(const void *sparse)
{
    if (!sparse) return 0;
    const unsigned *h = (const unsigned *)sparse;
    if (h[0] != kSparseMagic) return 0;
    return sparse_checked_bytes(sparse, h[1]);
}

cfb_error cfb_forward_host_sparse(cfb_codec *cd, int n, const void *const *h_frames, int frame_pitch,
                                  const cfb_quant *quant, void *const *h_sparse, size_t *sparse_bytes)
{
    if (!cd || !h_frames || !quant || !h_sparse) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (n < 1 || n > cd->max_batch) { set_error("batch %d exceeds codec max_batch %d", n, cd->max_batch); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_context *ctx = cd->ctx;
    for (int i = 0; i < n; i++) if (!h_sparse[i]) { set_error("null host buffer %d", i); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_error err = stage_fwd_upload(cd, n, h_frames, frame_pitch, ctx->stream);
    if (!err) err = stage_fwd_compute(cd, n, quant, true);
    if (err) return err;
    // Speculative single-pass D2H: copy as many bytes as recent frames needed (+12 %) right behind the kernels, without
    // a host round trip; only if a frame turns out to be larger is the remainder fetched.
    const unsigned guess = cd->value_guess ? cd->value_guess : sparse_initial_guess(cd);
    err = stage_fwd_download(cd, n, h_sparse, true, guess, ctx->stream);
    if (err) return err;
    CFB_CUDA(stream_wait(ctx));
    unsigned maxb = 0;
    bool more = false;
    size_t sizes[kMaxBatch];
    err = stage_fwd_tail(cd, n, h_sparse, guess, ctx->stream, sizes, &maxb, &more);
    if (err) return err;
    if (more) CFB_CUDA(stream_wait(ctx));
    if (sparse_bytes) for (int i = 0; i < n; i++) sparse_bytes[i] = sizes[i];
    cd->value_guess = sparse_next_guess(cd, maxb);
    return CFB_OK;
}

cfb_error cfb_inverse_host_sparse(cfb_codec *cd, int n, const void *const *h_sparse, const cfb_quant *quant,
                                  int out_format, void *const *h_frames, int frame_pitch)
{
    if (!cd || !h_sparse || !quant || !h_frames) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_context *ctx = cd->ctx;
    cfb_error err = stage_inv_upload(cd, n, h_sparse, true, ctx->stream);
    if (!err) err = stage_inv_compute(cd, n, quant, out_format, true);
    if (!err) err = stage_inv_download(cd, n, h_frames, frame_pitch, out_format, ctx->stream);
    if (err) return err;
    CFB_CUDA(stream_wait(ctx));
    return CFB_OK;
}

cfb_error cfb_sparse_expand(const cfb_layout *L, const void *sparse, void *dense_coded)
{
    if (!L || !sparse || !dense_coded) return CFB_ERROR_INVALID_ARGUMENT;
    const unsigned nwords = (unsigned)(L->coded_bytes / 2);
    const size_t total = sparse_checked_bytes(sparse, nwords);
    if (!total) { set_error("bad sparse header"); return CFB_ERROR_BADFORMAT; }
    const unsigned nblocks = sparse_nblocks(nwords);
    int16_t *out = (int16_t *)dense_coded;
    memset(out, 0, (size_t)nwords * 2);
    for (unsigned b = 0; b < nblocks; b++) {
        SparseChunk c;
        if (!sparse_chunk_open(sparse, total, b, &c)) { set_error("sparse block %u out of bounds", b); return CFB_ERROR_BADFORMAT; }
        unsigned gi = 0, vi = 0, ei = 0;
        for (unsigned g = 0; g < kSparseBlockGroups && c.groups; g++) {
            if (!((c.l1[g >> 3] >> (g & 7)) & 1u)) continue;
            if (gi >= c.groups) { set_error("sparse block %u: more groups than the table says", b); return CFB_ERROR_BADFORMAT; }
            unsigned m = c.masks[gi++];
            const size_t w = (size_t)b * kSparseBlockWords + (size_t)g * kSparseGroupWords;
            while (m) {
                const int k = __builtin_ctz(m);
                m &= m - 1;
                if (vi >= c.values || w + k >= nwords) { set_error("sparse block %u: value overrun", b); return CFB_ERROR_BADFORMAT; }
                int v = c.bytes[vi++];
                if (v == -128) {
                    if (ei >= c.escapes) { set_error("sparse block %u: escape overrun", b); return CFB_ERROR_BADFORMAT; }
                    v = c.wide[ei++];
                }
                out[w + k] = (int16_t)v;
            }
        }
        if (gi != c.groups || vi != c.values || ei != c.escapes) { set_error("sparse block %u: count mismatch", b); return CFB_ERROR_BADFORMAT; }
    }
    return CFB_OK;
}

cfb_error cfb_sparse_compact(const cfb_layout *L, const void *dense_coded, void *sparse, size_t *bytes)
{
    if (!L || !sparse || !dense_coded) return CFB_ERROR_INVALID_ARGUMENT;
    const unsigned nwords = (unsigned)(L->coded_bytes / 2);
    const int16_t *in = (const int16_t *)dense_coded;
    const size_t total = compact_all(nwords, sparse, [&](unsigned b, int16_t *) { return in + (size_t)b * kSparseBlockWords; });
    if (bytes) *bytes = total;
    return CFB_OK;
}

// The coded region as the entropy DEcoder leaves it: one buffer per band (pitch bytes per row; whatever lies between
// `width` and the pitch is ignored), e.g. the reference decoder's wavelet->band[] after Codec/decoder.c:19534-19808.
// Produces byte for byte what cfb_sparse_compact gives for the equivalent dense region -- the host-side half of
// "FSM output -> sparse upload" (SURVEY 8f rank 1): the host reads the bands once and uploads ~1/8 of them.
cfb_error cfb_sparse_compact_bands(const cfb_layout *L, const void *const *bands, const int32_t *pitches, void *sparse, size_t *bytes)
{
    if (!L || !bands || !pitches || !sparse) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    struct Seg { size_t w0, w1; const unsigned char *src; int pitch, width, lpitch; };
    Seg segs[CFB_MAX_CHANNELS * CFB_NUM_LEVELS * CFB_NUM_BANDS];
    int ns = 0;
    for (int c = 0; c < L->num_channels; c++)
        for (int k = CFB_NUM_LEVELS - 1; k >= 0; k--)
            for (int b = (k == CFB_NUM_LEVELS - 1 ? 0 : 1); b < CFB_NUM_BANDS; b++) {       // the coded region's order (cfb_layout_compute)
                const int idx = (c * CFB_NUM_LEVELS + k) * CFB_NUM_BANDS + b;
                const cfb_band_layout &bl = L->band[c][k][b];
                if (!bands[idx] || pitches[idx] < bl.width * 2) { set_error("band (%d, %d, %d): null or pitch too small", c, k, b); return CFB_ERROR_INVALID_ARGUMENT; }
                segs[ns++] = {(size_t)bl.offset / 2, (size_t)bl.offset / 2 + (size_t)(bl.pitch / 2) * bl.height, (const unsigned char *)bands[idx], pitches[idx], bl.width, bl.pitch / 2};
            }
    const unsigned nwords = (unsigned)(L->coded_bytes / 2);
    int cur = 0;
    const size_t total = compact_all(nwords, sparse, [&](unsigned b, int16_t *buf) {
        const size_t lo = (size_t)b * kSparseBlockWords, hi = lo + kSparseBlockWords;
        memset(buf, 0, kSparseBlockWords * sizeof(int16_t));
        while (cur < ns && segs[cur].w1 <= lo) cur++;
        for (int s = cur; s < ns && segs[s].w0 < hi; s++) {
            const Seg &g = segs[s];
            const size_t a = g.w0 > lo ? g.w0 : lo, z = g.w1 < hi ? g.w1 : hi;
            for (size_t row = (a - g.w0) / g.lpitch; row * g.lpitch + g.w0 < z; row++) {
                const size_t r0 = g.w0 + row * g.lpitch;                    // flat position of the row's first coefficient
                const size_t x0 = a > r0 ? a - r0 : 0;
                size_t x1 = (size_t)g.width;
                if (r0 + x1 > z) x1 = z - r0;
                if (x0 < x1) memcpy(buf + (r0 + x0 - lo), g.src + row * (size_t)g.pitch + 2 * x0, 2 * (x1 - x0));
            }
        }
        return (const int16_t *)buf;
    });
    if (bytes) *bytes = total;
    return CFB_OK;
}

}  // extern "C"
