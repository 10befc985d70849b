// cfb_host.h -- host-side internals shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <cstring>
#include <string>

#include "../../include/cfhd_b200.h"
#include "cfb_common.cuh"

namespace cfb {

void set_error(const char *fmt, ...);
cfb_error cuda_fail(cudaError_t e, const char *what);

#define CFB_CUDA(call)                                                  \
    do {                                                                \
        cudaError_t e_ = (call);                                        \
        if (e_ != cudaSuccess) return ::cfb::cuda_fail(e_, #call);      \
    } while (0)

QuantParam make_quant_param(int divisor, int midpoint_prequant, bool plain_midpoint = false);
// wait for everything queued on the context's stream without busy-waiting on a CPU core
cudaError_t stream_wait(cfb_context *ctx);
// rows per warp of a launch of `strips` x `planes` warp columns over `oh` rows (cfb_api.cu)
int pick_th(int strips, int oh, int planes, int sm_count, int largest = 16);

// Encode sources: one row per CFB_PIXEL_* input format (kFwdSources, cfb_api.cu).  The family fixes the planes: 4:2:2 =
// W x H luma + two W/2 x H chroma planes (the only family with an interlaced transform), 4:4:4 = three W x H planes,
// Bayer = four W/2 x H/2 planes.
enum CodecFamily { kAnyCodec, kCodec422, kCodec444, kCodecBayer };
struct FwdSource {
    int format;                 // CFB_PIXEL_*
    const char *name;
    CodecFamily family;
    int precision;              // bits of the coded planes
    bool alpha;                 // a fourth W x H channel with CFB_FRAME_ALPHA (RGBA 4:4:4:4)
    int group_px, group_bytes;  // frame row bytes: group_bytes per (partial) group of group_px pixels
    int lines_per_row;          // image lines per frame row (BYR5: 2, one packed row holds both Bayer lines of a plane row)
    int width_multiple;         // the frame width must be a multiple of it
    bool chroma_full;           // chroma quantised with the luma table (ChromaFullRes, encoder.c:1139)
    bool curve;                 // takes an encode-curve table (cfb_codec_set_bayer_curve)
    FwdSrc kernel;              // what level 1 reads
};
// the row of `pixel_format`, null for an unknown format
const FwdSource *fwd_source(int pixel_format);
// one channel of one level: band geometry from bands[0..3] (LL, LH, HL, HH), quantisers from the four divisors and the
// midpoint rule, LL left unquantised; the input plane (in_off, in_pitch) is the caller's
void fill_fwd_geom(PlaneGeom &g, const cfb_band_layout *bands, const int32_t *div, int midpoint);
// the same for the inverse: dequantisers from the divisors, LL carried as is; the output plane is the caller's
void fill_inv_geom(InvGeom &g, const cfb_band_layout *bands, const int32_t *div);

// kernel launchers (cfb_forward.cu / cfb_inverse.cu): each picks the rows per warp (p.th) of its own grid, launches on
// ctx->stream and counts what it launched (launch_kernel)
// nonneg: the planes are non-negative (LL bands of an unsigned source), so the prescaled level may use its packed taps
cudaError_t launch_fwd_plane(cfb_context *ctx, FwdParams &p, int prescale, bool nonneg);
cudaError_t launch_fwd_422(cfb_context *ctx, FwdParams &p);
// levels 1 and 2 of progressive packed 8-bit 4:2:2 in one pass (two launches: main rows, border rows); l2[3] = the
// level-2 geometry of the channels of p.ch
cudaError_t launch_fwd_422_l12(cfb_context *ctx, FwdParams &p, const PlaneGeom *l2);
cudaError_t launch_fwd_rg48(cfb_context *ctx, FwdParams &p);
cudaError_t launch_fwd_byr4(cfb_context *ctx, FwdParams &p);
cudaError_t launch_fwd_byr5(cfb_context *ctx, FwdParams &p);
// B64A (rg64 = false) / RG64 sources, p.nchan = 3 (RGB 4:4:4) or 4 (RGBA 4:4:4:4)
cudaError_t launch_fwd_rgba64(cfb_context *ctx, FwdParams &p, bool rg64);
cudaError_t launch_fwd_rgb30(cfb_context *ctx, FwdParams &p);
cudaError_t launch_inv_plane(cfb_context *ctx, InvParams &p, int descale);
// inverse levels 3 and 2 in one pass (two launches: main rows, border rows); descale3 = level 3's prescale, level 2's is 2
cudaError_t launch_inv_l32(cfb_context *ctx, InvL32Params &p, int descale3);
cudaError_t launch_inv_422(cfb_context *ctx, InvParams &p, InvOut out);
cudaError_t launch_inv_444(cfb_context *ctx, InvParams &p, InvOut out);
cudaError_t launch_lowpass(cfb_context *ctx, const InvParams &p, InvOut out);
cudaError_t launch_inv_fields(cfb_context *ctx, InvParams &p, const FieldsAux &a, bool planar);
// interlaced level 1 of every packed 4:2:2 source
cudaError_t launch_fwd_422_fields(cfb_context *ctx, FwdParams &p, FwdSrc src);
// progressive level 1 of YU64 / V210 (packed 8-bit runs launch_fwd_422 / launch_fwd_422_l12)
cudaError_t launch_fwd_422_src(cfb_context *ctx, FwdParams &p, FwdSrc src);
// opts the final 4:2:2 inverse kernels into the shared memory of their TMA ring on the current device (a per-device
// function attribute: cfb_context_create calls it for its device)
cudaError_t inv_opt_in_smem();
// range audit of the planes a forward level is about to read (cfb_audit.cu): ORs violation bits into ctx->d_range
cfb_error audit_level_input(cfb_context *ctx, const FwdParams &p, int prescale);
// forward level 1 of p.nframes frames d_frames[] (cfb_api.cu): p.nchan, p.nframes, p.out_base and p.ch[c] (fill_fwd_geom
// with the level's divisors div[c] and midpoint) set by the caller; sets the inputs and the interlaced midpoints and
// launches the kernels.  l2: the level-2 geometry when the caller asks for a prescaled level 2 too (null
// otherwise); *fused is set when level 1 ran it as well.
cfb_error launch_fwd_first(cfb_codec *cd, FwdParams &p, const void *const *d_frames, int frame_pitch, const int32_t *const *div,
                           int midpoint, int prescale, const PlaneGeom *l2, bool *fused);
// final inverse level of a progressive or interlaced frame into `out_format` (cfb_api.cu): p.nchan, p.nframes, p.ch[c]
// (band geometry of level 1) and the in / out bases set by the caller; fills the output fields of p and launches
cfb_error launch_inv_final(cfb_codec *cd, InvParams &p, int out_format, int prescale, int frame_pitch);
cfb_error range_status(cfb_context *ctx, int *flags);

// The host forms of the transform as three stages, each on a stream of the caller's choice, so that the frame pool can
// run uploads, kernels and downloads of different jobs on separate streams (copy engines + SMs all busy).  The compute
// stage always runs on cfb_context_stream(); the caller orders the stages with events.  Slots [0, n) of the codec's
// device staging are used.  The synchronous C-ABI calls are these three stages on one stream + a wait.
cfb_error stage_fwd_upload(cfb_codec *cd, int n, const void *const *h_frames, int frame_pitch, cudaStream_t s);
cfb_error stage_fwd_compute(cfb_codec *cd, int n, const cfb_quant *quant, bool sparse);
// sparse: copies the first `guess` bytes of every frame's sparse buffer (speculative single pass); dense: the coded region
cfb_error stage_fwd_download(cfb_codec *cd, int n, void *const *h_out, bool sparse, unsigned guess, cudaStream_t s);
// sparse only, after the download has completed: fetches the bytes beyond `guess` (if any frame has more), reports sizes
cfb_error stage_fwd_tail(cfb_codec *cd, int n, void *const *h_sparse, unsigned guess, cudaStream_t s, size_t *sizes,
                         unsigned *max_bytes, bool *more);
cfb_error stage_inv_upload(cfb_codec *cd, int n, const void *const *h_in, bool sparse, cudaStream_t s);
cfb_error stage_inv_compute(cfb_codec *cd, int n, const cfb_quant *quant, int out_format, bool sparse);
cfb_error stage_inv_download(cfb_codec *cd, int n, void *const *h_frames, int frame_pitch, int out_format, cudaStream_t s);
unsigned sparse_initial_guess(const cfb_codec *cd);
unsigned sparse_next_guess(const cfb_codec *cd, unsigned max_bytes);
// GPU compaction / expansion between the pyramids and the sparse staging buffers of slots [0, n) (kernels only)
cfb_error sparse_upload(cfb_codec *cd, int n, const void *const *h_sparse, cudaStream_t s);
cfb_error sparse_download(cfb_codec *cd, int n, void *const *h_sparse, unsigned guess, cudaStream_t s);
cfb_error sparse_compact_device(cfb_codec *cd, int n);
cfb_error sparse_expand_device(cfb_codec *cd, int n);

}  // namespace cfb

struct cfb_context {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;             // blocking-sync event: host threads sleep instead of spinning
    int sm_count = 0;
    int *d_range = nullptr;                 // device flag word of the range audit (cfb_audit.cu), allocated on first use
    int *h_range = nullptr;                 // pinned copy
    std::atomic<uint64_t> kernel_launches{0}, frames_forward{0}, frames_inverse{0}, h2d_bytes{0}, d2h_bytes{0};
};

struct cfb_codec {
    cfb_context *ctx = nullptr;
    cfb_frame_desc desc{};
    cfb_layout layout{};
    int max_batch = 0;
    unsigned char *d_frames = nullptr;      // max_batch packed frames
    unsigned char *d_pyramids = nullptr;    // max_batch pyramids
    size_t frame_stride = 0;                // bytes between device frame slots
    size_t pyramid_stride = 0;
    int bayer_phase = 0;                    // BAYER_FORMAT_* (0 RED_GRN, 1 GRN_RED, 2 GRN_BLU, 3 BLU_GRN), DemoasicFrames.h:30
    int fwd_mask = 7, inv_mask = 7;         // profiling aid: levels to run
    int interlaced = 0;                     // level 1 is the field transform (CFHD_ENCODING_FLAGS_YUV_INTERLACED)
    int *d_carry = nullptr;                 // interlaced inverse: HL row carries, kMaxBatch frames
    unsigned short *d_curve = nullptr;      // Bayer encode curve (1 << 14 entries), null = frame already curved
    unsigned short *d_restore = nullptr;    // BYR4 output: linear-restore table (1 << 14 entries), null = v & 0xfffe
    unsigned char *d_gop = nullptr;         // two-frame GOP buffer (cfb_gop2_layout.total_bytes), allocated on first use
    int carry_strips = 0;
    int decode_res = 1;                     // CFB_RESOLUTION_*: 1 full, 2 half (LL1), 3 quarter (LL2)
    // sparse transfer format staging (allocated on first use)
    unsigned char *d_sparse = nullptr;      // max_batch sparse buffers
    unsigned long long *d_status = nullptr; // max_batch * (nblocks + 1): look-back state of the one-pass packer
    unsigned *h_headers = nullptr;          // pinned, 4 u32 per slot
    size_t sparse_stride = 0;
    // B64A output (8 bytes per pixel) does not fit the frame staging of a 6-byte-per-pixel source: own staging, allocated on first use
    unsigned char *d_out64 = nullptr;
    size_t out64_stride = 0;
    unsigned value_guess = 0;               // running estimate of a frame's sparse size in bytes (speculative single-pass D2H)
};

namespace cfb {

// kernel<<<grid, block, smem, ctx->stream>>>(args...), counted in ctx->kernel_launches when the launch was accepted.
// Every kernel of the library is launched through it.
template <class... Params, class... Args>
cudaError_t launch_kernel(cfb_context *ctx, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, const Args &...args)
{
    kernel<<<grid, block, smem, ctx->stream>>>(args...);
    const cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) ctx->kernel_launches++;
    return e;
}

}  // namespace cfb
