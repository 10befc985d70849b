// cfb_api.cu -- C-ABI implementation (see include/cfhd_b200.h).
//
// Host side of the transform path: pyramid layout, quantisation schedule, CUDA
// context / staging management and the kernel launch sequences.  No transform
// arithmetic is ever done on the host: if no sm_90 device is usable every
// transform entry point fails with CFB_ERROR_NO_DEVICE.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <new>

#include "cfb_host.h"

#include <mutex>
#include <ctype.h>
#include <sched.h>
#include <stdio.h>

namespace cfb {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

cfb_error cuda_fail(cudaError_t e, const char *what)
{
    set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) return CFB_ERROR_NO_DEVICE;
    if (e == cudaErrorMemoryAllocation) return CFB_ERROR_OUTOFMEMORY;
    return CFB_ERROR_CUDA;
}

// Codec/quantize.c:1395-1427: multiplier = 65536/d, midpoint = d/g (g in [2,9)), minus one when g == 2.
QuantParam make_quant_param(int divisor, int g, bool plain_midpoint)
{
    QuantParam q;
    if (divisor <= 1) { q.m = 65536; q.cpos = 0; q.cneg = 65535; q.pad = 0; return q; }
    int mid = 0;
    // plain_midpoint: the difference-filtered HL band of the field transform rounds with divisor / g and has no
    // "-1" adjustment (spatial.c:5356-5358), unlike QuantizeRow16sTo16s (quantize.c:1415-1427)
    if (g >= 2 && g < 9) { mid = divisor / g; if (g == 2 && mid && !plain_midpoint) mid--; }
    q.m = 65536 / divisor;
    q.cpos = mid * q.m;
    q.cneg = 65535 - mid * q.m;
    q.pad = 0;
    return q;
}

cudaError_t stream_wait(cfb_context *ctx)
{
    cudaError_t e = cudaEventRecord(ctx->done, ctx->stream);
    if (e != cudaSuccess) return e;
    return cudaEventSynchronize(ctx->done);
}

static inline int align16(int x) { return (x + 15) & ~15; }
static inline int64_t align64(int64_t x) { return (x + 63) & ~(int64_t)63; }

// Rows per warp: the largest candidate that still gives >= 48 warps per SM over the launch, so that wave
// quantisation and the tail stay small, while the one-pair halo each warp re-reads stays <= 6-12 % (and is served by
// L2).  The candidates and the threshold have not been swept on an H100 (tools/microbench.py, CFB_TH), except for the
// fused forward levels 1 + 2, which takes candidates up to `largest` = 4 level-2 rows (see launch_fwd_422_l12), and the
// fused inverse levels 3 + 2, up to 6 level-2 rows (see launch_inv_l32).
int pick_th(int strips, int oh, int planes, int sm_count, int largest)
{
    static const int cand[] = {16, 12, 8, 6, 4};
    if (const char *e = getenv("CFB_TH")) { int v = atoi(e); if (v >= 2) return v; }     // tuning knob (development)
    const long long want = (long long)sm_count * 48;
    for (int th : cand) {
        if (th > largest) continue;
        long long warps = (long long)strips * ((oh + th - 1) / th) * planes;
        if (warps >= want) return th;
    }
    return 4;
}

}  // namespace cfb

using namespace cfb;

extern "C" {

int cfb_version(void) { return 100; }

const char *cfb_last_error_string(void) { return g_err; }

int cfb_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// NUMA placement.  Host<->device copies run at full PCIe rate only from memory (and threads) on the GPU's own NUMA
// node; the reference pins its worker threads too (Codec/thread.c SetThreadAffinityMask / the SDK's thread
// "capabilities" masks).  Linux sysfs only: /sys/bus/pci/devices/<bdf>/numa_node, /sys/devices/system/node/nodeN/cpulist.
int cfb_device_numa_node(int device)
{
    char bdf[32] = {0};
    if (cudaDeviceGetPCIBusId(bdf, sizeof(bdf), device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char *c = bdf; *c; c++) *c = (char)tolower((unsigned char)*c);
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bdf);
    FILE *f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

cfb_error cfb_bind_thread_to_device(int device)
{
    const int node = cfb_device_numa_node(device);
    if (node < 0) return CFB_OK;                    // no NUMA information (single node, container without sysfs): leave as is
    char path[128];
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    FILE *f = fopen(path, "r");
    if (!f) return CFB_OK;
    char list[4096] = {0};
    const size_t n = fread(list, 1, sizeof(list) - 1, f);
    fclose(f);
    list[n] = 0;
    cpu_set_t allowed, want;
    CPU_ZERO(&want);
    if (sched_getaffinity(0, sizeof(allowed), &allowed) != 0) return CFB_OK;
    int count = 0;
    for (char *tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
        int a = 0, b = 0;
        const int k = sscanf(tok, "%d-%d", &a, &b);
        if (k == 1) b = a;
        if (k < 1) continue;
        for (int c = a; c <= b && c < CPU_SETSIZE; c++)
            if (CPU_ISSET(c, &allowed)) { CPU_SET(c, &want); count++; }
    }
    if (count == 0) return CFB_OK;                  // the node's CPUs are outside this process's mask: keep the mask
    if (sched_setaffinity(0, sizeof(want), &want) != 0) { set_error("sched_setaffinity failed"); return CFB_ERROR_INVALID_ARGUMENT; }
    return CFB_OK;
}

// ---------------------------------------------------------------------------
// Layout: Codec/wavelet.c:1208-1283 (AllocTransform), :427 (AllocWaveletStack), :302 (InitWaveletStack)
cfb_error cfb_layout_compute(const cfb_frame_desc *desc, cfb_layout *out)
{
    if (!desc || !out) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    const int W = desc->width, H = desc->height, fmt = desc->pixel_format;
    if (W <= 0 || H <= 0) { set_error("bad dimensions %dx%d", W, H); return CFB_ERROR_INVALID_ARGUMENT; }
    const FwdSource *s = fwd_source(fmt);
    if (!s) { set_error("bad pixel format %d", fmt); return CFB_ERROR_BADFORMAT; }
    memset(out, 0, sizeof(*out));
    // RGBA 4:4:4:4 (ENCODED_FORMAT_RGBA_4444) when a 16-bit RGBA source asks for its alpha channel (Codec/codec.c:380-386)
    const int nc = (s->family == kCodecBayer ? 4 : 3) + (s->alpha && (desc->flags & CFB_FRAME_ALPHA) ? 1 : 0);
    out->num_channels = nc;
    out->precision = s->precision;
    out->frame_pitch = (W + s->group_px - 1) / s->group_px * s->group_bytes;
    if (W % s->width_multiple || (s->family == kCodecBayer && H % 2)) {
        set_error("%s width %d must be a multiple of %d%s", s->name, W, s->width_multiple, s->family == kCodecBayer ? ", its height even" : "");
        return CFB_ERROR_UNSUPPORTED;
    }
    int cw[CFB_MAX_CHANNELS], ch[CFB_MAX_CHANNELS];
    for (int c = 0; c < nc; c++) {
        const bool half = (s->family == kCodecBayer) || (s->family == kCodec422 && c > 0);
        cw[c] = half ? W / 2 : W;
        ch[c] = (s->family == kCodecBayer) ? H / 2 : H;
        if (ch[c] % 8 || ch[c] < 48) { set_error("channel height %d must be a multiple of 8 and >= 48", ch[c]); return CFB_ERROR_UNSUPPORTED; }
    }
    out->frame_bytes = (int64_t)out->frame_pitch * (H / s->lines_per_row) * (s->kernel == kFwdPlanes ? nc : 1);     // PLANAR16: planes stacked

    // coded region: per channel LL3, then highpass of level 3, 2, 1
    int64_t off = 0;
    for (int c = 0; c < nc; c++) {
        for (int k = CFB_NUM_LEVELS - 1; k >= 0; k--) {
            const int w = cw[c] >> (k + 1), h = ch[c] >> (k + 1);
            const int pitch = align16(w * 2);
            const int64_t bsz = align64((int64_t)pitch * h);
            for (int b = (k == CFB_NUM_LEVELS - 1 ? 0 : 1); b < CFB_NUM_BANDS; b++) {
                cfb_band_layout &bl = out->band[c][k][b];
                bl.offset = off; bl.width = w; bl.height = h; bl.pitch = pitch;
                off += bsz;
            }
        }
    }
    out->coded_bytes = off;
    // scratch region: LL1, LL2
    for (int c = 0; c < nc; c++) {
        for (int k = 0; k < CFB_NUM_LEVELS - 1; k++) {
            const int w = cw[c] >> (k + 1), h = ch[c] >> (k + 1);
            const int pitch = align16(w * 2);
            cfb_band_layout &bl = out->band[c][k][0];
            bl.offset = off; bl.width = w; bl.height = h; bl.pitch = pitch;
            off += align64((int64_t)pitch * h);
        }
    }
    out->total_bytes = off;
    return CFB_OK;
}

// ---------------------------------------------------------------------------
// Quantisation schedule for a fixed quality, GOP 1, progressive, rate control idle:
// Codec/quantize.c:186-584 (QuantizationSetQuality), :2865-3356 (SetTransformQuantization, spatial
// case with vbrscale 256 => VSCALE(q,m,256) = 256 q), Codec/wavelet.c:7022 (SetTransformScale:
// band scales {4,2,2,1}, {16,8,8,4}, {64,32,32,16}), Codec/wavelet.c:1710 (SetTransformPrescale).
cfb_error cfb_quant_for_quality(const cfb_frame_desc *desc, int quality, cfb_quant *out)
{
    return cfb_quant_for_source(desc, quality, 0, out);
}

// Subband divisor tables of one frame BEFORE they are mapped onto a transform: quantize.c:186 QuantizationSetQuality
// (tables, precision scaling, !progressive rescaling).  ql / qc: luma / chroma, index = subband number.
static cfb_error quant_tables(const cfb_frame_desc *desc, int quality, int interlaced, int *ql_out, int *qc_out, int *g_out,
                              int *precision_out, int *nchan_out)
{
    if (!desc) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_layout lay;
    cfb_error err = cfb_layout_compute(desc, &lay);
    if (err) return err;
    static const int luma_tab[4][17] = {
        {4, 4, 5, 5, 4, 5, 5, 9, 8, 8, 8, 4, 4, 4, 4, 4, 4},            // default
        {4, 8, 8, 12, 8, 8, 12, 9, 12, 12, 16, 32, 32, 48, 32, 32, 48},   // low
        {4, 6, 6, 8, 6, 6, 8, 5, 8, 8, 12, 16, 16, 24, 16, 16, 24},       // medium
        {4, 4, 4, 6, 4, 4, 6, 5, 8, 8, 8, 8, 8, 12, 8, 8, 12}};           // high
    static const int chroma_tab[4][17] = {
        {4, 4, 5, 5, 4, 5, 5, 9, 8, 8, 8, 8, 8, 8, 8, 8, 8},
        {4, 8, 8, 12, 8, 8, 12, 9, 12, 12, 16, 32, 32, 48, 32, 32, 48},
        {4, 6, 6, 8, 6, 6, 8, 5, 8, 8, 12, 16, 16, 32, 16, 16, 32},
        {4, 6, 6, 8, 6, 6, 8, 5, 8, 8, 8, 8, 8, 16, 8, 8, 16}};
    const int precision = lay.precision;
    const bool chroma_full = fwd_source(desc->pixel_format)->chroma_full;
    if (fwd_source(desc->pixel_format)->family == kCodecBayer) quality |= (3 << 25);     // encoder.c:2634 / :2674: no extra quant on channels 1-3
    int factor = quality & 0xff;
    const int detail = (quality & 0x0e0000) >> 17;
    int rgb_quality = (quality & 0x06000000) >> 25;
    if (rgb_quality > 2) rgb_quality = 2;
    int g = detail + 2;
    if (g > 8) g = 0;
    if (quality & 0x1f00) factor = 5;
    const int new_quality = factor;
    int limiter = 0;                                    // FSratelimiter on the first frame
    if (new_quality == 5) limiter = 8; else if (new_quality == 6) limiter = 4;
    if (factor < 1 || factor > 10) factor = 0;
    if (factor > 3) factor = 3;
    int ql[17], qc[17];
    memcpy(ql, luma_tab[factor], sizeof(ql));
    memcpy(qc, chroma_full ? luma_tab[factor] : chroma_tab[factor], sizeof(qc));
    int lowfreq = 4;
    if (precision >= 10) {
        int scale = 4 * 16;
        if (limiter > 16) limiter = 16;
        if (new_quality == 4) { lowfreq = 3; scale = 3 * 16; }
        else if (new_quality >= 5 && new_quality <= 10) { lowfreq = 2; scale = 16 + limiter * 2; }
        if (new_quality >= 5 && scale >= 4) scale >>= 1;
        if (new_quality == 10 && scale >= 6) { scale *= 2; scale /= 3; }
        if (new_quality >= 4) for (int i = 1; i < 7; i++) ql[i] = qc[i] = lowfreq;
        for (int i = 8; i < 17; i++) {
            ql[i] = (ql[i] * scale) >> 4; if (ql[i] < 2) ql[i] = 2;
            qc[i] = (qc[i] * scale) >> 4; if (qc[i] < 2) qc[i] = 2;
        }
        ql[7] = qc[7] = 4;
    }
    if (precision == 12) {
        if (new_quality >= 4) for (int i = 1; i < 7; i++) ql[i] = qc[i] = lowfreq;
        for (int i = 4; i < 7; i++) { ql[i] *= 4; qc[i] *= 4; }
        static const int gains[4] = {8, 6, 4, 4};
        const int chromagain = gains[rgb_quality];
        for (int i = 11; i < 17; i++) { ql[i] *= 4; qc[i] *= chromagain; }
    }
    if (interlaced) {       // quantize.c:490-541 (!progressive): LH of the field transform * 3/2, HL * 2/3
        ql[11] = ql[11] * 3 / 2; ql[12] = ql[12] * 2 / 3; ql[14] = ql[14] * 3 / 2; ql[15] = ql[15] * 2 / 3;
        qc[11] = qc[11] * 3 / 2; qc[12] = qc[12] * 2 / 3; qc[14] = qc[14] * 3 / 2; qc[15] = qc[15] * 2 / 3;
    }
    memcpy(ql_out, ql, sizeof(ql)); memcpy(qc_out, qc, sizeof(qc));
    *g_out = g; *precision_out = precision; *nchan_out = lay.num_channels;
    return CFB_OK;
}

cfb_error cfb_quant_for_source(const cfb_frame_desc *desc, int quality, int interlaced, cfb_quant *out)
{
    if (!desc || !out) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    int ql[17], qc[17], g = 0, precision = 0, nchan = 0;
    cfb_error err = quant_tables(desc, quality, interlaced, ql, qc, &g, &precision, &nchan);
    if (err) return err;
    memset(out, 0, sizeof(*out));
    // GOP length 1 (quantize.c:552-567)
    for (int i = 0; i < 3; i++) { ql[7 + i] = ql[11 + i]; qc[7 + i] = qc[11 + i]; }

    static const int scale[3][4] = {{4, 2, 2, 1}, {16, 8, 8, 4}, {64, 32, 32, 16}};
    out->midpoint_prequant = g;
    out->prescale[0] = 0; out->prescale[1] = 2; out->prescale[2] = (precision == 12) ? 2 : 0;
    for (int c = 0; c < nchan; c++) {
        const int *q = (c > 0) ? qc : ql;
        int subband = 1;
        for (int k = 2; k >= 0; k--) {
            out->divisor[c][k][0] = 1;
            for (int b = 1; b < 4; b++) {
                int d = (k == 0) ? q[subband] : ((q[subband] * scale[k][b]) >> 2);
                if (g) { d *= g; d /= (g - 1) * 2; } else d /= 2;
                out->divisor[c][k][b] = d;
                subband++;
            }
        }
    }
    return CFB_OK;
}

// Two-frame GOP (TRANSFORM_TYPE_FIELDPLUS): quantize.c:3480-3640 maps the subbands onto the six wavelets as
// 1-3 -> wavelet 5, 4-6 -> wavelet 4, 7 -> LL of wavelet 3 (forced to 1 for >= 10 bit, encoder.c:8487), 8-10 -> wavelet 3,
// 11-13 -> wavelet 1, 14-16 -> wavelet 0, with the band scales of wavelet.c:7135-7180 (SetTransformScale, FIELDPLUS):
// wavelet 3 {16,8,8,4}, wavelet 4 {32,16,16,8}, wavelet 5 {128,64,64,32}; frame wavelets take the table value itself.
// No GOP-1 copy of subbands 11-13 into 7-9 (quantize.c:552).  Prescale {0,0,0,0,2,0} (wavelet.c:1710, 10 bit).
cfb_error cfb_gop2_quant_for_quality(const cfb_frame_desc *desc, int quality, int interlaced, cfb_gop2_quant *out)
{
    if (!desc || !out) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    int ql[17], qc[17], g = 0, precision = 0, nchan = 0;
    cfb_error err = quant_tables(desc, quality, interlaced, ql, qc, &g, &precision, &nchan);
    if (err) return err;
    if (precision != 10) { set_error("two-frame GOP: 10-bit 4:2:2 sources"); return CFB_ERROR_UNSUPPORTED; }
    memset(out, 0, sizeof(*out));
    out->midpoint_prequant = g;
    out->prescale[4] = 2;
    static const int wavelet_of[5] = {5, 4, 3, 1, 0};
    static const int first_subband[5] = {1, 4, 8, 11, 14};
    static const int scale[6][4] = {{4, 2, 2, 1}, {4, 2, 2, 1}, {8, 4, 0, 0}, {16, 8, 8, 4}, {32, 16, 16, 8}, {128, 64, 64, 32}};
    for (int c = 0; c < nchan; c++) {
        const int *q = (c > 0) ? qc : ql;
        for (int k = 0; k < CFB_GOP2_WAVELETS; k++) out->divisor[c][k][0] = 1;
        out->divisor[c][2][1] = 1;
        for (int i = 0; i < 5; i++) {
            const int k = wavelet_of[i];
            for (int b = 1; b < 4; b++) {
                const int v = q[first_subband[i] + b - 1];
                int d = (k <= 1) ? v : ((v * scale[k][b]) >> 2);
                if (g) { d *= g; d /= (g - 1) * 2; } else d /= 2;
                out->divisor[c][k][b] = d;
            }
        }
    }
    return CFB_OK;
}

// ---------------------------------------------------------------------------
cfb_error cfb_context_create(int device, cfb_context **out)
{
    if (!out) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        set_error("no CUDA device available (%s): the transform path has no CPU fallback",
                  e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        return CFB_ERROR_NO_DEVICE;
    }
    if (device < 0 || device >= n) { set_error("device %d out of range [0,%d)", device, n); return CFB_ERROR_INVALID_ARGUMENT; }
    // three attributes, queried once per device: cudaGetDeviceProperties costs tens of milliseconds and serialises the
    // sixteen encoder threads of an SDK pool that all create their context at the same moment
    struct DevInfo { int major = -1, minor = 0, sms = 0; };
    static DevInfo info[64];
    static std::mutex info_mu;
    DevInfo di;
    {
        std::lock_guard<std::mutex> lk(info_mu);
        if (device < 64 && info[device].major >= 0) di = info[device];
        else {
            CFB_CUDA(cudaDeviceGetAttribute(&di.major, cudaDevAttrComputeCapabilityMajor, device));
            CFB_CUDA(cudaDeviceGetAttribute(&di.minor, cudaDevAttrComputeCapabilityMinor, device));
            CFB_CUDA(cudaDeviceGetAttribute(&di.sms, cudaDevAttrMultiProcessorCount, device));
            if (device < 64) info[device] = di;
        }
    }
    if (di.major != 9 || di.minor != 0) {
        set_error("device %d is sm_%d%d; this library carries sm_90a code only", device, di.major, di.minor);
        return CFB_ERROR_NO_DEVICE;
    }
    CFB_CUDA(cudaSetDevice(device));
    CFB_CUDA(inv_opt_in_smem());
    cfb_context *ctx = new (std::nothrow) cfb_context();
    if (!ctx) return CFB_ERROR_OUTOFMEMORY;
    ctx->device = device;
    ctx->sm_count = di.sms;
    e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->done, cudaEventBlockingSync | cudaEventDisableTiming);
    if (e != cudaSuccess) { if (ctx->stream) cudaStreamDestroy(ctx->stream); delete ctx; return cuda_fail(e, "cudaStreamCreate"); }
    *out = ctx;
    return CFB_OK;
}

void cfb_context_destroy(cfb_context *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->done) cudaEventDestroy(ctx->done);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->d_range) cudaFree(ctx->d_range);
    if (ctx->h_range) cudaFreeHost(ctx->h_range);
    delete ctx;
}

cfb_error cfb_context_synchronize(cfb_context *ctx)
{
    if (!ctx) return CFB_ERROR_INVALID_ARGUMENT;
    CFB_CUDA(cudaSetDevice(ctx->device));
    CFB_CUDA(stream_wait(ctx));
    return CFB_OK;
}

void *cfb_context_stream(cfb_context *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

cfb_error cfb_context_stats(cfb_context *ctx, cfb_stats *out)
{
    if (!ctx || !out) return CFB_ERROR_INVALID_ARGUMENT;
    out->kernel_launches = ctx->kernel_launches.load();
    out->frames_forward = ctx->frames_forward.load();
    out->frames_inverse = ctx->frames_inverse.load();
    out->h2d_bytes = ctx->h2d_bytes.load();
    out->d2h_bytes = ctx->d2h_bytes.load();
    return CFB_OK;
}

// ---------------------------------------------------------------------------
cfb_error cfb_codec_create(cfb_context *ctx, const cfb_frame_desc *desc, int max_batch, cfb_codec **out)
{
    if (!ctx || !desc || !out) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    *out = nullptr;
    if (max_batch < 1 || max_batch > CFB_MAX_BATCH) { set_error("max_batch %d out of range", max_batch); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_layout lay;
    cfb_error err = cfb_layout_compute(desc, &lay);
    if (err) return err;
    CFB_CUDA(cudaSetDevice(ctx->device));
    cfb_codec *cd = new (std::nothrow) cfb_codec();
    if (!cd) return CFB_ERROR_OUTOFMEMORY;
    cd->ctx = ctx; cd->desc = *desc; cd->layout = lay; cd->max_batch = max_batch;
    // frame staging must also hold the PLANAR16 rendition (channel planes stacked at the frame's luma pitch)
    int64_t planar_rows = 0;
    for (int c = 0; c < lay.num_channels; c++) planar_rows += lay.band[c][0][0].height * 2;
    int64_t fbytes = lay.frame_bytes;
    if (planar_rows * desc->width * 2 > fbytes) fbytes = planar_rows * desc->width * 2;
    cd->frame_stride = (size_t)((fbytes + 255) & ~(int64_t)255);
    cd->pyramid_stride = (size_t)((lay.total_bytes + 255) & ~(int64_t)255);
    cudaError_t e = cudaMalloc((void **)&cd->d_frames, cd->frame_stride * max_batch);
    if (e == cudaSuccess) e = cudaMalloc((void **)&cd->d_pyramids, cd->pyramid_stride * max_batch);
    if (e != cudaSuccess) { cfb_codec_destroy(cd); return cuda_fail(e, "cudaMalloc(codec staging)"); }
    // deterministic contents for the pitch padding (the reference's entropy coder walks it, encoder.c:5811)
    e = cudaMemsetAsync(cd->d_pyramids, 0, cd->pyramid_stride * max_batch, ctx->stream);
    if (e != cudaSuccess) { cfb_codec_destroy(cd); return cuda_fail(e, "cudaMemsetAsync"); }
    *out = cd;
    return CFB_OK;
}

void cfb_codec_destroy(cfb_codec *cd)
{
    if (!cd) return;
    if (cd->ctx) cudaSetDevice(cd->ctx->device);
    if (cd->d_frames) cudaFree(cd->d_frames);
    if (cd->d_pyramids) cudaFree(cd->d_pyramids);
    if (cd->d_carry) cudaFree(cd->d_carry);
    if (cd->d_gop) cudaFree(cd->d_gop);
    if (cd->d_curve) cudaFree(cd->d_curve);
    if (cd->d_restore) cudaFree(cd->d_restore);
    if (cd->d_sparse) cudaFree(cd->d_sparse);
    if (cd->d_out64) cudaFree(cd->d_out64);
    if (cd->d_status) cudaFree(cd->d_status);
    if (cd->h_headers) cudaFreeHost(cd->h_headers);
    delete cd;
}

cfb_error cfb_codec_layout(const cfb_codec *cd, cfb_layout *out)
{
    if (!cd || !out) return CFB_ERROR_INVALID_ARGUMENT;
    *out = cd->layout;
    return CFB_OK;
}

cfb_error cfb_codec_set_bayer_phase(cfb_codec *cd, int bayer_format)
{
    if (!cd || bayer_format < 0 || bayer_format > 3) { set_error("bayer format %d out of range 0..3", bayer_format); return CFB_ERROR_INVALID_ARGUMENT; }
    cd->bayer_phase = bayer_format;
    return CFB_OK;
}

cfb_error cfb_codec_set_bayer_curve(cfb_codec *cd, const uint16_t *curve, int entries)
{
    if (!cd) { set_error("null codec"); return CFB_ERROR_INVALID_ARGUMENT; }
    const FwdSource &s = *fwd_source(cd->desc.pixel_format);
    if (s.family != kCodecBayer) { set_error("the encode curve applies to Bayer (BYR4) codecs"); return CFB_ERROR_BADFORMAT; }
    if (!s.curve) { set_error("%s sources take no encode curve", s.name); return CFB_ERROR_UNSUPPORTED; }
    CFB_CUDA(cudaSetDevice(cd->ctx->device));
    if (!curve) {                                   // back to "curve already applied" (encode_curve_preset)
        if (cd->d_curve) { CFB_CUDA(stream_wait(cd->ctx)); cudaFree(cd->d_curve); cd->d_curve = nullptr; }
        return CFB_OK;
    }
    if (entries != (1 << 14)) { set_error("Bayer encode curve must have 1 << 14 entries (MAX_INPUT_PRECISION, frame.c:4843)"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (!cd->d_curve) CFB_CUDA(cudaMalloc((void **)&cd->d_curve, sizeof(uint16_t) << 14));
    CFB_CUDA(cudaMemcpyAsync(cd->d_curve, curve, sizeof(uint16_t) << 14, cudaMemcpyHostToDevice, cd->ctx->stream));
    CFB_CUDA(stream_wait(cd->ctx));                 // the caller's table may go away after this call
    return CFB_OK;
}

cfb_error cfb_codec_set_bayer_decode_curve(cfb_codec *cd, const uint16_t *table, int entries)
{
    if (!cd) { set_error("null codec"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (fwd_source(cd->desc.pixel_format)->family != kCodecBayer) { set_error("the linear-restore table applies to Bayer (BYR4, BYR5) codecs"); return CFB_ERROR_BADFORMAT; }
    CFB_CUDA(cudaSetDevice(cd->ctx->device));
    if (!table) {                                   // back to encode_curve_preset == 1: v & 0xfffe
        if (cd->d_restore) { CFB_CUDA(stream_wait(cd->ctx)); cudaFree(cd->d_restore); cd->d_restore = nullptr; }
        return CFB_OK;
    }
    if (entries != (1 << 14)) { set_error("the BYR4 linear-restore table must have 1 << 14 entries (decoder.c:10737)"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (!cd->d_restore) CFB_CUDA(cudaMalloc((void **)&cd->d_restore, sizeof(uint16_t) << 14));
    CFB_CUDA(cudaMemcpyAsync(cd->d_restore, table, sizeof(uint16_t) << 14, cudaMemcpyHostToDevice, cd->ctx->stream));
    CFB_CUDA(stream_wait(cd->ctx));                 // the caller's table may go away after this call
    return CFB_OK;
}

cfb_error cfb_codec_set_level_mask(cfb_codec *cd, int forward_mask, int inverse_mask)
{
    if (!cd) return CFB_ERROR_INVALID_ARGUMENT;
    cd->fwd_mask = forward_mask & 7; cd->inv_mask = inverse_mask & 7;
    return CFB_OK;
}

cfb_error cfb_codec_set_decode_resolution(cfb_codec *cd, int resolution)
{
    if (!cd) { set_error("null codec"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (resolution < CFB_RESOLUTION_FULL || resolution > CFB_RESOLUTION_QUARTER) {
        set_error("decode resolution %d not in {full=1, half=2, quarter=3}", resolution);
        return CFB_ERROR_INVALID_ARGUMENT;
    }
    cd->decode_res = resolution;
    return CFB_OK;
}

cfb_error cfb_codec_set_interlaced(cfb_codec *cd, int interlaced)
{
    if (!cd) { set_error("null codec"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (interlaced && fwd_source(cd->desc.pixel_format)->family != kCodec422) {
        set_error("the interlaced (field) transform is implemented for 4:2:2 sources (YUYV, UYVY, YU64, V210)");
        return CFB_ERROR_UNSUPPORTED;
    }
    if (interlaced && !cd->d_carry) {
        // per band row and strip carry-in of the difference-coded HL band, for up to kMaxBatch frames
        const cfb_band_layout &ll = cd->layout.band[0][0][0];
        cd->carry_strips = (ll.width + kInvStrip - 1) / kInvStrip;
        const size_t bytes = (size_t)kMaxBatch * 3 * ll.height * cd->carry_strips * sizeof(int);
        CFB_CUDA(cudaSetDevice(cd->ctx->device));
        cudaError_t e = cudaMalloc((void **)&cd->d_carry, bytes);
        if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(field carries)");
    }
    cd->interlaced = (interlaced == CFB_INTERLACED_HL_INTEGRATED) ? 2 : (interlaced ? 1 : 0);
    return CFB_OK;
}

cfb_error cfb_codec_decoded_size(const cfb_codec *cd, int *width, int *height)
{
    if (!cd || !width || !height) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (cd->decode_res == CFB_RESOLUTION_FULL) { *width = cd->desc.width; *height = cd->desc.height; }
    else {      // the lowpass image of level (res - 1) of channel 0: decoder.c:26078 (half), :17000 (quarter)
        const cfb_band_layout &ll = cd->layout.band[0][cd->decode_res - 2][0];
        *width = ll.width; *height = ll.height;
    }
    return CFB_OK;
}

void *cfb_codec_device_frame(cfb_codec *cd, int slot)
{
    return (cd && slot >= 0 && slot < cd->max_batch) ? cd->d_frames + cd->frame_stride * slot : nullptr;
}
void *cfb_codec_device_pyramid(cfb_codec *cd, int slot)
{
    return (cd && slot >= 0 && slot < cd->max_batch) ? cd->d_pyramids + cd->pyramid_stride * slot : nullptr;
}

// ---------------------------------------------------------------------------
// forward
cfb_error cfb_forward_device(cfb_codec *cd, int n, const void *const *d_frames, int frame_pitch,
                             const cfb_quant *quant, void *const *d_pyramids)
{
    if (!cd || !d_frames || !quant || !d_pyramids) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (n < 1 || n > kMaxBatch) { set_error("batch %d out of range [1,%d]", n, kMaxBatch); return CFB_ERROR_INVALID_ARGUMENT; }
    if (frame_pitch < cd->layout.frame_pitch || (frame_pitch & 15)) { set_error("frame pitch %d must be >= %d and 16-byte aligned", frame_pitch, cd->layout.frame_pitch); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_context *ctx = cd->ctx;
    const cfb_layout &L = cd->layout;
    CFB_CUDA(cudaSetDevice(ctx->device));
    for (int i = 0; i < n; i++)
        if (!d_frames[i] || !d_pyramids[i] || ((uintptr_t)d_frames[i] & 15) || ((uintptr_t)d_pyramids[i] & 15)) {
            set_error("frame/pyramid %d null or not 16-byte aligned", i);
            return CFB_ERROR_INVALID_ARGUMENT;
        }
    for (int lvl = 0; lvl < CFB_NUM_LEVELS; lvl++)
        if (quant->prescale[lvl] != 0 && quant->prescale[lvl] != 2) { set_error("prescale %d unsupported", quant->prescale[lvl]); return CFB_ERROR_UNSUPPORTED; }

    FwdParams p;
    memset(&p, 0, sizeof(p));
    p.nchan = L.num_channels; p.nframes = n;
    for (int i = 0; i < n; i++) p.out_base[i] = (unsigned char *)d_pyramids[i];
    bool level2_done = false;
    if (cd->fwd_mask & 1) {
        const int32_t *div[kMaxChannels];
        PlaneGeom l2[kMaxChannels] = {};
        for (int c = 0; c < L.num_channels; c++) {
            div[c] = quant->divisor[c][0];
            fill_fwd_geom(p.ch[c], L.band[c][0], div[c], quant->midpoint_prequant);
            fill_fwd_geom(l2[c], L.band[c][1], quant->divisor[c][1], quant->midpoint_prequant);
        }
        const bool with_l2 = (cd->fwd_mask & 2) && quant->prescale[1] == 2;
        cfb_error err = launch_fwd_first(cd, p, d_frames, frame_pitch, div, quant->midpoint_prequant, quant->prescale[0],
                                         with_l2 ? l2 : nullptr, &level2_done);
        if (err) return err;
    }
    // ---- levels 2, 3: input = LL of the previous level inside the pyramid ----
    for (int k = 1; k < CFB_NUM_LEVELS; k++) {
        if (!(cd->fwd_mask & (1 << k)) || (k == 1 && level2_done)) continue;
        for (int c = 0; c < L.num_channels; c++) {
            PlaneGeom &g = p.ch[c];
            fill_fwd_geom(g, L.band[c][k], quant->divisor[c][k], quant->midpoint_prequant);
            g.in_off = L.band[c][k - 1][0].offset; g.in_pitch = L.band[c][k - 1][0].pitch;
            g.quant_ll = (quant->prescale[k] == 0) && quant->divisor[c][k][0] > 1;
        }
        for (int i = 0; i < n; i++) p.in_base[i] = (const unsigned char *)d_pyramids[i];
        // the LL bands of every unsigned source format are non-negative (<= 4 * 4095): the prescaled level may use its
        // packed non-negative taps; caller-supplied planes (CFB_PIXEL_PLANAR16) carry no such promise
        const bool nonneg = fwd_source(cd->desc.pixel_format)->kernel != kFwdPlanes;
        CFB_CUDA(launch_fwd_plane(ctx, p, quant->prescale[k], nonneg));
    }
    ctx->frames_forward += n;
    return CFB_OK;
}

cfb_error cfb_forward_host(cfb_codec *cd, int n, const void *const *h_frames, int frame_pitch,
                           const cfb_quant *quant, void *const *h_coded)
{
    if (!cd || !h_frames || !quant || !h_coded) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_context *ctx = cd->ctx;
    cfb_error err = stage_fwd_upload(cd, n, h_frames, frame_pitch, ctx->stream);
    if (!err) err = stage_fwd_compute(cd, n, quant, false);
    if (!err) err = stage_fwd_download(cd, n, h_coded, false, 0, ctx->stream);
    if (err) return err;
    CFB_CUDA(stream_wait(ctx));
    return CFB_OK;
}

}  // extern "C"

namespace cfb {

cfb_error stage_fwd_upload(cfb_codec *cd, int n, const void *const *h_frames, int frame_pitch, cudaStream_t s)
{
    if (!cd || !h_frames) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (n < 1 || n > cd->max_batch) { set_error("batch %d exceeds codec max_batch %d", n, cd->max_batch); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_context *ctx = cd->ctx;
    const cfb_layout &L = cd->layout;
    if (frame_pitch < L.frame_pitch || (frame_pitch & 15)) { set_error("frame pitch %d must be >= %d and 16-byte aligned", frame_pitch, L.frame_pitch); return CFB_ERROR_INVALID_ARGUMENT; }
    CFB_CUDA(cudaSetDevice(ctx->device));
    const int rows = (int)(L.frame_bytes / L.frame_pitch);
    for (int i = 0; i < n; i++) {
        if (!h_frames[i]) { set_error("null host buffer %d", i); return CFB_ERROR_INVALID_ARGUMENT; }
        if (frame_pitch == L.frame_pitch)       // contiguous on both sides: one linear copy
            CFB_CUDA(cudaMemcpyAsync(cfb_codec_device_frame(cd, i), h_frames[i], (size_t)L.frame_pitch * rows, cudaMemcpyHostToDevice, s));
        else
            CFB_CUDA(cudaMemcpy2DAsync(cfb_codec_device_frame(cd, i), L.frame_pitch, h_frames[i], frame_pitch, L.frame_pitch, rows,
                                       cudaMemcpyHostToDevice, s));
        ctx->h2d_bytes += (uint64_t)L.frame_bytes;
    }
    return CFB_OK;
}

cfb_error stage_fwd_compute(cfb_codec *cd, int n, const cfb_quant *quant, bool sparse)
{
    if (!cd || !quant) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (n < 1 || n > cd->max_batch) { set_error("batch %d exceeds codec max_batch %d", n, cd->max_batch); return CFB_ERROR_INVALID_ARGUMENT; }
    const void *dfr[kMaxBatch];
    void *dpy[kMaxBatch];
    for (int i = 0; i < n; i++) { dfr[i] = cfb_codec_device_frame(cd, i); dpy[i] = cfb_codec_device_pyramid(cd, i); }
    cfb_error err = cfb_forward_device(cd, n, dfr, cd->layout.frame_pitch, quant, dpy);
    if (!err && sparse) err = sparse_compact_device(cd, n);
    return err;
}

}  // namespace cfb

namespace cfb {

// ---------------------------------------------------------------------------
// Encode sources: one row per CFB_PIXEL_* input.  cfb_layout_compute, the quantiser tables, the interlace and decode-output
// checks, cfb_gop2_layout_compute and the level-1 launch read it.
static const FwdSource kFwdSources[] = {
    // 4:2:2 widths: whole 16-pixel lanes (the reference's own row unpackers need them, convert.c:4701); V210 also whole
    // 6-pixel groups (the reference's unpacker reads row padding otherwise)
    {CFB_PIXEL_YUYV, "YUYV", kCodec422, 10, false, 1, 2, 1, 16, false, false, kFwdPacked8},
    {CFB_PIXEL_UYVY, "UYVY", kCodec422, 10, false, 1, 2, 1, 16, false, false, kFwdPacked8},
    {CFB_PIXEL_YU64, "YU64", kCodec422, 10, false, 1, 4, 1, 16, false, false, kFwdYU64},
    {CFB_PIXEL_V210, "V210", kCodec422, 10, false, 48, 128, 1, 48, false, false, kFwdV210},
    {CFB_PIXEL_PLANAR16, "PLANAR16", kCodec444, 12, false, 1, 2, 1, 8, true, false, kFwdPlanes},
    // ChromaFullRes = (format >= COLOR_FORMAT_BAYER) (encoder.c:1139): true for RG48 (120), RG64 (121) and BYR4 (104),
    // false for B64A (30), which reaches the quantiser under its own format (encoder.c:2484-2499 does not remap it)
    {CFB_PIXEL_RG48, "RG48", kCodec444, 12, false, 1, 6, 1, 8, true, false, kFwdRG48},
    {CFB_PIXEL_RG30, "RG30", kCodec444, 12, false, 1, 4, 1, 8, true, false, kFwdRGB10},
    {CFB_PIXEL_AB10, "AB10", kCodec444, 12, false, 1, 4, 1, 8, true, false, kFwdRGB10},
    {CFB_PIXEL_AR10, "AR10", kCodec444, 12, false, 1, 4, 1, 8, true, false, kFwdRGB10},
    {CFB_PIXEL_R210, "R210", kCodec444, 12, false, 1, 4, 1, 8, true, false, kFwdRGB10},
    {CFB_PIXEL_DPX0, "DPX0", kCodec444, 12, false, 1, 4, 1, 8, true, false, kFwdRGB10},
    // Codec/encoder.c:2484-2509 / :2734-2750: 12-bit planes G, R, B (+ A) of the frame's size
    {CFB_PIXEL_B64A, "B64A", kCodec444, 12, true, 1, 8, 1, 8, false, false, kFwdB64A},
    {CFB_PIXEL_RG64, "RG64", kCodec444, 12, true, 1, 8, 1, 8, true, false, kFwdRG64},
    {CFB_PIXEL_BYR4, "BYR4", kCodecBayer, 12, false, 1, 2, 1, 16, true, true, kFwdBYR4},
    // Codec/encoder.c:2648-2676: one packed row of 3 W bytes per plane row, no encode curve; ChromaFullRes (BYR5 = 105)
    {CFB_PIXEL_BYR5, "BYR5", kCodecBayer, 12, false, 1, 3, 2, 16, true, false, kFwdBYR5},
};

const FwdSource *fwd_source(int pixel_format)
{
    for (const FwdSource &s : kFwdSources)
        if (s.format == pixel_format) return &s;
    return nullptr;
}

// The 10-bit RGB words of RG30 / AB10 / AR10 / R210 / DPX0, in both directions: bit positions of R, G, B, and whether the
// word is stored byte-swapped (spatial.c:2118-2268 / InvertHorizontalStrip16s.c:15562-15613)
struct RGB10Word { int pos[3]; int byteswap; };
static const RGB10Word kRGB10Words[5] = {{{0, 10, 20}, 0}, {{0, 10, 20}, 0}, {{20, 10, 0}, 0}, {{20, 10, 0}, 1}, {{22, 12, 2}, 1}};

void fill_fwd_geom(PlaneGeom &g, const cfb_band_layout *bands, const int32_t *div, int midpoint)
{
    g.width = bands[0].width * 2; g.height = bands[0].height * 2;
    g.out_pitch = bands[0].pitch;
    for (int b = 0; b < 4; b++) {
        g.band_off[b] = bands[b].offset;
        g.q[b] = make_quant_param(div[b], midpoint);
    }
    // only the unprescaled planar filter ever quantises LL (spatial.c:10480; compiled out at :12942, absent at :14726)
    g.quant_ll = 0;
}

void fill_inv_geom(InvGeom &g, const cfb_band_layout *bands, const int32_t *div)
{
    g.width = bands[0].width; g.height = bands[0].height; g.pitch = bands[0].pitch;
    for (int b = 0; b < 4; b++) {
        g.band_off[b] = bands[b].offset;
        g.dq[b] = div[b] > 1 ? div[b] : 1;
    }
    g.dq[0] = 1;        // LL is carried unquantised through the pyramid (only LL3 is coded, raw)
}

cfb_error launch_fwd_first(cfb_codec *cd, FwdParams &p, const void *const *d_frames, int frame_pitch, const int32_t *const *div,
                           int midpoint, int prescale, const PlaneGeom *l2, bool *fused)
{
    cfb_context *ctx = cd->ctx;
    const FwdSource &s = *fwd_source(cd->desc.pixel_format);
    const int precision = cd->layout.precision;
    *fused = false;
    for (int i = 0; i < p.nframes; i++) p.in_base[i] = (const unsigned char *)d_frames[i];
    for (int c = 0; c < p.nchan; c++) {
        PlaneGeom &g = p.ch[c];
        g.in_pitch = frame_pitch;           // PLANAR16: the planes stacked at the frame's pitch
        g.in_off = (s.kernel == kFwdPlanes) ? (long long)c * frame_pitch * cd->desc.height : 0;
        g.quant_ll = s.kernel != kFwdPacked8 && div[c][0] > 1;     // planar filters: LL quantised when its divisor > 1
    }
    if (cd->interlaced) {
        // field transform (filter.c:273): the difference-filtered HL rounds with divisor / g and no "-1" (spatial.c:5356-5358);
        // the planar one (YU64, V210) also rounds LH with divisor / 2 (spatial.c:5856)
        for (int c = 0; c < p.nchan; c++) {
            if (s.kernel != kFwdPacked8) {
                if (div[c][0] > 1) { set_error("interlaced 16-bit / 10-bit 4:2:2 sources: a quantised level-1 lowpass band is not supported"); return CFB_ERROR_UNSUPPORTED; }
                p.ch[c].q[1] = make_quant_param(div[c][1], 2, true);
            }
            p.ch[c].q[2] = make_quant_param(div[c][2], midpoint, true);
        }
    }
    switch (s.kernel) {
    case kFwdPacked8:
        p.shift = precision - 8; p.uyvy = (s.format == CFB_PIXEL_UYVY);
        if (cd->interlaced) {
            CFB_CUDA(launch_fwd_422_fields(ctx, p, s.kernel));
        } else if (l2 && cd->desc.width % 32 == 0) {
            // levels 1 and 2 in one pass: LL1 stays in registers instead of a round trip through the scratch region.
            // Needs the prescaled level 2 (its non-negative filter) and whole level-2 lanes (LL1 chroma width a multiple
            // of 8, so no edge kernel); the layout's heights are multiples of 8, so LL2 has exactly half the LL1 rows.
            CFB_CUDA(launch_fwd_422_l12(ctx, p, l2));
            *fused = true;
        } else {
            CFB_CUDA(launch_fwd_422(ctx, p));
        }
        break;
    case kFwdYU64: case kFwdV210:
        p.shift = 16 - precision;
        CFB_CUDA(cd->interlaced ? launch_fwd_422_fields(ctx, p, s.kernel) : launch_fwd_422_src(ctx, p, s.kernel));
        break;
    case kFwdPlanes:
        CFB_CUDA(launch_fwd_plane(ctx, p, prescale, false));
        break;
    case kFwdRG48:
        // channel order of the reference: plane 0 = G, 1 = R, 2 = B (Codec/frame.c:6155-6157)
        p.shift = 16 - precision;
        CFB_CUDA(launch_fwd_rg48(ctx, p));
        break;
    case kFwdB64A: case kFwdRG64:
        p.shift = 16 - precision;
        CFB_CUDA(launch_fwd_rgba64(ctx, p, s.kernel == kFwdRG64));
        break;
    case kFwdRGB10: {
        static const int rgb_of[3] = {1, 0, 2};         // channel 0 = G, 1 = R, 2 = B
        const RGB10Word &w = kRGB10Words[s.format - CFB_PIXEL_RG30];
        for (int c = 0; c < 3; c++) {
            FwdParams q = p;
            q.nchan = 1; q.ch[0] = p.ch[c];
            q.shift = precision - 10; q.byteswap = w.byteswap; q.field_pos = w.pos[rgb_of[c]];
            CFB_CUDA(launch_fwd_rgb30(ctx, q));
        }
        break;
    }
    case kFwdBYR4:
        p.shift = 16 - precision; p.bayer_phase = cd->bayer_phase; p.lut = cd->d_curve;
        CFB_CUDA(launch_fwd_byr4(ctx, p));
        break;
    case kFwdBYR5:
        p.bayer_phase = cd->bayer_phase;
        CFB_CUDA(launch_fwd_byr5(ctx, p));
        break;
    }
    return CFB_OK;
}

// ---------------------------------------------------------------------------
// Decode outputs: one row per CFB_PIXEL_* output of the inverse.  The checks of cfb_inverse_device, the staging of
// inv_output_geometry / inv_frame_slot and the final-level launch read it.
struct InvOutputDesc {
    int format;                 // CFB_PIXEL_*
    const char *name;
    CodecFamily codec;          // the codec family it decodes
    bool needs12;               // 12-bit codec only
    int resolutions;            // the decode resolutions it is written at (kRes* bits)
    int interlaced_resolutions; // those of them at which it also decodes an interlaced codec
    bool min16;                 // full resolution: level-1 bands at least 16 coefficients wide
    int group_px, group_bytes;  // row bytes: group_bytes per (partial) group of group_px pixels
    bool fits_frame;            // its frame must fit the codec's frame staging
    bool own_staging;           // it has its own staging (wider than the codec's frames)
    InvOut kernel;              // what the final level writes
};
constexpr int kResFull = 1 << CFB_RESOLUTION_FULL, kResHalf = 1 << CFB_RESOLUTION_HALF, kResQuarter = 1 << CFB_RESOLUTION_QUARTER;
constexpr int kResAll = kResFull | kResHalf | kResQuarter;
// Reduced resolutions (k_lowpass_422 / k_lowpass_444): the reference's conversion of the lowpass image, see include/cfhd_b200.h
// at cfb_codec_set_decode_resolution for each rule and for the combinations that stay unsupported and why.  An interlaced
// 4:2:2 codec decodes at half resolution wherever a progressive one does: the reference's reduced paths run before its
// progressive / interlaced split (decoder.c:26075).
static const InvOutputDesc kInvOutputs[] = {
    {CFB_PIXEL_YUYV, "8-bit 4:2:2", kCodec422, false, kResAll, kResAll, false, 1, 2, false, false, kInvOut8},
    {CFB_PIXEL_UYVY, "8-bit 4:2:2", kCodec422, false, kResAll, kResAll, false, 1, 2, false, false, kInvOut8},
    // the 16-bit packed outputs of the reference's ...ToRow16u family
    {CFB_PIXEL_YU64, "YU64", kCodec422, false, kResFull | kResHalf, kResHalf, true, 1, 4, true, false, kInvOutYU64},
    {CFB_PIXEL_RG48, "RG48", kCodec444, false, kResFull, 0, true, 1, 6, true, false, kInvOutRG48},
    // 10-bit packed 4:2:2 (decoder.c:26303 -> convert.c:13526 ConvertPlanarYUVToV210)
    {CFB_PIXEL_V210, "V210", kCodec422, false, kResFull, 0, false, 6, 16, true, false, kInvOutV210},
    // 10-bit packed RGB of an RGB 4:4:4 sample (decoder.c:26893 -> InvertHorizontalStrip16s.c:14812 ...RGB2RG30); the
    // alpha channel of an RGBA sample does not enter (the routine's loops write R, G, B only)
    {CFB_PIXEL_RG30, "10-bit RGB", kCodec444, true, kResFull | kResQuarter, 0, true, 1, 4, true, false, kInvOutRGB10},
    {CFB_PIXEL_AB10, "10-bit RGB", kCodec444, true, kResFull | kResQuarter, 0, true, 1, 4, true, false, kInvOutRGB10},
    {CFB_PIXEL_AR10, "10-bit RGB", kCodec444, true, kResFull | kResQuarter, 0, true, 1, 4, true, false, kInvOutRGB10},
    {CFB_PIXEL_R210, "10-bit RGB", kCodec444, true, kResFull | kResQuarter, 0, true, 1, 4, true, false, kInvOutRGB10},
    {CFB_PIXEL_DPX0, "10-bit RGB", kCodec444, true, kResFull | kResQuarter, 0, true, 1, 4, true, false, kInvOutRGB10},
    // 16-bit A,R,G,B of an RGB 4:4:4 or RGBA 4:4:4:4 sample (decoder.c:26862 -> InvertHorizontalStrip16s.c:13298 ...RGB2B64A)
    {CFB_PIXEL_B64A, "B64A", kCodec444, true, kResFull, 0, true, 1, 8, false, true, kInvOutB64A},
    // the mosaic of a Bayer sample (BYR4 or BYR5 source), no demosaic (decoder.c:14629 ...ToRow16u rows -> bayer.c:13237
    // GenerateBYR2); 2 * W * H bytes fit the frame staging, which holds the four stacked planes at the mosaic's pitch
    {CFB_PIXEL_BYR4, "BYR4", kCodecBayer, true, kResFull, 0, true, 1, 2, true, false, kInvOutBYR4},
    // the int16 planes, stacked channel after channel at their own widths
    {CFB_PIXEL_PLANAR16, "PLANAR16", kAnyCodec, false, kResAll, kResAll, false, 1, 2, true, false, kInvOutPlanes},
};

static const InvOutputDesc *inv_output_desc(int out_format)
{
    for (const InvOutputDesc &d : kInvOutputs)
        if (d.format == out_format) return &d;
    set_error("output format %d not implemented", out_format);
    return nullptr;
}

static int inv_row_bytes(const InvOutputDesc &d, int width) { return (width + d.group_px - 1) / d.group_px * d.group_bytes; }

// The final level's output fields of InvParams for `out` (p.ch[c].width = the level-1 band widths)
static void inv_output_params(int out_format, InvOut out, int precision, InvParams &p)
{
    if (out == kInvOutRGB10) {
        const RGB10Word &w = kRGB10Words[out_format - CFB_PIXEL_RG30];
        for (int c = 0; c < 3; c++) p.rgb10.pos[c] = w.pos[c];
        p.rgb10.byteswap = w.byteswap;
        return;
    }
    if (out != kInvOutYU64 && out != kInvOutRG48 && out != kInvOutB64A && out != kInvOutB64AAlpha && out != kInvOutBYR4) return;
    p.up_shift = 16 - precision;
    p.hi_simd = ((1 << precision) - 1) << p.up_shift;
    for (int c = 0; c < p.nchan; c++) {
        const int w = p.ch[c].width;
        if (out == kInvOutB64A)
            // InvertHorizontalStrip16s.c:13319: the 8-column loop runs up to post_column = width - width % 8 and always leaves
            // the right border column to the scalar code, which saturates at 65535 instead of the 12-bit maximum
            p.tail_col[c] = (w % 8) ? w - w % 8 : w - 1;
        else
            // InvertHorizontalStrip16s.c:16589-16594: the 8-column loop ends at post_column = width - width % 8 - 16; one more
            // group of 7 columns is produced with the SIMD rule, everything right of it by the scalar code.  B64A with alpha
            // follows it: the reference decoder's active-metadata path (bayer.c:7144-7147) copies the ...ToRow16u rows.  So
            // does BYR4: its four RawBayer16 rows come from the same routine (InvertHorizontalStrip16s.c:17462 -> :16571).
            p.tail_col[c] = (w - (w % 8) - 16) + 7;
    }
}

cfb_error launch_inv_final(cfb_codec *cd, InvParams &p, int out_format, int prescale, int frame_pitch)
{
    cfb_context *ctx = cd->ctx;
    const cfb_layout &L = cd->layout;
    const InvOutputDesc *od = inv_output_desc(out_format);
    if (!od) return CFB_ERROR_UNSUPPORTED;
    const bool planar = (od->kernel == kInvOutPlanes);
    // PLANAR16: planes stacked channel after channel, each channel at its own width, pitch = frame_pitch
    long long off = 0;
    for (int c = 0; c < p.nchan; c++) {
        p.ch[c].out_pitch = frame_pitch;
        p.ch[c].out_off = planar ? off : 0;
        off += (long long)frame_pitch * p.ch[c].height * 2;
    }
    if (planar && !cd->interlaced) {
        CFB_CUDA(launch_inv_plane(ctx, p, prescale));
        return CFB_OK;
    }
    p.shift = L.precision - 8; p.uyvy = (out_format == CFB_PIXEL_UYVY);
    if (cd->interlaced) {
        FieldsAux aux;
        aux.carry = cd->d_carry; aux.nstrips = cd->carry_strips; aux.maxh = p.ch[0].height;
        aux.hl_integrated = (cd->interlaced == 2);      // the reference decoder's bands (decoder.c:20822): no carries
        CFB_CUDA(launch_inv_fields(ctx, p, aux, planar));
        return CFB_OK;
    }
    // four channels: channel 3 de-companded into the alpha word
    const InvOut out = (od->kernel == kInvOutB64A && L.num_channels == 4) ? kInvOutB64AAlpha : od->kernel;
    inv_output_params(out_format, out, L.precision, p);
    if (out == kInvOutBYR4) { p.bayer.phase = cd->bayer_phase; p.bayer.restore = cd->d_restore; }
    if (out == kInvOut8 || out == kInvOutYU64 || out == kInvOutV210) CFB_CUDA(launch_inv_422(ctx, p, out));
    else CFB_CUDA(launch_inv_444(ctx, p, out));
    return CFB_OK;
}

// Levels 3 and 2 run as one pass (launch_inv_l32) when the decode runs both (inverse mask bits 1 and 2; quarter resolution
// stops after level 3), level 2 is prescaled, and every channel's level-2 band is a multiple of 4 wide (no ragged edge
// columns) and exactly twice as wide and high as its level-3 band of at least 3 rows.  Otherwise the two levels keep
// their own launches.
static bool inv_l32_applies(const cfb_codec *cd, const cfb_quant *quant)
{
    const cfb_layout &L = cd->layout;
    if ((cd->inv_mask & 6) != 6 || cd->decode_res > CFB_RESOLUTION_HALF || quant->prescale[1] != 2) return false;
    for (int c = 0; c < L.num_channels; c++) {
        const cfb_band_layout &b2 = L.band[c][1][0], &b3 = L.band[c][2][0];
        if ((b2.width & 3) || b2.width != 2 * b3.width || b2.height != 2 * b3.height || b3.height < 3) return false;
    }
    return true;
}

}  // namespace cfb

extern "C" {

// ---------------------------------------------------------------------------
// inverse
cfb_error cfb_inverse_device(cfb_codec *cd, int n, void *const *d_pyramids, const cfb_quant *quant,
                             int out_format, void *const *d_frames, int frame_pitch)
{
    if (!cd || !d_pyramids || !quant || !d_frames) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (n < 1 || n > kMaxBatch) { set_error("batch %d out of range [1,%d]", n, kMaxBatch); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_context *ctx = cd->ctx;
    const cfb_layout &L = cd->layout;
    int out_w = 0, out_h = 0;
    cfb_codec_decoded_size(cd, &out_w, &out_h);
    const InvOutputDesc *od = inv_output_desc(out_format);
    if (!od) return CFB_ERROR_UNSUPPORTED;
    const CodecFamily family = fwd_source(cd->desc.pixel_format)->family;
    if ((od->codec != kAnyCodec && od->codec != family) || (od->needs12 && L.precision != 12)) {
        set_error("%s output needs a %s%s codec", od->name, od->needs12 ? "12-bit " : "",
                  od->codec == kCodec422 ? "4:2:2" : od->codec == kCodecBayer ? "Bayer" : "4:4:4");
        return CFB_ERROR_BADFORMAT;
    }
    static const char *const res_name[] = {"", "full", "half", "quarter"};
    if (!(od->resolutions & (1 << cd->decode_res))) {
        set_error("%s output: no %s-resolution decode", od->name, res_name[cd->decode_res]);
        return CFB_ERROR_UNSUPPORTED;
    }
    if (cd->interlaced && !(od->interlaced_resolutions & (1 << cd->decode_res))) {
        set_error("%s output: no %s-resolution decode of an interlaced codec", od->name, res_name[cd->decode_res]);
        return CFB_ERROR_UNSUPPORTED;
    }
    if (frame_pitch < inv_row_bytes(*od, out_w) || (frame_pitch & 15)) { set_error("bad output pitch %d", frame_pitch); return CFB_ERROR_INVALID_ARGUMENT; }
    if (od->min16 && cd->decode_res == CFB_RESOLUTION_FULL)
        for (int c = 0; c < L.num_channels; c++)
            if (L.band[c][0][0].width < 16) { set_error("%s output needs level-1 bands at least 16 coefficients wide", od->name); return CFB_ERROR_UNSUPPORTED; }
    for (int i = 0; i < n; i++)
        if (!d_frames[i] || !d_pyramids[i] || ((uintptr_t)d_frames[i] & 15) || ((uintptr_t)d_pyramids[i] & 15)) {
            set_error("frame/pyramid %d null or not 16-byte aligned", i);
            return CFB_ERROR_INVALID_ARGUMENT;
        }
    CFB_CUDA(cudaSetDevice(ctx->device));

    InvParams p;
    memset(&p, 0, sizeof(p));
    p.nchan = L.num_channels; p.nframes = n;
    // levels 3 and 2 in one pass when both run: LL2 stays in registers (the LL2 scratch region is then left as it was)
    const bool l32 = inv_l32_applies(cd, quant);
    if (l32) {
        InvL32Params q;
        memset(&q, 0, sizeof(q));
        q.nchan = L.num_channels; q.nframes = n;
        for (int c = 0; c < L.num_channels; c++) {
            fill_inv_geom(q.l3[c], L.band[c][2], quant->divisor[c][2]);
            fill_inv_geom(q.l2[c], L.band[c][1], quant->divisor[c][1]);
            q.l2[c].out_off = L.band[c][0][0].offset; q.l2[c].out_pitch = L.band[c][0][0].pitch;
        }
        for (int i = 0; i < n; i++) { q.in_base[i] = (const unsigned char *)d_pyramids[i]; q.out_base[i] = (unsigned char *)d_pyramids[i]; }
        CFB_CUDA(launch_inv_l32(ctx, q, quant->prescale[2]));
    }
    // levels 3 -> 2 -> 1: output = LL of the level below, inside the pyramid
    for (int k = l32 ? 0 : CFB_NUM_LEVELS - 1; k >= 1 && k >= cd->decode_res - 1; k--) {
        if (!(cd->inv_mask & (1 << k))) continue;
        for (int c = 0; c < L.num_channels; c++) {
            InvGeom &g = p.ch[c];
            fill_inv_geom(g, L.band[c][k], quant->divisor[c][k]);
            g.out_off = L.band[c][k - 1][0].offset; g.out_pitch = L.band[c][k - 1][0].pitch;
        }
        for (int i = 0; i < n; i++) { p.in_base[i] = (const unsigned char *)d_pyramids[i]; p.out_base[i] = (unsigned char *)d_pyramids[i]; }
        CFB_CUDA(launch_inv_plane(ctx, p, quant->prescale[k]));
    }
    if (cd->decode_res != CFB_RESOLUTION_FULL) {
        // reduced resolution: the output is the lowpass image of level kk+1 (decoder.c:26078-26160 half,
        // decoder.c:11818 + :17000 quarter); the levels below are never inverted
        const int kk = cd->decode_res - 2;
        for (int c = 0; c < L.num_channels; c++) fill_inv_geom(p.ch[c], L.band[c][kk], quant->divisor[c][kk]);
        if (out_format == CFB_PIXEL_PLANAR16) {
            for (int i = 0; i < n; i++) {
                long long off = 0;
                for (int c = 0; c < L.num_channels; c++) {
                    const InvGeom &g = p.ch[c];
                    CFB_CUDA(cudaMemcpy2DAsync((unsigned char *)d_frames[i] + off, frame_pitch,
                                               (const unsigned char *)d_pyramids[i] + g.band_off[0], g.pitch,
                                               (size_t)g.width * 2, g.height, cudaMemcpyDeviceToDevice, ctx->stream));
                    off += (long long)frame_pitch * g.height;
                }
            }
        } else {
            for (int i = 0; i < n; i++) { p.in_base[i] = (const unsigned char *)d_pyramids[i]; p.out_base[i] = (unsigned char *)d_frames[i]; }
            p.ch[0].out_pitch = frame_pitch;
            if (od->kernel == kInvOut8) {
                p.shift = 4;                                        // PRESCALE_LUMA10 / descale (frame.c:11742, temporal.c:11373)
                p.ll_unsigned = (cd->decode_res == CFB_RESOLUTION_QUARTER); // unsigned shift + packus in the quarter path
                p.uyvy = (out_format == CFB_PIXEL_UYVY);
            } else {
                // YU64 (half): 16 - precision - 2 (frame.c:11146 ConvertLowpass16sToYUV64: 4095 << 4 at 10 bits); the 10-bit
                // RGB words (quarter): 16 - precision - descale 2 (decoder.c:17000 ConvertQuarterFrameToBuffer)
                p.up_shift = 16 - L.precision - 2;
                if (od->kernel == kInvOutRGB10) inv_output_params(out_format, kInvOutRGB10, L.precision, p);
            }
            CFB_CUDA(launch_lowpass(ctx, p, od->kernel));
        }
        ctx->frames_inverse += n;
        return CFB_OK;
    }
    // level 1 -> pixels
    if (!(cd->inv_mask & 1)) { ctx->frames_inverse += n; return CFB_OK; }
    for (int c = 0; c < L.num_channels; c++) fill_inv_geom(p.ch[c], L.band[c][0], quant->divisor[c][0]);
    for (int i = 0; i < n; i++) { p.in_base[i] = (const unsigned char *)d_pyramids[i]; p.out_base[i] = (unsigned char *)d_frames[i]; }
    cfb_error err = launch_inv_final(cd, p, out_format, quant->prescale[0], frame_pitch);
    if (err) return err;
    ctx->frames_inverse += n;
    return CFB_OK;
}

cfb_error cfb_inverse_host(cfb_codec *cd, int n, const void *const *h_coded, const cfb_quant *quant,
                           int out_format, void *const *h_frames, int frame_pitch)
{
    if (!cd || !h_coded || !quant || !h_frames) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_context *ctx = cd->ctx;
    cfb_error err = stage_inv_upload(cd, n, h_coded, false, ctx->stream);
    if (!err) err = stage_inv_compute(cd, n, quant, out_format, false);
    if (!err) err = stage_inv_download(cd, n, h_frames, frame_pitch, out_format, ctx->stream);
    if (err) return err;
    CFB_CUDA(stream_wait(ctx));
    return CFB_OK;
}

}  // extern "C"

namespace cfb {

// geometry of what the inverse writes into the device frame staging / the caller's buffer at the current resolution
static cfb_error inv_output_geometry(const cfb_codec *cd, int out_format, int *rows, int *rowbytes, int *dpitch)
{
    const cfb_layout &L = cd->layout;
    const InvOutputDesc *od = inv_output_desc(out_format);
    if (!od) return CFB_ERROR_UNSUPPORTED;
    int out_w = 0, out_h = 0;
    cfb_codec_decoded_size(cd, &out_w, &out_h);
    const int kk = cd->decode_res - 1;          // lowest level that is inverted (0 = all three)
    *rowbytes = inv_row_bytes(*od, out_w);
    *dpitch = (*rowbytes + 15) & ~15;
    *rows = out_h;
    if (od->kernel == kInvOutPlanes) {
        *rows = 0;
        for (int c = 0; c < L.num_channels; c++) *rows += kk ? L.band[c][kk - 1][0].height : L.band[c][0][0].height * 2;
    }
    if (od->fits_frame && (size_t)*dpitch * *rows > cd->frame_stride) {
        set_error("%s output does not fit the codec's frame staging", od->name); return CFB_ERROR_UNSUPPORTED;
    }
    return CFB_OK;
}

// device frame slot the inverse writes for `out_format` (an output with its own staging: allocated on first use)
static cfb_error inv_frame_slot(cfb_codec *cd, int out_format, int dpitch, int rows, int slot, unsigned char **out)
{
    if (!inv_output_desc(out_format)->own_staging) { *out = (unsigned char *)cfb_codec_device_frame(cd, slot); return CFB_OK; }
    const size_t stride = ((size_t)dpitch * rows + 255) & ~(size_t)255;
    if (!cd->d_out64 || cd->out64_stride != stride) {
        CFB_CUDA(cudaSetDevice(cd->ctx->device));
        if (cd->d_out64) { CFB_CUDA(stream_wait(cd->ctx)); cudaFree(cd->d_out64); cd->d_out64 = nullptr; }
        CFB_CUDA(cudaMalloc((void **)&cd->d_out64, stride * cd->max_batch));
        cd->out64_stride = stride;
    }
    *out = cd->d_out64 + stride * slot;
    return CFB_OK;
}

cfb_error stage_inv_upload(cfb_codec *cd, int n, const void *const *h_in, bool sparse, cudaStream_t s)
{
    if (!cd || !h_in) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (n < 1 || n > cd->max_batch) { set_error("batch %d exceeds codec max_batch %d", n, cd->max_batch); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_context *ctx = cd->ctx;
    const cfb_layout &L = cd->layout;
    CFB_CUDA(cudaSetDevice(ctx->device));
    if (sparse) return sparse_upload(cd, n, h_in, s);
    const int kk = cd->decode_res - 1;
    for (int i = 0; i < n; i++) {
        if (!h_in[i]) { set_error("null host buffer %d", i); return CFB_ERROR_INVALID_ARGUMENT; }
        void *dpy = cfb_codec_device_pyramid(cd, i);
        if (kk == 0) {
            CFB_CUDA(cudaMemcpyAsync(dpy, h_in[i], (size_t)L.coded_bytes, cudaMemcpyHostToDevice, s));
            ctx->h2d_bytes += (uint64_t)L.coded_bytes;
        } else {
            // reduced resolution: each channel's bands are laid out LL3, level 3, level 2, level 1, so the levels a
            // half/quarter decode reads are one contiguous prefix per channel (the decoder skips the rest of the
            // sample the same way: decoder.c:1965-1984 decoded_subband_mask_half / _quarter)
            for (int c = 0; c < L.num_channels; c++) {
                const int64_t lo = L.band[c][CFB_NUM_LEVELS - 1][0].offset;
                const cfb_band_layout &last = L.band[c][kk][3];
                const int64_t hi = last.offset + (int64_t)last.pitch * last.height;
                CFB_CUDA(cudaMemcpyAsync((unsigned char *)dpy + lo, (const unsigned char *)h_in[i] + lo, (size_t)(hi - lo),
                                         cudaMemcpyHostToDevice, s));
                ctx->h2d_bytes += (uint64_t)(hi - lo);
            }
        }
    }
    return CFB_OK;
}

cfb_error stage_inv_compute(cfb_codec *cd, int n, const cfb_quant *quant, int out_format, bool sparse)
{
    if (!cd || !quant) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (n < 1 || n > cd->max_batch) { set_error("batch %d exceeds codec max_batch %d", n, cd->max_batch); return CFB_ERROR_INVALID_ARGUMENT; }
    int rows, rowbytes, dpitch;
    cfb_error err = inv_output_geometry(cd, out_format, &rows, &rowbytes, &dpitch);
    if (err) return err;
    if (sparse) { err = sparse_expand_device(cd, n); if (err) return err; }
    void *dpy[kMaxBatch], *dfr[kMaxBatch];
    for (int i = 0; i < n; i++) {
        dpy[i] = cfb_codec_device_pyramid(cd, i);
        unsigned char *slot = nullptr;
        err = inv_frame_slot(cd, out_format, dpitch, rows, i, &slot);
        if (err) return err;
        dfr[i] = slot;
    }
    return cfb_inverse_device(cd, n, dpy, quant, out_format, dfr, dpitch);
}

cfb_error stage_inv_download(cfb_codec *cd, int n, void *const *h_frames, int frame_pitch, int out_format, cudaStream_t s)
{
    if (!cd || !h_frames) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (n < 1 || n > cd->max_batch) { set_error("batch %d exceeds codec max_batch %d", n, cd->max_batch); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_context *ctx = cd->ctx;
    int rows, rowbytes, dpitch;
    cfb_error err = inv_output_geometry(cd, out_format, &rows, &rowbytes, &dpitch);
    if (err) return err;
    if (frame_pitch < rowbytes) { set_error("output pitch %d smaller than a row (%d bytes)", frame_pitch, rowbytes); return CFB_ERROR_INVALID_ARGUMENT; }
    CFB_CUDA(cudaSetDevice(ctx->device));
    const cfb_layout &L = cd->layout;
    const int kk = cd->decode_res - 1;
    for (int i = 0; i < n; i++) {
        if (!h_frames[i]) { set_error("null host buffer %d", i); return CFB_ERROR_INVALID_ARGUMENT; }
        unsigned char *slot = nullptr;
        err = inv_frame_slot(cd, out_format, dpitch, rows, i, &slot);
        if (err) return err;
        if (out_format == CFB_PIXEL_PLANAR16) {
            // each plane at its own width, as cfb_inverse_device writes it: the staging right of a narrower plane (4:2:2
            // chroma, the Bayer planes, reduced resolution) holds whatever an earlier job left there
            size_t doff = 0, hoff = 0;
            for (int c = 0; c < L.num_channels; c++) {
                const cfb_band_layout &b = kk ? L.band[c][kk - 1][0] : L.band[c][0][0];
                const int pw = kk ? b.width : 2 * b.width, ph = kk ? b.height : 2 * b.height;
                CFB_CUDA(cudaMemcpy2DAsync((unsigned char *)h_frames[i] + hoff, frame_pitch, slot + doff, dpitch, (size_t)pw * 2, ph,
                                           cudaMemcpyDeviceToHost, s));
                ctx->d2h_bytes += (uint64_t)pw * 2 * ph;
                doff += (size_t)dpitch * ph; hoff += (size_t)frame_pitch * ph;
            }
            continue;
        }
        if (frame_pitch == rowbytes && dpitch == rowbytes)
            CFB_CUDA(cudaMemcpyAsync(h_frames[i], slot, (size_t)rowbytes * rows, cudaMemcpyDeviceToHost, s));
        else
            CFB_CUDA(cudaMemcpy2DAsync(h_frames[i], frame_pitch, slot, dpitch, rowbytes, rows, cudaMemcpyDeviceToHost, s));
        ctx->d2h_bytes += (uint64_t)rowbytes * rows;
    }
    return CFB_OK;
}

cfb_error stage_fwd_download(cfb_codec *cd, int n, void *const *h_out, bool sparse, unsigned guess, cudaStream_t s)
{
    if (!cd || !h_out) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (n < 1 || n > cd->max_batch) { set_error("batch %d exceeds codec max_batch %d", n, cd->max_batch); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_context *ctx = cd->ctx;
    CFB_CUDA(cudaSetDevice(ctx->device));
    if (sparse) return sparse_download(cd, n, h_out, guess, s);
    for (int i = 0; i < n; i++) {
        if (!h_out[i]) { set_error("null host buffer %d", i); return CFB_ERROR_INVALID_ARGUMENT; }
        CFB_CUDA(cudaMemcpyAsync(h_out[i], cfb_codec_device_pyramid(cd, i), (size_t)cd->layout.coded_bytes, cudaMemcpyDeviceToHost, s));
        ctx->d2h_bytes += (uint64_t)cd->layout.coded_bytes;
    }
    return CFB_OK;
}

}  // namespace cfb
