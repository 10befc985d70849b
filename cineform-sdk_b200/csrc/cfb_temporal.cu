// cfb_temporal.cu -- two-frame GOP: temporal Haar between two int16 planes, sm_90a.
//
// Replaces (reference):
//   Codec/temporal.c:498  FilterTemporal16s       (16-bit branch :603-645)  -> k_temporal_fwd
//   Codec/temporal.c:9402 InvertTemporalQuant16s                            -> k_temporal_inv
// In the reference's TRANSFORM_TYPE_FIELDPLUS pyramid these run between the level-1 lowpass images of frame A and
// frame B (wavelet[2], Codec/encoder.c:8431 FinishFieldPlusTransformQuant / Codec/decoder.c:13109); the spatial
// levels either side are the same kernels as the intra-frame pyramid (k_fwd_plane / k_inv_plane).
//
// Pure streaming: one thread = 8 coefficients of each input (two 128-bit loads, two 128-bit stores), rows on
// blockIdx.y.  HBM-bound: 8 bytes moved per coefficient pair.
#include "cfb_host.h"

namespace cfb {

__device__ __forceinline__ int sat16i(int v) { return max(-32768, min(32767, v)); }

__global__ void __launch_bounds__(256) k_temporal_fwd(const unsigned char *a, const unsigned char *b, int in_pitch,
                                                       unsigned char *low, unsigned char *high, int out_pitch,
                                                       int width, int height)
{
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const uint4 va = __ldg(reinterpret_cast<const uint4 *>(a + (long long)y * in_pitch + x * 2));
    const uint4 vb = __ldg(reinterpret_cast<const uint4 *>(b + (long long)y * in_pitch + x * 2));
    // per-halfword saturating add / subtract == _mm_adds_epi16 / _mm_subs_epi16
    const uint4 lo = make_uint4(__vaddss2(va.x, vb.x), __vaddss2(va.y, vb.y), __vaddss2(va.z, vb.z), __vaddss2(va.w, vb.w));
    const uint4 hi = make_uint4(__vsubss2(vb.x, va.x), __vsubss2(vb.y, va.y), __vsubss2(vb.z, va.z), __vsubss2(vb.w, va.w));
    *reinterpret_cast<uint4 *>(low + (long long)y * out_pitch + x * 2) = lo;
    *reinterpret_cast<uint4 *>(high + (long long)y * out_pitch + x * 2) = hi;
}

// post = width - width % 40: columns below it follow the reference's SSE2 loop (saturating), the rest its scalar tail
__global__ void __launch_bounds__(256) k_temporal_inv(const unsigned char *low, const unsigned char *high, int in_pitch,
                                                       unsigned char *a, unsigned char *b, int out_pitch,
                                                       int width, int height, int post, int halftone)
{
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const uint4 vl = __ldg(reinterpret_cast<const uint4 *>(low + (long long)y * in_pitch + x * 2));
    const uint4 vh = __ldg(reinterpret_cast<const uint4 *>(high + (long long)y * in_pitch + x * 2));
    const unsigned l[4] = {vl.x, vl.y, vl.z, vl.w}, h[4] = {vh.x, vh.y, vh.z, vh.w};
    unsigned oa[4], ob[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        int e[2], o[2];
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int c = x + 2 * k + s;
            const int lv = s ? hi16(l[k]) : lo16(l[k]), hv = s ? hi16(h[k]) : lo16(h[k]);
            if (c < post) {
                const int t = halftone ? ((c + y + 1) & 1) : 0;
                e[s] = sat16i(lv - hv) >> 1;
                o[s] = sat16i(sat16i(lv + hv) + t) >> 1;
            } else {
                const int t = halftone ? ((c + y) & 1) : 0;
                e[s] = (lv - hv) >> 1;          // int arithmetic, truncated to int16 on store (temporal.c:9617-9640)
                o[s] = (lv + hv + t) >> 1;
            }
        }
        oa[k] = pack_lo(e[0], e[1]);
        ob[k] = pack_lo(o[0], o[1]);
    }
    *reinterpret_cast<uint4 *>(a + (long long)y * out_pitch + x * 2) = make_uint4(oa[0], oa[1], oa[2], oa[3]);
    *reinterpret_cast<uint4 *>(b + (long long)y * out_pitch + x * 2) = make_uint4(ob[0], ob[1], ob[2], ob[3]);
}

static cfb_error check_planes(const void *p0, const void *p1, const void *p2, const void *p3, int in_pitch, int out_pitch,
                              int width, int height)
{
    if (!p0 || !p1 || !p2 || !p3) { set_error("null plane"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (width <= 0 || height <= 0 || (width & 15)) { set_error("temporal transform: width %d must be a positive multiple of 16 (temporal.c:616)", width); return CFB_ERROR_INVALID_ARGUMENT; }
    if (in_pitch < width * 2 || out_pitch < width * 2 || (in_pitch & 15) || (out_pitch & 15)) { set_error("pitches must be >= 2*width and 16-byte aligned"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (((uintptr_t)p0 | (uintptr_t)p1 | (uintptr_t)p2 | (uintptr_t)p3) & 15) { set_error("planes must be 16-byte aligned"); return CFB_ERROR_INVALID_ARGUMENT; }
    return CFB_OK;
}

static inline dim3 plane_grid(int width, int height, dim3 block)
{
    return dim3((width / 8 + block.x - 1) / block.x, (height + block.y - 1) / block.y, 1);
}

}  // namespace cfb

using namespace cfb;

extern "C" {

cfb_error cfb_temporal_forward_device(cfb_context *ctx, const void *d_frame1, const void *d_frame2, int in_pitch,
                                      void *d_low, void *d_high, int out_pitch, int width, int height)
{
    if (!ctx) { set_error("null context"); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_error e = check_planes(d_frame1, d_frame2, d_low, d_high, in_pitch, out_pitch, width, height);
    if (e) return e;
    CFB_CUDA(cudaSetDevice(ctx->device));
    const dim3 block(32, 8);
    CFB_CUDA(launch_kernel(ctx, k_temporal_fwd, plane_grid(width, height, block), block, 0, (const unsigned char *)d_frame1,
                           (const unsigned char *)d_frame2, in_pitch, (unsigned char *)d_low, (unsigned char *)d_high, out_pitch,
                           width, height));
    return CFB_OK;
}

cfb_error cfb_temporal_inverse_device(cfb_context *ctx, const void *d_low, const void *d_high, int in_pitch,
                                      void *d_frame1, void *d_frame2, int out_pitch, int width, int height, int precision)
{
    if (!ctx) { set_error("null context"); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_error e = check_planes(d_low, d_high, d_frame1, d_frame2, in_pitch, out_pitch, width, height);
    if (e) return e;
    if (precision != 8 && precision != 10 && precision != 12) { set_error("precision %d not in {8, 10, 12}", precision); return CFB_ERROR_INVALID_ARGUMENT; }
    CFB_CUDA(cudaSetDevice(ctx->device));
    const dim3 block(32, 8);
    CFB_CUDA(launch_kernel(ctx, k_temporal_inv, plane_grid(width, height, block), block, 0, (const unsigned char *)d_low,
                           (const unsigned char *)d_high, in_pitch, (unsigned char *)d_frame1, (unsigned char *)d_frame2, out_pitch,
                           width, height, width - (width % 40), precision == 8));
    return CFB_OK;
}

// Host-buffer convenience forms: stage both planes through stream-ordered device allocations.
static cfb_error temporal_host(cfb_context *ctx, bool forward, const void *in0, const void *in1, int in_pitch,
                               void *out0, void *out1, int out_pitch, int width, int height, int precision)
{
    if (!ctx || !in0 || !in1 || !out0 || !out1) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (width <= 0 || height <= 0 || in_pitch < width * 2 || out_pitch < width * 2) { set_error("bad geometry"); return CFB_ERROR_INVALID_ARGUMENT; }
    CFB_CUDA(cudaSetDevice(ctx->device));
    const int dp = (width * 2 + 15) & ~15;
    const size_t plane = (size_t)dp * height;
    unsigned char *d = nullptr;
    CFB_CUDA(cudaMallocAsync((void **)&d, 4 * plane, ctx->stream));
    cfb_error err = CFB_OK;
    cudaError_t ce = cudaMemcpy2DAsync(d, dp, in0, in_pitch, (size_t)width * 2, height, cudaMemcpyHostToDevice, ctx->stream);
    if (ce == cudaSuccess) ce = cudaMemcpy2DAsync(d + plane, dp, in1, in_pitch, (size_t)width * 2, height, cudaMemcpyHostToDevice, ctx->stream);
    if (ce == cudaSuccess) {
        err = forward ? cfb_temporal_forward_device(ctx, d, d + plane, dp, d + 2 * plane, d + 3 * plane, dp, width, height)
                      : cfb_temporal_inverse_device(ctx, d, d + plane, dp, d + 2 * plane, d + 3 * plane, dp, width, height, precision);
    }
    if (ce == cudaSuccess && !err) ce = cudaMemcpy2DAsync(out0, out_pitch, d + 2 * plane, dp, (size_t)width * 2, height, cudaMemcpyDeviceToHost, ctx->stream);
    if (ce == cudaSuccess && !err) ce = cudaMemcpy2DAsync(out1, out_pitch, d + 3 * plane, dp, (size_t)width * 2, height, cudaMemcpyDeviceToHost, ctx->stream);
    cudaFreeAsync(d, ctx->stream);
    if (ce == cudaSuccess) ce = stream_wait(ctx);
    if (ce != cudaSuccess) return cuda_fail(ce, "temporal transform (host form)");
    if (!err) { ctx->h2d_bytes += 2 * (uint64_t)width * 2 * height; ctx->d2h_bytes += 2 * (uint64_t)width * 2 * height; }
    return err;
}

cfb_error cfb_temporal_forward_host(cfb_context *ctx, const void *frame1, const void *frame2, int in_pitch,
                                    void *low, void *high, int out_pitch, int width, int height)
{
    return temporal_host(ctx, true, frame1, frame2, in_pitch, low, high, out_pitch, width, height, 10);
}

cfb_error cfb_temporal_inverse_host(cfb_context *ctx, const void *low, const void *high, int in_pitch,
                                    void *frame1, void *frame2, int out_pitch, int width, int height, int precision)
{
    return temporal_host(ctx, false, low, high, in_pitch, frame1, frame2, out_pitch, width, height, precision);
}

}  // extern "C"
