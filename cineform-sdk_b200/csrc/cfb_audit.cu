// cfb_audit.cu -- range audit of a plane the forward level is about to transform ("Value range" in include/cfhd_b200.h).
//
// The level kernels compute in exact int32; the reference's SSE2 loops run saturating 16-bit chains
// (Codec/spatial.c:290-413 horizontal, :10290-10413 vertical: 0 -s x0 -s x1 +s x4 +s x5 +s 4, >> 3, +s (x2 -s x3)) and its
// scalar tails clamp or wrap once (SURVEY.md appendix A1 / A2 restate both).  All of them equal exact arithmetic when every
// chain input is at most 8190 in magnitude: the largest partial sum is then 4 * 8190 + 4 = 32764.  The horizontal
// chains read the plane (through the prescale taps (x + 3) >> 2 when prescale = 2), the vertical chains read the
// horizontal outputs, so the audit checks
//     bit 0   an input sample outside the bound (prescale 0: |x| <= 8190; prescale 2: |(x + 3) >> 2| <= 8190 and the
//             saturating lowpass sum |x0 + x1 + 6| <= 32767)
//     bit 1   a horizontal lowpass or highpass value (border filters included, clamped as the reference clamps them)
//             outside +-8190
// for every output pair of every row -- one streaming read of the plane, run only for free-standing planes
// (cfb_level_forward_*, wavelet 3 of the two-frame GOP); the codec's own sources are in range by construction.
#include "cfb_host.h"

namespace cfb {

constexpr int kChainBound = 8190;

template <int PRESCALE>
__global__ void __launch_bounds__(256) k_level_audit(const __grid_constant__ FwdParams p, int *flags)
{
    const int f = blockIdx.z / p.nchan, c = blockIdx.z - f * p.nchan;
    const PlaneGeom &g = p.ch[c];
    const int m = g.width >> 1;
    const int i = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (i >= m || r >= g.height) return;
    const short *row = reinterpret_cast<const short *>(p.in_base[f] + g.in_off + (long long)r * g.in_pitch);
    auto tap = [&](int k) { const int v = row[min(max(k, 0), g.width - 1)]; return PRESCALE ? (v + 3) >> 2 : v; };
    const int x0 = row[2 * i], x1 = row[2 * i + 1];
    int bad = 0;
    int low, high;
    if (PRESCALE) {
        if (abs(x0 + x1 + 6) > 32767) bad |= 1;
        low = (x0 + x1 + 3) >> 2;
    } else low = x0 + x1;
    const int t2 = tap(2 * i), t3 = tap(2 * i + 1);
    if (abs(t2) > kChainBound || abs(t3) > kChainBound) bad |= 1;
    if (i == 0)
        high = clamp16((5 * tap(0) - 11 * tap(1) + 4 * tap(2) + 4 * tap(3) - tap(4) - tap(5) + 4) >> 3);
    else if (i == m - 1) {
        const int n = g.width;
        high = clamp16((11 * tap(n - 2) - 5 * tap(n - 1) - 4 * tap(n - 3) - 4 * tap(n - 4) + tap(n - 5) + tap(n - 6) + 4) >> 3);
    } else
        high = ((-tap(2 * i - 2) - tap(2 * i - 1) + tap(2 * i + 2) + tap(2 * i + 3) + 4) >> 3) + t2 - t3;
    if (abs(low) > kChainBound || abs(high) > kChainBound) bad |= 2;
    if (bad) atomicOr(flags, bad);
}

cfb_error audit_level_input(cfb_context *ctx, const FwdParams &p, int prescale)
{
    if (!ctx->d_range) {
        CFB_CUDA(cudaMalloc((void **)&ctx->d_range, sizeof(int)));
        CFB_CUDA(cudaMemsetAsync(ctx->d_range, 0, sizeof(int), ctx->stream));
    }
    if (!ctx->h_range) CFB_CUDA(cudaHostAlloc((void **)&ctx->h_range, sizeof(int), cudaHostAllocPortable));
    int maxm = 0, maxh = 0;
    for (int c = 0; c < p.nchan; c++) { maxm = max(maxm, p.ch[c].width / 2); maxh = max(maxh, p.ch[c].height); }
    dim3 block(256), grid((maxm + 255) / 256, maxh, p.nframes * p.nchan);
    CFB_CUDA(launch_kernel(ctx, prescale ? k_level_audit<2> : k_level_audit<0>, grid, block, 0, p, ctx->d_range));
    return CFB_OK;
}

cfb_error range_status(cfb_context *ctx, int *flags)
{
    *flags = 0;
    if (!ctx->d_range) return CFB_OK;                   // nothing was ever audited on this context
    CFB_CUDA(cudaSetDevice(ctx->device));
    CFB_CUDA(cudaMemcpyAsync(ctx->h_range, ctx->d_range, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CFB_CUDA(cudaMemsetAsync(ctx->d_range, 0, sizeof(int), ctx->stream));
    CFB_CUDA(stream_wait(ctx));
    *flags = *ctx->h_range;
    return CFB_OK;
}

}  // namespace cfb
