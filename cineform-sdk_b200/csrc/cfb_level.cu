// cfb_level.cu -- one wavelet level on a free-standing int16 plane, behind the C ABI.
//
// The codec objects (cfb_api.cu) drive the fixed intra-frame pyramid.  Other transform graphs of the reference -- the
// two-frame-GOP FIELDPLUS pyramid (Codec/encoder.c:8431 FinishFieldPlusTransformQuant, Codec/decoder.c:13109) above all --
// are compositions of the SAME single-level transforms on other planes:
//   forward  = Codec/wavelet.c:2420 TransformForwardSpatial -> spatial.c:10026 FilterSpatialQuant16s      (prescale 0)
//                                                            / spatial.c:12942 FilterSpatialV210Quant16s  (prescale 2)
//   inverse  = Codec/wavelet.c:5685 TransformInverseSpatialQuantLowpass -> spatial.c:21877 / :22414
// These entry points expose the level kernels (k_fwd_plane / k_inv_plane) for such compositions; together with
// cfb_temporal_* they are enough to build the FIELDPLUS pyramid device-resident (tests/test_gop2.py::test_cuda_gop2_device_resident
// does, and checks every band against the reference's own two-frame-GOP encode).
#include "cfb_host.h"

using namespace cfb;

static cfb_error check_level(const cfb_level_desc *d, const void *plane, const void *const *bands)
{
    if (!d || !plane || !bands) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    if (d->width < 16 || d->height < 6 || (d->width & 1) || (d->height & 1)) {
        set_error("level plane %dx%d: width even (>= 16), height even (>= 6)", d->width, d->height);
        return CFB_ERROR_UNSUPPORTED;
    }
    if (d->prescale != 0 && d->prescale != 2) { set_error("prescale %d not in {0, 2}", d->prescale); return CFB_ERROR_INVALID_ARGUMENT; }
    if (d->plane_pitch < d->width * 2 || (d->plane_pitch & 15) || d->band_pitch < d->width || (d->band_pitch & 15)) {
        set_error("pitches must cover the row and be 16-byte aligned"); return CFB_ERROR_INVALID_ARGUMENT;
    }
    uintptr_t m = (uintptr_t)plane;
    for (int b = 0; b < 4; b++) { if (!bands[b]) { set_error("null band %d", b); return CFB_ERROR_INVALID_ARGUMENT; } m |= (uintptr_t)bands[b]; }
    if (m & 15) { set_error("plane and bands must be 16-byte aligned"); return CFB_ERROR_INVALID_ARGUMENT; }
    for (int b = 0; b < 4; b++) if (d->divisor[b] < 0) { set_error("negative divisor"); return CFB_ERROR_INVALID_ARGUMENT; }
    return CFB_OK;
}

extern "C" {

cfb_error cfb_level_forward_device(cfb_context *ctx, const cfb_level_desc *d, const void *d_plane, void *const *d_bands)
{
    if (!ctx) { set_error("null context"); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_error e = check_level(d, d_plane, (const void *const *)d_bands);
    if (e) return e;
    CFB_CUDA(cudaSetDevice(ctx->device));
    FwdParams p;
    memset(&p, 0, sizeof(p));
    p.nchan = 1; p.nframes = 1;
    PlaneGeom &g = p.ch[0];
    g.width = d->width; g.height = d->height; g.in_pitch = d->plane_pitch; g.out_pitch = d->band_pitch; g.in_off = 0;
    for (int b = 0; b < 4; b++) {
        g.band_off[b] = (long long)((const unsigned char *)d_bands[b] - (const unsigned char *)d_bands[0]);
        g.q[b] = make_quant_param(d->divisor[b], d->midpoint_prequant);
    }
    // only the unprescaled planar filter quantises LL (spatial.c:10480; compiled out at :12942)
    g.quant_ll = (d->prescale == 0 && d->divisor[0] > 1);
    p.in_base[0] = (const unsigned char *)d_plane;
    p.out_base[0] = (unsigned char *)d_bands[0];
    e = audit_level_input(ctx, p, d->prescale);        // a free-standing plane may be signed: see "Value range" in the header
    if (e) return e;
    CFB_CUDA(launch_fwd_plane(ctx, p, d->prescale, false));
    return CFB_OK;
}

cfb_error cfb_level_inverse_device(cfb_context *ctx, const cfb_level_desc *d, const void *const *d_bands, void *d_plane)
{
    if (!ctx) { set_error("null context"); return CFB_ERROR_INVALID_ARGUMENT; }
    cfb_error e = check_level(d, d_plane, d_bands);
    if (e) return e;
    CFB_CUDA(cudaSetDevice(ctx->device));
    InvParams p;
    memset(&p, 0, sizeof(p));
    p.nchan = 1; p.nframes = 1;
    InvGeom &g = p.ch[0];
    g.width = d->width / 2; g.height = d->height / 2; g.pitch = d->band_pitch; g.out_pitch = d->plane_pitch; g.out_off = 0;
    for (int b = 0; b < 4; b++) {
        g.band_off[b] = (long long)((const unsigned char *)d_bands[b] - (const unsigned char *)d_bands[0]);
        g.dq[b] = d->divisor[b] > 1 ? d->divisor[b] : 1;
    }
    if (g.dq[0] != 1) { set_error("the inverse level carries LL undequantised (divisor[0] must be <= 1)"); return CFB_ERROR_UNSUPPORTED; }
    p.in_base[0] = (const unsigned char *)d_bands[0];
    p.out_base[0] = (unsigned char *)d_plane;
    CFB_CUDA(launch_inv_plane(ctx, p, d->prescale));
    return CFB_OK;
}

// Host-buffer forms: stage the plane and the four bands through stream-ordered device allocations.
static cfb_error level_host(cfb_context *ctx, bool forward, const cfb_level_desc *d, void *plane, void *const *bands)
{
    if (!ctx || !d || !plane || !bands) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    for (int b = 0; b < 4; b++) if (!bands[b]) { set_error("null band %d", b); return CFB_ERROR_INVALID_ARGUMENT; }
    if (d->width <= 0 || d->height <= 0 || d->plane_pitch < d->width * 2 || d->band_pitch < d->width) { set_error("bad geometry"); return CFB_ERROR_INVALID_ARGUMENT; }
    CFB_CUDA(cudaSetDevice(ctx->device));
    cfb_level_desc dd = *d;
    dd.plane_pitch = (d->width * 2 + 15) & ~15;
    dd.band_pitch = (d->width + 15) & ~15;
    const size_t plane_bytes = (size_t)dd.plane_pitch * d->height, band_bytes = (((size_t)dd.band_pitch * (d->height / 2)) + 63) & ~(size_t)63;
    unsigned char *dev = nullptr;
    CFB_CUDA(cudaMallocAsync((void **)&dev, plane_bytes + 4 * band_bytes + 64, ctx->stream));
    unsigned char *dplane = dev, *db[4];
    for (int b = 0; b < 4; b++) db[b] = dev + ((plane_bytes + 63) & ~(size_t)63) + b * band_bytes;
    cudaError_t ce = cudaSuccess;
    cfb_error err = CFB_OK;
    const size_t prow = (size_t)d->width * 2, brow = (size_t)d->width;     // bytes per plane row / band row
    if (forward) {
        ce = cudaMemcpy2DAsync(dplane, dd.plane_pitch, plane, d->plane_pitch, prow, d->height, cudaMemcpyHostToDevice, ctx->stream);
        if (ce == cudaSuccess) err = cfb_level_forward_device(ctx, &dd, dplane, (void *const *)db);
        for (int b = 0; b < 4 && ce == cudaSuccess && !err; b++)
            ce = cudaMemcpy2DAsync(bands[b], d->band_pitch, db[b], dd.band_pitch, brow, d->height / 2, cudaMemcpyDeviceToHost, ctx->stream);
    } else {
        for (int b = 0; b < 4 && ce == cudaSuccess; b++)
            ce = cudaMemcpy2DAsync(db[b], dd.band_pitch, bands[b], d->band_pitch, brow, d->height / 2, cudaMemcpyHostToDevice, ctx->stream);
        if (ce == cudaSuccess) err = cfb_level_inverse_device(ctx, &dd, (const void *const *)db, dplane);
        if (ce == cudaSuccess && !err)
            ce = cudaMemcpy2DAsync(plane, d->plane_pitch, dplane, dd.plane_pitch, prow, d->height, cudaMemcpyDeviceToHost, ctx->stream);
    }
    cudaFreeAsync(dev, ctx->stream);
    if (ce == cudaSuccess) ce = stream_wait(ctx);
    if (ce != cudaSuccess) return cuda_fail(ce, "single-level transform (host form)");
    if (!err && forward) {
        int flags = 0;
        err = range_status(ctx, &flags);
        if (!err && flags) {
            set_error("plane outside the exact-arithmetic range (flags %d: 1 = input, 2 = horizontal output beyond +-8190): the reference's saturating chains would differ", flags);
            err = CFB_ERROR_RANGE;
        }
    }
    return err;
}

cfb_error cfb_level_forward_host(cfb_context *ctx, const cfb_level_desc *d, const void *plane, void *const *bands)
{
    return level_host(ctx, true, d, (void *)plane, bands);
}

cfb_error cfb_level_inverse_host(cfb_context *ctx, const cfb_level_desc *d, const void *const *bands, void *plane)
{
    return level_host(ctx, false, d, plane, (void *const *)bands);
}

cfb_error cfb_context_range_status(cfb_context *ctx, int *flags)
{
    if (!ctx || !flags) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    return range_status(ctx, flags);
}

}  // extern "C"
