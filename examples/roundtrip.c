/* roundtrip.c -- the C ABI from plain C: encode-side transform of one synthetic 4:2:2 frame to quantised bands,
 * decode-side transform back to pixels, PSNR.  No Python, no torch: this is what a C host (the reference SDK itself,
 * see INTEGRATION.md) links against.
 *
 *   gcc -O2 -I include examples/roundtrip.c -L cineform-sdk_b200 -lcfhd_b200 -Wl,-rpath,'$ORIGIN/../../cineform-sdk_b200' -lm
 *
 * Exit codes: 0 ok, 3 no usable GPU (the library has no CPU fallback and says so), 1 anything else. */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "cfhd_b200.h"

#define CHECK(call)                                                                                   \
    do {                                                                                              \
        cfb_error e_ = (call);                                                                        \
        if (e_ != CFB_OK) {                                                                           \
            fprintf(stderr, "%s failed: %d (%s)\n", #call, (int)e_, cfb_last_error_string());         \
            return e_ == CFB_ERROR_NO_DEVICE ? 3 : 1;                                                 \
        }                                                                                             \
    } while (0)

int main(int argc, char **argv)
{
    const int w = argc > 1 ? atoi(argv[1]) : 1920, h = argc > 2 ? atoi(argv[2]) : 1080;
    const int interlaced = argc > 3 ? atoi(argv[3]) : 0;
    cfb_frame_desc desc = {w, h, CFB_PIXEL_YUYV, 0};
    cfb_layout lay;
    cfb_quant quant;
    CHECK(cfb_layout_compute(&desc, &lay));                       /* host only: works without a GPU */
    CHECK(cfb_quant_for_source(&desc, 4 /* FILMSCAN1 */, interlaced, &quant));

    cfb_context *ctx = NULL;
    cfb_codec *codec = NULL;
    CHECK(cfb_context_create(0, &ctx));                           /* CFB_ERROR_NO_DEVICE without an sm_90 GPU */
    CHECK(cfb_codec_create(ctx, &desc, 1, &codec));
    if (interlaced) CHECK(cfb_codec_set_interlaced(codec, CFB_INTERLACED));

    void *frame = NULL, *coded = NULL, *out = NULL;
    CHECK(cfb_host_alloc((size_t)lay.frame_bytes, &frame));       /* pinned */
    CHECK(cfb_host_alloc((size_t)lay.coded_bytes, &coded));
    CHECK(cfb_host_alloc((size_t)lay.frame_bytes, &out));
    uint8_t *f = (uint8_t *)frame;
    uint32_t lcg = 12345u;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            lcg = lcg * 1664525u + 1013904223u;
            const int luma = 16 + (int)(100.0 + 80.0 * sin(x * 0.02) * cos(y * 0.03)) + (int)((lcg >> 24) & 3);
            f[(size_t)y * lay.frame_pitch + 2 * x] = (uint8_t)(luma > 235 ? 235 : luma);
            f[(size_t)y * lay.frame_pitch + 2 * x + 1] = (uint8_t)(128 + ((x & 2) ? 20 : -20) * ((y / 32) & 1 ? 1 : -1));
        }

    const void *frames[1] = {frame};
    void *codeds[1] = {coded};
    CHECK(cfb_forward_host(codec, 1, frames, lay.frame_pitch, &quant, codeds));
    size_t nonzero = 0;
    const int16_t *c16 = (const int16_t *)coded;
    for (int64_t i = 0; i < lay.coded_bytes / 2; i++) nonzero += c16[i] != 0;

    const void *in[1] = {coded};
    void *outs[1] = {out};
    CHECK(cfb_inverse_host(codec, 1, in, &quant, CFB_PIXEL_YUYV, outs, lay.frame_pitch));
    double mse = 0;
    const uint8_t *o = (const uint8_t *)out;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const double d = (double)o[(size_t)y * lay.frame_pitch + 2 * x] - (double)f[(size_t)y * lay.frame_pitch + 2 * x];
            mse += d * d;
        }
    mse /= (double)w * h;
    cfb_stats st;
    cfb_context_stats(ctx, &st);
    printf("{\"width\": %d, \"height\": %d, \"interlaced\": %d, \"coded_bytes\": %lld, \"nonzero_coefficients\": %zu, "
           "\"luma_psnr_db\": %.2f, \"kernel_launches\": %llu}\n",
           w, h, interlaced, (long long)lay.coded_bytes, nonzero, 10.0 * log10(255.0 * 255.0 / (mse + 1e-12)),
           (unsigned long long)st.kernel_launches);
    cfb_host_free(frame); cfb_host_free(coded); cfb_host_free(out);
    cfb_codec_destroy(codec);
    cfb_context_destroy(ctx);
    return 0;
}
