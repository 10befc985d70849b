// ref_probe_bayer.cpp -- TEST INFRASTRUCTURE ONLY.
//
// A shim beside ref_probe.cpp, compiled against the UNMODIFIED reference headers and linked to oracle/_ref/libcfhd_ref.so
// into oracle/_ref/libcfhd_ref_bayer.so (bayer.mk).  It contains no codec logic: it marshals buffers, sets two fields of
// the decoder's metadata and calls the reference's own decoder.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

extern "C" {
#include "config.h"
#include "image.h"
#include "wavelet.h"
#include "bitstream.h"
#include "codec.h"
#include "decoder.h"
}

extern "C" {

// Codec-level decode of a Bayer sample (Codec/decoder.c:1497 DecodeInit + :10078 DecodeSample) to DECODED_FORMAT_BYR4 (or any
// other decoded_format) at full resolution, with the Bayer phase (cfhddata.bayer_format) and curve mode
// (cfhddata.encode_curve_preset) given by the caller.  The encoder's own bayer.format / encode_curve_preset never reach the
// decoder: EncodeSample writes them only as metadata the SDK attaches (TAG_BAYER_FORMAT, TAG_ENCODE_PRESET), and the decoder
// resets both to 0 on its first sample (lutpath.cpp:980-982, :1301).  So the sample is decoded once, both fields are set on
// the decoder, and it is decoded again.  bayer_format < 0: one decode with the decoder's defaults.
// Outputs as ref_decode_sample_bands of ref_probe.cpp: dims[(c*3+k)*3] = {width, height, pitch}, quant[c*12 + k*4 + b], bands
// dense and concatenated in (c, level, band) order (highpass dequantised, LL3 raw), plus
//   state[3] = {bayer_format, encode_curve_preset the decoder holds after the decode, 1 if it built BYR4LinearRestore}
//   restore  = the 16384 entries of decoder->BYR4LinearRestore (decoder.c:10714-10785) when built.
// Returns 0 on success.
int ref_decode_bayer_bands(const uint8_t *sample, int64_t size, int width, int height, int decoded_format, int num_channels,
                           int bayer_format, int encode_curve_preset, uint8_t *out, int out_pitch,
                           int32_t *dims, int32_t *quant, int16_t *bands, int64_t bands_capacity, int32_t *state, uint16_t *restore)
{
    DECODER *dec = (DECODER *)calloc(1, DecoderSize());
    if (!dec || !DecodeInit(NULL, dec, width, height, decoded_format, DECODED_RESOLUTION_FULL, NULL)) return 1;
    SetDecoderColorFlags(dec, COLOR_SPACE_CG_709);
    SetDecoderFlags(dec, DECODER_FLAGS_RENDER);      // as CSampleDecoder::DecodeSample does (SampleDecoder.cpp:1507)
    void *smp = NULL, *o = NULL;
    const size_t obytes = (size_t)out_pitch * (height + 16) + 64;
    if (posix_memalign(&smp, 64, (size_t)size + 64) || posix_memalign(&o, 64, obytes)) return 1;
    memset(smp, 0, (size_t)size + 64);
    memset(o, 0, obytes);
    memcpy(smp, sample, (size_t)size);
    for (int pass = 0; pass < (bayer_format >= 0 ? 2 : 1); pass++) {
        if (pass) {
            dec->cfhddata.bayer_format = bayer_format;
            dec->cfhddata.encode_curve_preset = encode_curve_preset;
        }
        BITSTREAM bs;
        InitBitstreamBuffer(&bs, (uint8_t *)smp, (size_t)size, BITSTREAM_ACCESS_READ);
        if (!DecodeSample(dec, &bs, (uint8_t *)o, out_pitch, NULL, NULL)) return 2;
    }
    state[0] = (int32_t)dec->cfhddata.bayer_format;
    state[1] = (int32_t)dec->cfhddata.encode_curve_preset;
    state[2] = dec->BYR4LinearRestore ? 1 : 0;
    if (dec->BYR4LinearRestore) memcpy(restore, dec->BYR4LinearRestore, 16384 * sizeof(uint16_t));
    memcpy(out, o, (size_t)out_pitch * height);
    int64_t pos = 0;
    for (int c = 0; c < num_channels; c++) {
        for (int k = 0; k < 3; k++) {
            IMAGE *w = dec->transform[c]->wavelet[k];
            if (!w) return 3;
            dims[(c * 3 + k) * 3 + 0] = w->width; dims[(c * 3 + k) * 3 + 1] = w->height; dims[(c * 3 + k) * 3 + 2] = w->pitch;
            for (int b = 0; b < 4; b++) {
                quant[c * 12 + k * 4 + b] = w->quantization[b];
                if (pos + (int64_t)w->width * w->height > bands_capacity) return 4;
                for (int r = 0; r < w->height; r++)
                    memcpy(bands + pos + (int64_t)r * w->width, (uint8_t *)w->band[b] + (size_t)r * w->pitch, (size_t)w->width * 2);
                pos += (int64_t)w->width * w->height;
            }
        }
    }
    free(smp); free(o);
    return 0;
}

}  // extern "C"
