/* cfhd_oracle_bayer.h -- TEST INFRASTRUCTURE ONLY (as cfhd_oracle.h: never linked into the product).
 *
 * Scalar restatement of the Bayer reconstruction of the reference decoder's BYR4 output, built into
 * oracle/liboracle_bayer.so (bayer.mk) and pinned byte for byte to the unmodified reference by tests/test_output_byr4.py.
 * Paths and lines are those of the reference tree, as in cfhd_oracle.h.
 */
#ifndef CFHD_ORACLE_BAYER_H
#define CFHD_ORACLE_BAYER_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Bayer samples decoded to BYR4: the four unsigned 16-bit rows of the final inverse level -> the mosaic.
 * Codec/bayer.c:13237 GenerateBYR2 (the worker of DECODED_FORMAT_BYR2 / BYR4, decoder.c:14738-14767), one plane row ->
 * two mosaic rows.  g, rg, bg, gd = the ...ToRow16u rows of channels 0-3 (decoder.c:14629 -> InvertHorizontalStrip16s.c:17462
 * InvertHorizontalStrip16sToRow16uPlanar -> :16571; tests/parity_util.row16u restates them):
 *   d = GD - 32768;  r = ((RG - 32768) << 1) + G;  b = ((BG - 32768) << 1) + G;  g1 = G + d;  g2 = G - d,  each limited
 *   to [0, 65535]; then restore[v >> 2] (restore != NULL: the decoder's BYR4LinearRestore table, 16384 entries,
 *   decoder.c:10714-10785, used when encode_curve_preset == 0) or v & 0xfffe (restore == NULL: encode_curve_preset == 1).
 * The 2 x 2 cell is R G1 / G2 B, G1 R / B G2, G1 B / R G2, B G1 / G2 R for bayer_format 0-3 (BAYER_FORMAT_RED_GRN,
 * GRN_RED, GRN_BLU, BLU_GRN).  width / height = plane dimensions; out is 2 * width x 2 * height; pitches in bytes. */
void orc_bayer_to_byr4(const uint16_t *g, const uint16_t *rg, const uint16_t *bg, const uint16_t *gd, int plane_pitch,
                       int width, int height, int bayer_format, const uint16_t *restore, uint16_t *out, int out_pitch);

#ifdef __cplusplus
}
#endif
#endif
