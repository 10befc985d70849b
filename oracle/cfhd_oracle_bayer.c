/* cfhd_oracle_bayer.c -- TEST INFRASTRUCTURE ONLY, see cfhd_oracle_bayer.h. */
#include <stddef.h>

#include "cfhd_oracle_bayer.h"

static int clamp16u(int v) { return v < 0 ? 0 : (v > 0xffff ? 0xffff : v); }

void orc_bayer_to_byr4(const uint16_t *g, const uint16_t *rg, const uint16_t *bg, const uint16_t *gd, int plane_pitch,
                       int width, int height, int bayer_format, const uint16_t *restore, uint16_t *out, int out_pitch)
{
    int y, x;
    for (y = 0; y < height; y++) {
        const uint16_t *G = (const uint16_t *)((const uint8_t *)g + (size_t)y * plane_pitch);
        const uint16_t *RG = (const uint16_t *)((const uint8_t *)rg + (size_t)y * plane_pitch);
        const uint16_t *BG = (const uint16_t *)((const uint8_t *)bg + (size_t)y * plane_pitch);
        const uint16_t *GD = (const uint16_t *)((const uint8_t *)gd + (size_t)y * plane_pitch);
        uint16_t *a = (uint16_t *)((uint8_t *)out + (size_t)(2 * y) * out_pitch);
        uint16_t *b = (uint16_t *)((uint8_t *)out + (size_t)(2 * y + 1) * out_pitch);
        for (x = 0; x < width; x++) {
            const int d = (int)GD[x] - 32768;                              /* bayer.c:13291 */
            int r = clamp16u((((int)RG[x] - 32768) << 1) + G[x]);           /* :13293, :13302-13310 */
            int bl = clamp16u((((int)BG[x] - 32768) << 1) + G[x]);          /* :13294 */
            int g1 = clamp16u((int)G[x] + d);                               /* :13295 */
            int g2 = clamp16u((int)G[x] - d);                               /* :13296 */
            if (restore) {                                                  /* :13313-13319 */
                r = restore[r >> 2]; g1 = restore[g1 >> 2]; g2 = restore[g2 >> 2]; bl = restore[bl >> 2];
            } else {                                                        /* :13320-13326 */
                r &= 0xfffe; g1 &= 0xfffe; g2 &= 0xfffe; bl &= 0xfffe;
            }
            switch (bayer_format) {                                         /* :13329-13355 */
            case 0: a[2 * x] = (uint16_t)r; a[2 * x + 1] = (uint16_t)g1; b[2 * x] = (uint16_t)g2; b[2 * x + 1] = (uint16_t)bl; break;
            case 1: a[2 * x] = (uint16_t)g1; a[2 * x + 1] = (uint16_t)r; b[2 * x] = (uint16_t)bl; b[2 * x + 1] = (uint16_t)g2; break;
            case 2: a[2 * x] = (uint16_t)g1; a[2 * x + 1] = (uint16_t)bl; b[2 * x] = (uint16_t)r; b[2 * x + 1] = (uint16_t)g2; break;
            default: a[2 * x] = (uint16_t)bl; a[2 * x + 1] = (uint16_t)g1; b[2 * x] = (uint16_t)g2; b[2 * x + 1] = (uint16_t)r; break;
            }
        }
    }
}
