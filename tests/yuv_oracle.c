/* The YUV 4:2:0 -> RGBA8 conversion of DESIGN.md 2 ("YUV video"), restated in plain C for the tests, apart from the
 * library's code: floor division by 256 is written out, the coefficients come from a table indexed by colour value, and
 * chroma is addressed per plane.  Compiled by tests/test_yuv_host.py into a temporary directory. */
#include <stdint.h>

/* y0, cy, rv, gu, gv, bu = round(256 x the real coefficient); index = color (HT_YUV_BT709 = 1, HT_YUV_FULL_RANGE = 2) */
static const int COEF[4][6] = {
    {16, 298, 409, 100, 208, 516},   /* BT.601, limited range */
    {16, 298, 459, 55, 136, 541},    /* BT.709, limited range */
    {0, 256, 359, 88, 183, 454},     /* BT.601, full range */
    {0, 256, 403, 48, 120, 475},     /* BT.709, full range */
};

static int floor_div256(int v) {
  int q = v / 256;
  if (v % 256 != 0 && v < 0) q -= 1;
  return q;
}

static uint8_t sat(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

/* format 0 = NV12 (planes[1] interleaved U, V), 1 = I420 (planes[1] = U, planes[2] = V); pitch[] in bytes, all given */
void hto_yuv_to_rgba(const uint8_t *const planes[3], const int pitch[3], int width, int height, int format, int color,
                     uint8_t *rgba) {
  const int *k = COEF[color & 3];
  for (int y = 0; y < height; ++y) {
    for (int x = 0; x < width; ++x) {
      const int cx = x / 2, cy = y / 2;
      int Y = planes[0][y * pitch[0] + x], U, V;
      if (format == 0) {
        U = planes[1][cy * pitch[1] + 2 * cx];
        V = planes[1][cy * pitch[1] + 2 * cx + 1];
      } else {
        U = planes[1][cy * pitch[1] + cx];
        V = planes[2][cy * pitch[2] + cx];
      }
      const int c = k[1] * (Y - k[0]), d = U - 128, e = V - 128;
      uint8_t *o = rgba + 4 * ((long)y * width + x);
      o[0] = sat(floor_div256(c + k[2] * e + 128));
      o[1] = sat(floor_div256(c - k[3] * d - k[4] * e + 128));
      o[2] = sat(floor_div256(c + k[5] * d + 128));
      o[3] = 255;
    }
  }
}
