/* The video formats of ht_yuv_image (include/headtrackr_b200.h, DESIGN.md 2 "YUV video") -> RGBA8, restated in plain C
 * for the tests from the format table, apart from the library's code: every sample is addressed per format as the
 * table writes it, floor division by 256 is written out, and the coefficients come from a table indexed by colour.
 * Compiled by tests/test_formats_host.py into a temporary directory. */
#include <stdint.h>

/* y0, cy, rv, gu, gv, bu = round(256 x the real coefficient) */
static const int COEF[6][6] = {
    {16, 298, 409, 100, 208, 516},   /* 0: BT.601, limited range */
    {16, 298, 459, 55, 136, 541},    /* 1: BT.709, limited range */
    {0, 256, 359, 88, 183, 454},     /* 2: BT.601, full range */
    {0, 256, 403, 48, 120, 475},     /* 3: BT.709, full range */
    {16, 298, 430, 48, 167, 548},    /* 8: BT.2020, limited range */
    {0, 256, 377, 42, 146, 482},     /* 10: BT.2020, full range */
};

static const int *coef(int color) {
  switch (color) {
    case 8: return COEF[4];
    case 10: return COEF[5];
    default: return COEF[color & 3];
  }
}

static int floor_div256(int v) {
  int q = v / 256;
  if (v % 256 != 0 && v < 0) q -= 1;
  return q;
}

static uint8_t sat(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

/* a 16-bit little-endian sample reduced to 8 bits */
static int r10(const uint8_t *p) {
  const int s = p[0] | p[1] << 8;
  const int v = (s + 128) / 256;
  return v > 255 ? 255 : v;
}

static const uint8_t *at(const uint8_t *const planes[3], const int pitch[3], int p, int row, int col) {
  return planes[p] + (long)row * pitch[p] + col;
}

/* format: an HT_YUV_ value; pitch[] in bytes, all given */
void hto_format_to_rgba(const uint8_t *const planes[3], const int pitch[3], int width, int height, int format, int color,
                        uint8_t *rgba) {
  const int *k = coef(color);
  for (int y = 0; y < height; ++y) {
    for (int x = 0; x < width; ++x) {
      int Y = 0, U = 0, V = 0, R = -1, G = 0, B = 0, A = 255;
      const int hx = x / 2, hy = y / 2;
      switch (format) {
        case 0:   /* NV12 */
          Y = *at(planes, pitch, 0, y, x), U = *at(planes, pitch, 1, hy, 2 * hx), V = *at(planes, pitch, 1, hy, 2 * hx + 1);
          break;
        case 1:   /* I420 */
          Y = *at(planes, pitch, 0, y, x), U = *at(planes, pitch, 1, hy, hx), V = *at(planes, pitch, 2, hy, hx);
          break;
        case 16:  /* NV21 */
          Y = *at(planes, pitch, 0, y, x), V = *at(planes, pitch, 1, hy, 2 * hx), U = *at(planes, pitch, 1, hy, 2 * hx + 1);
          break;
        case 17:  /* I422 */
          Y = *at(planes, pitch, 0, y, x), U = *at(planes, pitch, 1, y, hx), V = *at(planes, pitch, 2, y, hx);
          break;
        case 18:  /* I444 */
          Y = *at(planes, pitch, 0, y, x), U = *at(planes, pitch, 1, y, x), V = *at(planes, pitch, 2, y, x);
          break;
        case 19:  /* YUYV */
          Y = *at(planes, pitch, 0, y, 2 * x), U = *at(planes, pitch, 0, y, 4 * hx + 1), V = *at(planes, pitch, 0, y, 4 * hx + 3);
          break;
        case 20:  /* UYVY */
          Y = *at(planes, pitch, 0, y, 2 * x + 1), U = *at(planes, pitch, 0, y, 4 * hx), V = *at(planes, pitch, 0, y, 4 * hx + 2);
          break;
        case 21:  /* P010: sample i of a row at byte 2i */
          Y = r10(at(planes, pitch, 0, y, 2 * x));
          U = r10(at(planes, pitch, 1, hy, 2 * (2 * hx)));
          V = r10(at(planes, pitch, 1, hy, 2 * (2 * hx + 1)));
          break;
        case 32:  /* BGRA */
          B = *at(planes, pitch, 0, y, 4 * x), G = *at(planes, pitch, 0, y, 4 * x + 1);
          R = *at(planes, pitch, 0, y, 4 * x + 2), A = *at(planes, pitch, 0, y, 4 * x + 3);
          break;
        case 33:  /* BGR24 */
          B = *at(planes, pitch, 0, y, 3 * x), G = *at(planes, pitch, 0, y, 3 * x + 1), R = *at(planes, pitch, 0, y, 3 * x + 2);
          break;
        default:  /* 34, RGB24 */
          R = *at(planes, pitch, 0, y, 3 * x), G = *at(planes, pitch, 0, y, 3 * x + 1), B = *at(planes, pitch, 0, y, 3 * x + 2);
          break;
      }
      uint8_t *o = rgba + 4 * ((long)y * width + x);
      if (R >= 0) {
        o[0] = (uint8_t)R, o[1] = (uint8_t)G, o[2] = (uint8_t)B, o[3] = (uint8_t)A;
        continue;
      }
      const int c = k[1] * (Y - k[0]), d = U - 128, e = V - 128;
      o[0] = sat(floor_div256(c + k[2] * e + 128));
      o[1] = sat(floor_div256(c - k[3] * d - k[4] * e + 128));
      o[2] = sat(floor_div256(c + k[5] * d + 128));
      o[3] = 255;
    }
  }
}
