/* An independent restatement of the YUV face crop conversion (DESIGN.md 2, "Face crops", item 5), for
 * tests/test_face_crop_yuv_host.py: the coefficient rows derived at run time from Kr / Kb by the rule the design states,
 * integer arithmetic with explicit floor division, and an RGBA8 image turned into NV12 or I420 planes. */
#include <math.h>
#include <stdint.h>

/* floor(a / 2^s) for any sign, without relying on >> of negative numbers */
static int floor_shift(int a, int s) {
  const int d = 1 << s;
  return a >= 0 ? a / d : -((-a + d - 1) / d);
}

static int clamp255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

/* One row: round(256 x real) each, then while the sum misses `target`, the coefficient (other than `keep`) whose
 * rounding error is largest among those that can move toward their real value moves one step. */
static void derive_row(const double real[3], int target, int keep, int out[3]) {
  for (int i = 0; i < 3; ++i) out[i] = (int)floor(256.0 * real[i] + 0.5);
  for (;;) {
    const int sum = out[0] + out[1] + out[2];
    if (sum == target) return;
    const int step = sum < target ? 1 : -1;
    int best = -1;
    double err = -1.0;
    for (int i = 0; i < 3; ++i) {
      const double e = 256.0 * real[i] - out[i];
      if (i == keep || (step > 0 ? e <= 0.0 : e >= 0.0)) continue;
      if (fabs(e) > err) err = fabs(e), best = i;
    }
    out[best] += step;
  }
}

/* color (bit 0 BT.709, bit 1 full range) -> y0, yr, yg, yb, ur, ug, ub, vr, vg, vb */
void hcyo_rows(int color, int out[10]) {
  const int bt709 = color & 1, full = (color & 2) != 0;
  const double kr = bt709 ? 0.2126 : 0.299, kb = bt709 ? 0.0722 : 0.114, kg = 1.0 - kr - kb;
  const double ys = full ? 1.0 : 219.0 / 255.0, cs = full ? 1.0 : 224.0 / 255.0;
  const double y[3] = {kr * ys, kg * ys, kb * ys};
  const double u[3] = {-kr / (1.0 - kb) / 2.0 * cs, -kg / (1.0 - kb) / 2.0 * cs, 0.5 * cs};
  const double v[3] = {0.5 * cs, -kg / (1.0 - kr) / 2.0 * cs, -kb / (1.0 - kr) / 2.0 * cs};
  out[0] = full ? 0 : 16;
  derive_row(y, full ? 256 : 220, -1, out + 1);
  derive_row(u, 0, 2, out + 4);
  derive_row(v, 0, 0, out + 7);
}

/* the luma of one pixel and the chroma of one block's sums */
static int luma(const int k[10], int r, int g, int b) { return k[0] + floor_shift(k[1] * r + k[2] * g + k[3] * b + 128, 8); }
static int chroma(const int *k, int sr, int sg, int sb) { return clamp255(128 + floor_shift(k[0] * sr + k[1] * sg + k[2] * sb + 512, 10)); }

/* n 2 x 2 blocks of RGBA8 words (p00, p01, p10, p11 each) -> 6 bytes each: the four Y, U, V */
void hcyo_blocks(int color, const uint32_t *blocks, long long n, uint8_t *out) {
  int k[10];
  hcyo_rows(color, k);
  for (long long i = 0; i < n; ++i) {
    int sr = 0, sg = 0, sb = 0;
    for (int p = 0; p < 4; ++p) {
      const uint32_t w = blocks[4 * i + p];
      const int r = w & 255, g = (w >> 8) & 255, b = (w >> 16) & 255;
      out[6 * i + p] = (uint8_t)luma(k, r, g, b);
      sr += r, sg += g, sb += b;
    }
    out[6 * i + 4] = (uint8_t)chroma(k + 4, sr, sg, sb);
    out[6 * i + 5] = (uint8_t)chroma(k + 7, sr, sg, sb);
  }
}

/* An even w x h RGBA8 image (rows of `pitch` bytes) -> planes: Y (rows of yp bytes); NV12 (nv12 = 1): U, V interleaved
 * in u (rows of up bytes); I420: U in u, V in v (rows of up and vp bytes).  Nothing else is written. */
void hcyo_convert(int color, int nv12, const uint8_t *rgba, int w, int h, int pitch, uint8_t *y, int yp, uint8_t *u,
                  int up, uint8_t *v, int vp) {
  int k[10];
  hcyo_rows(color, k);
  for (int by = 0; by < h / 2; ++by)
    for (int bx = 0; bx < w / 2; ++bx) {
      int sr = 0, sg = 0, sb = 0;
      for (int dy = 0; dy < 2; ++dy)
        for (int dx = 0; dx < 2; ++dx) {
          const uint8_t *p = rgba + (long)(2 * by + dy) * pitch + 4 * (2 * bx + dx);
          y[(long)(2 * by + dy) * yp + 2 * bx + dx] = (uint8_t)luma(k, p[0], p[1], p[2]);
          sr += p[0], sg += p[1], sb += p[2];
        }
      const int U = chroma(k + 4, sr, sg, sb), V = chroma(k + 7, sr, sg, sb);
      if (nv12) {
        u[(long)by * up + 2 * bx] = (uint8_t)U;
        u[(long)by * up + 2 * bx + 1] = (uint8_t)V;
      } else {
        u[(long)by * up + bx] = (uint8_t)U;
        v[(long)by * vp + bx] = (uint8_t)V;
      }
    }
}
