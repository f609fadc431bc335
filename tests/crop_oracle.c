/* An independent C restatement of the face crops (DESIGN.md 2, "Face crops"), built by the tests with
 * -ffp-contract=off.  It shares no code with the library: the map is evaluated from the definition's formulas in
 * plain C (every operation rounded as written), the view is applied from the orientation formulas of the header
 * (not from a resolved permutation), and pixels are sampled from the view's source rectangle cut out of the oriented
 * frame by the caller, with floor divisions instead of shifts.  sin / cos are stroke_oracle.c's restatement.
 *
 *   hco_map(rec, cw, ch, w, h, o, rect, Sw, Sh, scale, mr, mv)
 *       rec = {detection, x, y, width, height, angle}; a cw x ch canvas drawn from source rectangle rect = {sx, sy,
 *       sw, sh} of orientation o of a w x h video -> 1 and the map in the rectangle's tap coordinates (mr) and in the
 *       video's (mv), or 0 when the record makes no crop
 *   hco_crop(rgba, sw, sh, mr, dst, Sw, Sh, pitch)
 *       the crop from the sw x sh RGBA8 rectangle (tightly packed) through map mr */
#include "stroke_oracle.c"

static long long quantise(double v) { return (long long)floor(v * 65536.0 + 0.5); }

/* oriented pixel (x, y) of orientation o -> the video pixel (header: ht_video_view) */
static void video_of(int o, int w, int h, long long x, long long y, long long *vx, long long *vy) {
  const long long W = (o & 1) ? h : w;
  if (o & 4) x = W - 1 - x;
  switch (o & 3) {
    case 0: *vx = x; *vy = y; break;
    case 1: *vx = y; *vy = h - 1 - x; break;
    case 2: *vx = w - 1 - x; *vy = h - 1 - y; break;
    default: *vx = w - 1 - y; *vy = x; break;
  }
}

int hco_map(const double *rec, int cw, int ch, int w, int h, int o, const int *rect, int Sw, int Sh, double scale,
            long long *mr, long long *mv) {
  const double x = rec[1], y = rec[2], bw = rec[3], bh = rec[4], angle = rec[5];
  if ((int)rec[0] != 2 || !(bw > 0) || !(bh > 0)) return 0;
  if (!(fabs(x) <= 65536 && fabs(y) <= 65536 && fabs(bw) <= 65536 && fabs(bh) <= 65536)) return 0;
  const int sw = rect[2], sh = rect[3];
  double s, c;
  hso_sincos(angle - 1.5707963267948966, &s, &c);
  /* the stroked rectangle [rx, rx + w] x [ry, ry + h] and its centre */
  const double rx = trunc(-(bw / 2)), ry = trunc(-(bh / 2));
  const double cx = rx + bw * 0.5, cy = ry + bh * 0.5;
  /* scaled about the centre, then the shorter side grown to Sw : Sh */
  double hw = bw * scale * 0.5, hh = bh * scale * 0.5;
  const double aw = hw * Sh, ah = hh * Sw;
  if (aw < ah) hw = ah / Sh;
  else if (ah < aw) hh = aw / Sw;
  /* crop pixel centre (i + 1/2, j + 1/2) -> local (lx0 + i px, ly0 + j py) */
  const double px = hw * 2.0 / Sw, py = hh * 2.0 / Sh;
  const double lx0 = (cx - hw) + px * 0.5, ly0 = (cy - hh) + py * 0.5;
  /* translate . rotate, then the canvas -> rectangle scale, then u = x - 1/2 */
  const double X0 = x + (c * lx0 - s * ly0), Y0 = y + (s * lx0 + c * ly0);
  const double kx = (double)sw / cw, ky = (double)sh / ch;
  mr[0] = quantise(X0 * kx - 0.5);
  mr[1] = quantise(Y0 * ky - 0.5);
  mr[2] = quantise(c * px * kx);
  mr[3] = quantise(s * px * ky);
  mr[4] = quantise(-(s * py) * kx);
  mr[5] = quantise(c * py * ky);
  /* rectangle tap coordinates + (sx, sy) are oriented pixel indices; the orientation is affine on them */
  long long ax, ay, bx, by, dx, dy;
  video_of(o, w, h, rect[0], rect[1], &ax, &ay);
  video_of(o, w, h, rect[0] + 1, rect[1], &bx, &by);
  video_of(o, w, h, rect[0], rect[1] + 1, &dx, &dy);
  const long long mxx = bx - ax, myx = by - ay, mxy = dx - ax, myy = dy - ay;
  mv[0] = ax * 65536 + mxx * mr[0] + mxy * mr[1];
  mv[1] = ay * 65536 + myx * mr[0] + myy * mr[1];
  mv[2] = mxx * mr[2] + mxy * mr[3];
  mv[3] = myx * mr[2] + myy * mr[3];
  mv[4] = mxx * mr[4] + mxy * mr[5];
  mv[5] = myx * mr[4] + myy * mr[5];
  return 1;
}

static long long floor_div(long long a, long long b) {
  long long q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) --q;
  return q;
}

static const uint8_t *texel(const uint8_t *rgba, int sw, int sh, long long x, long long y) {
  static const uint8_t zero[4] = {0, 0, 0, 0};
  if (x < 0 || y < 0 || x >= sw || y >= sh) return zero;
  return rgba + 4 * ((size_t)y * sw + (size_t)x);
}

void hco_crop(const uint8_t *rgba, int sw, int sh, const long long *mr, uint8_t *dst, int Sw, int Sh, int pitch) {
  for (int j = 0; j < Sh; ++j)
    for (int i = 0; i < Sw; ++i) {
      const long long U = mr[0] + (long long)i * mr[2] + (long long)j * mr[4];
      const long long V = mr[1] + (long long)i * mr[3] + (long long)j * mr[5];
      const long long x0 = floor_div(U, 65536), y0 = floor_div(V, 65536);
      const long long fx = floor_div(U - 65536 * x0, 256), fy = floor_div(V - 65536 * y0, 256);
      const uint8_t *t[4] = {texel(rgba, sw, sh, x0, y0), texel(rgba, sw, sh, x0 + 1, y0), texel(rgba, sw, sh, x0, y0 + 1),
                             texel(rgba, sw, sh, x0 + 1, y0 + 1)};
      const long long wt[4] = {(256 - fx) * (256 - fy), fx * (256 - fy), (256 - fx) * fy, fx * fy};
      uint8_t *p = dst + (size_t)j * pitch + 4 * (size_t)i;
      for (int k = 0; k < 4; ++k) {
        long long acc = 32768;
        for (int q = 0; q < 4; ++q) acc += wt[q] * t[q][k];
        p[k] = (uint8_t)(acc / 65536);
      }
    }
}
