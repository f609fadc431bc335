/* An independent C restatement of the debug-canvas strokes (DESIGN.md 2, "Strokes"), built by the tests with
 * -ffp-contract=off.  It shares no code with the library: the rotation is evaluated from the definition's formulas,
 * and coverage is counted by brute force, every sample of every pixel in the outer quad's bounding box tested against
 * all edges with a multiplication, no span walk and no incremental stepping.
 *
 *   hso_sincos(t, &s, &c)              stroke_sincos
 *   hso_rect_corners(tx, ty, theta, x, y, w, h, out)
 *                                      -> number of quads (0..2); out[q][corner] = {x, y} in 1/256 px
 *   hso_stroke_rect(..., green, rgba, dw, dh, pitch), hso_stroke(rec, rgba, dw, dh, pitch)
 *                                      a stroke from main.js's calls, or from a tracker record, onto a canvas */
#include <math.h>
#include <stdint.h>
#include <string.h>

static const double PIO2_HI = 1.57079632673412561417e+00, PIO2_MID = 6.07710050630396597660e-11,
                    PIO2_LO = 2.02226624879595063154e-21, TWO_OVER_PI = 6.36619772367581382433e-01;

static double poly_sin(double r) {
  const double z = r * r, w = z * z;
  const double tail = (8.33333333332248946124e-03 + z * (-1.98412698298579493134e-04 + z * 2.75573137070700676789e-06)) +
                      (z * w) * (-2.50507602534068634195e-08 + z * 1.58969099521155010221e-10);
  return r + (z * r) * (-1.66666666666666324348e-01 + z * tail);
}

static double poly_cos(double r) {
  const double z = r * r, w = z * z;
  const double tail = z * (4.16666666666666019037e-02 + z * (-1.38888888888741095749e-03 + z * 2.48015872894767294178e-05)) +
                      (w * w) * (-2.75573143513906633035e-07 + z * (2.08757232129817482790e-09 + z * -1.13596475577881948265e-11));
  const double half = 0.5 * z, lead = 1.0 - half;
  return lead + (((1.0 - lead) - half) + z * tail);
}

void hso_sincos(double t, double *s, double *c) {
  if (!isfinite(t)) {
    *s = 0.0;
    *c = 1.0;
    return;
  }
  const double k = rint(t * TWO_OVER_PI);
  const double r = ((t - k * PIO2_HI) - k * PIO2_MID) - k * PIO2_LO;
  const double sr = poly_sin(r), cr = poly_cos(r);
  const double q4 = k - 4.0 * floor(k / 4.0);
  if (q4 == 0.0) { *s = sr; *c = cr; }
  else if (q4 == 1.0) { *s = cr; *c = -sr; }
  else if (q4 == 2.0) { *s = -sr; *c = -cr; }
  else { *s = -cr; *c = sr; }
}

static int64_t fix8(double v) { return (int64_t)floor(v * 256.0 + 0.5); }

/* one rectangle [x0, x1] x [y0, y1] of local coordinates through translate(tx, ty) . rotate */
static void place(double tx, double ty, double s, double c, double x0, double y0, double x1, double y1, int64_t q[4][2]) {
  const double xs[4] = {x0, x1, x1, x0}, ys[4] = {y0, y0, y1, y1};
  for (int i = 0; i < 4; ++i) {
    q[i][0] = fix8(tx + (c * xs[i] - s * ys[i]));
    q[i][1] = fix8(ty + (s * xs[i] + c * ys[i]));
  }
}

/* strokeRect(x, y, w, h) under translate(tx, ty) . rotate(theta) (no rotation for a non-finite theta) */
int hso_rect_corners(double tx, double ty, double theta, double x, double y, double w, double h, int64_t out[2][4][2]) {
  double s, c;
  hso_sincos(theta, &s, &c);
  if (w < 0) { x += w; w = -w; }
  if (h < 0) { y += h; h = -h; }
  if (w == 0 && h == 0) return 0;
  if (h == 0) { place(tx, ty, s, c, x, y - 0.5, x + w, y + 0.5, out[0]); return 1; }
  if (w == 0) { place(tx, ty, s, c, x - 0.5, y, x + 0.5, y + h, out[0]); return 1; }
  place(tx, ty, s, c, x - 0.5, y - 0.5, (x + w) + 0.5, (y + h) + 0.5, out[0]);
  if (w <= 1 || h <= 1) return 1;
  place(tx, ty, s, c, x + 0.5, y + 0.5, (x + w) - 0.5, (y + h) - 0.5, out[1]);
  return 2;
}

/* inside a quad whose corners run clockwise on the canvas: every cross product > 0, or == 0 on a top or left edge */
static int inside(int64_t q[4][2], int64_t px, int64_t py) {
  for (int i = 0; i < 4; ++i) {
    const int64_t ax = q[i][0], ay = q[i][1], dx = q[(i + 1) % 4][0] - ax, dy = q[(i + 1) % 4][1] - ay;
    const int64_t e = dx * (py - ay) - dy * (px - ax);
    const int top_left = dy < 0 || (dy == 0 && dx > 0);
    if (e < 0 || (e == 0 && !top_left)) return 0;
  }
  return 1;
}

/* the stroke of hso_rect_corners in #00CC00 (green) or #0000CC onto a dw x dh canvas -> the number of pixels written */
int hso_stroke_rect(double tx, double ty, double theta, double x, double y, double w, double h, int green, uint8_t *rgba,
                    int dw, int dh, int pitch) {
  int64_t q[2][4][2];
  const int nq = hso_rect_corners(tx, ty, theta, x, y, w, h, q);
  if (!nq) return 0;
  const unsigned cr = 0, cg = green ? 204 : 0, cb = green ? 0 : 204;
  int64_t x0 = q[0][0][0], x1 = x0, y0 = q[0][0][1], y1 = y0;
  for (int i = 1; i < 4; ++i) {
    if (q[0][i][0] < x0) x0 = q[0][i][0];
    if (q[0][i][0] > x1) x1 = q[0][i][0];
    if (q[0][i][1] < y0) y0 = q[0][i][1];
    if (q[0][i][1] > y1) y1 = q[0][i][1];
  }
  int64_t X0 = (int64_t)floor((double)x0 / 256.0), X1 = (int64_t)floor((double)x1 / 256.0);
  int64_t Y0 = (int64_t)floor((double)y0 / 256.0), Y1 = (int64_t)floor((double)y1 / 256.0);
  if (X0 < 0) X0 = 0;
  if (Y0 < 0) Y0 = 0;
  if (X1 > dw - 1) X1 = dw - 1;
  if (Y1 > dh - 1) Y1 = dh - 1;
  int written = 0;
  for (int64_t Y = Y0; Y <= Y1; ++Y)
    for (int64_t X = X0; X <= X1; ++X) {
      unsigned n = 0;
      for (int j = 0; j < 16; ++j)
        for (int i = 0; i < 16; ++i) {
          const int64_t px = 256 * X + 16 * i + 8, py = 256 * Y + 16 * j + 8;
          n += inside(q[0], px, py) && !(nq == 2 && inside(q[1], px, py));
        }
      if (!n) continue;
      uint8_t *p = rgba + Y * pitch + 4 * X;
      const unsigned a = (255 * n + 128) >> 8, da = p[3], A = a * 255 + da * (255 - a);
      const unsigned src[3] = {cr, cg, cb};
      for (int k = 0; k < 3; ++k) p[k] = (uint8_t)((src[k] * a * 255 + p[k] * da * (255 - a) + A / 2) / A);
      p[3] = (uint8_t)((A + 127) / 255);
      ++written;
    }
  return written;
}

/* rec = {detection, confidence, x, y, width, height, angle}: main.js's call for it (nothing when the confidence is 0,
 * the pass is not "VJ" (1) or "CS" (2), or a box field is not finite or beyond 65536 px) -> pixels written */
int hso_stroke(const double *rec, uint8_t *rgba, int dw, int dh, int pitch) {
  const int det = (int)rec[0];
  const double x = rec[2], y = rec[3], w = rec[4], h = rec[5];
  if (rec[1] == 0.0 || (det != 1 && det != 2)) return 0;
  if (!(fabs(x) <= 65536.0 && fabs(y) <= 65536.0 && fabs(w) <= 65536.0 && fabs(h) <= 65536.0)) return 0;
  if (det == 1) return hso_stroke_rect(0, 0, 0, x, y, w, h, 0, rgba, dw, dh, pitch);
  return hso_stroke_rect(x, y, rec[6] - 3.141592653589793 / 2, trunc(-(w / 2)), trunc(-(h / 2)), w, h, 1, rgba, dw, dh,
                         pitch);
}
