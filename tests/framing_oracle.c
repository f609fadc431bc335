/* An independent C restatement of a stream's framing (DESIGN.md 2, "Face crops", item 7), built by the tests with
 * -ffp-contract=off.  It shares no code with the library: the update is evaluated from the definition's formulas in
 * plain C (every operation rounded as written), the box layout is restated from the header's byte offsets, and the
 * framed crop's map is crop_oracle.c's map with the framed geometry (local centre 0, no rotation, the box's centre
 * and size).  sin / cos are stroke_oracle.c's restatement.
 *
 *   hfo_step(box, alpha, dead_zone, rec, cw, ch)
 *       box: 48 bytes of ht_framed_box; rec = {detection, x, y, width, height, angle} on a cw x ch canvas
 *       -> 1 on a crop tick (box updated), 0 otherwise (box unchanged)
 *   hfo_map(box, cw, ch, w, h, o, rect, Sw, Sh, scale, mr, mv)
 *       as crop_oracle.c's hco_map, for a crop cut from the framed box -> 1, or 0 for a box that is not valid */
#include "crop_oracle.c"

typedef struct {
  double v[4];            /*  0 cx, cy, width, height */
  int32_t cw, ch;         /* 32 canvas_w, canvas_h */
  uint32_t updates;       /* 40 */
  int32_t valid;          /* 44 */
} hfo_box;

static int makes_crop(int det, double x, double y, double w, double h) {
  return det == 2 && w > 0 && h > 0 && fabs(x) <= 65536 && fabs(y) <= 65536 && fabs(w) <= 65536 && fabs(h) <= 65536;
}

/* v moved towards t: only by the part of the error outside the band, times alpha */
static double glide(double v, double t, double band, double alpha) {
  const double e = t - v;
  if (!(fabs(e) > band)) return v;
  return v + alpha * (e - (e < 0 ? -band : band));
}

int hfo_step(void *box, double alpha, double dead_zone, const double *rec, int cw, int ch) {
  hfo_box b;
  memcpy(&b, box, sizeof b);
  const double x = rec[1], y = rec[2], w = rec[3], h = rec[4];
  if (!makes_crop((int)rec[0], x, y, w, h)) return 0;
  double s, c;
  hso_sincos(rec[5] - 1.5707963267948966, &s, &c);
  /* the green rectangle [trunc(-w/2), + w] x [trunc(-h/2), + h] about (x, y): its centre */
  const double lx = trunc(-(w / 2)) + w * 0.5, ly = trunc(-(h / 2)) + h * 0.5;
  const double tx = x + (c * lx - s * ly), ty = y + (s * lx + c * ly);
  const int snap = !b.valid || b.cw != cw || b.ch != ch || fabs(tx - b.v[0]) > b.v[2] / 2 || fabs(ty - b.v[1]) > b.v[3] / 2;
  if (snap) {
    b.v[0] = tx; b.v[1] = ty; b.v[2] = w; b.v[3] = h;
    b.cw = cw; b.ch = ch; b.valid = 1;
  } else {
    const double W = b.v[2], H = b.v[3];
    const double t[4] = {tx, ty, w, h}, band[4] = {dead_zone * W, dead_zone * H, dead_zone * W, dead_zone * H};
    for (int i = 0; i < 4; ++i) b.v[i] = glide(b.v[i], t[i], band[i], alpha);
  }
  b.updates += 1;
  memcpy(box, &b, sizeof b);
  return 1;
}

int hfo_map(const void *box, int cw, int ch, int w, int h, int o, const int *rect, int Sw, int Sh, double scale,
            long long *mr, long long *mv) {
  hfo_box b;
  memcpy(&b, box, sizeof b);
  if (!b.valid || !makes_crop(2, b.v[0], b.v[1], b.v[2], b.v[3])) return 0;
  const int sw = rect[2], sh = rect[3];
  double hw = b.v[2] * scale * 0.5, hh = b.v[3] * scale * 0.5;
  const double aw = hw * Sh, ah = hh * Sw;
  if (aw < ah) hw = ah / Sh;
  else if (ah < aw) hh = aw / Sw;
  const double px = hw * 2.0 / Sw, py = hh * 2.0 / Sh;
  /* upright: the crop's first pixel centre is the box's corner plus half a crop pixel */
  const double X0 = b.v[0] + ((0.0 - hw) + px * 0.5), Y0 = b.v[1] + ((0.0 - hh) + py * 0.5);
  const double kx = (double)sw / cw, ky = (double)sh / ch;
  mr[0] = quantise(X0 * kx - 0.5);
  mr[1] = quantise(Y0 * ky - 0.5);
  mr[2] = quantise(px * kx);
  mr[3] = 0;
  mr[4] = 0;
  mr[5] = quantise(py * ky);
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
