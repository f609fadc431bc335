/* An independent C restatement of face redaction (DESIGN.md 2, "Face redaction", items 2-7), built by the tests with
 * -ffp-contract=off.  It shares no code with the library: the region is evaluated from the definition's formulas in
 * plain C (every operation rounded as written), the view from its orientation table (crop_oracle.c's video_of), each
 * format's sample channels from the header's format table, and the cells by walking the grid row by row.  sin / cos
 * are stroke_oracle.c's restatement.
 *
 *   hro_rect(rec, cw, ch, w, h, o, rect, B, scale, out)
 *       rec = {detection, x, y, width, height, angle, confidence} on a cw x ch canvas drawn from a w x h video through
 *       orientation o and the resolved source rectangle rect = {sx, sy, sw, sh} -> 1 with the redacted video pixels
 *       out = {x0, y0, x1, y1} (half-open), or 0 for no face tick or an empty region
 *   hro_hold(state, hold, rec, cw, ch)
 *       state = {double x, y, width, height, angle; int32 detection, cw, ch, remaining}, all 0 at first; -> 1 if the
 *       tick redacts (state then holds the box it redacts, in rec's order), 0 if not
 *   hro_redact(format, planes, pitch, r, mode, B, fill_rgb, fill_yuv)
 *       the cells of video rectangle r of a frame of HT_YUV_ format `format` (-1: an RGBA8 frame, planes[0] with rows
 *       of pitch[0] bytes): mode 1 the integer mean of each cell's samples per channel, 2 the fill */
#include "crop_oracle.c"

static int face_tick(const double *rec) {
  const int det = (int)rec[0];
  if (det != 1 && det != 2) return 0;
  if (rec[6] == 0.0) return 0;
  if (!(rec[3] > 0) || !(rec[4] > 0)) return 0;
  for (int i = 1; i <= 4; ++i)
    if (!(fabs(rec[i]) <= 65536)) return 0;
  return 1;
}

int hro_rect(const double *rec, int cw, int ch, int w, int h, int o, const int *rect, int B, double scale, int *out) {
  out[0] = out[1] = out[2] = out[3] = 0;
  if (!face_tick(rec)) return 0;
  const double x = rec[1], y = rec[2], bw = rec[3], bh = rec[4];
  /* the box's centre in its local frame: VJ upright at (x, y) + (w/2, h/2), CS the green rectangle's */
  double s = 0.0, c = 1.0, lx = bw * 0.5, ly = bh * 0.5;
  if ((int)rec[0] == 2) {
    hso_sincos(rec[5] - 1.5707963267948966, &s, &c);
    lx = trunc(-(bw / 2)) + bw * 0.5;
    ly = trunc(-(bh / 2)) + bh * 0.5;
  }
  const double hw = bw * scale * 0.5, hh = bh * scale * 0.5;
  const int sw = rect[2], sh = rect[3];
  const double kx = (double)sw / cw, ky = (double)sh / ch;
  double lo_x = INFINITY, hi_x = -INFINITY, lo_y = INFINITY, hi_y = -INFINITY;
  const double ax[4] = {lx - hw, lx + hw, lx - hw, lx + hw}, ay[4] = {ly - hh, ly - hh, ly + hh, ly + hh};
  for (int i = 0; i < 4; ++i) {
    const double X = (x + (c * ax[i] - s * ay[i])) * kx, Y = (y + (s * ax[i] + c * ay[i])) * ky;
    lo_x = fmin(lo_x, X); hi_x = fmax(hi_x, X);
    lo_y = fmin(lo_y, Y); hi_y = fmax(hi_y, Y);
  }
  long long x0 = (long long)floor(lo_x), x1 = (long long)ceil(hi_x), y0 = (long long)floor(lo_y), y1 = (long long)ceil(hi_y);
  if (x0 < 0) x0 = 0;
  if (y0 < 0) y0 = 0;
  if (x1 > sw) x1 = sw;
  if (y1 > sh) y1 = sh;
  if (x0 >= x1 || y0 >= y1) return 0;
  /* the pixel rectangle and the whole source rectangle in video pixels: their corner pixels through the view */
  long long a[2][2], b[2][2], v[4], q[4];
  video_of(o, w, h, rect[0] + x0, rect[1] + y0, &a[0][0], &a[0][1]);
  video_of(o, w, h, rect[0] + x1 - 1, rect[1] + y1 - 1, &a[1][0], &a[1][1]);
  video_of(o, w, h, rect[0], rect[1], &b[0][0], &b[0][1]);
  video_of(o, w, h, rect[0] + sw - 1, rect[1] + sh - 1, &b[1][0], &b[1][1]);
  for (int k = 0; k < 2; ++k) {
    v[k] = a[0][k] < a[1][k] ? a[0][k] : a[1][k];
    v[k + 2] = (a[0][k] > a[1][k] ? a[0][k] : a[1][k]) + 1;
    q[k] = b[0][k] < b[1][k] ? b[0][k] : b[1][k];
    q[k + 2] = (b[0][k] > b[1][k] ? b[0][k] : b[1][k]) + 1;
  }
  /* every grid cell the rectangle meets, clipped to the source rectangle */
  for (int k = 0; k < 2; ++k) {
    long long lo = (v[k] / B) * B, hi = ((v[k + 2] + B - 1) / B) * B;
    out[k] = (int)(lo > q[k] ? lo : q[k]);
    out[k + 2] = (int)(hi < q[k + 2] ? hi : q[k + 2]);
  }
  return 1;
}

typedef struct {
  double box[5];
  int32_t det, cw, ch, remaining;
} hro_state;

int hro_hold(void *state, int hold, const double *rec, int cw, int ch) {
  hro_state st;
  memcpy(&st, state, sizeof st);
  int on = 0;
  if (face_tick(rec)) {
    for (int i = 0; i < 5; ++i) st.box[i] = rec[1 + i];
    st.det = (int)rec[0]; st.cw = cw; st.ch = ch; st.remaining = hold;
    on = 1;
  } else if ((int)rec[0] == 0 || cw != st.cw || ch != st.ch) {
    st.remaining = 0;
  } else if (st.remaining > 0) {
    st.remaining -= 1;
    on = 1;
  }
  memcpy(state, &st, sizeof st);
  return on;
}

/* one sample channel: first sample, bytes between horizontal samples, chroma shifts, 16-bit samples, RGB */
typedef struct {
  uint8_t *p;
  int pitch, step, sx, sy, wide, rgb;
} chan;

static int channels(int f, uint8_t *const *P, const int *pitch, chan out[3]) {
  /* offsets within their plane of channels 0, 1, 2, their planes, steps, shifts */
  int plane[3] = {0, 1, 2}, off[3] = {0, 0, 0}, ystep = 1, cstep = 1, sx = 1, sy = 1, wide = 0, rgb = 0;
  switch (f) {
    case -1: plane[1] = plane[2] = 0; off[1] = 1; off[2] = 2; ystep = cstep = 4; sx = sy = 0; rgb = 1; break;
    case 0: plane[2] = 1; cstep = 2; off[2] = 1; break;                                  /* NV12 */
    case 1: break;                                                                       /* I420 */
    case 16: plane[2] = 1; cstep = 2; off[1] = 1; break;                                 /* NV21 */
    case 17: sy = 0; break;                                                              /* I422 */
    case 18: sx = sy = 0; break;                                                         /* I444 */
    case 19: plane[1] = plane[2] = 0; off[1] = 1; off[2] = 3; ystep = 2; cstep = 4; sy = 0; break;   /* YUYV */
    case 20: plane[1] = plane[2] = 0; off[0] = 1; off[2] = 2; ystep = 2; cstep = 4; sy = 0; break;   /* UYVY */
    case 21: plane[2] = 1; off[2] = 2; ystep = 2; cstep = 4; wide = 1; break;            /* P010 */
    case 32: plane[1] = plane[2] = 0; off[0] = 2; off[1] = 1; ystep = cstep = 4; sx = sy = 0; rgb = 1; break;
    case 33: plane[1] = plane[2] = 0; off[0] = 2; off[1] = 1; ystep = cstep = 3; sx = sy = 0; rgb = 1; break;
    case 34: plane[1] = plane[2] = 0; off[1] = 1; off[2] = 2; ystep = cstep = 3; sx = sy = 0; rgb = 1; break;
    default: return 0;
  }
  for (int k = 0; k < 3; ++k) {
    out[k].p = P[plane[k]] + off[k];
    out[k].pitch = pitch[plane[k]];
    out[k].step = k == 0 ? ystep : cstep;
    out[k].sx = k == 0 ? 0 : sx;
    out[k].sy = k == 0 ? 0 : sy;
    out[k].wide = wide;
    out[k].rgb = rgb;
  }
  return 1;
}

static uint32_t get(const chan *c, int i, int j) {
  const uint8_t *p = c->p + (size_t)j * c->pitch + (size_t)i * c->step;
  return c->wide ? (uint32_t)p[0] | (uint32_t)p[1] << 8 : p[0];
}

static void put(const chan *c, int i, int j, uint32_t v) {
  uint8_t *p = c->p + (size_t)j * c->pitch + (size_t)i * c->step;
  p[0] = (uint8_t)v;
  if (c->wide) p[1] = (uint8_t)(v >> 8);
}

int hro_redact(int format, uint8_t *const *planes, const int *pitch, const int *r, int mode, int B,
               const uint8_t *fill_rgb, const uint8_t *fill_yuv) {
  chan ch[3];
  if (!channels(format, planes, pitch, ch)) return 0;
  for (int cy = r[1] - r[1] % B; cy < r[3]; cy += B)
    for (int cx = r[0] - r[0] % B; cx < r[2]; cx += B) {
      const int X0 = cx > r[0] ? cx : r[0], Y0 = cy > r[1] ? cy : r[1];
      const int X1 = cx + B < r[2] ? cx + B : r[2], Y1 = cy + B < r[3] ? cy + B : r[3];
      for (int k = 0; k < 3; ++k) {
        const chan *c = &ch[k];
        const int i0 = X0 >> c->sx, i1 = ((X1 - 1) >> c->sx) + 1, j0 = Y0 >> c->sy, j1 = ((Y1 - 1) >> c->sy) + 1;
        uint32_t v;
        if (mode == 1) {
          unsigned long long sum = 0, cnt = 0;
          for (int j = j0; j < j1; ++j)
            for (int i = i0; i < i1; ++i) sum += get(c, i, j), ++cnt;
          v = (uint32_t)((sum + cnt / 2) / cnt);
        } else {
          v = c->rgb ? fill_rgb[k] : fill_yuv[k];
          if (c->wide) v <<= 8;
        }
        for (int j = j0; j < j1; ++j)
          for (int i = i0; i < i1; ++i) put(c, i, j, v);
      }
    }
  return 1;
}
