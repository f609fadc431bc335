/* Independent C restatement of a stream's best shot (DESIGN.md 2, "Best shots"), for tests/test_best_shot_host.py.
 * Written from the definition, not from the library: the score of an RGBA8 image and one tick of the state.
 *
 *   gray      ccv.grayscale: R 0.3 + G 0.59 + B 0.11 in fp64, left to right, stored round-half-even (rint), at most 255
 *   score     sum over 1 <= i <= w-2, 1 <= j <= h-2 of L^2, L = 4 g(i,j) - g(i-1,j) - g(i+1,j) - g(i,j-1) - g(i,j+1),
 *             for the pixels whose alpha and whose four neighbours' alphas are all 255; uint64
 *   tick      a crop tick ("CS" = 2, width > 0, height > 0, x, y, width, height finite and within 65536) begins a
 *             track when none is open (ended == track), and sets the best on the track's first tick or when its
 *             score is strictly above the best; any other tick ends the open track.
 * Build: cc -O2 -ffp-contract=off -shared -fPIC -o libbest_shot_oracle.so best_shot_oracle.c -lm */
#include <math.h>
#include <stdint.h>
#include <string.h>

typedef struct {            /* ht_best_shot_state, 96 bytes */
  uint64_t best_score, score;
  double x, y, width, height, angle, now_ms;
  int32_t canvas_w, canvas_h;
  uint32_t track, ended, ticks, best_tick;
  int32_t buffer;
  uint32_t flags;
} hbo_state;

enum { BEGAN = 1, IMPROVED = 2, ENDED = 4 };

static int hbo_gray(const uint8_t *p) {
  volatile double r = p[0], g = p[1], b = p[2];
  volatile double t0 = r * 0.3, t1 = g * 0.59, t2 = b * 0.11;
  volatile double s = t0 + t1;
  volatile double v = s + t2;
  double q = rint(v);
  return q > 255.0 ? 255 : (int)q;
}

/* the score of a w x h RGBA8 image with rows of `pitch` bytes */
uint64_t hbo_score(const uint8_t *rgba, int w, int h, int pitch) {
  uint64_t sum = 0;
  for (int j = 1; j + 1 < h; ++j)
    for (int i = 1; i + 1 < w; ++i) {
      const uint8_t *c = rgba + (size_t)j * pitch + 4 * (size_t)i;
      const uint8_t *n[4] = {c - 4, c + 4, c - pitch, c + pitch};
      if (c[3] != 255 || n[0][3] != 255 || n[1][3] != 255 || n[2][3] != 255 || n[3][3] != 255) continue;
      const int64_t L = 4 * (int64_t)hbo_gray(c) - hbo_gray(n[0]) - hbo_gray(n[1]) - hbo_gray(n[2]) - hbo_gray(n[3]);
      sum += (uint64_t)(L * L);
    }
  return sum;
}

static int hbo_crop_tick(int det, const double f[4]) {
  if (det != 2 || !(f[2] > 0.0) || !(f[3] > 0.0)) return 0;
  for (int i = 0; i < 4; ++i)
    if (!(fabs(f[i]) <= 65536.0)) return 0;
  return 1;
}

/* ht_tracker_import on a stream with a best shot */
void hbo_end(hbo_state *s) {
  if (s->track != s->ended) {
    s->ended = s->track;
    s->flags = ENDED;
  }
}

/* one tick: rec = {detection, x, y, width, height, angle}; two: the best shot has two images -> 1 if it writes */
int hbo_step(hbo_state *s, int two, uint64_t score, const double rec[6], double now_ms, int cw, int ch) {
  s->flags = 0;
  if (!hbo_crop_tick((int)rec[0], rec + 1)) {
    hbo_end(s);
    return 0;
  }
  int began = 0;
  if (s->track == s->ended) {          /* no open track: this tick begins track t = track + 1 */
    s->track += 1;
    s->ticks = 0;
    s->buffer = two ? (int32_t)((s->track + 1u) % 2u) : 0;   /* (t - 1) mod 2 */
    began = 1;
  }
  s->score = score;
  int improved = 0;
  if (s->ticks == 0 || score > s->best_score) {
    improved = 1;
    s->best_score = score;
    s->x = rec[1]; s->y = rec[2]; s->width = rec[3]; s->height = rec[4]; s->angle = rec[5];
    s->now_ms = now_ms;
    s->canvas_w = cw; s->canvas_h = ch;
    s->best_tick = s->ticks;
  }
  s->ticks += 1;
  s->flags = (began ? BEGAN : 0) | (improved ? IMPROVED : 0);
  return improved;
}

int hbo_state_bytes(void) { return (int)sizeof(hbo_state); }
