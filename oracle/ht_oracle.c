/*
 * ht_oracle.c — CPU oracle (plain C restatement of the reference JavaScript).  See ht_oracle.h:
 * TEST INFRASTRUCTURE ONLY; never linked into or called from the product library.
 * Build: gcc -O2 -ffp-contract=off -fPIC -shared (oracle/Makefile).
 */
#include "ht_oracle.h"

#include <malloc.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* Many host threads run this oracle concurrently in bench.py's CPU baseline.  The restatement allocates
 * multi-megabyte temporaries per call (whole-frame pdf, pyramid planes) like the reference does; keep them in the
 * per-thread malloc arenas instead of mmap/munmap'ing each one, which serialises all threads in the kernel. */
__attribute__((constructor)) static void hto_init_malloc(void) {
  mallopt(M_MMAP_THRESHOLD, 1 << 30);
  mallopt(M_TRIM_THRESHOLD, 1 << 30);
  mallopt(M_ARENA_MAX, 256);
}

/* ------------------------------------------------------------------------------------------ */
/* JS number helpers                                                                           */

/* Uint8ClampedArray store (ES ToUint8Clamp): NaN->0, clamp, round half to even. */
static uint8_t js_to_uint8_clamp(double v) {
  if (!(v > 0.0)) return 0; /* NaN, negatives, -0 */
  if (v >= 255.0) return 255;
  return (uint8_t)nearbyint(v); /* default rounding mode: ties-to-even */
}

/* ES ToInt32 (used by `>> 0` and `<< 2`) */
static int32_t js_to_int32(double v) {
  if (isnan(v) || isinf(v)) return 0;
  double t = trunc(v);
  double m = fmod(t, 4294967296.0);
  if (m < 0) m += 4294967296.0;
  return (int32_t)(uint32_t)m;
}

/* ------------------------------------------------------------------------------------------ */
/* grayscale — src/ccv.js:22-32                                                                */

void hto_grayscale(const uint8_t *rgba, int w, int h, uint8_t *gray) {
  size_t n = (size_t)w * (size_t)h;
  /* the reference walks pixels last->first (ccv.js:28); per-pixel results are independent */
  for (size_t i = n; i-- > 0;) {
    double r = rgba[4 * i + 0], g = rgba[4 * i + 1], b = rgba[4 * i + 2];
    double v = r * 0.3 + g * 0.59 + b * 0.11; /* ccv.js:29, left-to-right */
    gray[i] = js_to_uint8_clamp(v);
  }
}

/* ------------------------------------------------------------------------------------------ */
/* canvas shim drawImage (defined in ht_oracle.h header comment)                               */

static inline int64_t floordiv64(int64_t a, int64_t b) { /* b > 0 */
  int64_t q = a / b;
  if ((a % b) < 0) --q;
  return q;
}

void hto_draw_image(const uint8_t *src, int src_pitch, int sx, int sy, int sw, int sh,
                    uint8_t *dst, int dst_pitch, int dw, int dh) {
  if (dw <= 0 || dh <= 0 || sw <= 0 || sh <= 0) return;
  const int64_t Dx = 2 * (int64_t)dw, Dy = 2 * (int64_t)dh;
  for (int Y = 0; Y < dh; ++Y) {
    int64_t vn = (2 * (int64_t)Y + 1) * sh - dh;
    int64_t y0 = floordiv64(vn, Dy);
    int64_t fy = vn - y0 * Dy;
    int64_t ya = y0 < 0 ? 0 : (y0 > sh - 1 ? sh - 1 : y0);
    int64_t yb = y0 + 1 < 0 ? 0 : (y0 + 1 > sh - 1 ? sh - 1 : y0 + 1);
    const uint8_t *ra = src + (size_t)(sy + ya) * src_pitch + sx;
    const uint8_t *rb = src + (size_t)(sy + yb) * src_pitch + sx;
    for (int X = 0; X < dw; ++X) {
      int64_t un = (2 * (int64_t)X + 1) * sw - dw;
      int64_t x0 = floordiv64(un, Dx);
      int64_t fx = un - x0 * Dx;
      int64_t xa = x0 < 0 ? 0 : (x0 > sw - 1 ? sw - 1 : x0);
      int64_t xb = x0 + 1 < 0 ? 0 : (x0 + 1 > sw - 1 ? sw - 1 : x0 + 1);
      int64_t num = (Dx - fx) * (Dy - fy) * ra[xa] + fx * (Dy - fy) * ra[xb] +
                    (Dx - fx) * fy * rb[xa] + fx * fy * rb[xb];
      dst[(size_t)Y * dst_pitch + X] = (uint8_t)((num + 2 * (int64_t)dw * dh) / (4 * (int64_t)dw * dh));
    }
  }
}

/* ------------------------------------------------------------------------------------------ */
/* pyramid — src/ccv.js:110-147                                                                */

struct hto_pyramid {
  hto_geom g;
  uint8_t *plane[128][4];
};

int hto_geometry(int W, int H, int interval, hto_geom *g) {
  if (W <= 0 || H <= 0 || interval < 0) return -1;
  memset(g, 0, sizeof(*g));
  double scale = pow(2.0, 1.0 / (interval + 1.0));                  /* ccv.js:110 */
  int next = interval + 1;                                           /* ccv.js:111 */
  /* cascade.width == cascade.height == 24 (ccv.js:112) */
  int scale_upto = (int)floor(log(24.0) / log(scale));
  int n_slots = scale_upto + next * 2;                               /* ccv.js:113 */
  if (n_slots > 128) return -2;
  g->interval = interval; g->next = next; g->scale_upto = scale_upto; g->n_slots = n_slots;
  g->w[0] = W; g->h[0] = H;
  for (int i = 1; i <= interval; ++i) {                              /* ccv.js:117-120 */
    g->w[i] = (int)floor((double)W / pow(scale, (double)i));
    g->h[i] = (int)floor((double)H / pow(scale, (double)i));
  }
  for (int i = next; i < n_slots; ++i) {                             /* ccv.js:124-127 */
    g->w[i] = g->w[i - next] / 2; /* Math.floor(w/2), w >= 0 */
    g->h[i] = g->h[i - next] / 2;
  }
  for (int i = 0; i < n_slots; ++i)
    if (g->w[i] <= 0 || g->h[i] <= 0) return -3; /* a browser throws on 0-sized getImageData */
  return 0;
}

hto_pyramid *hto_pyramid_build(const uint8_t *gray, int W, int H, int interval) {
  hto_geom g;
  if (hto_geometry(W, H, interval, &g) != 0) return NULL;
  hto_pyramid *p = (hto_pyramid *)calloc(1, sizeof(*p));
  p->g = g;
  const int next = g.next;
  p->plane[0][0] = (uint8_t *)malloc((size_t)W * H);
  memcpy(p->plane[0][0], gray, (size_t)W * H);
  for (int i = 1; i <= g.interval; ++i) {                            /* ccv.js:117-123 */
    p->plane[i][0] = (uint8_t *)calloc((size_t)g.w[i] * g.h[i], 1);
    hto_draw_image(p->plane[0][0], W, 0, 0, W, H, p->plane[i][0], g.w[i], g.w[i], g.h[i]);
  }
  for (int i = next; i < g.n_slots; ++i) {                           /* ccv.js:124-130 */
    const int s = i - next;
    p->plane[i][0] = (uint8_t *)calloc((size_t)g.w[i] * g.h[i], 1);
    hto_draw_image(p->plane[s][0], g.w[s], 0, 0, g.w[s], g.h[s], p->plane[i][0], g.w[i], g.w[i], g.h[i]);
  }
  for (int i = next * 2; i < g.n_slots; ++i) {                       /* ccv.js:131-147 */
    const int s = i - next;
    const int w = g.w[i], h = g.h[i]; /* == floor(w[s]/2), floor(h[s]/2) */
    for (int q = 1; q < 4; ++q) p->plane[i][q] = (uint8_t *)calloc((size_t)w * h, 1);
    /* ccv.js:135  drawImage(src, 1,0, W-1,H,   0,0, w-2,h)   */
    hto_draw_image(p->plane[s][0], g.w[s], 1, 0, g.w[s] - 1, g.h[s], p->plane[i][1], w, w - 2, h);
    /* ccv.js:140  drawImage(src, 0,1, W,H-1,   0,0, w,h-2)   */
    hto_draw_image(p->plane[s][0], g.w[s], 0, 1, g.w[s], g.h[s] - 1, p->plane[i][2], w, w, h - 2);
    /* ccv.js:145  drawImage(src, 1,1, W-1,H-1, 0,0, w-2,h-2) */
    hto_draw_image(p->plane[s][0], g.w[s], 1, 1, g.w[s] - 1, g.h[s] - 1, p->plane[i][3], w, w - 2, h - 2);
  }
  return p;
}

void hto_pyramid_free(hto_pyramid *p) {
  if (!p) return;
  for (int i = 0; i < 128; ++i)
    for (int q = 0; q < 4; ++q) free(p->plane[i][q]);
  free(p);
}

const hto_geom *hto_pyramid_geom(const hto_pyramid *p) { return &p->g; }

const uint8_t *hto_pyramid_plane(const hto_pyramid *p, int slot, int q, int *w, int *h) {
  if (slot < 0 || slot >= p->g.n_slots || q < 0 || q > 3 || !p->plane[slot][q]) return NULL;
  if (w) *w = p->g.w[slot];
  if (h) *h = p->g.h[slot];
  return p->plane[slot][q];
}

/* ------------------------------------------------------------------------------------------ */
/* cascade blob (HTC1, tools/pack_cascade.py)                                                  */

typedef struct {
  uint8_t size, pad;
  int8_t pz[5]; uint8_t px[5], py[5];
  int8_t nz[5]; uint8_t nx[5], ny[5];
} blob_feature;

typedef struct {
  uint32_t n_stages, n_features, width, height;
  const uint8_t *stages;    /* 16 B each */
  const blob_feature *feat; /* 32 B each */
  const uint8_t *alpha;     /* 16 B each */
} blob_view;

static int blob_open(const void *blob, size_t len, blob_view *v) {
  const uint8_t *b = (const uint8_t *)blob;
  if (len < 24 || memcmp(b, "HTC1", 4) != 0) return -1;
  memcpy(&v->n_stages, b + 4, 4); memcpy(&v->n_features, b + 8, 4);
  memcpy(&v->width, b + 12, 4); memcpy(&v->height, b + 16, 4);
  size_t need = 24 + (size_t)v->n_stages * 16 + (size_t)v->n_features * 48;
  if (len < need || v->n_stages > 64) return -2;
  v->stages = b + 24;
  v->feat = (const blob_feature *)(v->stages + (size_t)v->n_stages * 16);
  v->alpha = (const uint8_t *)v->feat + (size_t)v->n_features * 32;
  return 0;
}
static uint32_t st_count(const blob_view *v, int j) { uint32_t c; memcpy(&c, v->stages + 16 * j, 4); return c; }
static uint32_t st_first(const blob_view *v, int j) { uint32_t c; memcpy(&c, v->stages + 16 * j + 4, 4); return c; }
static double st_thr(const blob_view *v, int j) { double c; memcpy(&c, v->stages + 16 * j + 8, 8); return c; }
static double alpha_at(const blob_view *v, uint32_t feat, int which) {
  double c; memcpy(&c, v->alpha + 16 * (size_t)feat + 8 * which, 8); return c;
}

/* ------------------------------------------------------------------------------------------ */
/* window loop — src/ccv.js:148-246                                                            */

int hto_cascade_raw(const hto_pyramid *p, const void *blob, size_t blob_len,
                    hto_rect *raw_out, int raw_cap, hto_detect_stats *stats) {
  blob_view cv;
  if (blob_open(blob, blob_len, &cv) != 0) return -1;
  const hto_geom *g = &p->g;
  const int next = g->next;
  const double scale = pow(2.0, 1.0 / (g->interval + 1.0));
  double scale_x = 1, scale_y = 1;                                    /* ccv.js:150 */
  static const int dx[4] = {0, 1, 0, 1}, dy[4] = {0, 0, 1, 1};        /* ccv.js:151-152 */
  int n_raw = 0;
  if (stats) memset(stats, 0, sizeof(*stats));
  for (int i = 0; i < g->scale_upto; ++i) {                           /* ccv.js:154 */
    const int s0 = i, s1 = i + next, s2 = i + 2 * next;
    const int qw = g->w[s2] - (int)(cv.width / 4);                    /* ccv.js:155 */
    const int qh = g->h[s2] - (int)(cv.height / 4);                   /* ccv.js:156 */
    /* ccv.js:157 step[] are RGBA byte pitches; on single-channel planes the pitch is the width */
    const int step[3] = {g->w[s0], g->w[s1], g->w[s2]};
    for (int q = 0; q < 4; ++q) {                                     /* ccv.js:178 */
      const uint8_t *u8[3] = {p->plane[s0][0], p->plane[s1][0], p->plane[s2][q]};
      const size_t plane_len[3] = {(size_t)g->w[s0] * g->h[s0], (size_t)g->w[s1] * g->h[s1],
                                   (size_t)g->w[s2] * g->h[s2]};
      for (int y = 0; y < qh; ++y) {                                  /* ccv.js:181 */
        for (int x = 0; x < qw; ++x) {                                /* ccv.js:182 */
          /* ccv.js:180,235-241: running byte offsets u8o[] == these pixel offsets */
          const size_t u8o[3] = {(size_t)(4 * x + 2 * dx[q]) + (size_t)(4 * y + 2 * dy[q]) * step[0],
                                 (size_t)(2 * x + dx[q]) + (size_t)(2 * y + dy[q]) * step[1],
                                 (size_t)x + (size_t)y * step[2]};
          double sum = 0;
          int flag = 1;
          if (stats) stats->windows++;
          for (uint32_t j = 0; j < cv.n_stages; ++j) {               /* ccv.js:185 */
            sum = 0;
            if (stats) stats->stage_entries[j]++;
            const uint32_t cnt = st_count(&cv, j), first = st_first(&cv, j);
            for (uint32_t k = 0; k < cnt; ++k) {                      /* ccv.js:189 */
              const blob_feature *f = &cv.feat[first + k];
              if (stats) stats->feature_evals++;
#define PIX(z, xx, yy) (u8o[z] + (size_t)(xx) + (size_t)(yy) * step[z])
              size_t o = PIX(f->pz[0], f->px[0], f->py[0]);
              if (o >= plane_len[f->pz[0]]) return -10; /* reference would read undefined */
              int pmin = u8[f->pz[0]][o];                             /* ccv.js:191 */
              o = PIX(f->nz[0], f->nx[0], f->ny[0]);
              if (o >= plane_len[f->nz[0]]) return -10;
              int nmax = u8[f->nz[0]][o];                             /* ccv.js:192 */
              if (pmin <= nmax) {                                     /* ccv.js:193 */
                sum += alpha_at(&cv, first + k, 0);
              } else {
                int shortcut = 1;
                for (int fi = 0; fi < f->size; ++fi) {                /* ccv.js:197 */
                  if (f->pz[fi] >= 0) {
                    o = PIX(f->pz[fi], f->px[fi], f->py[fi]);
                    if (o >= plane_len[f->pz[fi]]) return -10;
                    int pv = u8[f->pz[fi]][o];
                    if (pv < pmin) {
                      if (pv <= nmax) { shortcut = 0; break; }
                      pmin = pv;
                    }
                  }
                  if (f->nz[fi] >= 0) {
                    o = PIX(f->nz[fi], f->nx[fi], f->ny[fi]);
                    if (o >= plane_len[f->nz[fi]]) return -10;
                    int nv = u8[f->nz[fi]][o];
                    if (nv > nmax) {
                      if (pmin <= nv) { shortcut = 0; break; }
                      nmax = nv;
                    }
                  }
                }
                sum += shortcut ? alpha_at(&cv, first + k, 1) : alpha_at(&cv, first + k, 0); /* :219 */
              }
#undef PIX
            }
            if (sum < st_thr(&cv, j)) { flag = 0; break; }            /* ccv.js:222-225 */
          }
          if (flag) {                                                 /* ccv.js:227-234 */
            if (raw_out && n_raw < raw_cap) {
              hto_rect *r = &raw_out[n_raw];
              r->x = (double)(x * 4 + dx[q] * 2) * scale_x;
              r->y = (double)(y * 4 + dy[q] * 2) * scale_y;
              r->width = (double)cv.width * scale_x;
              r->height = (double)cv.height * scale_y;
              r->neighbors = 1;
              r->confidence = sum;
              r->pad_ = 0;
            }
            ++n_raw;
          }
        }
      }
    }
    scale_x *= scale;                                                 /* ccv.js:244-245 */
    scale_y *= scale;
  }
  if (stats) stats->n_raw = n_raw;
  return n_raw;
}

/* ------------------------------------------------------------------------------------------ */
/* grouping — src/ccv.js:34-107 (array_group), 249-332                                         */

static int group_pred(const hto_rect *r1, const hto_rect *r2) {       /* ccv.js:252-261 */
  double distance = floor(r1->width * 0.25 + 0.5);
  return r2->x <= r1->x + distance && r2->x >= r1->x - distance &&
         r2->y <= r1->y + distance && r2->y >= r1->y - distance &&
         r2->width <= floor(r1->width * 1.5 + 0.5) &&
         floor(r2->width * 1.5 + 0.5) >= r1->width;
}

int hto_group(const hto_rect *seq, int n, int min_neighbors, hto_rect *out, int max_out) {
  if (!(min_neighbors > 0)) {                                         /* ccv.js:249-250 */
    for (int i = 0; i < n && i < max_out; ++i) out[i] = seq[i];
    return n;
  }
  int *parent = (int *)malloc(sizeof(int) * (size_t)(n + 1));
  int *rank = (int *)malloc(sizeof(int) * (size_t)(n + 1));
  int *idx = (int *)malloc(sizeof(int) * (size_t)(n + 1));
  for (int i = 0; i < n; ++i) { parent[i] = -1; rank[i] = 0; }        /* ccv.js:37-40 */
  for (int i = 0; i < n; ++i) {                                       /* ccv.js:41-89 */
    int root = i;
    while (parent[root] != -1) root = parent[root];
    for (int j = 0; j < n; ++j) {
      if (i != j && group_pred(&seq[i], &seq[j])) {
        int root2 = j;
        while (parent[root2] != -1) root2 = parent[root2];
        if (root2 != root) {
          if (rank[root] > rank[root2]) parent[root2] = root;
          else {
            parent[root] = root2;
            if (rank[root] == rank[root2]) rank[root2]++;
            root = root2;
          }
          int temp, node2 = j;
          while (parent[node2] != -1) { temp = node2; node2 = parent[node2]; parent[temp] = root; }
          node2 = i;
          while (parent[node2] != -1) { temp = node2; node2 = parent[node2]; parent[temp] = root; }
        }
      }
    }
  }
  int class_idx = 0;                                                  /* ccv.js:90-105 */
  for (int i = 0; i < n; ++i) {
    int node1 = i;
    while (parent[node1] != -1) node1 = parent[node1];
    if (rank[node1] >= 0) rank[node1] = ~class_idx++;
    idx[i] = ~rank[node1];
  }
  const int ncomp = class_idx;
  hto_rect *comps = (hto_rect *)calloc((size_t)ncomp + 1, sizeof(hto_rect)); /* ccv.js:264-271 */
  for (int i = 0; i < n; ++i) {                                       /* ccv.js:274-289 */
    const hto_rect *r1 = &seq[i];
    hto_rect *c = &comps[idx[i]];
    if (c->neighbors == 0) c->confidence = r1->confidence;
    ++c->neighbors;
    c->x += r1->x; c->y += r1->y; c->width += r1->width; c->height += r1->height;
    c->confidence = (c->confidence > r1->confidence) ? c->confidence : r1->confidence; /* Math.max, no NaNs */
  }
  hto_rect *seq2 = (hto_rect *)calloc((size_t)ncomp + 1, sizeof(hto_rect));
  int n2 = 0;
  for (int i = 0; i < ncomp; ++i) {                                   /* ccv.js:293-303 */
    int nn = comps[i].neighbors;
    if (nn >= min_neighbors) {
      hto_rect *r = &seq2[n2++];
      r->x = (comps[i].x * 2 + nn) / (2 * nn);
      r->y = (comps[i].y * 2 + nn) / (2 * nn);
      r->width = (comps[i].width * 2 + nn) / (2 * nn);
      r->height = (comps[i].height * 2 + nn) / (2 * nn);
      r->neighbors = comps[i].neighbors;
      r->confidence = comps[i].confidence;
    }
  }
  int n_out = 0;
  for (int i = 0; i < n2; ++i) {                                      /* ccv.js:307-330 */
    const hto_rect *r1 = &seq2[i];
    int flag = 1;
    for (int j = 0; j < n2; ++j) {
      const hto_rect *r2 = &seq2[j];
      double distance = floor(r2->width * 0.25 + 0.5);
      int mx = r1->neighbors > 3 ? r1->neighbors : 3;
      if (i != j && r1->x >= r2->x - distance && r1->y >= r2->y - distance &&
          r1->x + r1->width <= r2->x + r2->width + distance &&
          r1->y + r1->height <= r2->y + r2->height + distance &&
          (r2->neighbors > mx || r1->neighbors < 3)) {
        flag = 0;
        break;
      }
    }
    if (flag) {
      if (n_out < max_out) out[n_out] = *r1;
      ++n_out;
    }
  }
  free(parent); free(rank); free(idx); free(comps); free(seq2);
  return n_out;
}

int hto_detect(const uint8_t *rgba, int W, int H, const void *blob, size_t blob_len,
               int interval, int min_neighbors, hto_rect *out, int max_out,
               hto_rect *raw_out, int raw_cap, hto_detect_stats *stats) {
  uint8_t *gray = (uint8_t *)malloc((size_t)W * H);
  hto_grayscale(rgba, W, H, gray);
  hto_pyramid *p = hto_pyramid_build(gray, W, H, interval);
  free(gray);
  if (!p) return -3;
  int cap = raw_cap;
  hto_rect *raw = raw_out;
  hto_rect *own = NULL;
  int n_raw;
  if (!raw) {
    cap = 1024;
    own = raw = (hto_rect *)malloc(sizeof(hto_rect) * (size_t)cap);
  }
  for (;;) {
    n_raw = hto_cascade_raw(p, blob, blob_len, raw, cap, stats);
    if (n_raw < 0 || n_raw <= cap) break;
    if (!own) { n_raw = cap; break; } /* caller's buffer too small: group what fits (documented) */
    cap = n_raw;
    own = raw = (hto_rect *)realloc(own, sizeof(hto_rect) * (size_t)cap);
  }
  hto_pyramid_free(p);
  int n = n_raw < 0 ? n_raw : hto_group(raw, n_raw, min_neighbors, out, max_out);
  free(own);
  return n;
}

/* ------------------------------------------------------------------------------------------ */
/* camshift — src/camshift.js                                                                  */

void hto_histogram(const uint8_t *d, size_t n_px, uint32_t *bins) {  /* camshift.js:49-72 */
  memset(bins, 0, 4096 * sizeof(uint32_t));
  for (size_t i = 0; i < n_px; ++i) {
    unsigned r = d[4 * i + 0] >> 4, g = d[4 * i + 1] >> 4, b = d[4 * i + 2] >> 4;
    bins[256 * r + 16 * g + b] += 1;
  }
}

void hto_weights(const uint32_t *mh, const uint32_t *ch, double *w) { /* camshift.js:314-330 */
  for (int i = 0; i < 4096; ++i) {
    double p;
    if (ch[i] != 0) {
      p = (double)mh[i] / (double)ch[i];
      if (!(p < 1)) p = 1; /* Math.min(p,1) */
    } else p = 0;
    w[i] = p;
  }
}

int hto_tracker_init(hto_tracker *t, const uint8_t *rgba, int W, int H,
                     int x, int y, int w, int h, int calc_angles) { /* camshift.js:198-211 */
  if (w <= 0 || h <= 0) return -1; /* canvas getImageData throws IndexSizeError */
  memset(t, 0, sizeof(*t));
  /* getImageData(tax,tay,taw,tah): pixels outside the canvas are transparent black */
  for (int yy = 0; yy < h; ++yy)
    for (int xx = 0; xx < w; ++xx) {
      int cx = x + xx, cy = y + yy;
      unsigned r = 0, g = 0, b = 0;
      if (cx >= 0 && cx < W && cy >= 0 && cy < H) {
        const uint8_t *p = rgba + 4 * ((size_t)cy * W + cx);
        r = p[0] >> 4; g = p[1] >> 4; b = p[2] >> 4;
      }
      t->model_hist[256 * r + 16 * g + b] += 1;
    }
  t->sx = x; t->sy = y; t->sw = w; t->sh = h;      /* _searchWindow = trackedArea.clone() */
  t->tx = t->ty = t->tw = t->th = 0; t->angle = 0; /* new TrackObj() */
  t->calc_angles = calc_angles;
  t->initialised = 1;
  return 0;
}

typedef struct { double m00, m01, m10, m11, m02, m20, invM00, xc, yc, mu20, mu02, mu11; } moments_t;

/* camshift.js:79-120 ; data is the column-major pdf: data[i][j] = pdf[i*H + j] */
static moments_t moments(const double *pdf, int H, int x, int y, int w, int h, int second) {
  moments_t m;
  memset(&m, 0, sizeof(m));
  for (int i = x; i < w; ++i) {
    const double *a = pdf + (size_t)i * H;
    double vx = i - x;
    for (int j = y; j < h; ++j) {
      double val = a[j];
      double vy = j - y;
      m.m00 += val;
      m.m01 += vy * val;
      m.m10 += vx * val;
      if (second) {
        m.m11 += vx * vy * val;
        m.m02 += vy * vy * val;
        m.m20 += vx * vx * val;
      }
    }
  }
  m.invM00 = 1 / m.m00;
  m.xc = m.m10 * m.invM00;
  m.yc = m.m01 * m.invM00;
  if (second) {
    m.mu20 = m.m20 - m.m10 * m.xc;
    m.mu02 = m.m02 - m.m01 * m.yc;
    m.mu11 = m.m11 - m.m01 * m.xc;
  } else {
    m.mu20 = m.mu02 = m.mu11 = NAN; /* `undefined` in the reference; never consumed */
  }
  return m;
}

static int imax(int a, int b) { return a > b ? a : b; }
static int imin(int a, int b) { return a < b ? a : b; }

int hto_tracker_track(hto_tracker *t, const uint8_t *rgba, int W, int H, hto_track_trace *trace) {
  if (!t->initialised) return -1;
  if (W == 0 || H == 0) return 0;                                     /* camshift.js:219 */
  /* ---- meanShift, camshift.js:261-312 ---- */
  uint32_t *cur = (uint32_t *)malloc(4096 * sizeof(uint32_t));
  double *weights = (double *)malloc(4096 * sizeof(double));
  hto_histogram(rgba, (size_t)W * H, cur);                            /* :268 */
  hto_weights(t->model_hist, cur, weights);                           /* :270 */
  /* getBackProjectionData, :332-353 : column-major whole-frame pdf */
  double *pdf = (double *)malloc(sizeof(double) * (size_t)W * H);
  for (int x = 0; x < W; ++x)
    for (int y = 0; y < H; ++y) {
      const uint8_t *p = rgba + 4 * ((size_t)y * W + x);
      pdf[(size_t)x * H + y] = weights[256 * (p[0] >> 4) + 16 * (p[1] >> 4) + (p[2] >> 4)];
    }
  moments_t m;
  memset(&m, 0, sizeof(m));
  const int iters = 10;                                               /* :277 */
  int prevx = t->sx, prevy = t->sy;                                   /* :280-281 */
  if (trace) memset(trace, 0, sizeof(*trace));
  for (int i = 0; i < iters; ++i) {                                   /* :284 */
    int wadx = imax(t->sx, 0);
    int wady = imax(t->sy, 0);
    int wadw = imin(wadx + t->sw, W);
    int wadh = imin(wady + t->sh, H);
    m = moments(pdf, H, wadx, wady, wadw, wadh, i == iters - 1);      /* :291 */
    double x = m.xc, y = m.yc;
    t->sx += js_to_int32(x - t->sw / 2.0);                            /* :295 */
    t->sy += js_to_int32(y - t->sh / 2.0);                            /* :296 */
    if (trace) { trace->wx[i] = t->sx; trace->wy[i] = t->sy; trace->n_iter = i + 1; }
    if (t->sx == prevx && t->sy == prevy) {                           /* :299 */
      m = moments(pdf, H, wadx, wady, wadw, wadh, 1);
      if (trace) trace->converged = 1;
      break;
    } else {
      prevx = t->sx;
      prevy = t->sy;
    }
  }
  t->sx = imax(0, imin(t->sx, W));                                    /* :308 */
  t->sy = imax(0, imin(t->sy, H));                                    /* :309 */
  free(cur); free(weights); free(pdf);
  if (trace) {
    trace->m00 = m.m00; trace->m10 = m.m10; trace->m01 = m.m01;
    trace->m11 = m.m11; trace->m20 = m.m20; trace->m02 = m.m02;
  }
  /* ---- camShift, camshift.js:222-259 ---- */
  double a = m.mu20 * m.invM00;
  double c = m.mu02 * m.invM00;
  if (t->calc_angles) {
    double b = m.mu11 * m.invM00;
    double d = a + c;
    double e = sqrt((4 * b * b) + ((a - c) * (a - c)));
    t->tw = (int32_t)((uint32_t)js_to_int32(sqrt((d - e) * 0.5)) << 2);
    t->th = (int32_t)((uint32_t)js_to_int32(sqrt((d + e) * 0.5)) << 2);
    t->angle = atan2(2 * b, a - c + e);
    if (t->angle < 0) t->angle = t->angle + M_PI;
  } else {
    t->tw = (int32_t)((uint32_t)js_to_int32(sqrt(a)) << 2);
    t->th = (int32_t)((uint32_t)js_to_int32(sqrt(c)) << 2);
    t->angle = M_PI / 2;
  }
  {
    double cx = t->sx + t->sw / 2.0, cy = t->sy + t->sh / 2.0;        /* :253-254 */
    double mx = cx < W ? cx : W; /* Math.min */
    double my = cy < H ? cy : H;
    t->tx = (int32_t)floor(mx > 0 ? mx : 0);
    t->ty = (int32_t)floor(my > 0 ? my : 0);
  }
  t->sw = (int32_t)floor(1.1 * t->tw);                                /* :257 */
  t->sh = (int32_t)floor(1.1 * t->th);                                /* :258 */
  return 0;
}

void hto_backprojection_img(const hto_tracker *t, const uint8_t *rgba, int W, int H, uint8_t *out) {
  uint32_t *cur = (uint32_t *)malloc(4096 * sizeof(uint32_t));
  double *weights = (double *)malloc(4096 * sizeof(double));
  hto_histogram(rgba, (size_t)W * H, cur);
  hto_weights(t->model_hist, cur, weights);
  for (size_t i = 0; i < (size_t)W * H; ++i) {                        /* camshift.js:185-194 */
    const uint8_t *p = rgba + 4 * i;
    double val = floor(255 * weights[256 * (p[0] >> 4) + 16 * (p[1] >> 4) + (p[2] >> 4)]);
    uint8_t v = js_to_uint8_clamp(val);
    out[4 * i] = v; out[4 * i + 1] = v; out[4 * i + 2] = v; out[4 * i + 3] = 255;
  }
  free(cur); free(weights);
}

/* One facetrackr VJ frame followed by its CS frames (src/facetrackr.js:67-126) in a single C call, so that the
 * CPU baseline can run one frame per host thread without Python in the loop:
 * detect -> first max-confidence candidate (:157-165) -> confidence > -10 (:97) -> floor (:101-106) ->
 * initTracker -> n_calls x track().  Returns the number of detections; *found = 1 if a tracker was seeded. */
int hto_detect_track(const uint8_t *rgba, int W, int H, const void *blob, size_t blob_len, int interval,
                     int min_neighbors, int calc_angles, int n_calls, hto_tracker *t_out, int *found) {
  hto_rect res_small[256], *res = res_small;
  int n = hto_detect(rgba, W, H, blob, blob_len, interval, min_neighbors, res, 256, NULL, 0, NULL);
  if (found) *found = 0;
  if (n <= 0) return n;
  if (n > 256) {   /* the pick is over the whole list: detect again into a list that holds it */
    res = (hto_rect *)malloc(sizeof(hto_rect) * (size_t)n);
    if (!res) return -1;
    hto_detect(rgba, W, H, blob, blob_len, interval, min_neighbors, res, n, NULL, 0, NULL);
  }
  int best = 0;
  for (int i = 1; i < n; ++i)
    if (res[i].confidence > res[best].confidence) best = i;
  const hto_rect cand = res[best];
  if (res != res_small) free(res);
  if (!(cand.confidence > -10)) return n;
  hto_tracker t;
  if (hto_tracker_init(&t, rgba, W, H, (int)floor(cand.x), (int)floor(cand.y), (int)floor(cand.width),
                       (int)floor(cand.height), calc_angles) != 0)
    return n;
  for (int c = 0; c < n_calls; ++c) hto_tracker_track(&t, rgba, W, H, NULL);
  if (t_out) *t_out = t;
  if (found) *found = 1;
  return n;
}

/* ------------------------------------------------------------------------------------------ */
/* whitebalance — src/whitebalance.js:5-29                                                     */

double hto_whitebalance(const uint8_t *rgba, int W, int H) {
  double r = 0, g = 0, b = 0;
  size_t n = (size_t)W * H;
  for (size_t i = 0; i < n; ++i) { r += rgba[4 * i]; g += rgba[4 * i + 1]; b += rgba[4 * i + 2]; }
  double avgr = r / (double)n, avgg = g / (double)n, avgb = b / (double)n;
  return (avgr + avgg + avgb) / 3;
}
