// ht_track.cuh — sm_90a kernels for camshift.Tracker (src/camshift.js) and
// getWhitebalance (src/whitebalance.js) of the reference.
//
// The reference materialises a whole-frame back-projection (307,200 doubles in nested arrays,
// src/camshift.js:332-353) on every track(); here the weight of a pixel is looked up on the fly
// inside the search window, so a track() costs one streaming histogram pass over the frame plus a
// few window passes that stay in L2.
#pragma once
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstring>
#include <limits>

#include "ht_common.cuh"

namespace ht {

// rgb_bin() (src/camshift.js:63-66, 345-348) is defined in ht_detect.cuh: the fused gray pass uses it too.

// ------------------------------------------------------------------------------------------------
// K1'  4096-bin RGB histogram of whole frames — src/camshift.js:49-72 via :268 — plus the per-pixel
// bin plane (u16) that k_track's window passes read instead of re-decoding RGBA (half the bytes).  The plane
// holds 8 * bin: the byte offset of the pixel's weight in k_track's fp64 table (8 * 4095 < 2^16).
// grid = (chunks, n_frames).  Shared-memory histogram per CTA, flushed to hist[frame][4096].
__global__ void __launch_bounds__(256) k_hist(const uint8_t *__restrict__ rgba, size_t frame_bytes, int n_px,
                                              uint32_t *__restrict__ hist, uint16_t *__restrict__ bins, int chunks,
                                              const uint8_t *__restrict__ enable) {
  __shared__ uint32_t sh[4096];
  if (enable && !enable[blockIdx.y]) return;   // ht_stream_step: only the streams that are tracking
  for (int i = threadIdx.x; i < 4096; i += 256) sh[i] = 0;
  __syncthreads();
  const uint32_t *px = reinterpret_cast<const uint32_t *>(rgba + (size_t)blockIdx.y * frame_bytes);
  uint16_t *bout = bins ? bins + (size_t)blockIdx.y * n_px : nullptr;
  const int n_pair = (n_px + 1) / 2;
  const int per = (n_pair + chunks - 1) / chunks;
  const int beg = blockIdx.x * per, end = min(n_pair, beg + per);
  // the 8 B load / 4 B store of the paired path need this FRAME's pointers aligned: with an odd w*h every odd frame
  // index starts at 4 mod 8 (and its bin plane at 2 mod 4), and the caller's pointer is only 4-byte aligned
  const bool paired = ((reinterpret_cast<uintptr_t>(px) & 7u) == 0) && (!bout || (reinterpret_cast<uintptr_t>(bout) & 3u) == 0);
  for (int i = beg + threadIdx.x; i < end; i += 256) {
    const int p0 = 2 * i;
    if (!paired) {
      for (int p = p0; p < min(p0 + 2, n_px); ++p) {
        const uint32_t b0 = rgb_bin(__ldg(px + p));
        atomicAdd(&sh[b0], 1u);
        if (bout) bout[p] = (uint16_t)(b0 << 3);
      }
    } else if (p0 + 1 < n_px) {
      const uint2 v = __ldg(reinterpret_cast<const uint2 *>(px + p0));
      const uint32_t b0 = rgb_bin(v.x), b1 = rgb_bin(v.y);
      atomicAdd(&sh[b0], 1u);
      atomicAdd(&sh[b1], 1u);
      if (bout) *reinterpret_cast<uint32_t *>(bout + p0) = (b0 << 3) | (b1 << 19);
    } else {
      const uint32_t b0 = rgb_bin(__ldg(px + p0));
      atomicAdd(&sh[b0], 1u);
      if (bout) bout[p0] = (uint16_t)(b0 << 3);
    }
  }
  __syncthreads();
  uint32_t *out = hist + (size_t)blockIdx.y * 4096;
  if (chunks == 1) {
    for (int i = threadIdx.x; i < 4096; i += 256) out[i] = sh[i];
  } else {
    for (int i = threadIdx.x; i < 4096; i += 256)
      if (sh[i]) atomicAdd(&out[i], sh[i]);
  }
}

// ------------------------------------------------------------------------------------------------
// initTracker — src/camshift.js:198-211.  One CTA per slot: model histogram of the rectangle
// (pixels outside the canvas read as 0,0,0,0 -> bin 0, like getImageData), _searchWindow := rect,
// _trackObj := new TrackObj().  rects == NULL -> take the rectangle from det_pick (device pick).
// calc_angles < 0 (ht_tracker_step / feed): per entry, enable[k] & 2 (k_tracker_update sets it from the stream's
// parameters).  geo (ht_tracker_feed, else NULL): per-entry canvas size and place in the arena, instead of W, H and
// frame k at k * frame_bytes.  cost (ht_tracker_step / feed, else NULL): a seeded slot's k_track scheduling history
// starts over, so that the whole camshift section of a tracker stream follows from its last hand-off (tracker records).
__global__ void __launch_bounds__(256) k_track_init(const uint8_t *__restrict__ rgba, size_t frame_bytes, int W, int H,
                                                    const int32_t *__restrict__ slots,
                                                    const int32_t *__restrict__ rects, int calc_angles,
                                                    uint32_t *__restrict__ model_hist, TrackState *__restrict__ state,
                                                    int32_t *__restrict__ found, const uint8_t *__restrict__ enable,
                                                    const EntryCanvas *__restrict__ geo = nullptr,
                                                    int32_t *__restrict__ cost = nullptr) {
  __shared__ uint32_t sh[4096];
  const int k = blockIdx.x;
  if (enable && !enable[k]) return;            // ht_stream_step: only the streams that just found a face
  if (calc_angles < 0) calc_angles = (enable[k] >> 1) & 1;
  const uint8_t *frame = rgba + (size_t)k * frame_bytes;
  if (geo) {
    const EntryCanvas &e = geo[k];
    frame = rgba + e.base;
    W = e.w;
    H = e.h;
  }
  const int slot = slots ? slots[k] : k;
  const int rx = rects[4 * k + 0], ry = rects[4 * k + 1], rw = rects[4 * k + 2], rh = rects[4 * k + 3];
  if (rw <= 0 || rh <= 0) {  // no candidate (device pick): the slot becomes uninitialised
    if (threadIdx.x == 0) {
      state[slot].initialised = 0;
      if (found) found[k] = 0;
    }
    return;
  }
  for (int i = threadIdx.x; i < 4096; i += 256) sh[i] = 0;
  __syncthreads();
  const uint32_t *px = reinterpret_cast<const uint32_t *>(frame);
  for (int yy = threadIdx.x >> 5; yy < rh; yy += 8) {
    const int cy = ry + yy;
    for (int xx = threadIdx.x & 31; xx < rw; xx += 32) {
      const int cx = rx + xx;
      uint32_t bin = 0;
      if (cx >= 0 && cx < W && cy >= 0 && cy < H) bin = rgb_bin(__ldg(px + (size_t)cy * W + cx));
      atomicAdd(&sh[bin], 1u);
    }
  }
  __syncthreads();
  uint32_t *out = model_hist + (size_t)slot * 4096;
  for (int i = threadIdx.x; i < 4096; i += 256) out[i] = sh[i];
  if (threadIdx.x == 0) {
    TrackState s;
    s.sx = rx; s.sy = ry; s.sw = rw; s.sh = rh;
    s.tx = s.ty = s.tw = s.th = 0;
    s.angle = 0.0;
    s.calc_angles = calc_angles;
    s.initialised = 1;
    state[slot] = s;
    if (found) found[k] = 1;
    if (cost) cost[2 * slot] = cost[2 * slot + 1] = 0;
  }
}

// facetrackr's VJ->CS hand-off on the device — src/facetrackr.js:157-165 (first max-confidence
// candidate), :97 (confidence > -10), :101-106 (Math.floor of x,y,width,height).
// Frame k's candidates are det[k * stride, k * stride + min(counts[k], cap)): a caller's lists (stride = cap = K), or
// k_group's first-maximum records (stride = cap = 1), which stand for the whole grouped list when counts[k] > 0.
__global__ void k_pick_face(const Rect *__restrict__ det, int stride, const int32_t *__restrict__ counts, int cap, int n,
                            int32_t *__restrict__ rects) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int c = min(counts[k], cap);
  int32_t r[4] = {0, 0, 0, 0};
  if (c > 0) {
    const Rect *d = det + (size_t)k * stride;
    int best = 0;
    for (int i = 1; i < c; ++i)
      if (d[i].confidence > d[best].confidence) best = i;
    if (d[best].confidence > -10.0) {
      r[0] = (int32_t)floor(d[best].x); r[1] = (int32_t)floor(d[best].y);
      r[2] = (int32_t)floor(d[best].width); r[3] = (int32_t)floor(d[best].height);
    }
  }
  rects[4 * k + 0] = r[0]; rects[4 * k + 1] = r[1]; rects[4 * k + 2] = r[2]; rects[4 * k + 3] = r[3];
}

// ------------------------------------------------------------------------------------------------
// Zero-weight marking of the bin plane.  getWeights (src/camshift.js:314-330) gives a pixel the weight
// min(model[bin] / current[bin], 1): it is exactly +0.0 for every colour bin that does not occur in the model
// histogram, i.e. in the face rectangle of initTracker - the vast majority of a frame's pixels (a face has a few
// dozen to a few hundred of the 4096 bins).  Adding +0.0 to a moment sum never changes it,
// so those pixels can be skipped.  This pass rewrites their plane entries to ZERO (0x8000 = 8 * 4096, the table's
// extra +0.0 entry): k_track then skips every 128-pixel row segment whose entries are all ZERO with one warp vote.
// One read + one write of the u16 plane per frame, worth it when several track() calls follow on the same frame.
constexpr uint32_t BIN_ZERO = 8u * 4096u;          // byte offset of wsm[4096]
constexpr uint32_t BIN_ZERO2 = BIN_ZERO | (BIN_ZERO << 16);
__global__ void __launch_bounds__(256) k_bins_mask(uint16_t *__restrict__ bins, int n_px, const uint32_t *__restrict__ model_hist,
                                                   const int32_t *__restrict__ slots, const TrackState *__restrict__ state,
                                                   int chunks, const uint8_t *__restrict__ enable,
                                                   // cost != NULL: only the streams whose previous launch visited more than
                                                   // min_px256 * 256 pixels (k_track's scheduling history) - the pass over
                                                   // the plane is repaid by streams that sweep large windows many times
                                                   const int32_t *__restrict__ cost, int min_px256) {
  __shared__ uint32_t bm[128];                     // bit b set: model histogram bin b is non-zero
  const int k = blockIdx.y;
  if (enable && !enable[k]) return;
  const int slot = slots ? slots[k] : k;
  if (!state[slot].initialised) return;            // k_track refuses such a slot anyway
  if (cost && cost[2 * slot + 1] < min_px256) return;
  const uint32_t *mh = model_hist + (size_t)slot * 4096;
  if (threadIdx.x < 128) {
    uint32_t w = 0;
#pragma unroll 8
    for (int i = 0; i < 32; ++i) w |= (__ldg(mh + 32 * threadIdx.x + i) != 0u ? 1u : 0u) << i;
    bm[threadIdx.x] = w;
  }
  __syncthreads();
  uint16_t *pl = bins + (size_t)k * n_px;
  auto mask2 = [&](uint32_t v) {                   // two u16 entries (8 * bin each)
    const uint32_t b0 = (v & 0xffffu) >> 3, b1 = v >> 19;
    uint32_t o = v;
    if (b0 < 4096u && !((bm[b0 >> 5] >> (b0 & 31u)) & 1u)) o = (o & 0xffff0000u) | BIN_ZERO;
    if (b1 < 4096u && !((bm[b1 >> 5] >> (b1 & 31u)) & 1u)) o = (o & 0x0000ffffu) | (BIN_ZERO << 16);
    return o;
  };
  const bool vec = ((reinterpret_cast<uintptr_t>(pl) & 15u) == 0);
  const int n_grp = vec ? n_px / 8 : 0;            // groups of 8 entries (16 bytes)
  const int per = (n_grp + chunks - 1) / chunks;
  const int beg = blockIdx.x * per, end = min(n_grp, beg + per);
  for (int g = beg + threadIdx.x; g < end; g += 256) {
    uint4 v = *reinterpret_cast<const uint4 *>(pl + 8 * (size_t)g);
    const uint4 o = make_uint4(mask2(v.x), mask2(v.y), mask2(v.z), mask2(v.w));
    if (o.x != v.x || o.y != v.y || o.z != v.z || o.w != v.w) *reinterpret_cast<uint4 *>(pl + 8 * (size_t)g) = o;
  }
  if (blockIdx.x == 0)                             // tail (and unaligned planes): entry by entry
    for (int p = 8 * n_grp + threadIdx.x; p < n_px; p += 256) {
      const uint32_t b = pl[p] >> 3;
      if (b < 4096u && !((bm[b >> 5] >> (b & 31u)) & 1u)) pl[p] = (uint16_t)BIN_ZERO;
    }
}

// ------------------------------------------------------------------------------------------------
// track() — src/camshift.js:213-312.  One CTA per slot runs getWeights, the <=10 mean-shift
// iterations and the camShift epilogue for n_calls successive track() calls on the same frame.

struct Mom {
  double m00, m10, m01, m11, m20, m02;
};

__device__ __forceinline__ int32_t js_to_int32(double v) {  // ES ToInt32 for |v| < 2^31; NaN/Inf -> 0
  if (!isfinite(v)) return 0;
  return (int32_t)v;  // cvt.rzi: truncation toward zero
}

// true when truncating v could flip under the summation-order error of a parallel reduction: v lies within tol of an
// integer (trunc_tolerance gives tol)
__host__ __device__ __forceinline__ bool trunc_ambiguous(double v, double tol) {
  return isfinite(v) && fabs(v - rint(v)) < tol;
}

// How far apart k_track's parallel-order values and the reference's serial-order values of one window can lie, for
// each decision a pass makes (DESIGN.md §4 item 2).  Every term of every moment is >= 0, so ANY order of summing the
// window's n non-zero pixels - the serial one, or the kernel's per-thread chains, trees and FMAs (adding a zero term
// is exact) - is within gamma(n) * m of the exact sum (a term meets at most n roundings on its way; +64 covers the
// fixed trees and the products).  That relative error eps is carried through the reference's formulas with the
// magnitudes of THIS window: the mass centre X (from the window's origin), the raw second moments X2 = m20 / m00, Y2,
// and m10 * xc <= m20, |m11|, m01 * xc <= sqrt(m20 m02) (Cauchy-Schwarz).  a = (m20 - m10 xc) / m00 is a difference of
// two numbers of size X2, so its error scales with X2, not with a.  Each bound E is for one evaluation against exact;
// two evaluations differ by up to 2E.
constexpr double TRUNC_U = 1.1102230246251565e-16;                 // 2^-53
__host__ __device__ __forceinline__ double sum_eps(double n_px) {   // n_px: an upper bound of n
  const double nu = (n_px + 64.0) * TRUNC_U;
  return nu * (1.0 + 2.0 * nu) + TRUNC_U;                           // >= gamma(n + 64) (nu <= 1/2), plus one rounding
}
// the shift xc - half (half = sw / 2): xc = m10 * (1 / m00) has two moments and two roundings, then one rounding of
// the subtraction.  Cheap: k_track evaluates it for every shift within the frame's cap (trunc_cap) of an integer.
__host__ __device__ __forceinline__ double shift_tolerance(double eps, double xc, double half) {
  return 2.0 * (4.0 * eps * fabs(xc) + 2.0 * TRUNC_U * (fabs(xc) + half));
}
//   vx, vy : xc - sw/2, yc - sh/2        l1, l2 : the square roots that are truncated (<< 2)
//   b      : mu11 / m00, whose sign picks the angle's branch
struct TruncTol { double vx, vy, l1, l2, b; };
__host__ __device__ inline TruncTol trunc_tolerance(const Mom &m, double n_px, double sw, double sh, bool calc_angles) {
  const double u = TRUNC_U;
  const double eps = sum_eps(n_px);
  const double inv = 1.0 / m.m00;
  const double X = m.m10 * inv, Y = m.m01 * inv, X2 = m.m20 * inv, Y2 = m.m02 * inv;
  TruncTol t;
  t.vx = shift_tolerance(eps, X, 0.5 * sw);
  t.vy = shift_tolerance(eps, Y, 0.5 * sh);
  // a, c, b: the moments (eps each) and about six roundings, all on the scale of X2, Y2 and sqrt(X2 Y2)
  const double ea = 8.0 * eps * X2, ec = 8.0 * eps * Y2, eb = 8.0 * eps * sqrt(X2 * Y2);
  const double a = (m.m20 - m.m10 * X) * inv, c = (m.m02 - m.m01 * Y) * inv;
  double lam1, lam2, e1, e2;                                  // the two radicands and their error bounds
  if (calc_angles) {
    // lambda = (a + c -+ e) / 2 with e = |(2b, a - c)| (1-Lipschitz): errors ea + ec + eb, plus the roundings of d
    // and e (e <= a + c <= X2 + Y2)
    const double b = (m.m11 - m.m01 * X) * inv;
    const double e = sqrt(4 * b * b + (a - c) * (a - c));
    lam1 = (a + c - e) * 0.5; lam2 = (a + c + e) * 0.5;
    e1 = e2 = ea + ec + eb + 4.0 * u * (X2 + Y2);
  } else {
    lam1 = a; lam2 = c;
    e1 = ea; e2 = ec;
  }
  // sqrt: two radicands 2E apart give square roots min(sqrt(2E), 2E / l) apart - the first form near l = 0; plus the
  // rounding of each sqrt
  const double l1 = sqrt(fmax(lam1, 0.0)), l2 = sqrt(fmax(lam2, 0.0));
  t.l1 = fmin(sqrt(2.0 * e1), 2.0 * e1 / l1) + 4.0 * u * l1;
  t.l2 = fmin(sqrt(2.0 * e2), 2.0 * e2 / l2) + 4.0 * u * l2;
  t.b = 2.0 * eb;
  return t;
}
// Upper bounds of those radii over every window of a W x H frame (n <= W H; xc, yc <= M = max(W, H); X2, Y2 <= M^2):
// one comparison screens out the values far from an integer, only the rest need the window's own radius.
//   shift: shift_tolerance(eps, M, max(sw, sh) / 2)    l1, l2: root + 4u l    b: b
struct TruncCap { double eps, M, root, b; };
__host__ __device__ inline TruncCap trunc_cap(int W, int H) {
  TruncCap c;
  c.eps = sum_eps((double)W * (double)H);
  c.M = (double)(W > H ? W : H);
  c.root = sqrt(2.0 * (24.0 * c.eps + 8.0 * TRUNC_U) * c.M * c.M);
  c.b = 16.0 * c.eps * c.M * c.M;
  return c;
}

// Moments in the reference's exact order (x outer, y inner, one accumulator each) —
// src/camshift.js:90-107.  Used by one thread only when a truncation decision is ambiguous.
__device__ __noinline__ Mom moments_serial(const uint16_t *__restrict__ px, int W, int x, int y, int w, int h,
                                           const double *__restrict__ wsm) {
  Mom m = {0, 0, 0, 0, 0, 0};
  for (int i = x; i < w; ++i) {
    const double vx = (double)(i - x);
    for (int j = y; j < h; ++j) {
      const double val = wsm[px[(size_t)j * W + i] >> 3];
      const double vy = (double)(j - y);
      m.m00 += val;
      m.m01 += vy * val;
      m.m10 += vx * val;
      m.m11 += vx * vy * val;
      m.m02 += vy * vy * val;
      m.m20 += vx * vx * val;
    }
  }
  return m;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// One thread-block CLUSTER per slot: TRACK_CLUSTER CTAs split the rows of every window pass and
// combine their partial moments through distributed shared memory.  Mean-shift is a serial chain
// of passes per stream (up to 10 per track() call); spreading one pass over several SMs shortens
// the chain of the streams with large windows, which otherwise set the kernel's duration.
constexpr int TRACK_CLUSTER_MAX = 16;  // the cluster size is a launch-time choice (1, 2, 4, 8 or - non-portable - 16 CTAs per stream)

// Longest-chain-first launch order.  A stream's mean-shift passes form a serial chain whose length grows with its
// search window, and a launch holds only a few hundred streams at a time, so the streams with the largest windows
// are started first (and may be given a larger cluster): otherwise one of them starting in the last wave sets the
// duration of the whole launch.  area[i] = search-window area of stream i; order = indices by descending area
// (ties by index, so the order is deterministic).
__global__ void k_track_area(const TrackState *__restrict__ state, const int32_t *__restrict__ slots, int n,
                             const int32_t *__restrict__ cost, int32_t *__restrict__ area) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int slot = slots ? slots[i] : i;
  const TrackState *s = state + slot;
  long long a = 0;
  if (s->initialised) {
    // History first: what this stream cost in its previous launch (k_track's leader records {passes, window pixels
    // / 256}) predicts the chain it is about to run far better than its current window does - the windows that end
    // up covering the frame start small.  Units: one pass = 120, one pixel per thread of a 256-thread CTA = 1
    // (3 us vs 0.025 us, tools/track_chain_probe.py).  Streams without history: the window area of a typical
    // 70-pass chain.
    const int passes = cost ? cost[2 * slot] : 0;
    if (passes > 0) a = 120ll * passes + cost[2 * slot + 1];
    else a = 120ll * 70 + 70ll * (((long long)max(s->sw, 0) * (long long)max(s->sh, 0)) >> 8);
  }
  area[i] = (int32_t)min(a, (long long)0x7fffffff);
}
__global__ void k_track_rank(const int32_t *__restrict__ area, int n, int32_t *__restrict__ order) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t a = area[i];
  int rank = 0;
  for (int j = 0; j < n; ++j) {
    const int32_t b = __ldg(area + j);
    rank += (b > a || (b == a && j < i)) ? 1 : 0;
  }
  order[rank] = i;
}

// ld.shared.f64 from a 32-bit shared-window address (indexing the __shared__ array through its generic address
// makes the compiler rebuild the cluster-window base, an S2R, for every access)
__device__ __forceinline__ double lds_f64(uint32_t saddr) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(saddr));
  return v;
}

__device__ __forceinline__ void row_partial(const uint16_t *__restrict__ row, const double *__restrict__ wsm, int lane,
                                            int wx, int xbeg, int xend, bool vec4, double &r0, double &r1, double &r2) {
  if (vec4) {
    for (int x4 = xbeg + 4 * lane; x4 < xend; x4 += 128) {
      const uint2 v = __ldg(reinterpret_cast<const uint2 *>(row + x4));
      const uint32_t b[4] = {(v.x & 0xffffu) >> 3, v.x >> 19, (v.y & 0xffffu) >> 3, v.y >> 19};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int x = x4 + i;
        const double val = (x >= wx && x < xend) ? wsm[b[i]] : 0.0;   // +0.0 terms leave the sums unchanged
        const double vx = (double)(x - wx);
        r0 += val;
        r1 += vx * val;
        r2 += (vx * vx) * val;
      }
    }
  } else {
    for (int x = wx + lane; x < xend; x += 32) {
      const double val = wsm[row[x] >> 3];
      const double vx = (double)(x - wx);
      r0 += val;
      r1 += vx * val;
      r2 += (vx * vx) * val;
    }
  }
}

// __launch_bounds__: three resident 256-thread CTAs per SM (80 registers)
template <int TRACK_CLUSTER, int NT>
__global__ void __launch_bounds__(NT, (NT >= 1024) ? 1 : (NT >= 512 ? 2 : (NT >= 256 ? 3 : 6)))
k_track(const uint16_t *__restrict__ bins, int W, int H, const int32_t *__restrict__ slots,
        const uint32_t *__restrict__ model_hist, const uint32_t *__restrict__ cur_hist, TrackState *__restrict__ state,
        int n_calls, int32_t *__restrict__ out_objs /* 6 x i32 per frame */, int32_t *__restrict__ out_windows,
        int32_t *__restrict__ err_flag, unsigned long long *__restrict__ stats,
        // order != NULL: the k-th cluster runs stream order[list_off + k] (k_track_rank's order); NULL: stream k
        const int32_t *__restrict__ order, int list_off,
        // optional timeline (HT_TRACK_TRACE=1): per stream {globaltimer at start, at end, SM id, passes}
        unsigned long long *__restrict__ trace, size_t trace_stride,
        // memo != 0: moments are a pure function of (frame, weights, window) and all three are fixed for the calls of
        // one launch, so the leader keeps the moments of the last windows it has seen and re-uses them when
        // mean-shift returns to one of them (a converged stream, or one oscillating between two windows)
        int memo,
        // force_serial != 0 (ht_debug_set_exactness bit 2): every pass takes the strict-order fallback
        int force_serial,
        // per slot {passes, window pixels / 256} of this launch: the scheduling key of the next one (k_track_area)
        int32_t *__restrict__ cost,
        // enable != NULL (ht_stream_step): streams with enable[k] == 0 are not in tracking mode and are skipped
        const uint8_t *__restrict__ enable) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ double wsm[4096 + 1];   // [4096] = +0.0: the weight of pixels outside the window
  constexpr int NW = NT / 32;   // warps per CTA
  __shared__ double red[NW][6];
  // Every CTA of the cluster keeps its OWN copy of the reference's loop state and runs the scalar mean-shift step
  // redundantly (same inputs, same operations -> bit-identical windows), so a pass needs ONE cluster barrier - the
  // exchange of the partial moments - instead of two (partials to rank 0, barrier, rank 0 publishes the
  // next window, barrier).  cpart is double-buffered by pass parity: a CTA that is already exchanging pass p+1
  // cannot overwrite what a slower CTA still reads for pass p.
  __shared__ double cpart[2][TRACK_CLUSTER_MAX][6];  // partial moments of every CTA of the cluster (written remotely)
  __shared__ int win[4];                         // wadx, wady, wadw, wadh of the next pass
  __shared__ int ctrl;                            // 0 = run another pass over win[], 1 = this stream is finished
  constexpr int MEMO_N = 8;
  struct MemoEnt { int w[4]; int exact; int valid; Mom m; };
  __shared__ MemoEnt memo_tab[MEMO_N];            // thread 0 of every CTA
  __shared__ int memo_next;
  __shared__ unsigned long long st_memo_sh;
  const int crank = (int)cluster.block_rank();
  int k = blockIdx.x / TRACK_CLUSTER;
  if (order) k = order[list_off + k];
  if (enable && !enable[k]) return;               // uniform over the cluster, before any cluster barrier
  const int slot = slots ? slots[k] : k;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool leader = (crank == 0 && tid == 0);   // the one thread that writes results, state and statistics
  const bool stepper = (tid == 0);                 // thread 0 of EVERY CTA runs the mean-shift step
  // The reference's loop state lives in shared memory: only the leader thread touches it after this point, and
  // keeping it out of registers leaves them to the pipelined pass loop.
  struct Lead { TrackState s; unsigned long long st_pass, st_serial, st_px; int call, it, prevx, prevy;
                double shift_cap; };
  __shared__ Lead lead_sh;
  if (tid == 0) {
    lead_sh.s = state[slot];
    lead_sh.st_pass = lead_sh.st_serial = lead_sh.st_px = 0;
    lead_sh.call = 0; lead_sh.it = 0; lead_sh.prevx = lead_sh.s.sx; lead_sh.prevy = lead_sh.s.sy;
    memo_next = 0; st_memo_sh = 0;
    for (int i = 0; i < MEMO_N; ++i) memo_tab[i].valid = 0;
  }
  __syncthreads();
  TrackState &s = lead_sh.s;
  if (trace && leader) {
    unsigned long long t; unsigned smid;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    trace[4 * (size_t)k] = t; trace[4 * (size_t)k + 2] = smid;
  }
  if (!s.initialised) {   // uniform over the cluster
    if (leader) {
      atomicOr(err_flag, 1);
      int32_t *o = out_objs + 6 * (size_t)k;
      o[0] = o[1] = o[2] = o[3] = o[4] = o[5] = 0;  // TrackObj() defaults
      if (out_windows) { int32_t *w4 = out_windows + 4 * (size_t)k; w4[0] = w4[1] = w4[2] = w4[3] = 0; }
    }
    return;
  }
  // getWeights — src/camshift.js:314-330 (every CTA keeps its own copy)
  // The smallest non-zero weight (per warp here): a window has at most m00 / wmin non-zero pixels, which bounds its
  // summation error (trunc_tolerance) far below its area when the weights are sparse.
  __shared__ double wmin[NW];
  __shared__ double nz_per_mass;                  // (1 + 1e-6) / wmin, set by the stepper; 1e-6 covers m00's own error
  __shared__ TruncCap cap;                        // (stepper) the frame's caps of the radii
  {
    const uint32_t *mh = model_hist + (size_t)slot * 4096, *ch = cur_hist + (size_t)k * 4096;
    double wm = INFINITY;
    for (int i = tid; i < 4096; i += NT) {
      const uint32_t c = ch[i], m = mh[i];
      double p = 0.0;
      // (a bin absent from the model gives 0 / c = +0.0: no division for it - that is nearly all of the 4096 bins)
      if (c != 0 && m != 0) p = fmin((double)m / (double)c, 1.0);
      wsm[i] = p;
      if (p > 0.0) wm = fmin(wm, p);
    }
    if (tid == 0) wsm[4096] = 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wm = fmin(wm, __shfl_xor_sync(0xffffffffu, wm, o));
    if (lane == 0) wmin[warp] = wm;
  }
  const uint16_t *px = bins + (size_t)k * W * H;   // 12-bit colour bin of every pixel of this slot's frame (k_hist)
  const bool vec4 = (W & 3) == 0;
  int parity = 0;

  // leader-only bookkeeping of the reference's loops (src/camshift.js:213-312)
  unsigned long long &st_pass = lead_sh.st_pass, &st_serial = lead_sh.st_serial, &st_px = lead_sh.st_px;
  double &shift_cap = lead_sh.shift_cap;
  int &call = lead_sh.call, &it = lead_sh.it, &prevx = lead_sh.prevx, &prevy = lead_sh.prevy;
  auto publish = [&](int done) {   // stepper: next window (or the finish flag) for this CTA
    const int w0 = max(s.sx, 0), w1 = max(s.sy, 0);                // :286-289
    const int w2 = min(w0 + s.sw, W), w3 = min(w1 + s.sh, H);
    win[0] = w0; win[1] = w1; win[2] = w2; win[3] = w3;
    ctrl = done;
  };
  auto start_call = [&]() {        // leader: returns true when the stream stops here (all calls done)
    if (call >= n_calls) return true;
    it = 0; prevx = s.sx; prevy = s.sy;                            // :280-281
    shift_cap = shift_tolerance(cap.eps, cap.M, 0.5 * fmax((double)s.sw, (double)s.sh));   // (trunc_cap)
    return false;
  };
  if (TRACK_CLUSTER > 1) cluster.sync();  // every CTA is resident before the first remote access
  if (stepper) {
    cap = trunc_cap(W, H);           // (start_call reads it)
    publish(start_call() ? 1 : 0);
  }
  __syncthreads();
  if (stepper) {                     // (only the stepper reads nz_per_mass)
    double wm = wmin[0];
    for (int i = 1; i < NW; ++i) wm = fmin(wm, wmin[i]);
    nz_per_mass = (1.0 + 1e-6) / wm;
  }

#ifndef HT_TRACK_PASSTRACE
#define HT_TRACK_PASSTRACE 0   // 1 (profiling build): the leader thread accumulates the clock cycles of each phase of a pass
#endif
#if HT_TRACK_PASSTRACE
  long long pt_acc[5] = {0, 0, 0, 0, 0};
  long long pt_t = 0;
#define HT_PT_MARK(i) do { if (trace && leader) { const long long now_ = clock64(); pt_acc[i] += now_ - pt_t; pt_t = now_; } } while (0)
#else
#define HT_PT_MARK(i) do { } while (0)
#endif
  constexpr int ROW_STRIDE = NW * TRACK_CLUSTER;
  while (!ctrl) {
    const int wx = win[0], wy = win[1], ww = win[2] - win[0], wh = win[3] - win[1];
#if HT_TRACK_PASSTRACE
    if (trace && leader) pt_t = clock64();
#endif
    // Each lane reads 4 adjacent pixels (one 8 B load of 4 colour bins) of 4 rows per step.  Rows are assigned by
    // ABSOLUTE frame row (a CTA keeps hitting its own L1 lines when the window shifts between passes).  The steps of
    // a pass (row group x 128-pixel column block) are software-pipelined: the four loads of step t+1 are issued
    // before the arithmetic of step t, so a pass exposes one L2 latency instead of one per step (a pass is a short
    // serial chain: 3-25 steps per thread).  Per step and row: r0 = sum v, r1 = sum vx v; the vy factors are
    // applied once per row and step.
    double a00 = 0, a10 = 0, a01 = 0, a11 = 0, a20 = 0, a02 = 0;
    const int xbeg = wx & ~3, xend = wx + ww;
    const int mine = crank * NW + warp;                          // rows with (wy+yy) % ROW_STRIDE == mine
    const int yy0 = (mine - (wy % ROW_STRIDE) + ROW_STRIDE) % ROW_STRIDE;
    if (vec4) {
      const int n_x = (xend - xbeg + 127) >> 7;
      const int n_rg = (yy0 < wh) ? (wh - yy0 + 4 * ROW_STRIDE - 1) / (4 * ROW_STRIDE) : 0;
      const int total = n_rg * n_x;
      const uint16_t *col = px + (size_t)wy * W + xbeg + 4 * lane;
      const uint32_t wsm_base = (uint32_t)__cvta_generic_to_shared(wsm);
      constexpr uint32_t ZERO_W = 8u * 4096u;   // byte offset of wsm[4096]
      auto issue = [&](int rg, int xi, uint2 (&v)[4]) {
        const int x4 = xbeg + 4 * lane + 128 * xi;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int y = yy0 + (4 * rg + j) * ROW_STRIDE;
          v[j] = (y < wh && x4 < xend) ? __ldg(reinterpret_cast<const uint2 *>(col + (size_t)y * W + 128 * xi))
                                       : make_uint2(ZERO_W | (ZERO_W << 16), ZERO_W | (ZERO_W << 16));
        }
      };
      auto consume = [&](int rg, int xi, const uint2 (&v)[4]) {
        const int x4 = xbeg + 4 * lane + 128 * xi;
        double vx[4], vx2[4];
        bool in[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int x = x4 + i;
          in[i] = (x >= wx && x < xend);
          vx[i] = (double)(x - wx);
          vx2[i] = vx[i] * vx[i];
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          // a 128-pixel row segment whose entries are all ZERO (k_bins_mask: colours absent from the model; rows below
          // the window) adds +0.0 to every sum: skip it with one vote (uniform over the warp)
          if (!__any_sync(0xffffffffu, v[j].x != BIN_ZERO2 || v[j].y != BIN_ZERO2)) continue;
          const int y = yy0 + (4 * rg + j) * ROW_STRIDE;
          // table offsets (the plane holds 8 * bin); rows below the window were "loaded" as ZERO_W by issue()
          const uint32_t b[4] = {v[j].x & 0xffffu, v[j].x >> 16, v[j].y & 0xffffu, v[j].y >> 16};
          double r0 = 0.0, r1 = 0.0, r2 = 0.0;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            // pixels outside the window read the extra table entry wsm[4096] == +0.0, which leaves the sums unchanged
            const double val = lds_f64(wsm_base + (in[i] ? b[i] : ZERO_W));
            r0 += val;
            r1 = fma(vx[i], val, r1);     // fused: this fast path is validated by trunc_ambiguous, the strict
            r2 = fma(vx2[i], val, r2);    // reference order (separate multiply and add) is moments_serial
          }
          const double vy = (double)y;
          a00 += r0; a10 += r1; a20 += r2;
          a01 = fma(vy, r0, a01); a11 = fma(vy, r1, a11); a02 = fma(vy * vy, r0, a02);
        }
      };
      uint2 va[4], vb[4];
      int rg = 0, xi = 0;
      if (total > 0) issue(0, 0, va);
      for (int t = 0; t < total; t += 2) {
        int rg1 = rg, xi1 = xi + 1;
        if (xi1 == n_x) { xi1 = 0; ++rg1; }
        if (t + 1 < total) issue(rg1, xi1, vb);
        consume(rg, xi, va);
        int rg2 = rg1, xi2 = xi1 + 1;
        if (xi2 == n_x) { xi2 = 0; ++rg2; }
        if (t + 2 < total) issue(rg2, xi2, va);
        if (t + 1 < total) consume(rg1, xi1, vb);
        rg = rg2; xi = xi2;
      }
    } else {
      for (int yy = yy0; yy < wh; yy += 4 * ROW_STRIDE) {
        double r[4][3];
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j][0] = r[j][1] = r[j][2] = 0.0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int y = yy + j * ROW_STRIDE;
          if (y < wh) row_partial(px + (size_t)(wy + y) * W, wsm, lane, wx, xbeg, xend, false, r[j][0], r[j][1], r[j][2]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const double vy = (double)(yy + j * ROW_STRIDE);
          a00 += r[j][0]; a10 += r[j][1]; a20 += r[j][2];
          a01 += vy * r[j][0]; a11 += vy * r[j][1]; a02 += (vy * vy) * r[j][0];
        }
      }
    }
    HT_PT_MARK(0);                     // pixel loop of this thread (loads, lookups, FMAs)
    a00 = warp_sum(a00); a10 = warp_sum(a10); a01 = warp_sum(a01);
    a11 = warp_sum(a11); a20 = warp_sum(a20); a02 = warp_sum(a02);
    if (lane == 0) {
      red[warp][0] = a00; red[warp][1] = a10; red[warp][2] = a01;
      red[warp][3] = a11; red[warp][4] = a20; red[warp][5] = a02;
    }
    __syncthreads();
    HT_PT_MARK(1);                     // warp sums + wait for the CTA's slowest warp
    if (tid < 6 * TRACK_CLUSTER) {   // fixed-order sums (run-to-run deterministic), one copy into every CTA
      const int q = tid % 6, r = tid / 6;
      double t = 0;
      for (int w8 = 0; w8 < NW; ++w8) t += red[w8][q];
      cluster.map_shared_rank(&cpart[0][0][0], r)[(parity * TRACK_CLUSTER_MAX + crank) * 6 + q] = t;
    }
    if (TRACK_CLUSTER > 1) cluster.sync(); else __syncthreads();
    HT_PT_MARK(2);                     // cross-warp sum, remote stores, cluster barrier (wait for the slowest CTA)
    if (stepper) {
      Mom m = {0, 0, 0, 0, 0, 0};
      for (int r = 0; r < TRACK_CLUSTER; ++r) {
        m.m00 += cpart[parity][r][0]; m.m10 += cpart[parity][r][1]; m.m01 += cpart[parity][r][2];
        m.m11 += cpart[parity][r][3]; m.m20 += cpart[parity][r][4]; m.m02 += cpart[parity][r][5];
      }
      bool exact = false;          // m is in the reference's strict summation order (moments_serial)
      bool fresh = true;           // m was computed by this pass (false: taken from the memo)
      int cw0 = win[0], cw1 = win[1], cw2 = win[2], cw3 = win[3];   // the window m belongs to
      ++st_pass;
      st_px += (unsigned long long)(max(ww, 0)) * (unsigned long long)(max(wh, 0));
      // non-zero pixels of window cw, the one the parallel-order moments m belong to: at most its area, and at most
      // m00 / wmin - the n of the decisions' radii (trunc_tolerance)
      auto window_n = [&]() { return fmin((double)(cw2 - cw0) * (double)(cw3 - cw1), m.m00 * nz_per_mass); };
      for (;;) {
        double inv = 1.0 / m.m00;                                    // :109-111
        double vxf = m.m10 * inv - s.sw / 2.0, vyf = m.m01 * inv - s.sh / 2.0;
        bool amb_shift = force_serial;
        if (!exact && !amb_shift && (trunc_ambiguous(vxf, shift_cap) || trunc_ambiguous(vyf, shift_cap))) {
          const double eps = sum_eps(window_n());
          amb_shift = trunc_ambiguous(vxf, shift_tolerance(eps, m.m10 * inv, s.sw / 2.0)) ||
                      trunc_ambiguous(vyf, shift_tolerance(eps, m.m01 * inv, s.sh / 2.0));
        }
        if (!exact && amb_shift) {
          m = moments_serial(px, W, cw0, cw1, cw2, cw3, wsm);
          exact = true;
          ++st_serial;
          inv = 1.0 / m.m00;
          vxf = m.m10 * inv - s.sw / 2.0;
          vyf = m.m01 * inv - s.sh / 2.0;
        }
        s.sx += js_to_int32(vxf);                                    // :295-296
        s.sy += js_to_int32(vyf);
        const bool conv = (s.sx == prevx && s.sy == prevy);         // :299
        bool done = false;
        if (conv || it == 9) {
          // final moments (second == true) are those of this window.  camShift epilogue - src/camshift.js:230-258 -
          // computed once; when the moments are in the parallel order and a `<< 2` truncation (or, with angles, the sign
          // of b) is not safe, the strict moments replace them and the epilogue is recomputed from those.
          s.sx = max(0, min(s.sx, W));                                   // :308-309
          s.sy = max(0, min(s.sy, H));
          for (;;) {
            const double invM00 = 1.0 / m.m00;
            const double xc = m.m10 * invM00, yc = m.m01 * invM00;
            const double mu20 = m.m20 - m.m10 * xc, mu02 = m.m02 - m.m01 * yc, mu11 = m.m11 - m.m01 * xc;
            const double a = mu20 * invM00, c = mu02 * invM00;
            double l1, l2, b = 0.0, e = 0.0, ang = 3.141592653589793 / 2;
            if (s.calc_angles) {
              b = mu11 * invM00;
              const double d = a + c;
              e = sqrt((4 * b * b) + ((a - c) * (a - c)));
              l1 = sqrt((d - e) * 0.5); l2 = sqrt((d + e) * 0.5);
            } else {
              l1 = sqrt(a); l2 = sqrt(c);
            }
            // `if (ang < 0) ang += PI` (src/camshift.js:244) follows the SIGN of b = mu11 / m00: for a symmetric blob
            // b is rounding residue and the parallel summation order may flip it (angle off by PI, far outside the
            // 1e-4 tolerance) - so b within its radius of 0 takes the strict order too
            if (!exact && ((s.calc_angles && fabs(b) <= cap.b) || trunc_ambiguous(l1, cap.root + 4.0 * TRUNC_U * l1) ||
                           trunc_ambiguous(l2, cap.root + 4.0 * TRUNC_U * l2))) {
              const TruncTol tol = trunc_tolerance(m, window_n(), s.sw, s.sh, s.calc_angles);
              if ((s.calc_angles && fabs(b) <= tol.b) || trunc_ambiguous(l1, tol.l1) || trunc_ambiguous(l2, tol.l2)) {
                m = moments_serial(px, W, cw0, cw1, cw2, cw3, wsm); exact = true; ++st_serial;
                continue;
              }
            }
            if (s.calc_angles) {
              ang = atan2(2 * b, a - c + e);
              if (ang < 0) ang = ang + 3.141592653589793;
            }
            s.tw = (int32_t)((uint32_t)js_to_int32(l1) << 2);
            s.th = (int32_t)((uint32_t)js_to_int32(l2) << 2);
            s.angle = ang;
            break;
          }
          s.tx = (int32_t)floor(fmax(0.0, fmin(s.sx + s.sw / 2.0, (double)W)));   // :253-254
          s.ty = (int32_t)floor(fmax(0.0, fmin(s.sy + s.sh / 2.0, (double)H)));
          s.sw = (int32_t)floor(1.1 * s.tw);                             // :257-258
          s.sh = (int32_t)floor(1.1 * s.th);
          ++call;
          done = start_call();
        } else {
          prevx = s.sx;
          prevy = s.sy;
          ++it;
        }
        if (memo && fresh) {        // remember this window's moments (the strict ones if they had to be computed)
          MemoEnt &e = memo_tab[memo_next];
          memo_next = (memo_next + 1) % MEMO_N;
          e.w[0] = cw0; e.w[1] = cw1; e.w[2] = cw2; e.w[3] = cw3;
          e.exact = exact ? 1 : 0; e.m = m; e.valid = 1;
        }
        if (done) { publish(1); break; }
        if (memo) {                 // the next window (src/camshift.js:286-289) may be one whose moments are known
          const int n0 = max(s.sx, 0), n1 = max(s.sy, 0);
          const int n2 = min(n0 + s.sw, W), n3 = min(n1 + s.sh, H);
          int hit = -1;
          for (int i = 0; i < MEMO_N; ++i) {
            const MemoEnt &e = memo_tab[i];
            if (e.valid && e.w[0] == n0 && e.w[1] == n1 && e.w[2] == n2 && e.w[3] == n3) hit = i;
          }
          if (hit >= 0) {
            m = memo_tab[hit].m; exact = memo_tab[hit].exact != 0; fresh = false;
            cw0 = n0; cw1 = n1; cw2 = n2; cw3 = n3;
            ++st_memo_sh;
            continue;
          }
        }
        publish(0);
        break;
      }
    }
    HT_PT_MARK(3);                     // scalar mean-shift step
    parity ^= 1;
    __syncthreads();
    HT_PT_MARK(4);                     // CTA barrier that publishes the next window
  }
  if (leader) {
    if (cost) {
      cost[2 * slot] = (int32_t)min(st_pass, 0x7fffffffull);
      cost[2 * slot + 1] = (int32_t)min(st_px >> 8, 0x7fffffffull);
    }
    if (stats) {
      atomicAdd(&stats[0], st_pass); atomicAdd(&stats[1], st_serial);
      atomicAdd(&stats[2], st_px); atomicAdd(&stats[3], (unsigned long long)call);
      atomicAdd(&stats[4], st_memo_sh);
    }
    state[slot] = s;
    if (trace) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      trace[4 * (size_t)k + 1] = t; trace[4 * (size_t)k + 3] = st_pass;
#if HT_TRACK_PASSTRACE
      // phase totals (SM clock cycles) behind the per-stream records: [max_frames x 4][max_frames x 8]
      for (int i = 0; i < 5; ++i) trace[trace_stride + 8 * (size_t)k + i] = (unsigned long long)pt_acc[i];
#endif
    }
    int32_t *o = out_objs + 6 * (size_t)k;
    o[0] = s.tx; o[1] = s.ty; o[2] = s.tw; o[3] = s.th;
    *reinterpret_cast<double *>(o + 4) = s.angle;
    if (out_windows) {
      int32_t *w4 = out_windows + 4 * (size_t)k;
      w4[0] = s.sx; w4[1] = s.sy; w4[2] = s.sw; w4[3] = s.sh;
    }
  }
  if (TRACK_CLUSTER > 1) cluster.sync();  // no CTA may exit while another one can still address its shared memory
}

// ------------------------------------------------------------------------------------------------
// facetrackr's per-frame state machine on the device (src/facetrackr.js:67-126 with whitebalancing off, plus the
// lost-face rule of src/main.js:230-244) for n independent streams: ht_stream_step.
//   mode[k] : 0 = "VJ" (detect on this frame), 1 = "CS" (camshift on this frame)
// k_stream_plan runs before the frame's kernels and turns the modes into the masks they take; k_stream_update runs
// after them, writes the frame's event record and applies the transitions.
struct StreamEvent {       // == ht_stream_event (include/headtrackr_b200.h)
  int32_t detection;       // 1 = "VJ", 2 = "CS"  (facetrackr TrackObj.detection, src/facetrackr.js:233-241)
  int32_t status;          // bit 0: VJ found a face, the stream switches to CS (src/facetrackr.js:97-108)
                           // bit 1: CS lost the face (width or height 0), the stream re-detects (src/main.js:230-244)
  double x, y, width, height, angle, confidence;
};

// ------------------------------------------------------------------------------------------------
// What src/main.js does with a "CS" result after facetrackr: "found" status, Smoother (src/smoother.js:25-87),
// the wait for a stable head diagonal (src/main.js:262-281) and headposition.Tracker (src/headposition.js:35-191),
// as a per-stream epilogue of the state machine - one `headtrackingEvent {x, y, z}` record per stream and frame
// (SURVEY.md 8f-3).  Scalar fp64 code, operation for operation as the JavaScript (the library is built with
// -fmad=false); only atan / tan come from CUDA's libm instead of V8's (<= 2 ulp).
struct HeadParams {            // == ht_head_params (include/headtrackr_b200.h)
  int32_t smoothing;           // src/main.js:39   (default 1)
  int32_t head_position;       // src/main.js:55   (default 1)
  int32_t edgecorrection;      // src/headposition.js:44-48 (default 1)
  int32_t pad_;
  double alpha;                // Smoother(0.35, ...)            src/main.js:163
  double fov_deg;              // params.fov; <= 0: estimate it  src/main.js:283-288
  double camera_offset;        // params.cameraOffset (11.5)     src/main.js:53
  double distance_to_screen;   // 60                             src/headposition.js:75-79
  // constants of the 16 x 19 cm head model, filled by the library with the host's libm (src/headposition.js:53-63)
  double sin_hsa, cos_hsa, tan_hsa, head_diag_cm;
};
struct HeadState {
  int32_t face_found, sm_init, n_diag, hp_init, first_run, pad_;
  double sp[5];                // Smoother state: x, y, z, width, height (sp2 IS sp: src/smoother.js:28)
  double diag[6];              // headDiagonal
  double fov_saved_deg;        // `fov` of src/main.js:59,288
  double tan_fov_width, head_diag_cam;   // headposition.Tracker
};
struct HeadEvent {             // == ht_head_event
  int32_t valid;               // 1: a headtrackingEvent was dispatched on this frame
  int32_t status;              // bit 0: headtrackrStatus "found" on this frame (src/main.js:246-249)
  double x, y, z;              // src/headposition.js:183-188
  double fx, fy, fwidth, fheight;   // the (smoothed) face object the position was computed from
};

__host__ __device__ inline double js_nan() {
#ifdef __CUDA_ARCH__
  return __longlong_as_double(0x7ff8000000000000ll);
#else
  return std::numeric_limits<double>::quiet_NaN();
#endif
}

__host__ __device__ inline void head_new_state(HeadState &s) {
  s.face_found = s.sm_init = s.n_diag = s.hp_init = 0;
  s.first_run = 1; s.pad_ = 0;
  for (int i = 0; i < 5; ++i) s.sp[i] = 0.0;
  for (int i = 0; i < 6; ++i) s.diag[i] = 0.0;
  s.fov_saved_deg = 0.0; s.tan_fov_width = 0.0; s.head_diag_cam = 0.0;
}

// one frame of one stream: (x, y, w, h) = the CS TrackObj, lost = width or height 0.  retry: what a lost face does -
// with retryDetection (src/main.js:231-238) faceFound and headposition start over; without it (src/main.js:246-247,
// stop() :347-355) only faceFound does: smoother, head diagonals, firstRun, fov and headposition survive.
__host__ __device__ inline void head_step(HeadState &s, const HeadParams &p, bool is_cs, double x, double y, double w, double h,
                                          bool lost, double camw, double camh, HeadEvent &out, bool retry = true) {
  const double PI = 3.141592653589793;
  out.valid = 0; out.status = 0; out.x = out.y = out.z = 0.0; out.fx = out.fy = out.fwidth = out.fheight = 0.0;
  if (!is_cs) return;
  if (lost) {
    s.face_found = 0;
    if (retry) s.hp_init = 0;
    return;
  }
  if (!s.face_found) { out.status |= 1; s.face_found = 1; }          // :246-249
  if (p.smoothing) {                                                  // :255-261
    const double nan = js_nan();                 // faceObj.z is undefined (src/main.js:259) -> NaN
    if (!s.sm_init) { s.sm_init = 1; s.sp[0] = x; s.sp[1] = y; s.sp[2] = nan; s.sp[3] = w; s.sp[4] = h; }
    const double pos[5] = {x, y, nan, w, h};
    const double a = p.alpha;
    for (int i = 0; i < 5; ++i) {                                     // src/smoother.js:39-42 with sp2 === sp
      s.sp[i] = a * pos[i] + (1 - a) * s.sp[i];
      s.sp[i] = a * s.sp[i] + (1 - a) * s.sp[i];
    }
    // predict(0): step = 0, ratio = (alpha * 0) / (1 - alpha), a = 2 + ratio, b = 1 + ratio (src/smoother.js:77-84)
    const double ratio = (a * 0.0) / (1 - a), A = 2 + ratio, B = 1 + ratio;
    x = A * s.sp[0] - B * s.sp[0]; y = A * s.sp[1] - B * s.sp[1];
    w = A * s.sp[3] - B * s.sp[3]; h = A * s.sp[4] - B * s.sp[4];
  }
  out.fx = x; out.fy = y; out.fwidth = w; out.fheight = h;
  if (!p.head_position) return;
  bool track_now = s.hp_init != 0;
  if (!s.hp_init) {                                                   // src/main.js:264-294
    bool stable = false;
    const double headdiag = sqrt(w * w + h * h);
    if (s.n_diag < 6) s.diag[s.n_diag++] = headdiag;
    else {
      for (int i = 0; i < 5; ++i) s.diag[i] = s.diag[i + 1];
      s.diag[5] = headdiag;
      double mx = s.diag[0], mn = s.diag[0];
      bool any_nan = false;
      for (int i = 0; i < 6; ++i) { any_nan = any_nan || (s.diag[i] != s.diag[i]); mx = s.diag[i] > mx ? s.diag[i] : mx; mn = s.diag[i] < mn ? s.diag[i] : mn; }
      if (!any_nan && (mx - mn) < 5) stable = true;                   // Math.max/min are NaN if any element is
    }
    if (stable) {                                                     // new headposition.Tracker(faceObj, W, H, {...})
      s.head_diag_cam = sqrt((w * w) + (h * h));                      // src/headposition.js:66-68
      double fov_width;
      if (s.first_run) {
        if (!(p.fov_deg > 0.0)) {                                     // :69-84
          const double head_width_cam = p.sin_hsa * s.head_diag_cam;
          const double camwidth_at_default_face_cm = (camw / head_width_cam) * 16;
          fov_width = atan((camwidth_at_default_face_cm / 2) / p.distance_to_screen) * 2;
        } else {
          fov_width = p.fov_deg * PI / 180;
        }
        s.fov_saved_deg = fov_width * 180 / PI;                       // getFOV(), src/main.js:288
        s.first_run = 0;
      } else {
        fov_width = s.fov_saved_deg * PI / 180;                       // {fov : fov}, src/main.js:291
      }
      s.tan_fov_width = 2 * tan(fov_width / 2);                       // src/headposition.js:87
      s.hp_init = 1;
      track_now = true;
    }
  }
  if (!track_now) return;
  // headposition.Tracker.track — src/headposition.js:91-191
  double fx = x, fy = y, hdc = s.head_diag_cam;
  const double sin_hsa = p.sin_hsa, cos_hsa = p.cos_hsa, tan_hsa = p.tan_hsa;
  if (p.edgecorrection) {
    const double margin = 11;
    const double leftDistance = fx - (w / 2), rightDistance = camw - (fx + (w / 2));
    const double topDistance = fy - (h / 2), bottomDistance = camh - (fy + (h / 2));
    const bool onVerticalEdge = (leftDistance < margin || rightDistance < margin);
    const bool onHorizontalEdge = (topDistance < margin || bottomDistance < margin);
    if (onHorizontalEdge) {
      if (onVerticalEdge) {                                           // corner: keep the previous diagonal
        if (leftDistance < margin) fx = w - (hdc * sin_hsa / 2); else fx = fx - (w / 2) + (hdc * sin_hsa / 2);
        if (topDistance < margin) fy = h - (hdc * cos_hsa / 2); else fy = fy - (h / 2) + (hdc * cos_hsa / 2);
      } else if (topDistance < margin) {
        const double ow = topDistance / margin, ew = (margin - topDistance) / margin;
        fy = h - (ow * (h / 2) + ew * ((w / tan_hsa) / 2));
        hdc = ew * (w / sin_hsa) + ow * (sqrt((w * w) + (h * h)));
      } else {
        const double ow = bottomDistance / margin, ew = (margin - bottomDistance) / margin;
        fy = fy - (h / 2) + (ow * (h / 2) + ew * ((w / tan_hsa) / 2));
        hdc = ew * (w / sin_hsa) + ow * (sqrt((w * w) + (h * h)));
      }
    } else if (onVerticalEdge) {
      if (leftDistance < margin) {
        const double ow = leftDistance / margin, ew = (margin - leftDistance) / margin;
        hdc = ew * (h / cos_hsa) + ow * (sqrt((w * w) + (h * h)));
        fx = w - (ow * (w / 2) + (ew) * (h * tan_hsa / 2));
      } else {
        const double ow = rightDistance / margin, ew = (margin - rightDistance) / margin;
        hdc = ew * (h / cos_hsa) + ow * (sqrt((w * w) + (h * h)));
        fx = fx - (w / 2) + (ow * (w / 2) + ew * (h * tan_hsa / 2));
      }
    } else {
      hdc = sqrt((w * w) + (h * h));
    }
  } else {
    hdc = sqrt((w * w) + (h * h));
  }
  s.head_diag_cam = hdc;
  const double z = (p.head_diag_cm * camw) / (s.tan_fov_width * hdc);              // :165
  const double hx = -((fx / camw) - 0.5) * z * s.tan_fov_width;                    // :170
  double hy = -((fy / camh) - 0.5) * z * s.tan_fov_width * (camh / camw);
  hy = hy + p.camera_offset;                                                      // :175-180
  out.valid = 1; out.x = hx; out.y = hy; out.z = z;
}

__global__ void k_stream_plan(const int32_t *__restrict__ mode, int n, uint8_t *__restrict__ vj_quad_mask,
                              uint8_t *__restrict__ cs_enable, uint8_t *__restrict__ init_enable) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  cs_enable[k] = mode[k] == 1 ? 1 : 0;
  init_enable[k] = 0;
  if ((k & 3) == 0) {
    unsigned m = 0;
    for (int f = 0; f < 4 && k + f < n; ++f) m |= (mode[k + f] == 0 ? 1u : 0u) << f;
    vj_quad_mask[k >> 2] = (uint8_t)m;
  }
}

// One "VJ" or "CS" pass of facetrackr for one stream (shared by ht_stream_step and ht_tracker_step).
//   vj: pick from the ccv result list det[0, count); else read the camshift TrackObj obj = {x, y, w, h, angle (fp64)}.
// Fills the TrackObj record e (status bit 0: face found, bit 1: face lost) and returns the next mode (0 = "VJ",
// 1 = "CS").  seed: the tracker must be seeded with rect on this same frame.
__host__ __device__ inline int facetrackr_pass(bool vj, const Rect *det, int count, const int32_t *obj, StreamEvent &e,
                                               int32_t rect[4], bool &seed) {
  seed = false;
  e.status = 0;
  e.x = e.y = e.width = e.height = e.angle = 0.0;     // new TrackObj(), src/facetrackr.js:233-241
  e.confidence = -10000.0;
  if (vj) {                                            // doVJDetection, src/facetrackr.js:137-175
    e.detection = 1;
    if (count > 0) {
      int best = 0;
      for (int i = 1; i < count; ++i)
        if (det[i].confidence > det[best].confidence) best = i;   // first maximum, :161-165
      e.x = det[best].x; e.y = det[best].y; e.width = det[best].width; e.height = det[best].height;
      e.confidence = det[best].confidence;
    }
    if (e.confidence > -10.0) {                        // :97: switch to camshift, initTracker on THIS frame
      rect[0] = (int32_t)floor(e.x); rect[1] = (int32_t)floor(e.y);
      rect[2] = (int32_t)floor(e.width); rect[3] = (int32_t)floor(e.height);
      seed = true;
      e.status |= 1;
      return 1;
    }
    return 0;
  }
  e.detection = 2;                                     // doCSDetection, src/facetrackr.js:178-209
  e.x = obj[0]; e.y = obj[1]; e.width = obj[2]; e.height = obj[3];
  double angle;
  memcpy(&angle, obj + 4, sizeof(angle));
  e.angle = angle;
  e.confidence = 1.0;
  if (obj[2] == 0 || obj[3] == 0) {                    // src/main.js:230: lost -> a fresh facetrackr without whitebalancing
    e.status |= 2;
    return 0;
  }
  return 1;
}

// best[k], counts[k]: k_group's first-maximum record of stream k's grouped list and the list's copied-out length
// (> 0 exactly when the list is not empty)
__global__ void k_stream_update(int32_t *__restrict__ mode, int n, const Rect *__restrict__ best,
                                const int32_t *__restrict__ counts, const int32_t *__restrict__ objs,
                                int32_t *__restrict__ rects, uint8_t *__restrict__ init_enable,
                                StreamEvent *__restrict__ events,
                                // optional head-position epilogue (ht_stream_head_config): per-stream state, parameters,
                                // one HeadEvent per stream; camw / camh = the canvas size
                                HeadState *__restrict__ head_state, const HeadParams *__restrict__ head_params,
                                HeadEvent *__restrict__ head_events, int camw, int camh) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  StreamEvent e;
  const bool vj = mode[k] == 0;
  bool seed;
  int32_t rect[4];
  mode[k] = facetrackr_pass(vj, best + k, (vj && counts[k] > 0) ? 1 : 0, objs + 6 * (size_t)k, e, rect, seed);
  if (seed) {
    for (int i = 0; i < 4; ++i) rects[4 * k + i] = rect[i];
    init_enable[k] = 1;
  }
  events[k] = e;
  if (head_state) {
    HeadState hs = head_state[k];
    HeadEvent he;
    head_step(hs, *head_params, e.detection == 2, e.x, e.y, e.width, e.height, (e.status & 2) != 0, (double)camw, (double)camh, he);
    head_state[k] = hs;
    if (head_events) head_events[k] = he;
  }
}

// getBackProjectionImg's grey level of a pixel whose colour bin has m model and c current counts: Math.floor(255 *
// weight), the weight of getWeights (src/camshift.js:177-196, 314-330) in fp64.  An integer floor(255 * m / c) would
// differ where fl(m / c) rounds across k / 255.
__host__ __device__ __forceinline__ uint32_t backproj_value(uint32_t m, uint32_t c) {
  double p = 0.0;
  if (c != 0) p = fmin((double)m / (double)c, 1.0);
  return (uint32_t)floor(255 * p);
}

// getBackProjectionImg — src/camshift.js:177-196 (debug path)
__global__ void k_backproj(const uint8_t *__restrict__ rgba, int n_px, const uint32_t *__restrict__ mh,
                           const uint32_t *__restrict__ ch, uint8_t *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_px) return;
  const uint32_t bin = rgb_bin(reinterpret_cast<const uint32_t *>(rgba)[i]);
  const uint32_t v = backproj_value(mh[bin], ch[bin]);
  reinterpret_cast<uint32_t *>(out)[i] = v | (v << 8) | (v << 16) | 0xff000000u;
}

// ------------------------------------------------------------------------------------------------
// The debug canvas of a headtrackr.Tracker stream (ht_tracker_set_debug): on every CS pass facetrackr puts
// getBackProjectionImg() at (0, 0) of params.debug (src/facetrackr.js:193-196), clipped to that canvas.
// Layout of ht_debug_canvas, with the pitch resolved; rgba NULL: the stream has none.  strokes (the header's pad word):
// ht_tracker_set_debug_strokes's flag, which belongs to the stream whether or not it has a canvas.
struct DebugCanvas {
  uint8_t *rgba;
  int32_t w, h, pitch, strokes;
};
constexpr int DBG_TAB = 4112;                     // bytes per value table: 4096 bins + BIN_ZERO's 0, padded to 16 B
constexpr int DBG_TX = 128, DBG_TY = 32;          // pixels per tile of k_debug_backproj

// Value table of one stream's tick: table[b] = backproj_value(model[b], current[b]) for the 4096 colour bins, and
// table[4096] = 0 for the BIN_ZERO entries k_bins_mask writes (bins that are absent from the model: value 0, exact).
__host__ __device__ __forceinline__ void debug_table_entry(const uint32_t *mh, const uint32_t *ch, uint8_t *table, int b) {
  table[b] = b < 4096 ? (uint8_t)backproj_value(mh[b], ch[b]) : 0;
}

// pixels [x, min(x + 4, cw)) of one row: bin-plane entries (8 * bin) -> RGBA (v, v, v, 255).  vec: dst + 4 * x is
// 16-byte aligned (then four whole pixels go in one store).
__host__ __device__ __forceinline__ void debug_px4(const uint16_t *src, const uint8_t *table, uint8_t *dst, int x, int cw,
                                                   bool vec) {
  const int m = cw - x < 4 ? cw - x : 4;
  uint32_t o[4] = {0, 0, 0, 0};
  for (int i = 0; i < m; ++i) o[i] = (uint32_t)table[src[x + i] >> 3] * 0x010101u | 0xff000000u;
  if (vec && m == 4) {
    *reinterpret_cast<uint4 *>(dst + 4 * (size_t)x) = make_uint4(o[0], o[1], o[2], o[3]);
  } else {
    for (int i = 0; i < m; ++i) reinterpret_cast<uint32_t *>(dst)[x + i] = o[i];
  }
}

// ------------------------------------------------------------------------------------------------
// The strokes main.js draws on the debug canvas after a tick (src/main.js:199-219), rasterized by one definition
// (DESIGN.md 2, "Strokes"): lineWidth 1, miter joins, butt caps; corners through translate . rotate in fp64, quantised
// to 1/256 px; 16 x 16 samples per pixel tested with integer edge functions and the top-left rule; alpha
// (255 c + 128) >> 8 of the c covered samples; non-premultiplied source-over.  Host and device round alike: products
// are rounded before they are added (no contraction), so both give the same corners.
__host__ __device__ __forceinline__ double sk_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  volatile double p = a * b;   // a host compiler with FMA could otherwise fuse it into the next add
  return p;
#endif
}
__host__ __device__ __forceinline__ double sk_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

// sin and cos of theta: fdlibm's kernels (k_sin.c, k_cos.c) after a three-part Cody-Waite reduction by pi/2, every
// operation rounded as written.  (0, 1) exactly at 0; within 2 ulp of sin / cos on [-pi/2, pi/2]; a non-finite theta
// is no rotation, as the 2D context ignores rotate(NaN).
__host__ __device__ inline void stroke_sincos(double t, double &s, double &c) {
  if (!isfinite(t)) { s = 0.0; c = 1.0; return; }
  const double k = rint(sk_mul(t, 6.36619772367581382433e-01));
  double r = sk_add(t, -sk_mul(k, 1.57079632673412561417e+00));
  r = sk_add(r, -sk_mul(k, 6.07710050630396597660e-11));
  r = sk_add(r, -sk_mul(k, 2.02226624879595063154e-21));
  const double z = sk_mul(r, r), w = sk_mul(z, z);
  const double S1 = -1.66666666666666324348e-01, S2 = 8.33333333332248946124e-03, S3 = -1.98412698298579493134e-04,
               S4 = 2.75573137070700676789e-06, S5 = -2.50507602534068634195e-08, S6 = 1.58969099521155010221e-10;
  const double C1 = 4.16666666666666019037e-02, C2 = -1.38888888888741095749e-03, C3 = 2.48015872894767294178e-05,
               C4 = -2.75573143513906633035e-07, C5 = 2.08757232129817482790e-09, C6 = -1.13596475577881948265e-11;
  // sin r = r + r^3 (S1 + z (S2 + z (S3 + z S4) + z w (S5 + z S6)))
  const double sr = sk_add(sk_add(S2, sk_mul(z, sk_add(S3, sk_mul(z, S4)))), sk_mul(sk_mul(z, w), sk_add(S5, sk_mul(z, S6))));
  const double sn = sk_add(r, sk_mul(sk_mul(z, r), sk_add(S1, sk_mul(z, sr))));
  // cos r = (1 - z/2) + (((1 - (1 - z/2)) - z/2) + z cr)
  const double cr = sk_add(sk_mul(z, sk_add(C1, sk_mul(z, sk_add(C2, sk_mul(z, C3))))),
                           sk_mul(sk_mul(w, w), sk_add(C4, sk_mul(z, sk_add(C5, sk_mul(z, C6))))));
  const double hz = sk_mul(0.5, z), one_hz = sk_add(1.0, -hz);
  const double cs = sk_add(one_hz, sk_add(sk_add(sk_add(1.0, -one_hz), -hz), sk_mul(z, cr)));
  switch ((int)(k - 4.0 * floor(k * 0.25))) {   // the quadrant, k mod 4
    case 0: s = sn; c = cs; break;
    case 1: s = cs; c = -sn; break;
    case 2: s = -sn; c = -cs; break;
    default: s = -cs; c = sn; break;
  }
}

// One quad of a stroke: corners in 1/256 px, in the order (x0, y0), (x1, y0), (x1, y1), (x0, y1) of the rectangle's
// local coordinates, so its inside is E > 0 for every edge function E(p) = d x (p - a) of edge a -> a + d.  bias: 0
// for a top or left edge (a sample on it is inside), 1 otherwise.
struct StrokeQuad {
  long long ax[4], ay[4], dx[4], dy[4];
  int32_t bias[4];
};
// One tick's stroke on one debug canvas: the outer quad and the inner one (n_q == 2), the colour, and the canvas rows
// [y0, y1) that the outer quad's bounding box meets.
struct Stroke {
  StrokeQuad q[2];
  int32_t n_q, y0, y1;
  uint32_t rgb;   // 0x00BBGGRR
};

__host__ __device__ inline void stroke_quad(StrokeQuad &q, double tx, double ty, double s, double c, double x0, double y0,
                                            double x1, double y1) {
  const double lx[4] = {x0, x1, x1, x0}, ly[4] = {y0, y0, y1, y1};
  long long px[4], py[4];
  for (int i = 0; i < 4; ++i) {
    const double X = sk_add(tx, sk_add(sk_mul(c, lx[i]), -sk_mul(s, ly[i])));
    const double Y = sk_add(ty, sk_add(sk_mul(s, lx[i]), sk_mul(c, ly[i])));
    px[i] = (long long)floor(sk_add(sk_mul(X, 256.0), 0.5));
    py[i] = (long long)floor(sk_add(sk_mul(Y, 256.0), 0.5));
  }
  for (int i = 0; i < 4; ++i) {
    const int e = (i + 1) & 3;
    q.ax[i] = px[i]; q.ay[i] = py[i];
    q.dx[i] = px[e] - px[i]; q.dy[i] = py[e] - py[i];
    q.bias[i] = (q.dy[i] < 0 || (q.dy[i] == 0 && q.dx[i] > 0)) ? 0 : 1;
  }
}

// The stroke of one ht_tracker_event on a dw x dh debug canvas: the rule of streams.debug_calls (nothing when
// confidence is 0 or the pass is not "VJ" / "CS"; a VJ box as it is; a CS box rotated by angle - pi/2 about (x, y)
// at ToInt32(-w/2), ToInt32(-h/2)).  Boxes with a field that is not finite or beyond 65536 px draw nothing, as the
// 2D context ignores non-finite arguments; the tracker produces neither.  -> whether anything may be drawn.
__host__ __device__ inline bool stroke_make(int detection, double confidence, double x, double y, double w, double h,
                                            double angle, int dw, int dh, Stroke &S) {
  S.n_q = 0; S.y0 = S.y1 = 0; S.rgb = 0;
  if (confidence == 0.0 || (detection != 1 && detection != 2)) return false;
  const double v[4] = {x, y, w, h};
  for (int i = 0; i < 4; ++i)
    if (!(fabs(v[i]) <= 65536.0)) return false;
  double tx = 0.0, ty = 0.0, s = 0.0, c = 1.0, rx = x, ry = y;
  S.rgb = 0xCC0000u;                                 // "#0000CC"
  if (detection == 2) {
    tx = x; ty = y;
    stroke_sincos(sk_add(angle, -1.5707963267948966), s, c);
    rx = trunc(-(w / 2)); ry = trunc(-(h / 2));      // ToInt32 of values within +-32768
    S.rgb = 0x00CC00u;                               // "#00CC00"
  }
  if (w < 0) { rx = sk_add(rx, w); w = -w; }
  if (h < 0) { ry = sk_add(ry, h); h = -h; }
  if (w == 0 && h == 0) return false;
  const double xe = sk_add(rx, w), ye = sk_add(ry, h);
  if (h == 0) {                                      // a butt-capped line
    stroke_quad(S.q[0], tx, ty, s, c, rx, sk_add(ry, -0.5), xe, sk_add(ry, 0.5));
    S.n_q = 1;
  } else if (w == 0) {
    stroke_quad(S.q[0], tx, ty, s, c, sk_add(rx, -0.5), ry, sk_add(rx, 0.5), ye);
    S.n_q = 1;
  } else {
    stroke_quad(S.q[0], tx, ty, s, c, sk_add(rx, -0.5), sk_add(ry, -0.5), sk_add(xe, 0.5), sk_add(ye, 0.5));
    S.n_q = 1;
    if (w > 1 && h > 1) {
      stroke_quad(S.q[1], tx, ty, s, c, sk_add(rx, 0.5), sk_add(ry, 0.5), sk_add(xe, -0.5), sk_add(ye, -0.5));
      S.n_q = 2;
    }
  }
  long long lo = S.q[0].ay[0], hi = lo;
  for (int i = 1; i < 4; ++i) { lo = S.q[0].ay[i] < lo ? S.q[0].ay[i] : lo; hi = S.q[0].ay[i] > hi ? S.q[0].ay[i] : hi; }
  const long long r0 = lo >= 0 ? lo / 256 : -((255 - lo) / 256), r1 = (hi >= 0 ? hi / 256 : -((255 - hi) / 256)) + 1;
  S.y0 = (int)(r0 < 0 ? 0 : r0);
  S.y1 = (int)(r1 > dh ? dh : r1);
  return S.y0 < S.y1 && dw > 0;
}

// x-range of quad q at height y (1/256 px units), over its edges that reach y.  -> false if no edge does.
__host__ __device__ inline bool stroke_cross(const StrokeQuad &q, double y, double &l, double &r) {
  l = 1e300; r = -1e300;
  for (int i = 0; i < 4; ++i) {
    const double ay = (double)q.ay[i], by = (double)(q.ay[i] + q.dy[i]), ax = (double)q.ax[i], bx = (double)(q.ax[i] + q.dx[i]);
    if (y < fmin(ay, by) || y > fmax(ay, by)) continue;
    if (ay == by) {
      l = fmin(l, fmin(ax, bx)); r = fmax(r, fmax(ax, bx));
    } else {
      const double xc = ax + (y - ay) * (bx - ax) / (by - ay);
      l = fmin(l, xc); r = fmax(r, xc);
    }
  }
  return l <= r;
}

// The pixels of row Y that the kernel visits: [seg[0], seg[1]] and [seg[2], seg[3]] (empty when first > last).  They
// cover every pixel whose square meets the outer quad in this row, less those whose square lies inside the inner quad
// by 1/16 px or more (all their samples are inside it: c = 0).  Floating point only decides which pixels are visited,
// with a 1/16 px margin against its rounding; coverage itself is stroke_row_count's exact integer count.
__host__ __device__ inline void stroke_row_spans(const Stroke &S, int Y, int dw, int seg[4]) {
  const double y0 = 256.0 * Y, y1 = y0 + 256.0;
  double lo = 1e300, hi = -1e300;
  const StrokeQuad &o = S.q[0];
  for (int i = 0; i < 4; ++i) {                       // each edge clipped to the band [y0, y1]
    const double ay = (double)o.ay[i], by = (double)(o.ay[i] + o.dy[i]), ax = (double)o.ax[i], bx = (double)(o.ax[i] + o.dx[i]);
    const double ylo = fmax(fmin(ay, by), y0), yhi = fmin(fmax(ay, by), y1);
    if (ylo > yhi) continue;
    if (ay == by) {
      lo = fmin(lo, fmin(ax, bx)); hi = fmax(hi, fmax(ax, bx));
    } else {
      const double xa = ax + (ylo - ay) * (bx - ax) / (by - ay), xb = ax + (yhi - ay) * (bx - ax) / (by - ay);
      lo = fmin(lo, fmin(xa, xb)); hi = fmax(hi, fmax(xa, xb));
    }
  }
  seg[0] = 0; seg[1] = -1; seg[2] = 0; seg[3] = -1;
  if (lo > hi) return;
  const double a = floor((lo - 16.0) / 256.0), b = floor((hi + 16.0) / 256.0);
  if (b < 0.0 || a > dw - 1.0) return;
  seg[0] = a < 0.0 ? 0 : (int)a;
  seg[1] = b > dw - 1.0 ? dw - 1 : (int)b;
  double l0, r0, l1, r1;
  if (S.n_q == 2 && stroke_cross(S.q[1], y0, l0, r0) && stroke_cross(S.q[1], y1, l1, r1)) {
    const double sa = ceil((fmax(l0, l1) + 16.0) / 256.0), sb = floor((fmin(r0, r1) - 16.0) / 256.0) - 1.0;
    if (sa <= sb && sb >= seg[0] && sa <= seg[1]) {
      seg[2] = sb + 1.0 > seg[0] ? (int)sb + 1 : seg[0];
      seg[3] = seg[1];
      seg[1] = sa - 1.0 < seg[1] ? (int)sa - 1 : seg[1];
    }
  }
}

// Samples of sample row j of pixel (X, Y) inside quad q: edges that every sample of the row passes are skipped, the
// others stepped sample by sample with adds.
__host__ __device__ __forceinline__ int stroke_quad_row(const StrokeQuad &q, long long px, long long py) {
  uint32_t m = 0xffffu;
  for (int i = 0; i < 4; ++i) {
    const long long b = q.bias[i], step = -16 * q.dy[i];
    long long e = q.dx[i] * (py - q.ay[i]) - q.dy[i] * (px - q.ax[i]);
    const long long e15 = e + 15 * step;
    if (e >= b && e15 >= b) continue;
    if (e < b && e15 < b) return 0;
    uint32_t mk = 0;
    for (int s = 0; s < 16; ++s) {
      mk |= (uint32_t)(e >= b) << s;
      e += step;
    }
    m &= mk;
  }
#ifdef __CUDA_ARCH__
  return __popc(m);
#else
  return __builtin_popcount(m);
#endif
}

// c of sample row j (0..15) of pixel (X, Y): samples at (X + (2i+1)/32, Y + (2j+1)/32) in the outer quad and not in the
// inner one (which lies inside the outer).
__host__ __device__ __forceinline__ int stroke_row_count(const Stroke &S, int X, int Y, int j) {
  const long long px = 256LL * X + 8, py = 256LL * Y + 16 * j + 8;
  int c = stroke_quad_row(S.q[0], px, py);
  if (c && S.n_q == 2) c -= stroke_quad_row(S.q[1], px, py);
  return c;
}

// Source-over of colour rgb at coverage c (1..256) onto one non-premultiplied RGBA pixel, rounding half up.
__host__ __device__ __forceinline__ void stroke_blend(uint8_t *p, int c, uint32_t rgb) {
  const uint32_t a = (255u * (uint32_t)c + 128u) >> 8;
  const uint32_t d = *reinterpret_cast<const uint32_t *>(p), da = d >> 24;
  const uint32_t A = a * 255u + da * (255u - a);
  uint32_t o = ((A + 127u) / 255u) << 24;
  for (int ch = 0; ch < 3; ++ch) {
    const uint32_t s = (rgb >> (8 * ch)) & 0xffu, v = (d >> (8 * ch)) & 0xffu;
    o |= ((s * a * 255u + v * da * (255u - a) + A / 2u) / A) << (8 * ch);
  }
  *reinterpret_cast<uint32_t *>(p) = o;
}

// One CTA per batch entry: the value table of each entry that ran track() (cs_en) on a stream with a debug canvas.
// ids: the entries' stream ids (NULL: entry j is stream j); ch: the entries' current histograms.
__global__ void __launch_bounds__(256) k_debug_table(const int32_t *__restrict__ ids, const uint8_t *__restrict__ cs_en,
                                                     const DebugCanvas *__restrict__ dbg, const uint32_t *__restrict__ model_hist,
                                                     const uint32_t *__restrict__ ch, uint8_t *__restrict__ tables) {
  const int j = blockIdx.x;
  if (!cs_en[j]) return;
  const int id = ids ? ids[j] : j;
  if (!dbg[id].rgba) return;
  const uint32_t *mh = model_hist + (size_t)id * 4096, *c = ch + (size_t)j * 4096;
  for (int b = threadIdx.x; b < DBG_TAB; b += 256) debug_table_entry(mh, c, tables + (size_t)j * DBG_TAB, b);
}

// putImageData(getBackProjectionImg(), 0, 0) on the debug canvases of one canvas-size group, from its bin plane (2 B
// per pixel instead of the canvas's 4).  grid = (tiles of DBG_TX x DBG_TY over w x h, entries); pixels outside
// min(w, Dw) x min(h, Dh) are not written.
__global__ void __launch_bounds__(256) k_debug_backproj(const uint16_t *__restrict__ bins, int w, int h, int tiles_x,
                                                        const int32_t *__restrict__ ids, const uint8_t *__restrict__ cs_en,
                                                        const DebugCanvas *__restrict__ dbg, const uint8_t *__restrict__ tables) {
  const int j = blockIdx.y;
  if (!cs_en[j]) return;
  const DebugCanvas d = dbg[ids ? ids[j] : j];
  if (!d.rgba) return;
  const int cw = min(w, d.w), chh = min(h, d.h);
  const int x0 = (blockIdx.x % tiles_x) * DBG_TX, y0 = (blockIdx.x / tiles_x) * DBG_TY;
  if (x0 >= cw || y0 >= chh) return;
  __shared__ uint4 tab4[DBG_TAB / 16];
  const uint4 *src = reinterpret_cast<const uint4 *>(tables + (size_t)j * DBG_TAB);
  for (int i = threadIdx.x; i < DBG_TAB / 16; i += 256) tab4[i] = src[i];
  __syncthreads();
  const uint8_t *table = reinterpret_cast<const uint8_t *>(tab4);
  const bool vec = ((reinterpret_cast<uintptr_t>(d.rgba) | (uintptr_t)d.pitch) & 15u) == 0;
  const int x = x0 + 4 * (threadIdx.x & 31);
  if (x >= cw) return;
  const uint16_t *plane = bins + (size_t)j * w * h;
  const int y1 = min(y0 + DBG_TY, chh);
  for (int y = y0 + (threadIdx.x >> 5); y < y1; y += 8)
    debug_px4(plane + (size_t)y * w, table, d.rgba + (size_t)y * d.pitch, x, cw, vec);
}

// ------------------------------------------------------------------------------------------------
// getWhitebalance — src/whitebalance.js:17-26.  The reference sums bytes in fp64; the sums are
// exact integers, so integer accumulation in any order is bit-identical.
// enable (ht_tracker_step): per frame, 0 = no whitebalance wanted (the frame is not read); NULL = every frame
// geo (ht_tracker_feed, else NULL): per-entry canvas size and place in the arena
__global__ void __launch_bounds__(256) k_wb_sums(const uint8_t *__restrict__ rgba, size_t frame_bytes, int n_px,
                                                 unsigned long long *__restrict__ sums, int chunks,
                                                 const uint8_t *__restrict__ enable = nullptr,
                                                 const EntryCanvas *__restrict__ geo = nullptr) {
  if (enable && !enable[blockIdx.y]) return;
  const uint32_t *px = reinterpret_cast<const uint32_t *>(rgba + (size_t)blockIdx.y * frame_bytes);
  if (geo) {
    const EntryCanvas &e = geo[blockIdx.y];
    px = reinterpret_cast<const uint32_t *>(rgba + e.base);
    n_px = e.w * e.h;
  }
  const int per = (n_px + chunks - 1) / chunks;
  const int beg = blockIdx.x * per, end = min(n_px, beg + per);
  unsigned long long r = 0, g = 0, b = 0;
  for (int i = beg + threadIdx.x; i < end; i += 256) {
    const uint32_t p = __ldg(px + i);
    r += p & 0xffu; g += (p >> 8) & 0xffu; b += (p >> 16) & 0xffu;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    r += __shfl_down_sync(0xffffffffu, r, o);
    g += __shfl_down_sync(0xffffffffu, g, o);
    b += __shfl_down_sync(0xffffffffu, b, o);
  }
  if ((threadIdx.x & 31) == 0) {
    unsigned long long *s = sums + 3 * (size_t)blockIdx.y;
    atomicAdd(&s[0], r); atomicAdd(&s[1], g); atomicAdd(&s[2], b);
  }
}

__host__ __device__ inline double wb_value(const unsigned long long *s, int n_px) {
  const double sz = (double)n_px;
  const double avgr = (double)s[0] / sz, avgg = (double)s[1] / sz, avgb = (double)s[2] / sz;
  return (avgr + avgg + avgb) / 3;  // src/whitebalance.js:23-26
}

__global__ void k_wb_final(const unsigned long long *__restrict__ sums, int n, int n_px, double *__restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  out[k] = wb_value(sums + 3 * (size_t)k, n_px);
}

// ------------------------------------------------------------------------------------------------
// headtrackr.Tracker's lifecycle per stream on the device (src/main.js:168-355 with facetrackr.js:67-126): the starter's
// content check, the whitebalance gate, VJ -> CS, the status events, lost-face handling with and without
// retryDetection, start() / stop(), and the head-position epilogue - ht_tracker_step.
enum { TM_IDLE = 0, TM_STARTING = 1, TM_WB = 2, TM_VJ = 3, TM_CS = 4 };
// headtrackrStatus bits of one frame, in the order src/main.js dispatches them (:182,183,193,233,246,350,251)
enum { ST_WHITEBALANCE = 1, ST_DETECTING = 2, ST_HINTS = 4, ST_REDETECTING = 8, ST_LOST = 16, ST_STOPPED = 32, ST_FOUND = 64 };
constexpr int WB_WINDOW = 15;                  // pwbLength, src/facetrackr.js:59

struct TrackerParams {          // ht_tracker_params with the head parameters as make_head_params completes them
  int32_t retry_detection;      // src/main.js:40
  int32_t calc_angles;          // src/main.js:54
  HeadParams head;
};
struct TrackerState {
  int32_t mode;                 // TM_*
  int32_t n_wb;                 // previousWhitebalances.length
  int32_t timer_set, pad_;      // detectionTimer !== undefined (src/main.js:188-193)
  double timer_ms;
  double wb[WB_WINDOW];         // previousWhitebalances, newest first
  HeadState head;               // faceFound, firstRun, smoother, head diagonals, fov, headposition
};
struct TrackerEvent {           // == ht_tracker_event (include/headtrackr_b200.h)
  int32_t detection;            // 0 = no pass, 1 = "VJ", 2 = "CS", 3 = "WB"
  int32_t status;               // ST_* bits
  double x, y, width, height, angle, confidence;
  double wb;
  int32_t running, pad_;
  double fov;
  HeadEvent head;
};

__host__ __device__ inline void tracker_new_state(TrackerState &s) {   // new headtrackr.Tracker + init(): not running
  s.mode = TM_IDLE; s.n_wb = 0; s.timer_set = 0; s.pad_ = 0; s.timer_ms = 0.0;
  for (int i = 0; i < WB_WINDOW; ++i) s.wb[i] = 0.0;
  head_new_state(s.head);
}
// start() (src/main.js:328-345): the next frame goes through starter().  On a stream that is already running the
// reference would run an extra, unscheduled pass; here it does nothing.
__host__ __device__ inline void tracker_start(TrackerState &s) {
  if (s.mode == TM_IDLE) s.mode = TM_STARTING;
}
// stop() (src/main.js:347-355): clears the track() timer and faceFound.  A pending starter() retry is another timer and
// survives, as in the reference; the detection timer survives too.
__host__ __device__ inline void tracker_stop(TrackerState &s) {
  if (s.mode != TM_STARTING) s.mode = TM_IDLE;
  s.head.face_found = 0;
}

// One frame of one stream.  Inputs, as the stream's mode asks for them: wb = getWhitebalance (TM_STARTING, TM_WB),
// det[0, count) = detect_objects(frame, cascade, 5, 1) (TM_VJ), obj = camshift TrackObj after track() (TM_CS).
// seed: initTracker(frame, rect) must follow on this frame.
__host__ __device__ inline void tracker_step(TrackerState &s, const TrackerParams &p, double wb, const Rect *det, int count,
                                             const int32_t *obj, double now_ms, double camw, double camh, TrackerEvent &out,
                                             int32_t rect[4], bool &seed) {
  seed = false;
  out.detection = 0; out.status = 0; out.pad_ = 0;
  out.x = out.y = out.width = out.height = out.angle = 0.0;
  out.confidence = -10000.0;
  out.wb = 0.0;
  int mode = s.mode;
  head_step(s.head, p.head, false, 0.0, 0.0, 0.0, 0.0, false, camw, camh, out.head);   // clears out.head
  if (mode == TM_STARTING) {                   // starter(), src/main.js:307-326
    out.wb = wb;
    if (wb > 0) {                              // run = true; track(): a new facetrackr with whitebalancing (:173-176)
      s.n_wb = 0;
      mode = TM_WB;
    }
  }
  if (mode == TM_WB) {                         // checkWhitebalance + the gate, src/facetrackr.js:79-95,220-227
    out.detection = 3; out.wb = wb;
    if (s.n_wb >= WB_WINDOW) s.n_wb = WB_WINDOW - 1;                    // pop()
    for (int i = s.n_wb; i > 0; --i) s.wb[i] = s.wb[i - 1];            // unshift(wb)
    s.wb[0] = wb;
    ++s.n_wb;
    if (s.n_wb == WB_WINDOW) {
      double mx = s.wb[0], mn = s.wb[0];
      for (int i = 1; i < WB_WINDOW; ++i) { mx = s.wb[i] > mx ? s.wb[i] : mx; mn = s.wb[i] < mn ? s.wb[i] : mn; }
      if ((mx - mn) < 2) mode = TM_VJ;
    }
    out.status |= ST_WHITEBALANCE;                                     // src/main.js:182
  } else if (mode == TM_VJ || mode == TM_CS) {
    const bool vj = mode == TM_VJ;
    StreamEvent e;
    const int next = facetrackr_pass(vj, det, count, obj, e, rect, seed);
    out.detection = e.detection;
    out.x = e.x; out.y = e.y; out.width = e.width; out.height = e.height; out.angle = e.angle; out.confidence = e.confidence;
    mode = next == 1 ? TM_CS : TM_VJ;
    if (vj && s.head.first_run) out.status |= ST_DETECTING;            // :183
    if (!(e.confidence == 0)) {                                        // :186
      if (vj) {
        if (!s.timer_set) { s.timer_set = 1; s.timer_ms = now_ms; }   // :187-194
        if ((now_ms - s.timer_ms) > 5000) out.status |= ST_HINTS;
      } else {
        s.timer_set = 0;                                               // :209
        const bool lost = (e.status & 2) != 0;
        const bool retry = p.retry_detection != 0;
        if (lost) {
          if (retry) out.status |= ST_REDETECTING;                     // :231-244
          else { out.status |= ST_LOST | ST_STOPPED; mode = TM_IDLE; } // :245-248, stop()
        }
        head_step(s.head, p.head, true, e.x, e.y, e.width, e.height, lost, camw, camh, out.head, retry);
        if (out.head.status & 1) out.status |= ST_FOUND;               // :250-253
      }
    }
  }
  s.mode = mode;
  out.running = (mode != TM_IDLE && mode != TM_STARTING) ? 1 : 0;
  out.fov = s.head.fov_saved_deg;                                      // getFOV(), :363-365
}

// modes -> the masks of the frame's kernels (a TM_IDLE stream's frame is never read).  Batch entry k is stream ids[k]
// (ids == NULL: stream k); all masks are indexed by batch entry.  draw (ht_tracker_feed, else NULL): the entry's video
// is drawn onto its canvas - every stream that is not TM_IDLE.  The VJ frame quads are those of each canvas-size group
// (geo, ht_tracker_feed; NULL: one group [0, n) whose quads start at 0): no quad mixes canvas sizes.
__global__ void k_tracker_plan(const TrackerState *__restrict__ st, const int32_t *__restrict__ ids, int n,
                               uint8_t *__restrict__ vj_quad_mask, uint8_t *__restrict__ cs_enable,
                               uint8_t *__restrict__ init_enable, uint8_t *__restrict__ wb_enable,
                               uint8_t *__restrict__ draw, const EntryCanvas *__restrict__ geo) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int m = st[ids ? ids[k] : k].mode;
  cs_enable[k] = m == TM_CS ? 1 : 0;
  wb_enable[k] = (m == TM_STARTING || m == TM_WB) ? 1 : 0;
  init_enable[k] = 0;
  if (draw) draw[k] = m != TM_IDLE ? 1 : 0;
  const int g0 = geo ? geo[k].g0 : 0, g_end = geo ? geo[k].g_end : n, q0 = geo ? geo[k].q0 : 0;
  if (((k - g0) & 3) == 0) {
    unsigned mask = 0;
    for (int f = 0; f < 4 && k + f < g_end; ++f) mask |= (st[ids ? ids[k + f] : k + f].mode == TM_VJ ? 1u : 0u) << f;
    vj_quad_mask[q0 + ((k - g0) >> 2)] = (uint8_t)mask;
  }
}

// Batch entry k is stream ids[k] (NULL: stream k) with the parameters params[stream].
// now (ht_tracker_feed, else NULL): the clock of each batch entry; otherwise every entry ticks at now_ms.
// geo (ht_tracker_feed, else NULL): per entry the canvas size (whitebalance pixel count, headposition's camera size)
// and the record whose event it is; otherwise every entry is on camw x camh and its event is events[k].
// best, counts: as in k_stream_update, per batch entry.  init_enable[k] := 1 | 2 * calcAngles when initTracker follows.
__global__ void k_tracker_update(TrackerState *__restrict__ st, const int32_t *__restrict__ ids,
                                 const TrackerParams *__restrict__ params, int n,
                                 const unsigned long long *__restrict__ wb_sums, int n_px, const Rect *__restrict__ best,
                                 const int32_t *__restrict__ counts, const int32_t *__restrict__ objs,
                                 int32_t *__restrict__ rects, uint8_t *__restrict__ init_enable, double now_ms,
                                 const double *__restrict__ now, int camw, int camh, const EntryCanvas *__restrict__ geo,
                                 TrackerEvent *__restrict__ events) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  if (now) now_ms = now[k];
  int out = k;
  if (geo) {
    const EntryCanvas &g = geo[k];
    camw = g.w; camh = g.h; n_px = g.w * g.h; out = g.record;
  }
  const int id = ids ? ids[k] : k;
  TrackerState &s = st[id];                    // updated in place: the window and the head state stay in memory
  const TrackerParams &p = params[id];
  const bool wants_wb = s.mode == TM_STARTING || s.mode == TM_WB;
  const double wb = wants_wb ? wb_value(wb_sums + 3 * (size_t)k, n_px) : 0.0;
  TrackerEvent e;
  int32_t rect[4];
  bool seed;
  tracker_step(s, p, wb, best + k, (s.mode == TM_VJ && counts[k] > 0) ? 1 : 0, objs + 6 * (size_t)k, now_ms,
               (double)camw, (double)camh, e, rect, seed);
  if (seed) {
    for (int i = 0; i < 4; ++i) rects[4 * k + i] = rect[i];
    init_enable[k] = (uint8_t)(1 | (p.calc_angles ? 2 : 0));
  }
  events[out] = e;
}

// op: 0 = new state, 1 = start(), 2 = stop()
__global__ void k_tracker_control(TrackerState *st, int first, int n, int op) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  TrackerState &s = st[first + k];
  if (op == 0) tracker_new_state(s);
  else if (op == 1) tracker_start(s);
  else tracker_stop(s);
}

// ------------------------------------------------------------------------------------------------
// The head-coupled camera of a headtrackr.Tracker stream (ht_tracker_set_camera): realisticAbsoluteCameraControl
// (src/controllers.js:28-68) on an ht_camera in device memory, and three.js r48's updateProjectionMatrix as DESIGN.md
// 5.4 f10 restates it.  All in fp64 (the library builds with -fmad=false: every product rounds), the matrices rounded
// once to float32.
struct CameraCtl {              // one stream's controller; camera NULL: none
  ht_camera *camera;
  double scaling, damping;
  double wh, ww;                // screenHeight * scaling, wh * camera.aspect (src/controllers.js:45-46)
  double fixed[3];              // fixedPosition
  double fov, aspect, near_, far_;   // the camera's own
  double rot[9];                // R of lookAt(fixedPosition -> lookAt, up +y): columns x, y, z
};

// Matrix4.lookAt(eye, target, up = (0, 1, 0)) of r48 without its epsilon nudge: z = normalize(eye - target),
// x = normalize(up x z) = normalize((z2, 0, -z0)), y = z x x.  -> false for a degenerate lookAt (eye == target, a
// view direction parallel to up) or a non-finite axis.
__host__ __device__ inline bool camera_lookat(const double eye[3], const double target[3], double rot[9]) {
  double z[3] = {eye[0] - target[0], eye[1] - target[1], eye[2] - target[2]};
  const double zn = sqrt(z[0] * z[0] + z[1] * z[1] + z[2] * z[2]);
  if (!(zn > 0.0) || !(zn < HUGE_VAL)) return false;
  for (int i = 0; i < 3; ++i) z[i] = z[i] / zn;
  double x[3] = {z[2], 0.0, -z[0]};
  const double xn = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
  if (!(xn > 0.0)) return false;
  for (int i = 0; i < 3; ++i) x[i] = x[i] / xn;
  const double y[3] = {z[1] * x[2] - z[2] * x[1], z[2] * x[0] - z[0] * x[2], z[0] * x[1] - z[1] * x[0]};
  for (int i = 0; i < 3; ++i) {
    rot[i] = x[i]; rot[3 + i] = y[i]; rot[6 + i] = z[i];
  }
  for (int i = 0; i < 9; ++i)
    if (!(fabs(rot[i]) <= 1.0)) return false;
  return true;
}

// makeFrustum of r48 -> column-major float32
__host__ __device__ inline void camera_frustum(double l, double r, double b, double t, double n, double f, float m[16]) {
  for (int i = 0; i < 16; ++i) m[i] = 0.0f;
  m[0] = (float)(2 * n / (r - l));
  m[5] = (float)(2 * n / (t - b));
  m[8] = (float)((r + l) / (r - l));
  m[9] = (float)((t + b) / (t - b));
  m[10] = (float)(-(f + n) / (f - n));
  m[11] = -1.0f;
  m[14] = (float)(-2 * f * n / (f - n));
}

// updateProjectionMatrix (with or without the view offset) and the view matrix inverse(T(position) R) = R^T T(-position)
__host__ __device__ inline void camera_matrices(ht_camera &c, const CameraCtl &k) {
  const double PI = 3.141592653589793;
  if (c.has_view_offset) {
    const double fw = c.view[0], fh = c.view[1];
    const double aspect = fw / fh;
    const double top = tan(c.fov * PI / 360) * k.near_;
    const double left = -(aspect * top);
    const double width = 2 * (aspect * top), height = 2 * top;
    camera_frustum(left + c.view[2] * width / fw, left + (c.view[2] + c.view[4]) * width / fw,
                   top - (c.view[3] + c.view[5]) * height / fh, top - c.view[3] * height / fh, k.near_, k.far_,
                   c.projection);
  } else {                                     // makePerspective(fov, aspect, near, far)
    const double ymax = k.near_ * tan(c.fov * PI / 360);
    camera_frustum(-ymax * k.aspect, ymax * k.aspect, -ymax, ymax, k.near_, k.far_, c.projection);
  }
  const double *p = c.position;
  for (int r = 0; r < 3; ++r) {
    const double *a = k.rot + 3 * r;           // row r of R^T: axis r
    for (int col = 0; col < 3; ++col) c.view_matrix[4 * col + r] = (float)a[col];
    c.view_matrix[12 + r] = (float)(-(a[0] * p[0] + a[1] * p[1] + a[2] * p[2]));
    c.view_matrix[4 * r + 3] = 0.0f;
  }
  c.view_matrix[15] = 1.0f;
}

// the constructed camera (src/controllers.js:40-46): position = fixedPosition, the camera's own fov, no view offset
__host__ __device__ inline void camera_construct(ht_camera &c, const CameraCtl &k) {
  for (int i = 0; i < 3; ++i) c.position[i] = k.fixed[i];
  c.fov = k.fov;
  for (int i = 0; i < 6; ++i) c.view[i] = 0.0;
  c.events = 0; c.has_view_offset = 0; c.pad_[0] = c.pad_[1] = 0;
  camera_matrices(c, k);
}

// the headtrackingEvent listener (src/controllers.js:48-67) for the event (x, y, z), operation for operation
__host__ __device__ inline void camera_step(ht_camera &c, const CameraCtl &k, double x, double y, double z) {
  const double PI = 3.141592653589793;
  const double scaling = k.scaling, damping = k.damping;
  const double xOffset = x > 0 ? 0.0 : -x * 2 * damping * scaling;
  const double yOffset = y < 0 ? 0.0 : y * 2 * damping * scaling;
  c.view[0] = k.ww + fabs(x * 2 * damping * scaling);
  c.view[1] = k.wh + fabs(y * damping * 2 * scaling);
  c.view[2] = xOffset; c.view[3] = yOffset; c.view[4] = k.ww; c.view[5] = k.wh;
  c.has_view_offset = 1;
  c.position[0] = k.fixed[0] + (x * scaling * damping);
  c.position[1] = k.fixed[1] + (y * scaling * damping);
  c.position[2] = k.fixed[2] + (z * scaling);
  c.fov = atan((k.wh / 2 + fabs(y * scaling * damping)) / (fabs(z * scaling))) * 360 / PI;
  ++c.events;
  camera_matrices(c, k);
}

// After k_tracker_update: batch entry k (stream ids[k], NULL: k; its record events[geo[k].record], geo NULL: k) moves
// its stream's camera when its record has a headtrackingEvent.
__global__ void k_camera_update(const int32_t *__restrict__ ids, const EntryCanvas *__restrict__ geo, int n,
                                const TrackerEvent *__restrict__ events, const CameraCtl *__restrict__ ctl) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const CameraCtl &c = ctl[ids ? ids[k] : k];
  if (!c.camera) return;
  const HeadEvent &h = events[geo ? geo[k].record : k].head;
  if (!h.valid) return;
  ht_camera cam = *c.camera;
  camera_step(cam, c, h.x, h.y, h.z);
  *c.camera = cam;
}

// After k_tracker_update (and k_debug_backproj, so CS strokes land on the back-projection): one CTA per batch entry
// strokes its record (events[geo[k].record], geo NULL: k) onto its stream's debug canvas, if the stream has one and
// strokes on (DebugCanvas::strokes).  Warp w walks rows y0 + w, y0 + w + 8, ... of the stroke; each half-warp takes one
// visited pixel at a time, lane j its sample row j, and lane 0 of the half writes the pixel.
__global__ void __launch_bounds__(256, 1) k_debug_strokes(const int32_t *__restrict__ ids, const EntryCanvas *__restrict__ geo,
                                                       const TrackerEvent *__restrict__ events,
                                                       const DebugCanvas *__restrict__ dbg) {
  const int k = blockIdx.x;
  const DebugCanvas d = dbg[ids ? ids[k] : k];
  if (!d.rgba || !d.strokes) return;
  __shared__ Stroke S;
  __shared__ int draw;
  if (threadIdx.x == 0) {
    const TrackerEvent &e = events[geo ? geo[k].record : k];
    draw = stroke_make(e.detection, e.confidence, e.x, e.y, e.width, e.height, e.angle, d.w, d.h, S);
  }
  __syncthreads();
  if (!draw) return;
  const int half = (threadIdx.x >> 4) & 1, j = threadIdx.x & 15;
  for (int Y = S.y0 + (int)(threadIdx.x >> 5); Y < S.y1; Y += 8) {
    int seg[4];
    stroke_row_spans(S, Y, d.w, seg);
    const int na = seg[1] - seg[0] + 1 > 0 ? seg[1] - seg[0] + 1 : 0, nb = seg[3] - seg[2] + 1 > 0 ? seg[3] - seg[2] + 1 : 0;
    for (int p0 = 0; p0 < na + nb; p0 += 2) {
      const int p = p0 + half;
      const int X = p < na ? seg[0] + p : seg[2] + (p - na);
      int c = p < na + nb ? stroke_row_count(S, X, Y, j) : 0;
      c += __shfl_xor_sync(0xffffffffu, c, 8);
      c += __shfl_xor_sync(0xffffffffu, c, 4);
      c += __shfl_xor_sync(0xffffffffu, c, 2);
      c += __shfl_xor_sync(0xffffffffu, c, 1);
      if (j == 0 && c > 0) stroke_blend(d.rgba + (size_t)Y * d.pitch + 4 * (size_t)X, c, S.rgb);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Face crops (ht_tracker_set_face_crop; DESIGN.md 2, "Face crops"): after a tick whose record is "CS" with width > 0
// and height > 0, the rectangle main.js strokes in green, scaled about its centre, grown to the crop's aspect ratio and
// resampled upright from the tick's video at video resolution.
// Layout of ht_face_crop, with the pitch resolved; rgba NULL: the stream has none.  A YUV crop
// (ht_tracker_set_face_crop_yuv) keeps its Y plane in rgba / pitch, its layout in `layout` and the rest in the stream's
// CropPlanes.
enum : int32_t { CROP_RGBA = 0, CROP_NV12 = 1, CROP_I420 = 2 };
struct FaceCrop {
  uint8_t *rgba;
  int32_t w, h, pitch, layout;          // CROP_*
  double scale;
};
// The chroma planes and colour of a YUV crop, pitches resolved.  NV12 is v = u + 1 in one interleaved plane.
struct CropPlanes {
  uint8_t *u, *v;
  int32_t upitch, vpitch, color, pad_;
};
constexpr int CROP_TX = 64, CROP_TY = 16;        // crop pixels per tile of k_face_crop

__host__ __device__ __forceinline__ double sk_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

// The crop map of one record: M = {U0, V0, Ui, Vi, Uj, Vj}, so that crop pixel (i, j) samples tap coordinates
// (U0 + i Ui + j Uj, V0 + i Vi + j Vj) / 65536 of the sw x sh source rectangle (the whole video without a view) that a
// cw x ch canvas is drawn from.  fp64 in this order, every operation rounded as written, then each value quantised
// with floor(v 65536 + 1/2).  Records that are not "CS" with width > 0 and height > 0 make no crop; neither do boxes
// with a field that is not finite or beyond 65536 px (the tracker produces none), which also keeps every tap
// coordinate of a 2048 x 2048 crop within int64.  -> whether the record makes a crop.
// crop_tick: whether a record makes a crop, a crop tick
__host__ __device__ __forceinline__ bool crop_tick(int detection, double x, double y, double w, double h) {
  if (detection != 2 || !(w > 0.0) || !(h > 0.0)) return false;
  const double f[4] = {x, y, w, h};
  for (int i = 0; i < 4; ++i)
    if (!(fabs(f[i]) <= 65536.0)) return false;
  return true;
}
// The rotation (s, c) of a record's green rectangle and its local centre (cx, cy), as main.js strokes it (DESIGN.md 2,
// "Strokes")
__host__ __device__ __forceinline__ void crop_frame(double w, double h, double angle, double &s, double &c, double &cx,
                                                    double &cy) {
  stroke_sincos(sk_add(angle, -1.5707963267948966), s, c);
  const double rx = trunc(-(w / 2)), ry = trunc(-(h / 2));
  cx = sk_add(rx, sk_mul(w, 0.5));
  cy = sk_add(ry, sk_mul(h, 0.5));
}
// crop_map's steps from the rotation on: a w x h box about local centre (cx, cy), rotated by (s, c) and translated to
// (x, y)
__host__ __device__ __forceinline__ void crop_map_box(double x, double y, double cx, double cy, double s, double c, double w,
                                                      double h, int cw, int ch, int sw, int sh, int Sw, int Sh,
                                                      double scale, long long M[6]) {
  double hw = sk_mul(sk_mul(w, scale), 0.5), hh = sk_mul(sk_mul(h, scale), 0.5);
  const double aw = sk_mul(hw, (double)Sh), ah = sk_mul(hh, (double)Sw);
  if (aw < ah) hw = sk_div(ah, (double)Sh);                            // the shorter side grows to S_w : S_h
  else if (ah < aw) hh = sk_div(aw, (double)Sw);
  const double px = sk_div(sk_mul(hw, 2.0), (double)Sw), py = sk_div(sk_mul(hh, 2.0), (double)Sh);
  const double lx = sk_add(sk_add(cx, -hw), sk_mul(px, 0.5)), ly = sk_add(sk_add(cy, -hh), sk_mul(py, 0.5));
  const double X = sk_add(x, sk_add(sk_mul(c, lx), -sk_mul(s, ly)));
  const double Y = sk_add(y, sk_add(sk_mul(s, lx), sk_mul(c, ly)));
  const double kx = sk_div((double)sw, (double)cw), ky = sk_div((double)sh, (double)ch);
  const double v[6] = {sk_add(sk_mul(X, kx), -0.5), sk_add(sk_mul(Y, ky), -0.5), sk_mul(sk_mul(c, px), kx),
                       sk_mul(sk_mul(s, px), ky),   sk_mul(-sk_mul(s, py), kx),  sk_mul(sk_mul(c, py), ky)};
  for (int i = 0; i < 6; ++i) M[i] = (long long)floor(sk_add(sk_mul(v[i], 65536.0), 0.5));
}
__host__ __device__ inline bool crop_map(int detection, double x, double y, double w, double h, double angle, int cw, int ch,
                                         int sw, int sh, int Sw, int Sh, double scale, long long M[6]) {
  if (!crop_tick(detection, x, y, w, h)) return false;
  double s, c, cx, cy;
  crop_frame(w, h, angle, s, c, cx, cy);
  crop_map_box(x, y, cx, cy, s, c, w, h, cw, ch, sw, sh, Sw, Sh, scale, M);
  return true;
}

// Framing (ht_tracker_set_framing; DESIGN.md 2, "Face crops", item 7): a per-stream filter whose state, the framed box
// (ht_framed_box, in caller-owned device memory), moves only on crop ticks (crop_tick: the ticks that write crops).
// The target is the green rectangle's centre, as crop_map places it, and the record's size.  The box snaps to the
// target when it is not valid yet, lies on another canvas size, or no longer holds the target's centre; otherwise
// each of cx, cy, width, height glides by alpha times the part of its error outside the dead zone, dead_zone times
// the old width (cx, width) or height (cy, height).  fp64 from the old state, every operation rounded as written.
__host__ __device__ __forceinline__ double framing_glide(double v, double t, double size, double alpha, double dead_zone) {
  const double band = sk_mul(dead_zone, size), e = sk_add(t, -v);
  return fabs(e) > band ? sk_add(v, sk_mul(alpha, sk_add(e, -copysign(band, e)))) : v;
}
// -> whether the record is a crop tick (and the box moved)
__host__ __device__ inline bool framing_step(ht_framed_box &b, double alpha, double dead_zone, int detection, double x,
                                             double y, double w, double h, double angle, int cw, int ch) {
  if (!crop_tick(detection, x, y, w, h)) return false;
  double s, c, cx, cy;
  crop_frame(w, h, angle, s, c, cx, cy);
  const double tx = sk_add(x, sk_add(sk_mul(c, cx), -sk_mul(s, cy)));
  const double ty = sk_add(y, sk_add(sk_mul(s, cx), sk_mul(c, cy)));
  if (!b.valid || b.canvas_w != cw || b.canvas_h != ch || fabs(sk_add(tx, -b.cx)) > sk_mul(b.width, 0.5) ||
      fabs(sk_add(ty, -b.cy)) > sk_mul(b.height, 0.5)) {
    b.cx = tx; b.cy = ty; b.width = w; b.height = h;
    b.canvas_w = cw; b.canvas_h = ch; b.valid = 1;
  } else {
    const double ow = b.width, oh = b.height;
    b.cx = framing_glide(b.cx, tx, ow, alpha, dead_zone);
    b.cy = framing_glide(b.cy, ty, oh, alpha, dead_zone);
    b.width = framing_glide(ow, w, ow, alpha, dead_zone);
    b.height = framing_glide(oh, h, oh, alpha, dead_zone);
  }
  ++b.updates;
  return true;
}
// The crop map of a framed box: crop_map's with local centre (0, 0), no rotation, and the box's centre and size.
// -> false for a box that is not valid (or, as crop_map, has a field that is not finite or beyond 65536 px).
__host__ __device__ inline bool crop_map_framed(const ht_framed_box &b, int cw, int ch, int sw, int sh, int Sw, int Sh,
                                                double scale, long long M[6]) {
  if (!b.valid || !crop_tick(2, b.cx, b.cy, b.width, b.height)) return false;
  crop_map_box(b.cx, b.cy, 0.0, 0.0, 0.0, 1.0, b.width, b.height, cw, ch, sw, sh, Sw, Sh, scale, M);
  return true;
}

// Face redaction (ht_tracker_set_redact; DESIGN.md 2, "Face redaction"): after the tick's crops, the cells of a
// B x B grid anchored at video pixel (0, 0) that meet the tracked face are overwritten in the video itself, with their
// mean (mosaic) or a colour (fill).
// A face tick: a record main.js strokes ("VJ" or "CS" with confidence != 0) with width > 0 and height > 0, its box
// finite and within 65536 px as crop_tick bounds it.
__host__ __device__ __forceinline__ bool redact_tick(int detection, double confidence, double x, double y, double w, double h) {
  if ((detection != 1 && detection != 2) || confidence == 0.0) return false;
  return crop_tick(2, x, y, w, h);
}
// A stream's hold: the box of its last face tick (record fields and canvas size) and the ticks it may still redact
// without one.  All 0 when the redaction is set.
struct RedactHold {
  double x, y, w, h, angle;
  int32_t detection, cw, ch, remaining;
};
// One tick of the hold for a record on a cw x ch canvas.  A face tick stores its box and remaining = hold; any other
// tick redacts the stored box while remaining > 0, if it ran a pass (detection != 0) on the stored canvas size, and
// takes one from remaining; an IDLE tick or a canvas-size change ends the hold.  -> whether the tick redacts, s then
// holding the box it redacts.
__host__ __device__ inline bool redact_hold_step(RedactHold &s, int hold, int detection, double confidence, double x,
                                                 double y, double w, double h, double angle, int cw, int ch) {
  if (redact_tick(detection, confidence, x, y, w, h)) {
    s.x = x; s.y = y; s.w = w; s.h = h; s.angle = angle;
    s.detection = detection; s.cw = cw; s.ch = ch; s.remaining = hold;
    return true;
  }
  if (detection == 0 || s.cw != cw || s.ch != ch) {
    s.remaining = 0;
    return false;
  }
  if (s.remaining <= 0) return false;
  --s.remaining;
  return true;
}
// The video pixels [r0, r2) x [r1, r3) of source-rectangle pixels [s0, s2) x [s1, s3) through view record v: its map
// is a signed permutation, so the two opposite corner pixels give the rectangle
__host__ __device__ __forceinline__ void redact_to_video(const ViewFeedRec &v, int s0, int s1, int s2, int s3, int r[4]) {
  const int ax = v.bx + v.mxx * s0 + v.mxy * s1, ay = v.by + v.myx * s0 + v.myy * s1;
  const int bx = v.bx + v.mxx * (s2 - 1) + v.mxy * (s3 - 1), by = v.by + v.myx * (s2 - 1) + v.myy * (s3 - 1);
  r[0] = ax < bx ? ax : bx; r[1] = ay < by ? ay : by;
  r[2] = (ax > bx ? ax : bx) + 1; r[3] = (ay > by ? ay : by) + 1;
}
// The redacted video rectangle r = [r0, r2) x [r1, r3) of a face box (a face tick's record fields) on a cw x ch canvas
// drawn from view record v's sw x sh source rectangle.  The region's four corners in canvas pixels - a VJ box upright,
// a CS box as crop_frame places the green rectangle, each scaled by `scale` about its centre - are computed in fp64,
// every operation rounded as written, and scaled by sw / cw and sh / ch; pixels floor(min) .. ceil(max) - 1, clipped to
// the rectangle, go through the view, every B x B cell (grid at video pixel 0) they meet is taken, and that is
// clipped to the rectangle in video pixels.  -> false for an empty region.
__host__ __device__ inline bool redact_rect(int detection, double x, double y, double w, double h, double angle, int cw,
                                            int ch, const ViewFeedRec &v, int block, double scale, int r[4]) {
  double s = 0.0, c = 1.0, lx = sk_mul(w, 0.5), ly = sk_mul(h, 0.5);     // VJ: the upright box's centre
  if (detection == 2) crop_frame(w, h, angle, s, c, lx, ly);
  const double hw = sk_mul(sk_mul(w, scale), 0.5), hh = sk_mul(sk_mul(h, scale), 0.5);
  const double kx = sk_div((double)v.sw, (double)cw), ky = sk_div((double)v.sh, (double)ch);
  double x0 = 0.0, x1 = 0.0, y0 = 0.0, y1 = 0.0;
  for (int i = 0; i < 4; ++i) {
    const double ax = sk_add(lx, (i & 1) ? hw : -hw), ay = sk_add(ly, (i & 2) ? hh : -hh);
    const double X = sk_mul(sk_add(x, sk_add(sk_mul(c, ax), -sk_mul(s, ay))), kx);
    const double Y = sk_mul(sk_add(y, sk_add(sk_mul(s, ax), sk_mul(c, ay))), ky);
    x0 = i == 0 || X < x0 ? X : x0; x1 = i == 0 || X > x1 ? X : x1;
    y0 = i == 0 || Y < y0 ? Y : y0; y1 = i == 0 || Y > y1 ? Y : y1;
  }
  x0 = fmax(floor(x0), 0.0); y0 = fmax(floor(y0), 0.0);
  x1 = fmin(ceil(x1), (double)v.sw); y1 = fmin(ceil(y1), (double)v.sh);
  if (!(x0 < x1) || !(y0 < y1)) return false;
  int f[4], a[4];
  redact_to_video(v, (int)x0, (int)y0, (int)x1, (int)y1, f);
  redact_to_video(v, 0, 0, v.sw, v.sh, a);                          // the source rectangle in video pixels
  const int B = block;
  r[0] = f[0] / B * B; r[1] = f[1] / B * B;
  r[2] = (f[2] + B - 1) / B * B; r[3] = (f[3] + B - 1) / B * B;
  r[0] = r[0] > a[0] ? r[0] : a[0]; r[1] = r[1] > a[1] ? r[1] : a[1];
  r[2] = r[2] < a[2] ? r[2] : a[2]; r[3] = r[3] < a[3] ? r[3] : a[3];
  return true;
}
// Sample channel k (0..2) of a view record's video: sample (i, j) at p + j pitch + i step, one byte or (wide) one
// 16-bit word, covering luma pixels with x >> sx == i and y >> sy == j.  RGBA8 video: R, G, B at step 4.  rgb: the
// channels are R, G, B (fill_rgb), otherwise Y, U, V (fill_yuv).
struct RedactChan {
  uint8_t *p;
  int32_t pitch, step, sx, sy, wide, rgb;
};
__host__ __device__ __forceinline__ RedactChan redact_chan(const ViewFeedRec &v, int k) {
  const YuvFeedRec &r = v.src;
  if (v.kind == VIEW_RGBA) return RedactChan{const_cast<uint8_t *>(r.y) + k, r.ypitch, 4, 0, 0, 0, 1};
  const int wide = r.sample_bytes == 2, rgb = r.rgb;
  if (k == 0) return RedactChan{const_cast<uint8_t *>(r.y), r.ypitch, r.ystep, 0, 0, wide, rgb};
  return RedactChan{const_cast<uint8_t *>(k == 1 ? r.u : r.v), k == 1 ? r.upitch : r.vpitch, r.cstep, r.sx, r.sy, wide, rgb};
}
// Cell [X0, X1) x [Y0, Y1) (luma pixels) of channel c: its samples [X0 >> sx, ((X1 - 1) >> sx) + 1) x (likewise in y)
// become (sum + cnt / 2) / cnt of them (mosaic) or `fill` (P010: fill << 8).  Lane `lane` of `lanes` visits samples
// lane, lane + lanes, ... in row order; sum(v) is the lanes' total, given to every lane (on the host, one lane: v).
template <class Sum>
__host__ __device__ __forceinline__ void redact_cell(const RedactChan &c, int X0, int Y0, int X1, int Y1, bool mosaic,
                                                     uint32_t fill, int lane, int lanes, Sum sum) {
  const int x0 = X0 >> c.sx, y0 = Y0 >> c.sy, w = ((X1 - 1) >> c.sx) + 1 - x0, y1 = ((Y1 - 1) >> c.sy) + 1;
  auto walk = [&](auto visit) {
    int i = lane, j = y0;
    while (i >= w) i -= w, ++j;
    while (j < y1) {
      visit(c.p + (size_t)j * c.pitch + (size_t)(x0 + i) * c.step);
      i += lanes;
      while (i >= w) i -= w, ++j;
    }
  };
  uint32_t value = c.wide ? fill << 8 : fill;
  if (mosaic) {
    uint32_t part = 0;
    walk([&](const uint8_t *p) { part += c.wide ? *reinterpret_cast<const uint16_t *>(p) : *p; });
    const uint32_t cnt = (uint32_t)w * (uint32_t)(y1 - y0);
    value = (sum(part) + cnt / 2) / cnt;
  }
  walk([&](uint8_t *p) {
    if (c.wide) *reinterpret_cast<uint16_t *>(p) = (uint16_t)value;
    else *p = (uint8_t)value;
  });
}
// Every cell of redacted rectangle r for channels 0..2 of view record v, cell `first`, first + stride, ... of the row-
// major cell grid (also run on the host by ht_selftest_face_redact)
template <class Sum>
__host__ __device__ __forceinline__ void redact_cells(const ViewFeedRec &v, const ht_face_redact &d, const int r[4], int first,
                                                      int stride, int lane, int lanes, Sum sum) {
  const int B = d.block, gx = r[0] / B, gy = r[1] / B;
  const int nx = (r[2] - 1) / B - gx + 1, ny = (r[3] - 1) / B - gy + 1;
  for (int cell = first; cell < nx * ny; cell += stride) {
    const int cx = gx + cell % nx, cy = gy + cell / nx;
    const int X0 = cx * B > r[0] ? cx * B : r[0], Y0 = cy * B > r[1] ? cy * B : r[1];
    const int X1 = (cx + 1) * B < r[2] ? (cx + 1) * B : r[2], Y1 = (cy + 1) * B < r[3] ? (cy + 1) * B : r[3];
    for (int k = 0; k < 3; ++k) {
      const RedactChan c = redact_chan(v, k);
      redact_cell(c, X0, Y0, X1, Y1, d.mode == HT_REDACT_MOSAIC, c.rgb ? d.fill_rgb[k] : d.fill_yuv[k], lane, lanes, sum);
    }
  }
}
// A stream's redaction in the device table: the caller's record (mode HT_REDACT_OFF: none) and its hold, which only
// k_face_redact and the setter write.  ticket counts the CTAs of a tick's entry that have read the hold.
struct Redact {
  ht_face_redact d;
  RedactHold s;
  uint32_t ticket, pad_;
};

// Crop pixel (i, j) of the map M over view record v (map, source rectangle and texel source resolved): bilinear with
// 8-bit weights between the taps (U >> 16, V >> 16) and their right and lower neighbours, taken in the rectangle and
// mapped to the video through the view, so a turned or mirrored video samples the same taps with the same weights as
// its upright twin.  A tap outside the rectangle reads (0, 0, 0, 0).
template <int KIND>
__host__ __device__ __forceinline__ uint32_t crop_pixel(const ViewFeedRec &v, const long long M[6], int i, int j) {
  const long long U = M[0] + (long long)i * M[2] + (long long)j * M[4], V = M[1] + (long long)i * M[3] + (long long)j * M[5];
  const long long x0 = U >> 16, y0 = V >> 16;
  const uint32_t fx = (uint32_t)(U >> 8) & 255u, fy = (uint32_t)(V >> 8) & 255u;
  auto tap = [&](long long x, long long y) -> uint32_t {
    if (x < 0 || y < 0 || x >= v.sw || y >= v.sh) return 0u;
    const int xi = (int)x, yi = (int)y;
    return view_texel<KIND>(v.src, v.bx + v.mxx * xi + v.mxy * yi, v.by + v.myx * xi + v.myy * yi);
  };
  const uint32_t p00 = tap(x0, y0), p01 = tap(x0 + 1, y0), p10 = tap(x0, y0 + 1), p11 = tap(x0 + 1, y0 + 1);
  const uint32_t w00 = (256u - fx) * (256u - fy), w01 = fx * (256u - fy), w10 = (256u - fx) * fy, w11 = fx * fy;
  uint32_t out = 0;
#pragma unroll
  for (int ch = 0; ch < 4; ++ch) {
    const uint32_t num = w00 * byte_of(p00, ch) + w01 * byte_of(p01, ch) + w10 * byte_of(p10, ch) + w11 * byte_of(p11, ch);
    out |= ((num + 32768u) >> 16) << (8 * ch);
  }
  return out;
}

// Best shots (ht_tracker_set_best_shot; DESIGN.md 2, "Best shots"): per track, the crop tick whose candidate - the
// RGBA8 crop of the best shot's size and scale - has the highest Laplacian energy.
// A candidate pixel as the score reads it: its gray (gray_of), or -1 where its alpha is below 255
__host__ __device__ __forceinline__ int best_gray(uint32_t px) { return (px >> 24) == 255u ? (int)gray_of(px) : -1; }
// The score's term of one pixel from the best_gray of it and of its left, right, upper and lower neighbours: L^2 with
// L = 4 c - l - r - u - d, or 0 if one of the five is -1.  At most 1020^2.
__host__ __device__ __forceinline__ uint32_t best_term(int c, int l, int r, int u, int d) {
  if ((c | l | r | u | d) < 0) return 0u;
  const int L = 4 * c - l - r - u - d;
  return (uint32_t)(L * L);
}
// Ends the stream's open track, if one is open (flags HT_BEST_ENDED); otherwise changes nothing
__host__ __device__ __forceinline__ void best_shot_end(ht_best_shot_state &s) {
  if (s.ended != s.track) {
    s.ended = s.track;
    s.flags = HT_BEST_ENDED;
  }
}
// One tick of a stream's best shot (two: it has two images): a record on a cw x ch canvas at clock now_ms whose
// candidate scored `score` (read only on a crop tick).  A crop tick begins a track if none is open, and sets the
// track's best on its first tick or with a score strictly above best_score; any other tick ends an open track.
// flags become the tick's.  -> whether the tick set a new best (the candidate is then to be written to rgba[buffer]).
__host__ __device__ inline bool best_shot_step(ht_best_shot_state &s, bool two, unsigned long long score, int detection,
                                               double x, double y, double w, double h, double angle, double now_ms, int cw,
                                               int ch) {
  s.flags = 0;
  if (!crop_tick(detection, x, y, w, h)) {
    best_shot_end(s);
    return false;
  }
  if (s.ended == s.track) {
    ++s.track;
    s.ticks = 0;
    s.buffer = two ? (int32_t)((s.track - 1u) & 1u) : 0;
    s.flags = HT_BEST_BEGAN;
  }
  s.score = score;
  const bool best = s.ticks == 0 || score > s.best_score;
  if (best) {
    s.best_score = score;
    s.x = x; s.y = y; s.width = w; s.height = h; s.angle = angle;
    s.now_ms = now_ms;
    s.canvas_w = cw; s.canvas_h = ch;
    s.best_tick = s.ticks;
    s.flags |= HT_BEST_IMPROVED;
  }
  ++s.ticks;
  return best;
}

// The video of batch entry k as a view record: the tick's frames (ht_tracker_step: frame k, one canvas size, 1:1),
// or the feed table's record k as k_feed_draw / k_feed_draw_yuv / k_feed_draw_view drew it.
enum : int32_t { CROP_FRAMES = 0, CROP_FEED = 1, CROP_YUV = 2, CROP_VIEW = 3 };
struct CropSource {
  int32_t mode, fw, fh, pad_;          // CROP_*; the frames' size
  const void *recs;                    // FeedRec / YuvFeedRec / ViewFeedRec table, or the frames
};
__device__ __forceinline__ void crop_source(const CropSource &s, int k, ViewFeedRec &v) {
  if (s.mode == CROP_VIEW) { v = reinterpret_cast<const ViewFeedRec *>(s.recs)[k]; return; }
  v.src = YuvFeedRec{};
  v.bx = v.by = v.mxy = v.myx = 0;
  v.mxx = v.myy = 1;
  v.pad_ = 0;
  if (s.mode == CROP_YUV) {
    v.src = reinterpret_cast<const YuvFeedRec *>(s.recs)[k];
    v.kind = nv12_i420_path(v.src) ? VIEW_NV12_I420 : VIEW_FMT;
  } else if (s.mode == CROP_FEED) {
    const FeedRec r = reinterpret_cast<const FeedRec *>(s.recs)[k];
    v.src.y = r.src, v.src.ypitch = r.pitch, v.src.width = r.width, v.src.height = r.height;
    v.kind = VIEW_RGBA;
  } else {
    v.src.y = reinterpret_cast<const uint8_t *>(s.recs) + (size_t)k * s.fw * s.fh * 4;
    v.src.ypitch = 4 * s.fw, v.src.width = s.fw, v.src.height = s.fh;
    v.kind = VIEW_RGBA;
  }
  v.sw = v.src.width, v.sh = v.src.height;
}

// One 64 x 16 tile from (X0, Y0) of crop f: a warp writes 128 consecutive bytes of a crop row.  Out of line per texel
// source, as feed_draw_view, so that each keeps its own registers.  COPY: one instantiation per calling kernel
// (k_face_crop 0, k_best_write 1), since ptxas allocates an out-of-line function's registers across all its callers.
template <int KIND, int COPY = 0>
__device__ __noinline__ void face_crop_tile(const ViewFeedRec *__restrict__ vp, const long long *__restrict__ Mp,
                                            const FaceCrop f, int X0, int Y0) {
  const ViewFeedRec v = *vp;
  long long M[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) M[i] = Mp[i];
  const int X = X0 + (threadIdx.x & 63);
  if (X >= f.w) return;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int Y = Y0 + 4 * r + (threadIdx.x >> 6);
    if (Y < f.h) reinterpret_cast<uint32_t *>(f.rgba + (size_t)Y * f.pitch)[X] = crop_pixel<KIND>(v, M, X, Y);
  }
}

// Two bytes at p (an even address: one 16-bit store)
__host__ __device__ __forceinline__ void crop_put2(uint8_t *p, uint32_t lo, uint32_t hi) {
  if ((reinterpret_cast<uintptr_t>(p) & 1u) == 0) *reinterpret_cast<uint16_t *>(p) = (uint16_t)(lo | hi << 8);
  else p[0] = (uint8_t)lo, p[1] = (uint8_t)hi;
}
// The 2 x 2 block from even (X, Y) of YUV crop f / c: the four RGBA8 pixels of the crop of the same size and scale
// (crop_pixel), converted by rgba_to_yuv420 into their four Y samples and one U and one V sample.
template <int KIND, bool NV12>
__host__ __device__ __forceinline__ void crop_yuv_block(const ViewFeedRec &v, const long long M[6], const FaceCrop &f,
                                                        const CropPlanes &c, int X, int Y) {
  uint32_t uv;
  const uint32_t y4 = rgba_to_yuv420(c.color, crop_pixel<KIND>(v, M, X, Y), crop_pixel<KIND>(v, M, X + 1, Y),
                                     crop_pixel<KIND>(v, M, X, Y + 1), crop_pixel<KIND>(v, M, X + 1, Y + 1), uv);
  uint8_t *y = f.rgba + (size_t)Y * f.pitch + X;
  crop_put2(y, y4 & 0xffu, (y4 >> 8) & 0xffu);
  crop_put2(y + f.pitch, (y4 >> 16) & 0xffu, y4 >> 24);
  const size_t row = (size_t)(Y >> 1);
  if (NV12) {
    crop_put2(c.u + row * c.upitch + X, uv & 0xffu, uv >> 8);
  } else {
    c.u[row * c.upitch + (X >> 1)] = (uint8_t)uv;
    c.v[row * c.vpitch + (X >> 1)] = (uint8_t)(uv >> 8);
  }
}

// One 64 x 16 tile from (X0, Y0) of YUV crop f / c: each thread one 2 x 2 block, a warp 64 consecutive Y bytes of two
// rows.  Out of line per texel source and output layout, as face_crop_tile.  The view record and the map stay in
// k_face_crop's shared memory (vp, Mp): copied into registers, as face_crop_tile does, they would lift k_face_crop from
// 64 to 80 registers and cost every crop, RGBA included, a quarter of its resident CTAs.
template <int KIND, bool NV12>
__device__ __noinline__ void face_crop_yuv_tile(const ViewFeedRec *__restrict__ vp, const long long *__restrict__ Mp,
                                                const FaceCrop f, const CropPlanes c, int X0, int Y0) {
  const ViewFeedRec &v = *vp;
  const long long *M = Mp;
  const int X = X0 + 2 * (int)(threadIdx.x & 31), Y = Y0 + 2 * (int)(threadIdx.x >> 5);
  if (X < f.w && Y < f.h) crop_yuv_block<KIND, NV12>(v, M, f, c, X, Y);
}

// Face tensors (ht_tracker_set_face_tensor; DESIGN.md 2, "Face crops", item 6): a stream's face as a model's input, the
// RGBA8 crop of the same size and scale converted per pixel, alpha ignored.  Layout of ht_face_tensor (strides in
// elements); data NULL: the stream has none.
struct FaceTensor {
  void *data;
  long long row, plane;
  int32_t w, h, dtype, layout, channels, pad_;   // HT_TENSOR_*
  float mul[3], add[3];
  double scale;
};

// One channel value c of a face tensor as its element's bits: U8 c; F32 fmaf(c, mul, add), one rounding; F16 / BF16
// that float rounded to nearest even (overflow: +-inf).
__host__ __device__ __forceinline__ uint32_t tensor_value(int dtype, uint32_t c, float mul, float add) {
  if (dtype == HT_TENSOR_U8) return c;
#ifdef __CUDA_ARCH__
  const float v = __fmaf_rn((float)c, mul, add);     // explicit: the build contracts nothing (-fmad=false)
#else
  const float v = fmaf((float)c, mul, add);
#endif
  if (dtype == HT_TENSOR_F16) return __half_raw(__float2half_rn(v)).x;
  if (dtype == HT_TENSOR_BF16) return __nv_bfloat16_raw(__float2bfloat16_rn(v)).x;
#ifdef __CUDA_ARCH__
  return __float_as_uint(v);
#else
  uint32_t u;
  memcpy(&u, &v, 4);
  return u;
#endif
}

// Pixel (i, j) of face tensor t from px, the pixel (i, j) of the RGBA8 crop of its size and scale: channel k of
// HT_TENSOR_RGB is byte k of px, of HT_TENSOR_BGR byte 2 - k, and HT_TENSOR_GRAY's one channel is gray_of(px); each is
// converted by tensor_value and stored at k plane + j row + i (CHW) or j row + i C + k (HWC).
__host__ __device__ __forceinline__ void tensor_put(const FaceTensor &t, uint32_t px, int i, int j) {
  const bool gray = t.channels == HT_TENSOR_GRAY, bgr = t.channels == HT_TENSOR_BGR, hwc = t.layout == HT_TENSOR_HWC;
  const int C = gray ? 1 : 3;
  const long long at = (long long)j * t.row + (hwc ? (long long)i * C : (long long)i), step = hwc ? 1 : t.plane;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (k >= C) break;
    const uint32_t c = gray ? gray_of(px) : byte_of(px, bgr ? 2 - k : k);
    const uint32_t bits = tensor_value(t.dtype, c, t.mul[k], t.add[k]);
    const long long e = at + k * step;
    if (t.dtype == HT_TENSOR_U8) static_cast<uint8_t *>(t.data)[e] = (uint8_t)bits;
    else if (t.dtype == HT_TENSOR_F32) static_cast<uint32_t *>(t.data)[e] = bits;
    else static_cast<uint16_t *>(t.data)[e] = (uint16_t)bits;
  }
}

// One 64 x 16 tile from (X0, Y0) of face tensor *tp: a warp converts 32 consecutive pixels of one row, so each plane's
// stores (CHW) or the row's interleaved ones (HWC) are consecutive elements.  Out of line per texel source; dtype,
// layout and channel order are warp-uniform runtime branches.  The view record and the map stay in k_face_crop's shared
// memory and the tensor record in global memory, as face_crop_yuv_tile keeps them, so k_face_crop stays at 64
// registers.
template <int KIND>
__device__ __noinline__ void face_tensor_tile(const ViewFeedRec *__restrict__ vp, const long long *__restrict__ Mp,
                                              const FaceTensor *__restrict__ tp, int X0, int Y0) {
  const ViewFeedRec &v = *vp;
  const FaceTensor &t = *tp;
  const int X = X0 + (threadIdx.x & 63);
  if (X >= t.w) return;
#pragma unroll 1
  for (int r = 0; r < 4; ++r) {
    const int Y = Y0 + 4 * r + (threadIdx.x >> 6);
    if (Y < t.h) tensor_put(t, crop_pixel<KIND>(v, Mp, X, Y), X, Y);
  }
}

// After k_tracker_update: grid (tiles of the largest crop or tensor, batch entries, slices).  Slice tz is the face
// tensors' (tz = 1 while some stream has a crop, else 0; a grid without a tensor slice never reaches it), the other one
// the crops'.  Entry k's CTAs read its record (events[geo[k].record], geo NULL: k) and canvas size (geo[k], geo NULL:
// cw x ch), and write the tiles of its stream's crop or tensor on a crop tick; entries without one, without a crop tick,
// or past their own tiles exit at once.  An RGBA crop's tiles go to face_crop_tile, a YUV crop's (layout, then
// planes[id]) to face_crop_yuv_tile, a tensor's to face_tensor_tile.
// framing (NULL while no stream has one): a stream whose framing's `outputs` has the output's bit takes the map of
// its framed box (k_framing_update has moved it for this tick) in place of the record's.
__global__ void __launch_bounds__(256) k_face_crop(const int32_t *__restrict__ ids, const EntryCanvas *__restrict__ geo,
                                                   int cw, int ch, const TrackerEvent *__restrict__ events,
                                                   const FaceCrop *__restrict__ crops,
                                                   const CropPlanes *__restrict__ planes,
                                                   const FaceTensor *__restrict__ tensors, int tz, CropSource src,
                                                   const ht_framing *__restrict__ framing) {
  const int k = blockIdx.y, id = ids ? ids[k] : k;
  const bool tensor = (int)blockIdx.z == tz;
  FaceCrop f;
  if (tensor) {                        // only the geometry: the body reads the rest of the record
    const FaceTensor &t = tensors[id];
    f = FaceCrop{static_cast<uint8_t *>(t.data), t.w, t.h, 0, 0, t.scale};
  } else {
    f = crops[id];
  }
  if (!f.rgba) return;
  const int tiles_x = (f.w + CROP_TX - 1) / CROP_TX;
  if ((int)blockIdx.x >= tiles_x * ((f.h + CROP_TY - 1) / CROP_TY)) return;
  __shared__ ViewFeedRec v;
  __shared__ long long M[6];
  __shared__ int on;
  if (threadIdx.x == 0) {
    crop_source(src, k, v);
    const TrackerEvent &e = events[geo ? geo[k].record : k];
    const int ew = geo ? geo[k].w : cw, eh = geo ? geo[k].h : ch;
    on = crop_map(e.detection, e.x, e.y, e.width, e.height, e.angle, ew, eh, v.sw, v.sh, f.w, f.h, f.scale, M);
    if (on && framing) {
      const ht_framing &g = framing[id];
      if (g.box && (g.outputs & (tensor ? HT_FRAMING_TENSOR : HT_FRAMING_CROP)))
        on = crop_map_framed(*g.box, ew, eh, v.sw, v.sh, f.w, f.h, f.scale, M);
    }
  }
  __syncthreads();
  if (!on) return;
  const int X0 = ((int)blockIdx.x % tiles_x) * CROP_TX, Y0 = ((int)blockIdx.x / tiles_x) * CROP_TY;
  if (tensor) {
    if (v.kind == VIEW_RGBA) face_tensor_tile<VIEW_RGBA>(&v, M, tensors + id, X0, Y0);
    else if (v.kind == VIEW_NV12_I420) face_tensor_tile<VIEW_NV12_I420>(&v, M, tensors + id, X0, Y0);
    else face_tensor_tile<VIEW_FMT>(&v, M, tensors + id, X0, Y0);
    return;
  }
  if (f.layout == CROP_RGBA) {
    if (v.kind == VIEW_RGBA) face_crop_tile<VIEW_RGBA>(&v, M, f, X0, Y0);
    else if (v.kind == VIEW_NV12_I420) face_crop_tile<VIEW_NV12_I420>(&v, M, f, X0, Y0);
    else face_crop_tile<VIEW_FMT>(&v, M, f, X0, Y0);
    return;
  }
  const CropPlanes c = planes[id];
  if (f.layout == CROP_NV12) {
    if (v.kind == VIEW_RGBA) face_crop_yuv_tile<VIEW_RGBA, true>(&v, M, f, c, X0, Y0);
    else if (v.kind == VIEW_NV12_I420) face_crop_yuv_tile<VIEW_NV12_I420, true>(&v, M, f, c, X0, Y0);
    else face_crop_yuv_tile<VIEW_FMT, true>(&v, M, f, c, X0, Y0);
  } else {
    if (v.kind == VIEW_RGBA) face_crop_yuv_tile<VIEW_RGBA, false>(&v, M, f, c, X0, Y0);
    else if (v.kind == VIEW_NV12_I420) face_crop_yuv_tile<VIEW_NV12_I420, false>(&v, M, f, c, X0, Y0);
    else face_crop_yuv_tile<VIEW_FMT, false>(&v, M, f, c, X0, Y0);
  }
}

// After k_tracker_update, before k_face_crop: batch entry k (stream ids[k], NULL: k; its record events[geo[k].record]
// and canvas geo[k], geo NULL: k and cw x ch) moves its stream's framed box, if the stream has a framing.
__global__ void k_framing_update(const int32_t *__restrict__ ids, const EntryCanvas *__restrict__ geo, int n, int cw, int ch,
                                 const TrackerEvent *__restrict__ events, const ht_framing *__restrict__ framing) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const ht_framing &g = framing[ids ? ids[k] : k];
  if (!g.box) return;
  const TrackerEvent &e = events[geo ? geo[k].record : k];
  ht_framed_box b = *g.box;
  if (framing_step(b, g.alpha, g.dead_zone, e.detection, e.x, e.y, e.width, e.height, e.angle, geo ? geo[k].w : cw,
                   geo ? geo[k].h : ch))
    *g.box = b;
}

// ht_tracker_set_framing: one CTA makes the framed boxes of streams [first, first + n) that have a framing invalid,
// with no updates
__global__ void k_framing_reset(const ht_framing *__restrict__ framing, int first, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (framing[first + i].box) *framing[first + i].box = ht_framed_box{};
}

// The tick's last launch, after k_face_crop and k_track_init have read the video: grid (R, batch entries).  Thread 0
// of each of entry k's R CTAs resolves its video (src), its record (events[geo[k].record], geo NULL: k; canvas geo[k],
// geo NULL: cw x ch), the hold of its stream's redaction and the redacted rectangle; the CTAs then share out the cells,
// one warp per cell.  Each CTA reads the hold before it takes a ticket, and the entry's last ticket writes the hold
// back, so every CTA sees the hold as the tick found it.  Entries whose stream has no redaction exit at once.
__global__ void __launch_bounds__(256) k_face_redact(const int32_t *__restrict__ ids, const EntryCanvas *__restrict__ geo,
                                                     int cw, int ch, const TrackerEvent *__restrict__ events,
                                                     Redact *redact, CropSource src) {
  const int k = blockIdx.y, id = ids ? ids[k] : k;
  Redact &t = redact[id];
  if (t.d.mode == HT_REDACT_OFF) return;
  __shared__ ViewFeedRec v;
  __shared__ int r[4], on;
  if (threadIdx.x == 0) {
    crop_source(src, k, v);
    const TrackerEvent &e = events[geo ? geo[k].record : k];
    const int ew = geo ? geo[k].w : cw, eh = geo ? geo[k].h : ch;
    RedactHold s = t.s;
    on = redact_hold_step(s, t.d.hold, e.detection, e.confidence, e.x, e.y, e.width, e.height, e.angle, ew, eh) &&
         redact_rect(s.detection, s.x, s.y, s.w, s.h, s.angle, ew, eh, v, t.d.block, t.d.scale, r);
    __threadfence();
    if (atomicAdd(&t.ticket, 1u) == gridDim.x - 1) {
      t.s = s;
      t.ticket = 0;
    }
  }
  __syncthreads();
  if (!on) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  redact_cells(v, t.d, r, (int)blockIdx.x * 8 + warp, (int)gridDim.x * 8, lane, 32, [](uint32_t x) {
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
  });
}

// A stream's best shot in the device table: the caller's record with the pitch resolved (rgba[0] NULL: none), and the
// running sum and ticket of its tick, which only k_best_score writes (0 between ticks).
struct BestShot {
  ht_best_shot d;
  unsigned long long acc;
  uint32_t ticket, pad_;
};
constexpr int BEST_HX = CROP_TX + 2, BEST_HY = CROP_TY + 2;   // a score tile with its one-pixel halo

// The best_gray of the candidate pixels [X0 - 1, X0 + CROP_TX] x [Y0 - 1, Y0 + CROP_TY] inside the W x H candidate
// into g (k_best_score's shared memory; the others are never read).  Out of line per texel source, as face_crop_tile;
// the view record and the map stay in shared memory (vp, Mp), as face_tensor_tile keeps them, which holds the kernel
// to 64 registers.
template <int KIND>
__device__ __noinline__ void best_tile_gray(const ViewFeedRec *__restrict__ vp, const long long *__restrict__ Mp,
                                            int16_t (*g)[BEST_HX], int X0, int Y0, int W, int H) {
  const ViewFeedRec &v = *vp;
  const long long *M = Mp;
  for (int t = threadIdx.x; t < BEST_HX * BEST_HY; t += blockDim.x) {
    const int x = t % BEST_HX, y = t / BEST_HX, i = X0 - 1 + x, j = Y0 - 1 + y;
    if (i >= 0 && j >= 0 && i < W && j < H) g[y][x] = (int16_t)best_gray(crop_pixel<KIND>(v, M, i, j));
  }
}

// After k_face_crop, before k_face_redact: grid (tiles of the largest best shot, batch entries).  Entry k (stream
// ids[k], NULL: k; record events[geo[k].record] and canvas geo[k], geo NULL: k and cw x ch; clock now[k], NULL:
// now_ms) scores the candidate of its stream's best shot on a crop tick: each of its CTAs samples one 64 x 16 tile and
// its halo with crop_pixel, sums best_term over the tile's scored pixels and adds that to the stream's acc; the last
// ticket takes the total, steps the state and resets acc and ticket.  On any other tick CTA 0 alone steps the state.
// Streams without a best shot and CTAs past their own tiles exit at once.
__global__ void __launch_bounds__(256) k_best_score(const int32_t *__restrict__ ids, const EntryCanvas *__restrict__ geo,
                                                    int cw, int ch, const TrackerEvent *__restrict__ events, double now_ms,
                                                    const double *__restrict__ now, BestShot *best, CropSource src) {
  const int k = blockIdx.y, id = ids ? ids[k] : k;
  BestShot &b = best[id];
  if (!b.d.rgba[0]) return;
  const int W = b.d.width, H = b.d.height, tiles_x = (W + CROP_TX - 1) / CROP_TX;
  const unsigned tiles = (unsigned)(tiles_x * ((H + CROP_TY - 1) / CROP_TY));
  if (blockIdx.x >= tiles) return;
  const TrackerEvent &e = events[geo ? geo[k].record : k];
  const int ew = geo ? geo[k].w : cw, eh = geo ? geo[k].h : ch;
  const double t = now ? now[k] : now_ms;
  const bool two = b.d.rgba[1] != nullptr;
  if (!crop_tick(e.detection, e.x, e.y, e.width, e.height)) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      ht_best_shot_state s = *b.d.state;
      best_shot_step(s, two, 0, e.detection, e.x, e.y, e.width, e.height, e.angle, t, ew, eh);
      *b.d.state = s;
    }
    return;
  }
  __shared__ ViewFeedRec v;
  __shared__ long long M[6];
  __shared__ int16_t g[BEST_HY][BEST_HX];
  __shared__ uint32_t part[8];
  if (threadIdx.x == 0) {
    crop_source(src, k, v);
    crop_map(e.detection, e.x, e.y, e.width, e.height, e.angle, ew, eh, v.sw, v.sh, W, H, b.d.scale, M);
  }
  __syncthreads();
  const int X0 = ((int)blockIdx.x % tiles_x) * CROP_TX, Y0 = ((int)blockIdx.x / tiles_x) * CROP_TY;
  if (v.kind == VIEW_RGBA) best_tile_gray<VIEW_RGBA>(&v, M, g, X0, Y0, W, H);
  else if (v.kind == VIEW_NV12_I420) best_tile_gray<VIEW_NV12_I420>(&v, M, g, X0, Y0, W, H);
  else best_tile_gray<VIEW_FMT>(&v, M, g, X0, Y0, W, H);
  __syncthreads();
  // a CTA's sum stays below 2^32: 1024 pixels of at most 1020^2
  uint32_t sum = 0;
  const int x = threadIdx.x & 63, i = X0 + x;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int y = 4 * r + (threadIdx.x >> 6), j = Y0 + y;
    if (i >= 1 && i <= W - 2 && j >= 1 && j <= H - 2)
      sum += best_term(g[y + 1][x + 1], g[y + 1][x], g[y + 1][x + 2], g[y][x + 1], g[y + 2][x + 1]);
  }
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < 8; ++w) sum += part[w];
  atomicAdd(&b.acc, (unsigned long long)sum);
  __threadfence();
  if (atomicAdd(&b.ticket, 1u) != tiles - 1) return;
  __threadfence();
  const unsigned long long score = atomicExch(&b.acc, 0ull);
  b.ticket = 0;
  ht_best_shot_state s = *b.d.state;
  best_shot_step(s, two, score, e.detection, e.x, e.y, e.width, e.height, e.angle, t, ew, eh);
  *b.d.state = s;
}

// After k_best_score: grid (tiles of the largest best shot, batch entries).  Entry k's CTAs write the candidate (the
// crop of its best shot's size and scale, by face_crop_tile) into rgba[buffer] if its tick set a new best
// (HT_BEST_IMPROVED in the state k_best_score has just stepped).
__global__ void __launch_bounds__(256) k_best_write(const int32_t *__restrict__ ids, const EntryCanvas *__restrict__ geo,
                                                    int cw, int ch, const TrackerEvent *__restrict__ events,
                                                    const BestShot *__restrict__ best, CropSource src) {
  const int k = blockIdx.y, id = ids ? ids[k] : k;
  const BestShot &b = best[id];
  if (!b.d.rgba[0]) return;
  const int W = b.d.width, H = b.d.height, tiles_x = (W + CROP_TX - 1) / CROP_TX;
  if ((int)blockIdx.x >= tiles_x * ((H + CROP_TY - 1) / CROP_TY)) return;
  __shared__ ViewFeedRec v;
  __shared__ long long M[6];
  __shared__ int buffer;
  if (threadIdx.x == 0) {
    const ht_best_shot_state &s = *b.d.state;
    buffer = (s.flags & HT_BEST_IMPROVED) ? s.buffer : -1;
    if (buffer >= 0) {
      crop_source(src, k, v);
      const TrackerEvent &e = events[geo ? geo[k].record : k];
      crop_map(e.detection, e.x, e.y, e.width, e.height, e.angle, geo ? geo[k].w : cw, geo ? geo[k].h : ch, v.sw, v.sh, W,
               H, b.d.scale, M);
    }
  }
  __syncthreads();
  if (buffer < 0) return;
  const FaceCrop f{b.d.rgba[buffer], W, H, b.d.pitch, CROP_RGBA, b.d.scale};
  const int X0 = ((int)blockIdx.x % tiles_x) * CROP_TX, Y0 = ((int)blockIdx.x / tiles_x) * CROP_TY;
  if (v.kind == VIEW_RGBA) face_crop_tile<VIEW_RGBA, 1>(&v, M, f, X0, Y0);
  else if (v.kind == VIEW_NV12_I420) face_crop_tile<VIEW_NV12_I420, 1>(&v, M, f, X0, Y0);
  else face_crop_tile<VIEW_FMT, 1>(&v, M, f, X0, Y0);
}

// ht_tracker_set_best_shot: one CTA zeroes the states of streams [first, first + n) that have a best shot
__global__ void k_best_reset(const BestShot *__restrict__ best, int first, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (best[first + i].d.rgba[0]) *best[first + i].d.state = ht_best_shot_state{};
}

// ht_tracker_import: the n streams ids[0..n) that have a best shot end their open tracks
__global__ void k_best_end(const int32_t *__restrict__ ids, int n, const BestShot *__restrict__ best) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const BestShot &b = best[ids[k]];
  if (!b.d.rgba[0]) return;
  ht_best_shot_state s = *b.d.state;
  best_shot_end(s);
  *b.d.state = s;
}

// ht_tracker_set_camera: one CTA constructs the cameras of streams [first, first + n) that have a controller
__global__ void k_camera_construct(const CameraCtl *__restrict__ ctl, int first, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const CameraCtl &c = ctl[first + i];
    if (!c.camera) continue;
    ht_camera cam;
    camera_construct(cam, c);
    *c.camera = cam;
  }
}

// the parameter check of ht_tracker_config / ht_tracker_set_params, also applied to imported records
__host__ __device__ inline bool tracker_head_ok(double alpha, double distance_to_screen) {
  return alpha >= 0.0 && alpha <= 1.0 && distance_to_screen > 0.0;
}

// ------------------------------------------------------------------------------------------------
// Tracker records (ht_tracker_export / ht_tracker_import): one stream's whole headtrackr.Tracker as a fixed-size,
// position-independent, little-endian byte string, so that a stream can move to another slot, context or GPU and
// outlive its process.  Byte offsets (include/headtrackr_b200.h; every section 16-byte aligned, the gaps zero):
//   0           header: u32 magic "HTR1", u32 format version, u32 record bytes, u32 0, u64 checksum, u32 0, u32 0
//   REC_STATE   TrackerState, as tracker_step keeps it
//   REC_PARAMS  TrackerParams as the device holds them (the head-model constants travel: import does not recompute them)
//   REC_TRACK   camshift section: the slot's TrackState, then (REC_COST) its two d_track_cost words, then
//   REC_HIST    its 4096-bin model histogram
// checksum = sum of w_i * (2i + 1) mod 2^64 over the 32-bit words from byte 24 on (i = 0, 1, ...): a flipped bit changes
// it (2^b times an odd number is never 0 mod 2^64), and so does swapping two unequal words (2 |j - i| |w_i - w_j| <
// 2^64).  Canonical form: the camshift section of a stream that is not in CS is dead state (the next hand-off re-seeds
// it) and is written as zeros, so export(import(r)) == r and two exports of one state are byte-identical.
constexpr uint32_t REC_MAGIC = 0x31525448u;        // "HTR1"
constexpr uint32_t REC_VERSION = 1;
__host__ __device__ constexpr int rec_align16(size_t b) { return (int)((b + 15) / 16 * 16); }
constexpr int REC_STATE = 32;
constexpr int REC_PARAMS = rec_align16(REC_STATE + sizeof(TrackerState));
constexpr int REC_TRACK = rec_align16(REC_PARAMS + sizeof(TrackerParams));
constexpr int REC_COST = REC_TRACK + (int)sizeof(TrackState);
constexpr int REC_HIST = rec_align16(REC_COST + 2 * sizeof(int32_t));
constexpr int REC_BYTES = REC_HIST + 4096 * (int)sizeof(uint32_t);
constexpr int REC_HEAD_WORDS = REC_HIST / 4;       // the words before the histogram
constexpr int REC_SUM0 = 6;                        // the first word under the checksum
static_assert(sizeof(TrackerState) % 4 == 0 && sizeof(TrackerParams) % 4 == 0 && sizeof(TrackState) % 4 == 0 &&
                  REC_BYTES % 16 == 0, "tracker record sections are whole words, the record whole 16-byte vectors");
// import status of a record, in the order the checks run
enum { REC_OK = 0, REC_BAD_MAGIC, REC_BAD_VERSION, REC_BAD_SIZE, REC_BAD_CHECKSUM, REC_BAD_MODE, REC_BAD_WB, REC_BAD_DIAG,
       REC_BAD_PARAMS, REC_BAD_TRACK };

__host__ __device__ inline uint32_t rec_word(const void *p, int j) {
  uint32_t w;
  memcpy(&w, static_cast<const char *>(p) + 4 * j, 4);
  return w;
}
__host__ __device__ inline void rec_put(void *p, int j, uint32_t w) { memcpy(static_cast<char *>(p) + 4 * j, &w, 4); }
__host__ __device__ __forceinline__ unsigned long long rec_term(int i, uint32_t w) {   // word i's share of the checksum
  return (unsigned long long)w * (2ull * (unsigned)(i - REC_SUM0) + 1ull);
}

// word i < REC_HEAD_WORDS of a stream's record, the checksum words (4, 5) as 0.  cs: the stream is in CS, so its
// camshift section is live.
__host__ __device__ inline uint32_t tracker_record_head_word(int i, const TrackerState &s, const TrackerParams &p,
                                                             const TrackState &t, const int32_t *cost, bool cs) {
  const int b = 4 * i;
  if (i == 0) return REC_MAGIC;
  if (i == 1) return REC_VERSION;
  if (i == 2) return (uint32_t)REC_BYTES;
  if (b >= REC_STATE && b < REC_STATE + (int)sizeof(TrackerState)) return rec_word(&s, (b - REC_STATE) / 4);
  if (b >= REC_PARAMS && b < REC_PARAMS + (int)sizeof(TrackerParams)) return rec_word(&p, (b - REC_PARAMS) / 4);
  if (!cs) return 0;
  if (b >= REC_TRACK && b < REC_COST) return rec_word(&t, (b - REC_TRACK) / 4);
  if (b >= REC_COST && b < REC_COST + 8) return (uint32_t)cost[(b - REC_COST) / 4];
  return 0;
}

// word i < REC_HEAD_WORDS of a checked record, w, into the stream's sections; cs: the record's mode is CS (otherwise
// its camshift section is stored as zeros, whatever the record holds)
__host__ __device__ inline void tracker_record_unpack_word(int i, uint32_t w, bool cs, TrackerState &s, TrackerParams &p,
                                                           TrackState &t, int32_t *cost) {
  const int b = 4 * i;
  if (b >= REC_STATE && b < REC_STATE + (int)sizeof(TrackerState)) rec_put(&s, (b - REC_STATE) / 4, w);
  else if (b >= REC_PARAMS && b < REC_PARAMS + (int)sizeof(TrackerParams)) rec_put(&p, (b - REC_PARAMS) / 4, w);
  else if (b >= REC_TRACK && b < REC_COST) rec_put(&t, (b - REC_TRACK) / 4, cs ? w : 0u);
  else if (b >= REC_COST && b < REC_COST + 8) cost[(b - REC_COST) / 4] = cs ? (int32_t)w : 0;
}

// The whole record of a stream, sequentially (k_tracker_export does the same per word with one CTA).  hist: the
// slot's model histogram; track, hist and cost are read only when the stream is in CS.
__host__ __device__ inline void tracker_record_pack(uint8_t *rec, const TrackerState &s, const TrackerParams &p,
                                                    const TrackState &t, const uint32_t *hist, const int32_t *cost) {
  const bool cs = s.mode == TM_CS;
  unsigned long long sum = 0;
  for (int i = 0; i < REC_BYTES / 4; ++i) {
    const uint32_t w = i < REC_HEAD_WORDS ? tracker_record_head_word(i, s, p, t, cost, cs) : cs ? hist[i - REC_HEAD_WORDS] : 0u;
    rec_put(rec, i, w);
    if (i >= REC_SUM0) sum += rec_term(i, w);
  }
  memcpy(rec + 16, &sum, 8);
}

// the checksum of a record's words, sequentially (k_tracker_import_check sums them with one CTA)
__host__ __device__ inline unsigned long long tracker_record_sum(const uint8_t *rec) {
  unsigned long long sum = 0;
  for (int i = REC_SUM0; i < REC_BYTES / 4; ++i) sum += rec_term(i, rec_word(rec, i));
  return sum;
}

// The checks of import, given the checksum of the record's words: the header, the checksum, then every field that
// indexes an array or selects a branch.  -> REC_OK or the first failed check.
__host__ __device__ inline int tracker_record_check(const uint8_t *rec, unsigned long long sum) {
  if (rec_word(rec, 0) != REC_MAGIC) return REC_BAD_MAGIC;
  if (rec_word(rec, 1) != REC_VERSION) return REC_BAD_VERSION;
  if (rec_word(rec, 2) != (uint32_t)REC_BYTES || rec_word(rec, 3) != 0u) return REC_BAD_SIZE;
  unsigned long long stored;
  memcpy(&stored, rec + 16, 8);
  if (stored != sum) return REC_BAD_CHECKSUM;
  TrackerState s;
  TrackerParams p;
  TrackState t;
  memcpy(&s, rec + REC_STATE, sizeof(s));
  memcpy(&p, rec + REC_PARAMS, sizeof(p));
  memcpy(&t, rec + REC_TRACK, sizeof(t));
  if (s.mode < TM_IDLE || s.mode > TM_CS) return REC_BAD_MODE;
  if (s.n_wb < 0 || s.n_wb > WB_WINDOW) return REC_BAD_WB;
  if (s.head.n_diag < 0 || s.head.n_diag > 6) return REC_BAD_DIAG;              // head_step: s.diag[s.n_diag++]
  if (!tracker_head_ok(p.head.alpha, p.head.distance_to_screen)) return REC_BAD_PARAMS;
  if (s.mode == TM_CS && !(t.initialised == 1 && t.sw > 0 && t.sh > 0)) return REC_BAD_TRACK;   // k_track's window
  return REC_OK;
}

// sum of v over the CTA (256 threads), valid in thread 0
__device__ __forceinline__ unsigned long long cta_sum_u64(unsigned long long v, unsigned long long *part) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned long long s = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < 8; ++w) s += part[w];
  return s;
}

// Record k of `records` (16-byte aligned, REC_BYTES apart) := stream ids[k].  One CTA per record: the head word by word,
// the histogram in 16-byte vectors (zeros when the stream is not in CS), then the checksum.
__global__ void __launch_bounds__(256) k_tracker_export(const int32_t *__restrict__ ids, const TrackerState *__restrict__ st,
                                                        const TrackerParams *__restrict__ params,
                                                        const TrackState *__restrict__ track,
                                                        const uint32_t *__restrict__ model_hist,
                                                        const int32_t *__restrict__ cost, uint8_t *__restrict__ records) {
  __shared__ unsigned long long part[8];
  const int id = ids[blockIdx.x];
  uint8_t *rec = records + (size_t)blockIdx.x * REC_BYTES;
  const bool cs = st[id].mode == TM_CS;
  unsigned long long sum = 0;
  for (int i = threadIdx.x; i < REC_HEAD_WORDS; i += 256) {
    if (i == 4 || i == 5) continue;                // the checksum, written last
    const uint32_t w = tracker_record_head_word(i, st[id], params[id], track[id], cost + 2 * (size_t)id, cs);
    reinterpret_cast<uint32_t *>(rec)[i] = w;
    if (i >= REC_SUM0) sum += rec_term(i, w);
  }
  const uint4 *src = reinterpret_cast<const uint4 *>(model_hist + (size_t)id * 4096);
  uint4 *dst = reinterpret_cast<uint4 *>(rec + REC_HIST);
  for (int j = threadIdx.x; j < 1024; j += 256) {
    const uint4 v = cs ? src[j] : make_uint4(0u, 0u, 0u, 0u);
    dst[j] = v;
    const int i = REC_HEAD_WORDS + 4 * j;
    sum += rec_term(i, v.x) + rec_term(i + 1, v.y) + rec_term(i + 2, v.z) + rec_term(i + 3, v.w);
  }
  sum = cta_sum_u64(sum, part);
  if (threadIdx.x == 0) *reinterpret_cast<unsigned long long *>(rec + 16) = sum;
}

// status[k] := tracker_record_check of record k.  One CTA per record, the checksum in 16-byte vectors.
__global__ void __launch_bounds__(256) k_tracker_import_check(const uint8_t *__restrict__ records, int32_t *__restrict__ status) {
  __shared__ unsigned long long part[8];
  const uint8_t *rec = records + (size_t)blockIdx.x * REC_BYTES;
  const uint4 *v = reinterpret_cast<const uint4 *>(rec);
  unsigned long long sum = 0;
  for (int j = threadIdx.x; j < REC_BYTES / 16; j += 256) {
    const uint4 q = v[j];
    const int i = 4 * j;
    if (j == 1) sum += rec_term(6, q.z) + rec_term(7, q.w);          // words 4 and 5 are the checksum itself
    else if (j > 1) sum += rec_term(i, q.x) + rec_term(i + 1, q.y) + rec_term(i + 2, q.z) + rec_term(i + 3, q.w);
  }
  sum = cta_sum_u64(sum, part);
  if (threadIdx.x == 0) status[blockIdx.x] = tracker_record_check(rec, sum);
}

// stream ids[k] := record k (checked by k_tracker_import_check).  One CTA per record.
__global__ void __launch_bounds__(256) k_tracker_import(const int32_t *__restrict__ ids, const uint8_t *__restrict__ records,
                                                        TrackerState *__restrict__ st, TrackerParams *__restrict__ params,
                                                        TrackState *__restrict__ track, uint32_t *__restrict__ model_hist,
                                                        int32_t *__restrict__ cost) {
  const int id = ids[blockIdx.x];
  const uint8_t *rec = records + (size_t)blockIdx.x * REC_BYTES;
  const bool cs = rec_word(rec, REC_STATE / 4) == (uint32_t)TM_CS;   // TrackerState::mode
  for (int i = threadIdx.x; i < REC_HEAD_WORDS; i += 256)
    tracker_record_unpack_word(i, rec_word(rec, i), cs, st[id], params[id], track[id], cost + 2 * (size_t)id);
  const uint4 *src = reinterpret_cast<const uint4 *>(rec + REC_HIST);
  uint4 *dst = reinterpret_cast<uint4 *>(model_hist + (size_t)id * 4096);
  for (int j = threadIdx.x; j < 1024; j += 256) dst[j] = cs ? src[j] : make_uint4(0u, 0u, 0u, 0u);
}

}  // namespace ht
