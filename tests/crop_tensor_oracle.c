/* An independent restatement of the face tensor conversion (DESIGN.md 2, "Face crops", item 6), for
 * tests/test_face_tensor_host.py: the channel bytes of an RGBA8 crop (ccv's gray in fp64 for one channel), the value
 * c mul + add rounded once to float through a round-to-odd double sum, float to f16 / bf16 by explicit bit rounding to
 * nearest even, and the elements placed by the CHW or HWC strides.  Built with -ffp-contract=off. */
#include <math.h>
#include <stdint.h>
#include <string.h>

enum { U8 = 0, F16 = 1, BF16 = 2, F32 = 3 };
enum { CHW = 0, HWC = 1 };
enum { RGB = 0, BGR = 1, GRAY = 2 };

static uint32_t bits_of(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* p + a, both doubles, rounded to odd: exact sum if it is a double, otherwise the neighbour with an odd last bit.  A
 * float rounded from it is the exactly rounded p + a (53 >= 24 + 2). */
static double sum_to_odd(double p, double a) {
  const double s = p + a, bb = s - p;
  const double e = (p - (s - bb)) + (a - bb);     /* TwoSum: s + e == p + a exactly */
  if (e == 0.0) return s;
  uint64_t u;
  memcpy(&u, &s, 8);
  if (u & 1) return s;
  return nextafter(s, e > 0 ? INFINITY : -INFINITY);
}

/* c mul + add rounded once to float; c (at most 8 bits) times mul (24 bits) is exact in double */
static float value_f32(int c, float mul, float add) { return (float)sum_to_odd((double)c * (double)mul, (double)add); }

/* float -> binary16 bits, round to nearest even; overflow -> inf */
static uint16_t to_f16(float f) {
  uint32_t u = bits_of(f);
  const uint16_t sign = (uint16_t)((u >> 16) & 0x8000u);
  u &= 0x7fffffffu;
  if (u >= 0x7f800000u) return sign | 0x7c00u | (u > 0x7f800000u ? 0x200u : 0u);
  if (u < 0x00800000u) return sign;                  /* float subnormals are far below half's smallest */
  const int e = (int)(u >> 23) - 127;
  const uint32_t m = (u & 0x7fffffu) | 0x800000u;
  if (e > 15) return sign | 0x7c00u;
  const int shift = e >= -14 ? 13 : 13 + (-14 - e);
  if (shift > 24) return sign;
  uint32_t q = m >> shift;
  const uint32_t rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
  if (rem > half || (rem == half && (q & 1u))) ++q;
  const uint32_t r = e >= -14 ? ((uint32_t)(e + 14) << 10) + q : q;
  return sign | (uint16_t)(r >= 0x7c00u ? 0x7c00u : r);
}

/* float -> bfloat16 bits, round to nearest even (finite inputs) */
static uint16_t to_bf16(float f) {
  const uint32_t u = bits_of(f);
  return (uint16_t)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
}

/* ccv.grayscale: r 0.3 + g 0.59 + b 0.11 in double, left to right, stored round-half-even and clamped */
static int gray(int r, int g, int b) {
  const double v = (double)r * 0.3 + (double)g * 0.59 + (double)b * 0.11;
  const double q = rint(v);
  return q > 255.0 ? 255 : (int)q;
}

/* the element bits of channel value c */
static uint32_t element(int dtype, int c, float mul, float add) {
  if (dtype == U8) return (uint32_t)c;
  const float v = value_f32(c, mul, add);
  return dtype == F16 ? to_f16(v) : dtype == BF16 ? to_bf16(v) : bits_of(v);
}

/* n channel values c[] -> n elements of dtype in out (1, 2 or 4 bytes each) */
void hcto_values(int dtype, float mul, float add, const uint8_t *c, long long n, void *out) {
  for (long long i = 0; i < n; ++i) {
    const uint32_t b = element(dtype, c[i], mul, add);
    if (dtype == U8) ((uint8_t *)out)[i] = (uint8_t)b;
    else if (dtype == F32) ((uint32_t *)out)[i] = b;
    else ((uint16_t *)out)[i] = (uint16_t)b;
  }
}

/* n RGBA8 pixels -> their gray bytes */
void hcto_gray(const uint32_t *px, long long n, uint8_t *out) {
  for (long long i = 0; i < n; ++i) out[i] = (uint8_t)gray(px[i] & 255, (px[i] >> 8) & 255, (px[i] >> 16) & 255);
}

/* A w x h RGBA8 crop (rows of `pitch` bytes) -> the tensor at data: element (k, j, i) at k plane + j row + i (CHW) or
 * j row + i C + k (HWC), strides in elements.  Nothing else is written. */
void hcto_convert(const uint8_t *rgba, int w, int h, int pitch, int dtype, int layout, int channels, const float mul[3],
                  const float add[3], void *data, long long row, long long plane) {
  const int C = channels == GRAY ? 1 : 3;
  const int es = dtype == U8 ? 1 : dtype == F32 ? 4 : 2;
  for (int j = 0; j < h; ++j)
    for (int i = 0; i < w; ++i) {
      const uint8_t *p = rgba + (long)j * pitch + 4 * i;
      for (int k = 0; k < C; ++k) {
        const int c = channels == GRAY ? gray(p[0], p[1], p[2]) : channels == BGR ? p[2 - k] : p[k];
        const long long at = layout == CHW ? k * plane + j * row + i : j * row + (long long)i * C + k;
        const uint32_t b = element(dtype, c, mul[k], add[k]);
        uint8_t *dst = (uint8_t *)data + at * es;
        if (es == 1) *dst = (uint8_t)b;
        else if (es == 2) { const uint16_t v = (uint16_t)b; memcpy(dst, &v, 2); }
        else memcpy(dst, &b, 4);
      }
    }
}
