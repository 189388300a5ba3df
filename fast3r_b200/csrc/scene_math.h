// Host/device math of the viewer scene (scene.cu): the image-to-u8 conversion, OpenCV's 8-bit RGB -> HSV and the
// per-pixel sky rule of detect_sky_mask (fast3r/viz/viser_visualizer.py:24-53), and the sort key of the
// confidence order.  Kept in a header that also compiles as plain C++ so the CPU test suite checks exactly this code
// (tests/scene_math_host.cpp) against numpy and cv2.cvtColor + cv2.inRange on every RGB triplet.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define F3R_SCENE_HD __host__ __device__ __forceinline__
#else
#define F3R_SCENE_HD inline
#endif

namespace f3r {

// ((x + 1) * 127.5).astype(np.uint8) in float32: two separately rounded operations (never one fused multiply-add),
// then truncation towards zero and the int -> uint8 wrap of numpy's cast
F3R_SCENE_HD uint8_t scene_u8(float x) {
#if defined(__CUDA_ARCH__)
  const float v = __fmul_rn(__fadd_rn(x, 1.0f), 127.5f);
#else
  volatile float s = x + 1.0f;  // volatile: a contracting host compiler must not fuse the two operations either
  const float v = s * 127.5f;
#endif
  return static_cast<uint8_t>(static_cast<int>(v));
}

// cvRound of a positive double: round half to even
F3R_SCENE_HD int scene_round(double x) {
#if defined(__CUDA_ARCH__)
  return __double2int_rn(x);
#else
  return static_cast<int>(nearbyint(x));
#endif
}

// OpenCV's integer RGB2HSV_b (hsv_shift = 12, H in [0, 180)): S = round(diff * sdiv[v]), H = round(h' * hdiv[diff]) with
// sdiv[v] = cvRound((255 << 12) / v) and hdiv[d] = cvRound((180 << 12) / (6 d)), both 0 at 0.
F3R_SCENE_HD void scene_hsv(int r, int g, int b, int* h, int* s, int* v) {
  const int vmax = r > g ? (r > b ? r : b) : (g > b ? g : b);
  const int vmin = r < g ? (r < b ? r : b) : (g < b ? g : b);
  const int diff = vmax - vmin;
#if defined(__CUDA_ARCH__)
  const int sdiv = vmax ? scene_round(__ddiv_rn(static_cast<double>(255 << 12), static_cast<double>(vmax))) : 0;
  const int hdiv = diff ? scene_round(__ddiv_rn(static_cast<double>(180 << 12), __dmul_rn(6.0, diff))) : 0;
#else
  const int sdiv = vmax ? scene_round(static_cast<double>(255 << 12) / static_cast<double>(vmax)) : 0;
  const int hdiv = diff ? scene_round(static_cast<double>(180 << 12) / (6.0 * diff)) : 0;
#endif
  *s = (diff * sdiv + (1 << 11)) >> 12;
  int hh = vmax == r ? g - b : (vmax == g ? b - r + 2 * diff : r - g + 4 * diff);
  hh = (hh * hdiv + (1 << 11)) >> 12;
  *h = hh < 0 ? hh + 180 : hh;
  *v = vmax;
}

F3R_SCENE_HD bool scene_in(int h, int s, int v, int h0, int s0, int v0, int h1, int s1, int v1) {
  return h >= h0 && h <= h1 && s >= s0 && s <= s1 && v >= v0 && v <= v1;
}

// the sky colour boxes of detect_sky_mask (cv2.inRange, inclusive), and in the upper rows also S < 50 and V > 150
F3R_SCENE_HD bool scene_sky_pixel(int r, int g, int b, bool upper) {
  int h, s, v;
  scene_hsv(r, g, b, &h, &s, &v);
  return scene_in(h, s, v, 105, 50, 140, 135, 255, 255) || scene_in(h, s, v, 95, 5, 150, 145, 100, 255) ||
         scene_in(h, s, v, 0, 0, 235, 180, 10, 255) || (upper && s < 50 && v > 150);
}

// Ascending order of this key is the order of np.argsort(-conf, kind="stable") on the values: descending, -0.0 equal to
// +0.0, every NaN last (ties, and NaNs among themselves, keep their index order through the stable sort).
F3R_SCENE_HD uint32_t scene_desc_key(float c) {
  uint32_t u;
  memcpy(&u, &c, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0xffffffffu;  // NaN
  if ((u & 0x7fffffffu) == 0u) u = 0u;                       // -0.0 -> +0.0
  const uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~asc;
}

F3R_SCENE_HD float scene_desc_value(uint32_t key) {
  if (key == 0xffffffffu) return NAN;
  const uint32_t asc = ~key;
  const uint32_t u = (asc & 0x80000000u) ? (asc & 0x7fffffffu) : ~asc;
  float c;
  memcpy(&c, &u, 4);
  return c;
}

// ascending order-preserving image of a float (the percentile's radix select); NaNs land above +inf or below -inf
F3R_SCENE_HD uint32_t scene_asc_key(float c) {
  uint32_t u;
  memcpy(&u, &c, 4);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

F3R_SCENE_HD float scene_asc_value(uint32_t k) {
  const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float c;
  memcpy(&c, &u, 4);
  return c;
}

}  // namespace f3r
