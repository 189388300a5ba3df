// Host build of the per-pixel math the sky-mask and gather kernels run (fast3r_b200/csrc/scene_math.h), so the CPU suite
// checks that exact code against numpy and cv2.  Compiled by tests/test_scene_cpu.py with g++.
#include "scene_math.h"

extern "C" void f3r_test_scene_u8(const float* x, long long n, unsigned char* out) {
  for (long long i = 0; i < n; ++i) out[i] = f3r::scene_u8(x[i]);
}

// out[i] = bit 0: a colour box holds for triplet i = (r, g, b) = (i >> 16, i >> 8, i) & 255; bit 1: the box or the
// upper-rows rule; hsv [n][3] the HSV image
extern "C" void f3r_test_scene_hsv(long long n, unsigned char* out, unsigned char* hsv) {
  for (long long i = 0; i < n; ++i) {
    const int r = (i >> 16) & 255, g = (i >> 8) & 255, b = i & 255;
    int h, s, v;
    f3r::scene_hsv(r, g, b, &h, &s, &v);
    hsv[3 * i] = h;
    hsv[3 * i + 1] = s;
    hsv[3 * i + 2] = v;
    out[i] = (f3r::scene_sky_pixel(r, g, b, false) ? 1 : 0) | (f3r::scene_sky_pixel(r, g, b, true) ? 2 : 0);
  }
}

extern "C" void f3r_test_scene_keys(const float* x, long long n, unsigned int* desc, float* back) {
  for (long long i = 0; i < n; ++i) {
    desc[i] = f3r::scene_desc_key(x[i]);
    back[i] = f3r::scene_desc_value(desc[i]);
  }
}
