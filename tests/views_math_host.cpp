// Host build of the ground-truth view math (fast3r_b200/csrc/views_math.h), compiled with g++ -ffp-contract=off by
// tests/views_emulator.py: the per-axis nearest rule, the unprojection and the rotation for the CPU tests, and the whole
// of f3r_view_geometry over host records (depth pointers into host memory) for the CPU emulator of the entry point.
#include <stdint.h>

#include "../include/fast3r_b200.h"
#include "views_math.h"

namespace vw = f3r::vw;

extern "C" {
// out[i] = nearest(i, ssize, dsize) for i < dsize
void f3r_test_nearest(int ssize, int dsize, int32_t* out) {
  for (int i = 0; i < dsize; ++i) out[i] = vw::nearest(i, ssize, dsize);
}

// camera and world points of n pixels (u[i], v[i], z[i]) with k4 = (fu, fv, cu, cv) and pose rows [R | t]
void f3r_test_points(const int32_t* u, const int32_t* v, const float* z, long long n, const float* k4, const float* pose,
                     float* cam, float* world, uint8_t* valid) {
  for (long long i = 0; i < n; ++i) {
    cam[3 * i] = vw::unproject(u[i], k4[2], z[i], k4[0]);
    cam[3 * i + 1] = vw::unproject(v[i], k4[3], z[i], k4[1]);
    cam[3 * i + 2] = z[i];
    valid[i] = vw::point(u[i], v[i], z[i], k4, pose, world + 3 * i);
  }
}

// f3r_view_geometry on the host, pixel for pixel as the kernel does it
void f3r_test_view_geometry(const f3r_view_param* params, int count, float* out_pts, uint8_t* out_valid,
                            float* out_depth) {
  for (int i = 0; i < count; ++i) {
    const f3r_view_param& P = params[i];
    const int n = P.out_w * P.out_h;
    for (int p = 0; p < n; ++p) {
      const int u = P.transpose ? p / P.out_h : p % P.out_w;
      const int v = P.transpose ? p % P.out_h : p / P.out_w;
      const int sx = P.crop_x + vw::nearest(u + P.box_x, P.crop_w, P.rs_w);
      const int sy = P.crop_y + vw::nearest(v + P.box_y, P.crop_h, P.rs_h);
      const float z = P.depth[static_cast<long long>(sy) * P.src_w + sx];
      const long long o = P.out_offset + p;
      out_valid[o] = vw::point(u, v, z, P.k, P.pose, out_pts + 3 * o);
      out_depth[o] = z;
    }
  }
}

// sizeof and field offsets of f3r_view_param as this compiler lays it out (checked against lib.VIEW_PARAM)
void f3r_test_view_param_layout(int64_t* out) {
  const f3r_view_param p{};
  const char* b = reinterpret_cast<const char*>(&p);
  int i = 0;
  out[i++] = sizeof(f3r_view_param);
#define F(x) out[i++] = reinterpret_cast<const char*>(&p.x) - b
  F(depth); F(out_offset); F(src_w); F(src_h); F(crop_x); F(crop_y); F(crop_w); F(crop_h); F(rs_w); F(rs_h);
  F(box_x); F(box_y); F(out_w); F(out_h); F(transpose); F(reserved); F(k); F(pose);
#undef F
}
}
