// Host build of the RANSAC scoring math the CUDA kernel runs per point and hypothesis (fast3r_b200/csrc/pose_math.h), so
// the CPU suite checks that exact code against cv2.projectPoints.  Compiled by tests/test_pose_cpu.py with g++.
#include "pose_math.h"

extern "C" void f3r_test_pnp_project(const double* rt, const double* k, const float* pts, const float* ip, int n, float* uv,
                                     float* err) {
  for (int i = 0; i < n; ++i) {
    f3r::pnp_project(rt, rt + 9, k[0], k[1], k[2], k[3], pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], &uv[2 * i],
                     &uv[2 * i + 1]);
    err[i] = f3r::pnp_error(ip[2 * i], ip[2 * i + 1], uv[2 * i], uv[2 * i + 1]);
  }
}
