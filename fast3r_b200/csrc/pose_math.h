// Host/device math of the RANSAC scoring (pose.cu): OpenCV's reprojection error of one point under one PnP hypothesis,
// in OpenCV's operation order (cvProjectPoints2Internal with zero distortion, then PnPRansacCallback::computeError).
// Every double and float operation is an explicit round-to-nearest intrinsic on the device and a plain operation on
// the host, so no multiply-add is contracted (OpenCV's x86-64 build does not contract these).  Kept in a header that
// also compiles as plain C++ so the CPU test suite checks exactly this code (tests/pose_math_host.cpp) against
// cv2.projectPoints.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define F3R_POSE_HD __host__ __device__ __forceinline__
#else
#define F3R_POSE_HD inline
#endif

namespace f3r {

F3R_POSE_HD double pnp_dmul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
F3R_POSE_HD double pnp_dadd(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
F3R_POSE_HD float pnp_fmul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
F3R_POSE_HD float pnp_fadd(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
F3R_POSE_HD float pnp_fsub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}

// (u, v) = projectPoints of the fp32 point (X, Y, Z) under R (row-major, from Rodrigues of the hypothesis' rvec), t and
// K = (fx, fy, cx, cy), all double, stored as float:
//   x = ((r0 X + r1 Y) + r2 Z) + t0, likewise y and z;  w = z != 0 ? 1/z : 1;  x *= w;  y *= w;  u = x fx + cx.
// With zero distortion OpenCV still forms cdist = 1 + k1 r2 + k2 r4 + k3 r6 with r2 = x^2 + y^2, r4 = r2^2, r6 = r4 r2:
// for finite x, y that is exactly 1 unless r6 overflows, where 0 * inf makes both coordinates NaN; a non-finite x or y
// gives NaN the same way.
F3R_POSE_HD void pnp_project(const double* r, const double* t, double fx, double fy, double cx, double cy, float X, float Y,
                             float Z, float* u, float* v) {
  const double xd = X, yd = Y, zd = Z;
  double x = pnp_dadd(pnp_dadd(pnp_dadd(pnp_dmul(r[0], xd), pnp_dmul(r[1], yd)), pnp_dmul(r[2], zd)), t[0]);
  double y = pnp_dadd(pnp_dadd(pnp_dadd(pnp_dmul(r[3], xd), pnp_dmul(r[4], yd)), pnp_dmul(r[5], zd)), t[1]);
  const double z = pnp_dadd(pnp_dadd(pnp_dadd(pnp_dmul(r[6], xd), pnp_dmul(r[7], yd)), pnp_dmul(r[8], zd)), t[2]);
#if defined(__CUDA_ARCH__)
  const double w = z != 0.0 ? __drcp_rn(z) : 1.0;
#else
  const double w = z != 0.0 ? 1.0 / z : 1.0;
#endif
  x = pnp_dmul(x, w);
  y = pnp_dmul(y, w);
  // r6 < inf exactly when |x|, |y| are finite and below ~5e51; test the cheap bound first, the exact rule past it
  if (!(fabs(x) < 1e50 && fabs(y) < 1e50)) {
    const double r2 = pnp_dadd(pnp_dmul(x, x), pnp_dmul(y, y));
    const double r6 = pnp_dmul(pnp_dmul(r2, r2), r2);
    if (!(r6 <= 1.7976931348623157e308)) {
      x = y = NAN;
    }
  }
  *u = static_cast<float>(pnp_dadd(pnp_dmul(x, fx), cx));
  *v = static_cast<float>(pnp_dadd(pnp_dmul(y, fy), cy));
}

// err = |ip - proj|^2 as computeError forms it: a float difference, then normL2Sqr's float sum 0 + dx^2 + dy^2
F3R_POSE_HD float pnp_error(float ipx, float ipy, float u, float v) {
  const float dx = pnp_fsub(ipx, u), dy = pnp_fsub(ipy, v);
  return pnp_fadd(pnp_fadd(0.0f, pnp_fmul(dx, dx)), pnp_fmul(dy, dy));
}

}  // namespace f3r
