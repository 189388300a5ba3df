// Host/device math of the ground-truth view kernel (views.cu): one output pixel of the datasets' view pipeline
// (fast3r/dust3r/datasets/base/base_stereo_view_dataset.py:78-142, :165-221; fast3r/dust3r/utils/geometry.py:186-243).
//   nearest   cv2.resize(depthmap, dsize, interpolation=INTER_NEAREST) of the principal-point crop: per axis
//             src = min(floor(dst * (1.0 / (dsize / ssize))), ssize - 1), in double, as OpenCV's resizeNN
//   unproject depthmap_to_camera_coordinates: numpy promotes (u - cu) * z / fu to float64 (u is int64, the rest float32)
//             and the stack is cast back to float32; z is the depth itself
//   to_world  np.einsum("ik, vuk -> vui", R, X) + t in float32: ((r0 x + r1 y) + r2 z) + t, every product and sum
//             rounded on its own (no FMA)
// The host build (tests/views_math_host.cpp) runs this same code for the CPU tests and the emulator of the entry point.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define F3R_VW_HD __host__ __device__ __forceinline__
#else
#define F3R_VW_HD inline
#endif

namespace f3r {
namespace vw {

#if defined(__CUDA_ARCH__)
// The device rounds like the host but gives every NaN result as one canonical NaN.  numpy's results carry x86 SSE's
// NaNs, which pts3d shows for a missing pose (NaN pose) or an inf - inf: a NaN operand propagates quietened (the
// first one, in the expression's order, when both are NaN), an invalid operation gives the negative default NaN, and
// a conversion between float and double keeps the sign and the leading payload bits.  These wrappers restate that.
__device__ __forceinline__ float f_nan(float a, float b, float r) {
  if (isnan(a)) return __int_as_float(__float_as_int(a) | 0x00400000);
  if (isnan(b)) return __int_as_float(__float_as_int(b) | 0x00400000);
  return isnan(r) ? __int_as_float(static_cast<int>(0xffc00000u)) : r;
}
__device__ __forceinline__ double d_nan(double a, double b, double r) {
  const long long q = 0x0008000000000000ll;
  if (isnan(a)) return __longlong_as_double(__double_as_longlong(a) | q);
  if (isnan(b)) return __longlong_as_double(__double_as_longlong(b) | q);
  return isnan(r) ? __longlong_as_double(static_cast<long long>(0xfff8000000000000ull)) : r;
}
F3R_VW_HD float fmul(float a, float b) { return f_nan(a, b, __fmul_rn(a, b)); }
F3R_VW_HD float fadd(float a, float b) { return f_nan(a, b, __fadd_rn(a, b)); }
F3R_VW_HD double dmul(double a, double b) { return d_nan(a, b, __dmul_rn(a, b)); }
F3R_VW_HD double dsub(double a, double b) { return d_nan(a, b, __dsub_rn(a, b)); }
F3R_VW_HD double ddiv(double a, double b) { return d_nan(a, b, __ddiv_rn(a, b)); }
F3R_VW_HD double f2d(float a) {
  if (!isnan(a)) return static_cast<double>(a);
  const unsigned long long b = static_cast<unsigned int>(__float_as_int(a));
  return __longlong_as_double(static_cast<long long>(((b & 0x80000000ull) << 32) | 0x7ff8000000000000ull |
                                                     ((b & 0x7fffffull) << 29)));
}
F3R_VW_HD float d2f(double a) {
  if (!isnan(a)) return __double2float_rn(a);
  const unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(a));
  return __int_as_float(static_cast<int>(static_cast<unsigned int>(((b >> 32) & 0x80000000ull) | 0x7fc00000ull |
                                                                    ((b >> 29) & 0x7fffffull))));
}
#else
// the host build is compiled without contraction (-ffp-contract=off), so these are single rounded operations; on an
// x86 host they give numpy's NaNs by themselves
F3R_VW_HD float fmul(float a, float b) { return a * b; }
F3R_VW_HD float fadd(float a, float b) { return a + b; }
F3R_VW_HD double dmul(double a, double b) { return a * b; }
F3R_VW_HD double dsub(double a, double b) { return a - b; }
F3R_VW_HD double ddiv(double a, double b) { return a / b; }
F3R_VW_HD double f2d(float a) { return static_cast<double>(a); }
F3R_VW_HD float d2f(double a) { return static_cast<float>(a); }
#endif

// source index of destination index `dst` along an axis resized from ssize to dsize with INTER_NEAREST
F3R_VW_HD int nearest(int dst, int ssize, int dsize) {
  const double ifx = ddiv(1.0, ddiv(static_cast<double>(dsize), static_cast<double>(ssize)));
  const int s = static_cast<int>(floor(dmul(static_cast<double>(dst), ifx)));
  return s < ssize - 1 ? s : ssize - 1;
}

// camera coordinate of pixel coordinate u (column or row) at depth z for principal point c and focal f
F3R_VW_HD float unproject(int u, float c, float z, float f) {
  return d2f(ddiv(dmul(dsub(static_cast<double>(u), f2d(c)), f2d(z)), f2d(f)));
}

// world point of camera point x[3] through the row-major cam2world rows pose[12] = [R | t]
F3R_VW_HD void to_world(const float* pose, const float* x, float* out) {
  for (int i = 0; i < 3; ++i) {
    const float* r = pose + 4 * i;
    out[i] = fadd(fadd(fadd(fmul(r[0], x[0]), fmul(r[1], x[1])), fmul(r[2], x[2])), r[3]);
  }
}

// pixel (u, v) of the final crop: point, validity (depth > 0 and every coordinate finite)
F3R_VW_HD bool point(int u, int v, float z, const float* k4, const float* pose, float* out) {
  const float x[3] = {unproject(u, k4[2], z, k4[0]), unproject(v, k4[3], z, k4[1]), z};
  to_world(pose, x, out);
  return z > 0.f && isfinite(out[0]) && isfinite(out[1]) && isfinite(out[2]);
}

}  // namespace vw
}  // namespace f3r
