// Host/device math of the camera-pose metric (pose_metric.cu): the relative-pose errors of one view pair as the
// reference's camera_to_rel_deg computes them on the CPU (fast3r/eval/cam_pose_metric.py with
// fast3r/utils/so3_utils.py), in torch's CPU operation order:
//   * bmm of small matrices: a sequential sum from 0 per output element, no multiply-add;
//   * torch.sum(., dim=1) of 3 elements: sequential from 0;
//   * torch.norm(., dim=1) of a strided (P, 3) column: a sequential sum of squares, then sqrt;
//   * a Python-float scalar operand is first rounded to the tensor's type; `x * 180 / pi` is two roundings.
// Every operation is an explicit round-to-nearest intrinsic on the device and a plain operation on the host (built with
// -ffp-contract=off), so the CPU suite checks exactly this code (tests/pose_metric_host.cpp).  The two elementwise
// functions torch takes from a vector library, sqrt and acos, are not correctly rounded there; here sqrt is IEEE and
// acos is restated from basic operations (fdlibm's rational approximation in double), so host and device agree bit
// for bit and the angles are within a few ulp of torch's.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define F3R_PM_HD __host__ __device__ __forceinline__
#else
#define F3R_PM_HD inline
#endif

namespace f3r {
namespace pm {

F3R_PM_HD float add(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
F3R_PM_HD double add(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
F3R_PM_HD float sub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
F3R_PM_HD double sub(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
F3R_PM_HD float mul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
F3R_PM_HD double mul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
F3R_PM_HD float div(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
F3R_PM_HD double div(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
F3R_PM_HD float sqrt_(float a) {
#if defined(__CUDA_ARCH__)
  return __fsqrt_rn(a);
#else
  return sqrtf(a);
#endif
}
F3R_PM_HD double sqrt_(double a) {
#if defined(__CUDA_ARCH__)
  return __dsqrt_rn(a);
#else
  return sqrt(a);
#endif
}

// acos in double, fdlibm's e_acos.c (public domain, Sun Microsystems): |error| < 1 ulp.  NaN and |x| > 1 give NaN.
F3R_PM_HD double acos_d(double x) {
  const double pi = 3.14159265358979311600e+00, pio2_hi = 1.57079632679489655800e+00,
               pio2_lo = 6.12323399573676603587e-17;
  const double pS0 = 1.66666666666666657415e-01, pS1 = -3.25565818622400915405e-01, pS2 = 2.01212532134862925881e-01,
               pS3 = -4.00555345006794114027e-02, pS4 = 7.91534994289814532176e-04, pS5 = 3.47933107596021167570e-05;
  const double qS1 = -2.40339491173441421878e+00, qS2 = 2.02094576023350569471e+00, qS3 = -6.88283971605453293030e-01,
               qS4 = 7.70381505559019352791e-02;
  const double ax = fabs(x);
  if (!(ax < 1.0)) {
    if (x == 1.0) return 0.0;
    if (x == -1.0) return add(pi, mul(2.0, pio2_lo));
    return NAN;
  }
  if (ax < 0.5) {
    if (ax <= 6.938893903907228e-18) return add(pio2_hi, pio2_lo);  // 2^-57
    const double z = mul(x, x);
    const double p = mul(z, add(pS0, mul(z, add(pS1, mul(z, add(pS2, mul(z, add(pS3, mul(z, add(pS4, mul(z, pS5)))))))))));
    const double q = add(1.0, mul(z, add(qS1, mul(z, add(qS2, mul(z, add(qS3, mul(z, qS4))))))));
    const double r = div(p, q);
    return sub(pio2_hi, sub(x, sub(pio2_lo, mul(x, r))));
  }
  const double z = mul(add(1.0, -ax), 0.5);
  const double p = mul(z, add(pS0, mul(z, add(pS1, mul(z, add(pS2, mul(z, add(pS3, mul(z, add(pS4, mul(z, pS5)))))))))));
  const double q = add(1.0, mul(z, add(qS1, mul(z, add(qS2, mul(z, add(qS3, mul(z, qS4))))))));
  const double s = sqrt_(z);
  const double r = div(p, q);
  if (x < 0.0) {
    const double w = sub(mul(r, s), pio2_lo);
    return sub(pi, mul(2.0, add(s, w)));
  }
  uint64_t bits;
  memcpy(&bits, &s, 8);
  bits &= 0xFFFFFFFF00000000ull;
  double df;
  memcpy(&df, &bits, 8);
  const double c = div(sub(z, mul(df, df)), add(s, df));
  const double w = add(mul(r, s), c);
  return mul(2.0, add(df, w));
}
F3R_PM_HD float acos_(float x) { return static_cast<float>(acos_d(static_cast<double>(x))); }
F3R_PM_HD double acos_(double x) { return acos_d(x); }

// The scalars of so3_relative_angle(eps=1e-4, cos_bound=1e-4) and compare_translation_by_angle, as Python forms them
// in double (bound = 1 - 1e-4; slope = _dacos_dx(+-bound); math.acos(+-bound)); tests/test_pose_metric_cpu.py checks
// them against the reference's functions.
constexpr double TRACE_LO = -0x1.00068db8bac71p+0;  // -1 - 1e-4
constexpr double TRACE_HI = 0x1.800346dc5d639p+1;   // 3 + 1e-4
constexpr double BOUND = 0x1.fff2e48e8a71ep-1;      // 1 - 1e-4
constexpr double SLOPE = -0x1.1ad98b6e7e8fdp+6;     // -1 / sqrt(1 - bound^2)
constexpr double ACOS_HI = 0x1.cf69d216bd74bp-7;    // acos(bound)
constexpr double ACOS_LO = 0x1.90504b722c141p+1;    // acos(-bound)
constexpr double EPS_T = 1e-15;
constexpr double PI = 0x1.921fb54442d18p+1;         // np.pi
constexpr double DEFAULT_ERR = 1e6;

// closed_form_inverse of one SE(3) matrix p (row-major 4x4): inv (row-major 3x4) = [R^T | -(R^T t)]
template <typename T>
F3R_PM_HD void inverse(const T* p, T* inv) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) inv[4 * r + c] = p[4 * c + r];
    const T s = add(add(add(T(0), mul(p[r], p[3])), mul(p[4 + r], p[7])), mul(p[8 + r], p[11]));
    inv[4 * r + 3] = -s;
  }
}

// rows 0..2 of inv_i . pose_j (bmm of the (4, 4) inverse, whose row 3 is [0, 0, 0, 1], with the (4, 4) pose)
template <typename T>
F3R_PM_HD void relative(const T* inv, const T* p, T* rel) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c)
      rel[4 * r + c] = add(add(add(add(T(0), mul(inv[4 * r], p[c])), mul(inv[4 * r + 1], p[4 + c])),
                               mul(inv[4 * r + 2], p[8 + c])), mul(inv[4 * r + 3], p[12 + c]));
}

// so3_rotation_angle's trace of R12 = R_gt . R_pred^T (only its diagonal is formed)
template <typename T>
F3R_PM_HD T trace(const T* g, const T* q) {
  T d[3];
  for (int k = 0; k < 3; ++k)
    d[k] = add(add(add(T(0), mul(g[4 * k], q[4 * k])), mul(g[4 * k + 1], q[4 * k + 1])), mul(g[4 * k + 2], q[4 * k + 2]));
  return add(add(d[0], d[1]), d[2]);
}

template <typename T>
F3R_PM_HD bool trace_bad(T tr) { return tr < T(TRACE_LO) || tr > T(TRACE_HI); }

// acos_linear_extrapolation((trace - 1) * 0.5, (-bound, bound)) in degrees
template <typename T>
F3R_PM_HD T rotation_deg(T tr) {
  const T x = mul(sub(tr, T(1)), T(0.5));
  T a;
  if (x >= T(BOUND)) a = add(mul(sub(x, T(BOUND)), T(SLOPE)), T(ACOS_HI));
  else if (x <= T(-BOUND)) a = add(mul(sub(x, T(-BOUND)), T(SLOPE)), T(ACOS_LO));
  else a = acos_(x);
  return div(mul(a, T(180)), T(PI));
}

// compare_translation_by_angle(t_gt, t) in degrees; *u = 1 - loss_t, the argument of its sqrt.  torch.norm of the
// strided (P, 3) translation column takes the generic reduction: a sequential sum of squares, then a correctly
// rounded sqrt.  The elementwise torch.sqrt and torch.acos of the CPU build are vector-library routines that are not
// correctly rounded; here both are (sqrt by IEEE, acos to within fdlibm's bound), so the angle can differ from torch's
// by a few ulp while every value up to *u is bit-equal.
template <typename T>
F3R_PM_HD T translation_deg(const T* tg, const T* tp, T* u) {
  const T np_ = add(sqrt_(add(add(mul(tp[0], tp[0]), mul(tp[1], tp[1])), mul(tp[2], tp[2]))), T(EPS_T));
  const T ng = add(sqrt_(add(add(mul(tg[0], tg[0]), mul(tg[1], tg[1])), mul(tg[2], tg[2]))), T(EPS_T));
  T dot = T(0);
  for (int k = 0; k < 3; ++k) dot = add(dot, mul(div(tp[k], np_), div(tg[k], ng)));
  T loss = sub(T(1), mul(dot, dot));
  if (loss < T(EPS_T)) loss = T(EPS_T);  // clamp_min: NaN stays NaN
  *u = sub(T(1), loss);
  T e = acos_(sqrt_(*u));
  if (isnan(e) || isinf(e)) e = T(DEFAULT_ERR);
  return div(mul(e, T(180)), T(PI));
}

// torch.histc(x, bins, min=0, max=hmax) bin of x, or -1 where histc drops it (NaN, outside [0, hmax]); bins = hmax + 1
template <typename T>
F3R_PM_HD int hist_bin(T x, int hmax) {
  if (!(x >= T(0) && x <= T(hmax))) return -1;
  const long long pos = static_cast<long long>(div(mul(sub(x, T(0)), T(hmax + 1)), T(hmax)));
  return pos == hmax + 1 ? hmax : static_cast<int>(pos);
}

// torch.max(stack((r, t)), dim) propagates NaN
template <typename T>
F3R_PM_HD T max_nan(T r, T t) { return isnan(r) ? r : (isnan(t) ? t : (t > r ? t : r)); }

}  // namespace pm
}  // namespace f3r
