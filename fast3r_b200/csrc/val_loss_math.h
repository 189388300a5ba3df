// Host/device math of the validation criterion (val_loss.cu): ConfLossMultiviewV2(Regr3DMultiviewV4(L21Loss()))
// of fast3r/dust3r/losses.py:570-848 for one pixel of one (view, item), and the norm factors from the sums.
//   global term: gt in view 0's frame, inv(pose_0) gt, against pts3d_in_other_view; factors per item over all views
//   local term:  gt in its own view's frame, inv(pose_v) gt, against pts3d_local; factors per (view, item), or the
//                global ones with local_scale_consistent
// Per pixel the arithmetic is float32, as the reference's; the sums over pixels are float64.  The host build
// (tests/val_loss_host.cpp) runs this same code for the CPU emulator of the entry point.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define F3R_VL_HD __host__ __device__ __forceinline__
#else
#define F3R_VL_HD inline
#endif

namespace f3r {
namespace vl {

// launch-1 sums per (view, item): the sum of ||p|| (or log1p ||p||) over the valid pixels where it is not NaN, then
// the number of those pixels, for each of the four point sets
enum { PR_G = 0, GT_G = 1, PR_L = 2, GT_L = 3, SETS = 4, NORM_SUMS = 2 * SETS };
// launch-2 sums per (view, item), the entry point's output: sum of d and of d c - alpha log c for the global and the
// local term, and the number of valid pixels (the same for both terms)
enum { D_G = 0, C_G = 1, D_L = 2, C_L = 3, COUNT = 4, TERM_SUMS = 5 };

// inv(m) of a row-major 4x4 float matrix (a general inverse, as torch.linalg.inv): Gauss-Jordan elimination with
// partial pivoting in double, rounded to float.  A singular matrix gives inf / NaN entries (torch raises).
F3R_VL_HD void inverse(const float* m, float* out) {
  double a[4][8];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 8; ++c) a[r][c] = c < 4 ? static_cast<double>(m[4 * r + c]) : (c - 4 == r ? 1.0 : 0.0);
  for (int c = 0; c < 4; ++c) {
    int p = c;
    for (int r = c + 1; r < 4; ++r)
      if (fabs(a[r][c]) > fabs(a[p][c])) p = r;
    if (p != c)
      for (int k = 0; k < 8; ++k) {
        const double t = a[c][k];
        a[c][k] = a[p][k];
        a[p][k] = t;
      }
    const double d = a[c][c];
    for (int k = 0; k < 8; ++k) a[c][k] /= d;
    for (int r = 0; r < 4; ++r) {
      if (r == c) continue;
      const double f = a[r][c];
      for (int k = 0; k < 8; ++k) a[r][k] -= f * a[c][k];
    }
  }
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) out[4 * r + c] = static_cast<float>(a[r][4 + c]);
}

// geotrf(T, p) of one point: the 3x3 block times p plus the translation column
F3R_VL_HD void transform(const float* T, const float* p, float* q) {
  for (int i = 0; i < 3; ++i) q[i] = T[4 * i] * p[0] + T[4 * i + 1] * p[1] + T[4 * i + 2] * p[2] + T[4 * i + 3];
}

F3R_VL_HD float norm3(float x, float y, float z) { return sqrtf(x * x + y * y + z * z); }

// one point's contribution to a norm factor: ||p|| or log1p(||p||) (norm_mode avg_dis / avg_log1p); NaN is skipped
F3R_VL_HD void add_norm(const float* p, bool log1p, double* sum, double* count) {
  float d = norm3(p[0], p[1], p[2]);
  if (log1p) d = log1pf(d);
  if (d == d) {
    *sum += d;
    *count += 1.0;
  }
}

// nanmean(...).clip(min=1e-8) in float from the sum and the count (0 / 0 and NaN stay NaN)
F3R_VL_HD float factor(double sum, double count) {
  const float f = static_cast<float>(sum / count);
  return f < 1e-8f ? 1e-8f : f;
}

// L21 distance ||pr / fp - gt / fg|| of one pixel (fg = 1 with gt_scale: x / 1 is x)
F3R_VL_HD float dist(const float* pr, float fp, const float* gt, float fg) {
  return norm3(pr[0] / fp - gt[0] / fg, pr[1] / fp - gt[1] / fg, pr[2] / fp - gt[2] / fg);
}

// the confidence-weighted term d c - alpha log c
F3R_VL_HD float conf_term(float d, float c, float alpha) { return d * c - alpha * logf(c); }

}  // namespace vl
}  // namespace f3r
