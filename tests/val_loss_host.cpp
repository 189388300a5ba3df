// Host build of the validation criterion's math (fast3r_b200/csrc/val_loss_math.h), compiled with g++ by
// tests/val_loss_emulator.py: the sums of f3r_val_loss from the very per-pixel code the kernels run, summed
// sequentially per (view, item) (the kernels sum in another fixed order, so the float64 sums agree to rounding).
#include <stdint.h>

#include <vector>

#include "val_loss_math.h"

namespace vl = f3r::vl;

extern "C" {
// maps [views][items][n] as in f3r_val_loss; out [views][items][vl::TERM_SUMS]; mags [views][items][4] receives the
// sums of |d| and |d c - alpha log c| (the scale of the tests' bounds)
void f3r_test_val_loss(const float* gt, const uint8_t* valid, const float* pr, const float* pr_local, const float* conf,
                       const float* conf_local, const float* poses, int views, int items, int n, float alpha, int log1p,
                       int gt_scale, int local_scale_consistent, double* out, double* mags) {
  const bool has_local = pr_local != nullptr;
  const long long nvb = static_cast<long long>(views) * items;
  std::vector<float> inv(16 * nvb);
  for (long long vb = 0; vb < nvb; ++vb) vl::inverse(poses + 16 * vb, &inv[16 * vb]);
  std::vector<double> s1(vl::NORM_SUMS * nvb, 0.0), item(vl::NORM_SUMS * static_cast<size_t>(items), 0.0);
  for (long long vb = 0; vb < nvb; ++vb) {
    const float* tg = &inv[16 * (vb % items)];
    const float* tl = &inv[16 * vb];
    double* a = &s1[vl::NORM_SUMS * vb];
    for (long long i = vb * n; i < (vb + 1) * n; ++i) {
      if (!valid[i]) continue;
      float q[3];
      vl::transform(tg, gt + 3 * i, q);
      vl::add_norm(pr + 3 * i, log1p, &a[vl::PR_G], &a[vl::SETS + vl::PR_G]);
      vl::add_norm(q, log1p, &a[vl::GT_G], &a[vl::SETS + vl::GT_G]);
      if (has_local) {
        vl::transform(tl, gt + 3 * i, q);
        vl::add_norm(pr_local + 3 * i, log1p, &a[vl::PR_L], &a[vl::SETS + vl::PR_L]);
        vl::add_norm(q, log1p, &a[vl::GT_L], &a[vl::SETS + vl::GT_L]);
      }
    }
    for (int k = 0; k < vl::NORM_SUMS; ++k) item[vl::NORM_SUMS * (vb % items) + k] += a[k];
  }
  for (long long vb = 0; vb < nvb; ++vb) {
    const double* sg = &item[vl::NORM_SUMS * (vb % items)];
    const double* sl = &s1[vl::NORM_SUMS * vb];
    const float fpg = vl::factor(sg[vl::PR_G], sg[vl::SETS + vl::PR_G]);
    const float fgg = gt_scale ? 1.f : vl::factor(sg[vl::GT_G], sg[vl::SETS + vl::GT_G]);
    const float fpl = local_scale_consistent ? fpg : vl::factor(sl[vl::PR_L], sl[vl::SETS + vl::PR_L]);
    const float fgl = gt_scale ? 1.f : local_scale_consistent ? fgg : vl::factor(sl[vl::GT_L], sl[vl::SETS + vl::GT_L]);
    const float* tg = &inv[16 * (vb % items)];
    const float* tl = &inv[16 * vb];
    double* o = out + vl::TERM_SUMS * vb;
    double* g = mags + 4 * vb;
    for (int k = 0; k < vl::TERM_SUMS; ++k) o[k] = 0.0;
    for (int k = 0; k < 4; ++k) g[k] = 0.0;
    for (long long i = vb * n; i < (vb + 1) * n; ++i) {
      if (!valid[i]) continue;
      float q[3];
      vl::transform(tg, gt + 3 * i, q);
      const float dg = vl::dist(pr + 3 * i, fpg, q, fgg);
      const float cg = vl::conf_term(dg, conf[i], alpha);
      o[vl::D_G] += dg;
      o[vl::C_G] += cg;
      g[vl::D_G] += fabsf(dg);
      g[vl::C_G] += fabsf(cg);
      if (has_local) {
        vl::transform(tl, gt + 3 * i, q);
        const float dl = vl::dist(pr_local + 3 * i, fpl, q, fgl);
        const float cl = vl::conf_term(dl, conf_local[i], alpha);
        o[vl::D_L] += dl;
        o[vl::C_L] += cl;
        g[vl::D_L] += fabsf(dl);
        g[vl::C_L] += fabsf(cl);
      }
      o[vl::COUNT] += 1.0;
    }
  }
}

// the float32 inverses of val_loss_math.h for m [count][4][4]
void f3r_test_val_loss_inverse(const float* m, long long count, float* out) {
  for (long long i = 0; i < count; ++i) vl::inverse(m + 16 * i, out + 16 * i);
}
}
