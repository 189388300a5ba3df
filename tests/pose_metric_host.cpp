// Host build of the camera-pose metric math (fast3r_b200/csrc/pose_metric_math.h), compiled with g++ -ffp-contract=off
// by tests/pose_metric_emulator.py: the per-pair errors and counts of f3r_pose_metric / f3r_pose_metric_counts from the
// very code the kernels run, plus the intermediates the CPU tests hold against torch.
#include <vector>

#include "pose_metric_math.h"

namespace {

constexpr int FLAGS = 8, COUNTS = 72;

template <typename T>
void count(T r, T t, bool bad, int hmax, long long* c) {
  c[0] += r < T(5);
  c[1] += r < T(15);
  c[2] += r < T(30);
  c[3] += t < T(5);
  c[4] += t < T(15);
  c[5] += t < T(30);
  c[6] += bad;
  c[7] += 1;
  const int b = f3r::pm::hist_bin(f3r::pm::max_nan(r, t), hmax);
  if (b >= 0) c[FLAGS + b] += 1;
}

// per item: pairs in torch.combinations order; r, t, tr, s: [items][P] or NULL; counts [items][COUNTS]
template <typename T>
void metric(const T* pred, const T* gt, int items, int n, int hmax, T* r, T* t, T* tr, T* s, long long* counts) {
  const long long P = static_cast<long long>(n) * (n - 1) / 2;
  std::vector<T> ip(12 * static_cast<size_t>(n)), ig(12 * static_cast<size_t>(n));
  for (int b = 0; b < items; ++b) {
    const T* pp = pred + 16ll * n * b;
    const T* pg = gt + 16ll * n * b;
    for (int v = 0; v < n; ++v) {
      f3r::pm::inverse(pp + 16 * v, &ip[12 * v]);
      f3r::pm::inverse(pg + 16 * v, &ig[12 * v]);
    }
    long long* c = counts + static_cast<long long>(b) * COUNTS;
    for (int k = 0; k < COUNTS; ++k) c[k] = 0;
    long long p = 0;
    for (int i = 0; i < n; ++i)
      for (int j = i + 1; j < n; ++j, ++p) {
        T rp[12], rg[12], arg;
        f3r::pm::relative(&ig[12 * i], pg + 16 * j, rg);
        f3r::pm::relative(&ip[12 * i], pp + 16 * j, rp);
        const T trace = f3r::pm::trace(rg, rp);
        const T rd = f3r::pm::rotation_deg(trace);
        const T tg[3] = {rg[3], rg[7], rg[11]}, tp[3] = {rp[3], rp[7], rp[11]};
        const T td = f3r::pm::translation_deg(tg, tp, &arg);
        const long long o = b * P + p;
        if (r) r[o] = rd, t[o] = td;
        if (tr) tr[o] = trace, s[o] = arg;  // s: 1 - loss_t
        count(rd, td, f3r::pm::trace_bad(trace), hmax, c);
      }
  }
}

template <typename T>
void counts_of(const T* r, const T* t, long long n, int hmax, long long* c) {
  for (int k = 0; k < COUNTS; ++k) c[k] = 0;
  for (long long p = 0; p < n; ++p) count(r[p], t[p], false, hmax, c);
}

}  // namespace

extern "C" {
void f3r_test_pose_metric(int f64, const void* pred, const void* gt, int items, int n, int hmax, void* r, void* t,
                          void* tr, void* s, long long* counts) {
  if (f64)
    metric(static_cast<const double*>(pred), static_cast<const double*>(gt), items, n, hmax, static_cast<double*>(r),
           static_cast<double*>(t), static_cast<double*>(tr), static_cast<double*>(s), counts);
  else
    metric(static_cast<const float*>(pred), static_cast<const float*>(gt), items, n, hmax, static_cast<float*>(r),
           static_cast<float*>(t), static_cast<float*>(tr), static_cast<float*>(s), counts);
}

void f3r_test_pose_counts(int f64, const void* r, const void* t, long long n, int hmax, long long* counts) {
  if (f64) counts_of(static_cast<const double*>(r), static_cast<const double*>(t), n, hmax, counts);
  else counts_of(static_cast<const float*>(r), static_cast<const float*>(t), n, hmax, counts);
}

void f3r_test_acos(int f64, const void* x, long long n, void* out) {
  for (long long i = 0; i < n; ++i) {
    if (f64) static_cast<double*>(out)[i] = f3r::pm::acos_(static_cast<const double*>(x)[i]);
    else static_cast<float*>(out)[i] = f3r::pm::acos_(static_cast<const float*>(x)[i]);
  }
}
}
