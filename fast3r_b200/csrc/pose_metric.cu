// Camera-pose metric (evaluate_camera_poses' RRA / RTA / mAA, fast3r/eval/cam_pose_metric.py): the relative-pose errors
// of every view pair (i < j, torch.combinations order) of every batch item, in the reference's CPU arithmetic
// (pose_metric_math.h), reduced to exact integer counts per item:
//   pm_inverse  closed_form_inverse of every view of the prediction and the ground truth (once per view)
//   pm_pairs    all pairs of all items in one launch (grid.y = item): the two relative poses, the rotation and
//               translation angles in degrees (optionally stored), and the counts
//   pm_count    the same counts from given angle arrays (calculate_auc)
// Counts are integers summed by warp reductions, shared-memory and global atomics, so they do not depend on
// scheduling; the host forms the means from them.
#include <stdint.h>

#include "f3r_kernels.h"
#include "pose_metric_math.h"

namespace f3r {

namespace {

constexpr int PT = 256;       // threads per pair CTA
constexpr int MAX_GX = 1024;  // CTAs per item (grid-stride past that)

struct Counts {
  unsigned flag[PM_FLAGS];
  unsigned hist[PM_MAX_BINS];
};

__device__ __forceinline__ void counts_init(Counts& s) {
  for (int k = threadIdx.x; k < PM_FLAGS + PM_MAX_BINS; k += blockDim.x) reinterpret_cast<unsigned*>(&s)[k] = 0;
}

// one pair's contribution; every lane of the warp calls this (valid = false for lanes past the last pair)
template <typename T>
__device__ __forceinline__ void count_pair(Counts& s, bool valid, T r, T t, bool bad, int hmax) {
  const unsigned lane = threadIdx.x & 31;
  const bool f[PM_FLAGS] = {valid && r < T(5),  valid && r < T(15), valid && r < T(30), valid && t < T(5),
                            valid && t < T(15), valid && t < T(30), valid && bad,       valid};
#pragma unroll
  for (int k = 0; k < PM_FLAGS; ++k) {
    const unsigned c = __reduce_add_sync(0xffffffffu, f[k] ? 1u : 0u);
    if (lane == 0 && c) atomicAdd(&s.flag[k], c);
  }
  if (valid) {
    const int b = pm::hist_bin(pm::max_nan(r, t), hmax);
    if (b >= 0) atomicAdd(&s.hist[b], 1u);
  }
}

__device__ __forceinline__ void counts_flush(const Counts& s, int bins, unsigned long long* out) {
  __syncthreads();
  for (int k = threadIdx.x; k < PM_FLAGS + bins; k += blockDim.x) {
    const unsigned c = k < PM_FLAGS ? s.flag[k] : s.hist[k - PM_FLAGS];
    if (c) atomicAdd(&out[k], static_cast<unsigned long long>(c));
  }
}

template <typename T>
__global__ void __launch_bounds__(PT) pm_inverse_kernel(const T* __restrict__ pred, const T* __restrict__ gt, int n,
                                                        T* __restrict__ inv) {
  const int v = blockIdx.x * PT + threadIdx.x;
  if (v >= n) return;
  T p[16], q[12];
  for (int s = 0; s < 2; ++s) {
    const T* src = (s ? gt : pred) + 16ll * v;
    for (int k = 0; k < 16; ++k) p[k] = src[k];
    pm::inverse(p, q);
    for (int k = 0; k < 12; ++k) inv[(static_cast<long long>(s) * n + v) * 12 + k] = q[k];
  }
}

// the pair (i, j) of index p in torch.combinations(arange(n), 2) order: row i holds n - 1 - i pairs
__device__ __forceinline__ void pair_of(long long p, int n, int* i, int* j) {
  const double b = 2.0 * n - 1.0;
  long long r = static_cast<long long>((b - sqrt(b * b - 8.0 * static_cast<double>(p))) * 0.5);
  r = r < 0 ? 0 : (r > n - 2 ? n - 2 : r);
  auto start = [n](long long k) { return k * (2ll * n - k - 1) / 2; };
  while (r > 0 && start(r) > p) --r;
  while (r < n - 2 && start(r + 1) <= p) ++r;
  *i = static_cast<int>(r);
  *j = static_cast<int>(p - start(r) + r + 1);
}

template <typename T, bool kAngles>
__global__ void __launch_bounds__(PT) pm_pairs_kernel(const T* __restrict__ pred, const T* __restrict__ gt,
                                                      const T* __restrict__ inv, int n, int items, long long pairs,
                                                      int hmax, T* __restrict__ r_out, T* __restrict__ t_out,
                                                      unsigned long long* __restrict__ counts) {
  __shared__ Counts s;
  counts_init(s);
  __syncthreads();
  const int item = blockIdx.y;
  const long long v0 = static_cast<long long>(item) * n;
  const T* inv_p = inv + v0 * 12;
  const T* inv_g = inv + (static_cast<long long>(items) * n + v0) * 12;
  const long long stride = static_cast<long long>(gridDim.x) * PT;
  for (long long base = static_cast<long long>(blockIdx.x) * PT; base < pairs; base += stride) {
    const long long p = base + threadIdx.x;
    const bool valid = p < pairs;
    T r = T(0), t = T(0);
    bool bad = false;
    if (valid) {
      int i, j;
      pair_of(p, n, &i, &j);
      T a[16], ip[12], rel_p[12], rel_g[12], arg;
      for (int k = 0; k < 12; ++k) ip[k] = inv_g[12ll * i + k];
      for (int k = 0; k < 16; ++k) a[k] = gt[(v0 + j) * 16 + k];
      pm::relative(ip, a, rel_g);
      for (int k = 0; k < 12; ++k) ip[k] = inv_p[12ll * i + k];
      for (int k = 0; k < 16; ++k) a[k] = pred[(v0 + j) * 16 + k];
      pm::relative(ip, a, rel_p);
      const T tr = pm::trace(rel_g, rel_p);
      bad = pm::trace_bad(tr);
      r = pm::rotation_deg(tr);
      const T tg[3] = {rel_g[3], rel_g[7], rel_g[11]}, tp[3] = {rel_p[3], rel_p[7], rel_p[11]};
      t = pm::translation_deg(tg, tp, &arg);
      if (kAngles) {
        r_out[item * pairs + p] = r;
        t_out[item * pairs + p] = t;
      }
    }
    count_pair(s, valid, r, t, bad, hmax);
  }
  counts_flush(s, hmax + 1, counts + static_cast<long long>(item) * PM_COUNTS);
}

template <typename T>
__global__ void __launch_bounds__(PT) pm_count_kernel(const T* __restrict__ r, const T* __restrict__ t, long long n,
                                                      int hmax, unsigned long long* __restrict__ counts) {
  __shared__ Counts s;
  counts_init(s);
  __syncthreads();
  const long long stride = static_cast<long long>(gridDim.x) * PT;
  for (long long base = static_cast<long long>(blockIdx.x) * PT; base < n; base += stride) {
    const long long p = base + threadIdx.x;
    const bool valid = p < n;
    count_pair(s, valid, valid ? r[p] : T(0), valid ? t[p] : T(0), false, hmax);
  }
  counts_flush(s, hmax + 1, counts);
}

int grid_x(long long n) {
  const long long g = (n + PT - 1) / PT;
  return static_cast<int>(g < MAX_GX ? (g > 0 ? g : 1) : MAX_GX);
}

template <typename T>
cudaError_t run_pairs(const T* pred, const T* gt, int items, int n, int hmax, T* r_out, T* t_out,
                      unsigned long long* counts, void* workspace, cudaStream_t st) {
  cudaError_t e;
  if ((e = cudaMemsetAsync(counts, 0, sizeof(unsigned long long) * PM_COUNTS * items, st)) != cudaSuccess) return e;
  T* inv = static_cast<T*>(workspace);
  const int nv = items * n;
  if ((e = launch(pm_inverse_kernel<T>, (nv + PT - 1) / PT, PT, 0, st, false, pred, gt, nv, inv)) != cudaSuccess)
    return e;
  const long long pairs = static_cast<long long>(n) * (n - 1) / 2;
  const dim3 grid(grid_x(pairs), items);
  if (r_out)
    return launch(pm_pairs_kernel<T, true>, grid, PT, 0, st, false, pred, gt, static_cast<const T*>(inv), n, items,
                  pairs, hmax, r_out, t_out, counts);
  return launch(pm_pairs_kernel<T, false>, grid, PT, 0, st, false, pred, gt, static_cast<const T*>(inv), n, items,
                pairs, hmax, r_out, t_out, counts);
}

template <typename T>
cudaError_t run_count(const T* r, const T* t, long long n, int hmax, unsigned long long* counts, cudaStream_t st) {
  cudaError_t e;
  if ((e = cudaMemsetAsync(counts, 0, sizeof(unsigned long long) * PM_COUNTS, st)) != cudaSuccess) return e;
  return launch(pm_count_kernel<T>, grid_x(n), PT, 0, st, false, r, t, n, hmax, counts);
}

}  // namespace

size_t pose_metric_workspace(int f64, int items, int views) {
  return (f64 ? sizeof(double) : sizeof(float)) * 24 * static_cast<size_t>(items) * views;
}

cudaError_t launch_pose_metric(int f64, const void* pred, const void* gt, int items, int views, int hmax, void* r_out,
                               void* t_out, unsigned long long* counts, void* workspace, cudaStream_t st) {
  if (f64)
    return run_pairs(static_cast<const double*>(pred), static_cast<const double*>(gt), items, views, hmax,
                     static_cast<double*>(r_out), static_cast<double*>(t_out), counts, workspace, st);
  return run_pairs(static_cast<const float*>(pred), static_cast<const float*>(gt), items, views, hmax,
                   static_cast<float*>(r_out), static_cast<float*>(t_out), counts, workspace, st);
}

cudaError_t launch_pose_metric_counts(int f64, const void* r, const void* t, long long n, int hmax,
                                      unsigned long long* counts, cudaStream_t st) {
  if (f64) return run_count(static_cast<const double*>(r), static_cast<const double*>(t), n, hmax, counts, st);
  return run_count(static_cast<const float*>(r), static_cast<const float*>(t), n, hmax, counts, st);
}

}  // namespace f3r
