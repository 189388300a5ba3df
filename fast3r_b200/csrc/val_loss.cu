// Validation criterion ConfLossMultiviewV2(Regr3DMultiviewV4(L21Loss())) (fast3r/dust3r/losses.py:570-848), forward
// only, over maps stacked [views][items][n] (val_loss_math.h has the per-pixel math):
//   vl_inverse  inv(camera_pose) of every (view, item), once, in double rounded to float
//   vl_norms    one pass over the pixels: the sums behind the four norm factors (prediction and ground truth, global
//               and local) per (view, item); the CTA that finishes a (view, item) last sums its chunks, and the one that
//               finishes an item last sums its views (the global factors)
//   vl_terms    the factors from those sums, then one pass over the pixels: sum of d and of d c - alpha log c for both
//               terms and the valid-pixel count per (view, item), summed over the chunks the same way
// Every sum is float64 in a fixed order (thread, warp tree, warps, chunks, views); the only atomics are integer
// arrival counters, so two runs give the same bits.  The host forms the means, the loss and the details.
#include <stdint.h>

#include "f3r_kernels.h"
#include "val_loss_math.h"

namespace f3r {

namespace {

constexpr int VT = 256;   // threads per CTA
constexpr int VPX = 4096; // pixels per CTA (one chunk of a (view, item))

struct VlMaps {
  const float* gt;
  const uint8_t* valid;
  const float* pr;
  const float* pr_local;
  const float* conf;
  const float* conf_local;
  int items, views, n, chunks;
};

// sums acc over the CTA in a fixed order; thread k < K stores element k at out[k]
template <int K>
__device__ __forceinline__ void block_sum(double (&acc)[K], double* out) {
  __shared__ double warp_sums[VT / 32][K];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double v = acc[k];
    for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
    if (lane == 0) warp_sums[w][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double s = 0.0;
    for (int i = 0; i < VT / 32; ++i) s += warp_sums[i][threadIdx.x];
    out[threadIdx.x] = s;
  }
}

// Called by every thread of every CTA of a group after the CTA stored its K partials: the CTA that arrives last
// (per the integer counter) sums the group's `parts` partials, part i at parts_at[i * stride], in index order into
// out[0..K) and returns true; the others return false.
template <int K>
__device__ __forceinline__ bool finish_group(const double* parts_at, int parts, long long stride, unsigned* counter,
                                             double* out) {
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(counter, 1u) == static_cast<unsigned>(parts - 1);
  __syncthreads();
  if (!last) return false;
  __threadfence();
  if (threadIdx.x < K) {
    double s = 0.0;
    for (int i = 0; i < parts; ++i) s += __ldcg(parts_at + i * stride + threadIdx.x);
    out[threadIdx.x] = s;
  }
  return true;
}

__global__ void __launch_bounds__(VT) vl_inverse_kernel(const float* __restrict__ poses, int nvb, float* __restrict__ inv) {
  const int i = blockIdx.x * VT + threadIdx.x;
  if (i < nvb) vl::inverse(poses + 16ll * i, inv + 16ll * i);
}

__global__ void __launch_bounds__(VT) vl_norms_kernel(VlMaps m, const float* __restrict__ inv, bool log1p,
                                                      bool has_local, double* __restrict__ part,
                                                      double* __restrict__ vb_sums, double* __restrict__ item_sums,
                                                      unsigned* __restrict__ counters) {
  const int vb = blockIdx.x / m.chunks, chunk = blockIdx.x % m.chunks;
  const int b = vb % m.items;
  float tg[16], tl[16];
  for (int k = 0; k < 16; ++k) tg[k] = inv[16 * b + k], tl[k] = inv[16ll * vb + k];
  double acc[vl::NORM_SUMS] = {};
  const long long base = static_cast<long long>(vb) * m.n;
  for (int p = chunk * VPX + threadIdx.x, end = m.n - chunk * VPX > VPX ? chunk * VPX + VPX : m.n; p < end;
       p += VT) {
    const long long i = base + p;
    if (!m.valid[i]) continue;
    const float g[3] = {m.gt[3 * i], m.gt[3 * i + 1], m.gt[3 * i + 2]};
    float q[3];
    vl::transform(tg, g, q);
    vl::add_norm(m.pr + 3 * i, log1p, &acc[vl::PR_G], &acc[vl::SETS + vl::PR_G]);
    vl::add_norm(q, log1p, &acc[vl::GT_G], &acc[vl::SETS + vl::GT_G]);
    if (has_local) {
      vl::transform(tl, g, q);
      vl::add_norm(m.pr_local + 3 * i, log1p, &acc[vl::PR_L], &acc[vl::SETS + vl::PR_L]);
      vl::add_norm(q, log1p, &acc[vl::GT_L], &acc[vl::SETS + vl::GT_L]);
    }
  }
  block_sum(acc, part + static_cast<long long>(blockIdx.x) * vl::NORM_SUMS);
  const int nvb = m.views * m.items;
  if (!finish_group<vl::NORM_SUMS>(part + static_cast<long long>(vb) * m.chunks * vl::NORM_SUMS, m.chunks,
                                   vl::NORM_SUMS, counters + vb, vb_sums + static_cast<long long>(vb) * vl::NORM_SUMS))
    return;
  finish_group<vl::NORM_SUMS>(vb_sums + static_cast<long long>(b) * vl::NORM_SUMS, m.views,
                              static_cast<long long>(m.items) * vl::NORM_SUMS, counters + nvb + b,
                              item_sums + static_cast<long long>(b) * vl::NORM_SUMS);
}

__global__ void __launch_bounds__(VT) vl_terms_kernel(VlMaps m, const float* __restrict__ inv, float alpha,
                                                      bool gt_scale, bool local_scale_consistent, bool has_local,
                                                      const double* __restrict__ vb_sums,
                                                      const double* __restrict__ item_sums, double* __restrict__ part,
                                                      unsigned* __restrict__ counters, double* __restrict__ out) {
  const int vb = blockIdx.x / m.chunks, chunk = blockIdx.x % m.chunks;
  const int b = vb % m.items;
  const double* sg = item_sums + static_cast<long long>(b) * vl::NORM_SUMS;
  const double* sl = vb_sums + static_cast<long long>(vb) * vl::NORM_SUMS;
  const float fpg = vl::factor(sg[vl::PR_G], sg[vl::SETS + vl::PR_G]);
  const float fgg = gt_scale ? 1.f : vl::factor(sg[vl::GT_G], sg[vl::SETS + vl::GT_G]);
  const float fpl = local_scale_consistent ? fpg : vl::factor(sl[vl::PR_L], sl[vl::SETS + vl::PR_L]);
  const float fgl = gt_scale ? 1.f : local_scale_consistent ? fgg : vl::factor(sl[vl::GT_L], sl[vl::SETS + vl::GT_L]);
  float tg[16], tl[16];
  for (int k = 0; k < 16; ++k) tg[k] = inv[16 * b + k], tl[k] = inv[16ll * vb + k];
  double acc[vl::TERM_SUMS] = {};
  const long long base = static_cast<long long>(vb) * m.n;
  for (int p = chunk * VPX + threadIdx.x, end = m.n - chunk * VPX > VPX ? chunk * VPX + VPX : m.n; p < end;
       p += VT) {
    const long long i = base + p;
    if (!m.valid[i]) continue;
    const float g[3] = {m.gt[3 * i], m.gt[3 * i + 1], m.gt[3 * i + 2]};
    float q[3];
    vl::transform(tg, g, q);
    const float dg = vl::dist(m.pr + 3 * i, fpg, q, fgg);
    acc[vl::D_G] += dg;
    acc[vl::C_G] += vl::conf_term(dg, m.conf[i], alpha);
    if (has_local) {
      vl::transform(tl, g, q);
      const float dl = vl::dist(m.pr_local + 3 * i, fpl, q, fgl);
      acc[vl::D_L] += dl;
      acc[vl::C_L] += vl::conf_term(dl, m.conf_local[i], alpha);
    }
    acc[vl::COUNT] += 1.0;
  }
  block_sum(acc, part + static_cast<long long>(blockIdx.x) * vl::TERM_SUMS);
  finish_group<vl::TERM_SUMS>(part + static_cast<long long>(vb) * m.chunks * vl::TERM_SUMS, m.chunks, vl::TERM_SUMS,
                              counters + vb, out + static_cast<long long>(vb) * vl::TERM_SUMS);
}

// workspace carve-up, all offsets 8-byte aligned
struct VlLayout {
  size_t inv, part1, vb1, item1, part2, counters, total;
  VlLayout(int views, int items, int n) {
    const size_t nvb = static_cast<size_t>(views) * items, chunks = (static_cast<size_t>(n) + VPX - 1) / VPX;
    inv = 0;
    part1 = inv + sizeof(float) * 16 * nvb;
    vb1 = part1 + sizeof(double) * vl::NORM_SUMS * nvb * chunks;
    item1 = vb1 + sizeof(double) * vl::NORM_SUMS * nvb;
    part2 = item1 + sizeof(double) * vl::NORM_SUMS * items;
    counters = part2 + sizeof(double) * vl::TERM_SUMS * nvb * chunks;
    total = counters + sizeof(unsigned) * (2 * nvb + items);
  }
};

}  // namespace

size_t val_loss_workspace(int views, int items, int n) { return VlLayout(views, items, n).total; }

cudaError_t launch_val_loss(const float* gt, const uint8_t* valid, const float* pr, const float* pr_local,
                            const float* conf, const float* conf_local, const float* poses, int views, int items,
                            int n, float alpha, bool log1p, bool gt_scale, bool local_scale_consistent, bool has_local,
                            double* out, void* workspace, cudaStream_t st) {
  const VlLayout lay(views, items, n);
  char* ws = static_cast<char*>(workspace);
  float* inv = reinterpret_cast<float*>(ws + lay.inv);
  double* part1 = reinterpret_cast<double*>(ws + lay.part1);
  double* vb1 = reinterpret_cast<double*>(ws + lay.vb1);
  double* item1 = reinterpret_cast<double*>(ws + lay.item1);
  double* part2 = reinterpret_cast<double*>(ws + lay.part2);
  unsigned* counters = reinterpret_cast<unsigned*>(ws + lay.counters);
  const int nvb = views * items;
  const VlMaps m{gt, valid, pr, pr_local, conf, conf_local, items, views, n, (n + VPX - 1) / VPX};
  const unsigned grid = static_cast<unsigned>(nvb) * static_cast<unsigned>(m.chunks);
  cudaError_t e;
  if ((e = cudaMemsetAsync(counters, 0, lay.total - lay.counters, st)) != cudaSuccess) return e;
  if ((e = launch(vl_inverse_kernel, (nvb + VT - 1) / VT, VT, 0, st, false, poses, nvb, inv)) != cudaSuccess) return e;
  if ((e = launch(vl_norms_kernel, grid, VT, 0, st, false, m, static_cast<const float*>(inv), log1p, has_local, part1,
                  vb1, item1, counters)) != cudaSuccess)
    return e;
  return launch(vl_terms_kernel, grid, VT, 0, st, false, m, static_cast<const float*>(inv), alpha, gt_scale,
                local_scale_consistent, has_local, static_cast<const double*>(vb1), static_cast<const double*>(item1),
                part2, counters + nvb + items, out);
}

}  // namespace f3r
