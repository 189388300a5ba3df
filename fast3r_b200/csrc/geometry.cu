// Geometry tail that every caller runs right after the forward (SURVEY.md §8 row f2, first slice):
//   conf_quantile      torch.quantile(conf.reshape(-1), q) per view            (multiview_dust3r_module.py:477, :1093)
//   similarity_fit     mask = conf >= thr & valid (with the two "< 3 points" fallbacks) and the least-squares
//                      similarity y ~ s R x + t over the masked points        (multiview_dust3r_module.py:427-525;
//                      roma.rigid_points_registration(compute_scaling=True) = Umeyama / Kabsch)
//   similarity_apply   out = s (x R^T) + t on ALL points                       (multiview_dust3r_module.py:517-521)
//   focal_weiszfeld    IRLS focal from a pointmap                              (dust3r/post_process.py:19-79, :82-142)
// All of it is HBM-bound streaming / reduction work: one pass over 12-28 bytes per pixel per kernel, fp64 accumulators,
// fixed reduction order (no float atomics), so results do not depend on scheduling.
#include <cooperative_groups.h>
#include <math.h>

#include "f3r_kernels.h"
#include "geometry_math.h"

namespace f3r {

// ------------------------------------------------------------------------------------------------- quantile
// One 8-CTA cluster per view: 4-pass 8-bit radix select of the order statistic floor(q (n-1)) on the order-preserving
// integer image of the floats, one more pass for its successor, then ATen's lerp.  Each CTA histograms its eighth of the
// view (four keys per thread and iteration so that loads overlap); the eight histograms are summed through distributed
// shared memory and every CTA derives the same digit.  Histogram updates are warp-aggregated (confidences share their
// exponent byte, so naive shared atomics would serialise on one bin).  No global atomics, fixed result.  A NaN of either
// sign makes the view's result NaN, as in ATen (its key lies above fkey(+inf) or below fkey(-inf)): the first pass flags
// it and ORs the flag across the cluster with the histograms.
namespace {

namespace cg = cooperative_groups;

constexpr int QT = 1024;  // threads per CTA
constexpr int QC = 8;     // CTAs per view (one cluster)

__device__ __forceinline__ uint32_t fkey(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// keys of elements i .. i+3 (i a multiple of 4 past the slice start); elements at or past i1 are flagged invalid
__device__ __forceinline__ void load_keys4(const float* __restrict__ c, int i, int i1, bool vec, uint32_t u[4], bool ok[4]) {
  if (vec && i + 3 < i1) {
    const float4 v = *reinterpret_cast<const float4*>(c + i);
    u[0] = fkey(v.x); u[1] = fkey(v.y); u[2] = fkey(v.z); u[3] = fkey(v.w);
    ok[0] = ok[1] = ok[2] = ok[3] = true;
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      ok[e] = i + e < i1;
      u[e] = ok[e] ? fkey(c[i + e]) : 0u;
    }
  }
}

// warp-collective: every thread of the warp must call it
__device__ __forceinline__ void hist_add(uint32_t* hist, bool ok, uint32_t d) {
  const unsigned act = __ballot_sync(0xffffffffu, ok);
  if (ok) {
    const unsigned peers = __match_any_sync(act, d);
    if ((__ffs(peers) - 1) == static_cast<int>(threadIdx.x & 31)) atomicAdd(&hist[d], static_cast<uint32_t>(__popc(peers)));
  }
}

__global__ void __launch_bounds__(QT) conf_quantile_kernel(const float* __restrict__ conf, int n, float q,
                                                           float* __restrict__ thr, int vec_ok) {
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ uint32_t hist[256];
  __shared__ uint32_t total[256];
  __shared__ uint32_t s_prefix, s_k, s_cnt_le, s_min_gt, s_nan, s_any_nan;
  const int view = blockIdx.x / QC;
  const unsigned crank = cluster.block_rank();
  const float* c = conf + static_cast<size_t>(view) * n;
  const int tid = threadIdx.x;
  const bool vec = vec_ok != 0;
  const int per = (((n + QC - 1) / QC) + 3) & ~3;
  const int i0 = min(n, static_cast<int>(crank) * per), i1 = min(n, i0 + per);
  const float rank = __fmul_rn(q, static_cast<float>(n - 1));
  const int lo = static_cast<int>(floorf(rank));
  const int hi = static_cast<int>(ceilf(rank));
  const float w = __fsub_rn(rank, static_cast<float>(lo));

  uint32_t prefix = 0, mask = 0, k = static_cast<uint32_t>(lo);
  if (tid == 0) s_nan = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    bool nan = false;
    for (int base = i0; base < i1; base += QT * 4) {
      uint32_t u[4];
      bool ok[4];
      load_keys4(c, base + tid * 4, i1, vec, u, ok);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        hist_add(hist, ok[e] && (u[e] & mask) == prefix, (u[e] >> shift) & 255u);
        if (shift == 24) nan |= ok[e] && (u[e] > 0xff800000u || u[e] < 0x007fffffu);  // NaN: beyond fkey(+-inf)
      }
    }
    if (nan) s_nan = 1;
    cluster.sync();  // all eight histograms (and NaN flags) of this view are complete
    if (tid < 256) {
      uint32_t sum = 0;
      for (unsigned r = 0; r < QC; ++r) sum += cluster.map_shared_rank(hist, r)[tid];
      total[tid] = sum;
    }
    if (shift == 24 && tid == 256) {
      uint32_t any = 0;
      for (unsigned r = 0; r < QC; ++r) any |= *cluster.map_shared_rank(&s_nan, r);
      s_any_nan = any;
    }
    cluster.sync();  // remote reads done before any CTA clears its histogram for the next pass
    if (shift == 24 && s_any_nan) {  // the same in every CTA of the cluster, so all leave together
      if (crank == 0 && tid == 0) thr[view] = __uint_as_float(0x7fc00000u);
      return;
    }
    if (tid == 0) {
      uint32_t cum = 0;
      int d = 0;
      for (; d < 255; ++d) {
        const uint32_t h = total[d];
        if (cum + h > k) break;
        cum += h;
      }
      s_prefix = prefix | (static_cast<uint32_t>(d) << shift);
      s_k = k - cum;
    }
    __syncthreads();
    prefix = s_prefix;
    k = s_k;
    mask |= 0xffu << shift;
  }
  const uint32_t u_lo = prefix;
  if (hi == lo) {  // integral rank: ATen still evaluates lerp(a, a, 0) = fma(0, a - a, a), which is NaN for an infinite a
    if (crank == 0 && tid == 0) {
      const float a = fkey_inv(u_lo);
      thr[view] = fmaf(w, __fsub_rn(a, a), a);
    }
    return;
  }
  if (tid == 0) {
    s_cnt_le = 0;
    s_min_gt = 0xffffffffu;
  }
  __syncthreads();
  uint32_t cnt = 0, mn = 0xffffffffu;
  for (int base = i0; base < i1; base += QT * 4) {
    uint32_t u[4];
    bool ok[4];
    load_keys4(c, base + tid * 4, i1, vec, u, ok);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (!ok[e]) continue;
      if (u[e] <= u_lo) ++cnt;
      else mn = min(mn, u[e]);
    }
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  mn = __reduce_min_sync(0xffffffffu, mn);
  if ((tid & 31) == 0) {
    atomicAdd(&s_cnt_le, cnt);
    atomicMin(&s_min_gt, mn);
  }
  cluster.sync();
  if (crank == 0 && tid == 0) {
    uint32_t cnt_le = 0, min_gt = 0xffffffffu;
    for (unsigned r = 0; r < QC; ++r) {
      cnt_le += *cluster.map_shared_rank(&s_cnt_le, r);
      min_gt = min(min_gt, *cluster.map_shared_rank(&s_min_gt, r));
    }
    const uint32_t u_hi = (static_cast<uint32_t>(hi) < cnt_le) ? u_lo : min_gt;
    const float a = fkey_inv(u_lo), b = fkey_inv(u_hi);
    const float diff = __fsub_rn(b, a);
    // ATen lerp (Lerp.h; fused multiply-add on both the vectorised CPU path and CUDA):
    // |w| < 0.5 ? fma(w, b - a, a) : fma(w - 1, b - a, b)
    thr[view] = (fabsf(w) < 0.5f) ? fmaf(w, diff, a) : fmaf(__fsub_rn(w, 1.0f), diff, b);
  }
  cluster.sync();  // keep every CTA's shared memory alive until CTA 0 has read it
}

// ------------------------------------------------------------------------------------------------- similarity fit
// MOM (17 moments per point set) comes from geometry_math.h
constexpr int FIT_THREADS = 256;
constexpr int FIT_CHUNKS = 32;   // partial sums per view (fixed, so the reduction order is)

struct Moments {
  double v[MOM];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < MOM; ++i) v[i] = 0.0;
  }
  __device__ __forceinline__ void add(float x0, float x1, float x2, float y0, float y1, float y2) {
    const double a0 = x0, a1 = x1, a2 = x2, b0 = y0, b1 = y1, b2 = y2;
    v[0] += 1.0;
    v[1] += a0; v[2] += a1; v[3] += a2;
    v[4] += b0; v[5] += b1; v[6] += b2;
    v[7] += a0 * a0 + a1 * a1 + a2 * a2;
    v[8] += b0 * a0;  v[9] += b0 * a1;  v[10] += b0 * a2;
    v[11] += b1 * a0; v[12] += b1 * a1; v[13] += b1 * a2;
    v[14] += b2 * a0; v[15] += b2 * a1; v[16] += b2 * a2;
  }
};

// mode 0: moments of the pixels with conf >= thr & valid.  mode 1 (the reference's first fallback, only for the views
// the mode-0 solve flagged as having fewer than 3 such pixels): valid pixels only.  partial [views][FIT_CHUNKS][MOM].
// Four pixels per thread and iteration (3 + 3 + 1 sixteen-byte loads in flight) when the layout allows it.
__global__ void __launch_bounds__(FIT_THREADS) similarity_moments_kernel(
    const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ conf,
    const float* __restrict__ thr, const uint8_t* __restrict__ valid, int n, int vec_ok, int mode,
    const int* __restrict__ flags, double* __restrict__ partial) {
  __shared__ double red[FIT_THREADS / 32][MOM];
  const int view = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
  if (mode == 1 && flags[view] == 0) return;
  const size_t base = static_cast<size_t>(view) * n;
  const float* xv = x + base * 3;
  const float* yv = y + base * 3;
  const bool use_conf = mode == 0 && conf != nullptr && thr != nullptr;
  const float* cv = use_conf ? conf + base : nullptr;
  const uint8_t* vv = valid ? valid + base : nullptr;
  const float t = use_conf ? thr[view] : 0.f;
  const bool vec = vec_ok != 0;
  const int per = (((n + FIT_CHUNKS - 1) / FIT_CHUNKS) + 3) & ~3;
  const int i0 = min(n, chunk * per), i1 = min(n, i0 + per);
  Moments a;
  a.zero();
  for (int i = i0 + tid * 4; i < i1; i += FIT_THREADS * 4) {
    float px[12], py[12], pc[4];
    bool in[4];
    if (vec && i + 3 < i1) {
      const float4* xs = reinterpret_cast<const float4*>(xv + 3 * static_cast<size_t>(i));
      const float4* ys = reinterpret_cast<const float4*>(yv + 3 * static_cast<size_t>(i));
      const float4 x0 = xs[0], x1 = xs[1], x2 = xs[2], y0 = ys[0], y1 = ys[1], y2 = ys[2];
      px[0] = x0.x; px[1] = x0.y; px[2] = x0.z; px[3] = x0.w; px[4] = x1.x; px[5] = x1.y;
      px[6] = x1.z; px[7] = x1.w; px[8] = x2.x; px[9] = x2.y; px[10] = x2.z; px[11] = x2.w;
      py[0] = y0.x; py[1] = y0.y; py[2] = y0.z; py[3] = y0.w; py[4] = y1.x; py[5] = y1.y;
      py[6] = y1.z; py[7] = y1.w; py[8] = y2.x; py[9] = y2.y; py[10] = y2.z; py[11] = y2.w;
      if (cv) {
        const float4 cc = *reinterpret_cast<const float4*>(cv + i);
        pc[0] = cc.x; pc[1] = cc.y; pc[2] = cc.z; pc[3] = cc.w;
      } else {
        pc[0] = pc[1] = pc[2] = pc[3] = 0.f;
      }
      if (vv) {
        const uchar4 m = *reinterpret_cast<const uchar4*>(vv + i);
        in[0] = m.x != 0; in[1] = m.y != 0; in[2] = m.z != 0; in[3] = m.w != 0;
      } else {
        in[0] = in[1] = in[2] = in[3] = true;
      }
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = i + e;
        in[e] = j < i1 && (vv ? vv[j] != 0 : true);
        pc[e] = (in[e] && cv) ? cv[j] : 0.f;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          px[3 * e + d] = in[e] ? xv[3 * static_cast<size_t>(j) + d] : 0.f;
          py[3 * e + d] = in[e] ? yv[3 * static_cast<size_t>(j) + d] : 0.f;
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (in[e] && (!cv || pc[e] >= t)) a.add(px[3 * e], px[3 * e + 1], px[3 * e + 2], py[3 * e], py[3 * e + 1], py[3 * e + 2]);
  }
#pragma unroll
  for (int j = 0; j < MOM; ++j) {
    double va = a.v[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) va += __shfl_down_sync(0xffffffffu, va, o);
    if ((tid & 31) == 0) red[tid >> 5][j] = va;
  }
  __syncthreads();
  if (tid < MOM) {
    double s = 0.0;
#pragma unroll
    for (int wp = 0; wp < FIT_THREADS / 32; ++wp) s += red[wp][tid];
    partial[(static_cast<size_t>(view) * FIT_CHUNKS + chunk) * MOM + tid] = s;
  }
}

// mode 0: solve from the confidence-masked moments, or flag the view (fewer than 3 pixels) and write the identity;
// mode 1: for flagged views, solve from the valid-only moments (multiview_dust3r_module.py:493-501) or keep the identity (:504-509)
__global__ void __launch_bounds__(64) similarity_solve_kernel(const double* __restrict__ partial, float* __restrict__ rts,
                                                              int mode, int* __restrict__ flags) {
  __shared__ double tot[MOM];
  const int view = blockIdx.x, tid = threadIdx.x;
  if (mode == 1 && flags[view] == 0) return;
  if (tid < MOM) {
    double s = 0.0;
    for (int c = 0; c < FIT_CHUNKS; ++c) s += partial[(static_cast<size_t>(view) * FIT_CHUNKS + c) * MOM + tid];
    tot[tid] = s;
  }
  __syncthreads();
  if (tid != 0) return;
  float* out = rts + static_cast<size_t>(view) * 13;
  if (tot[0] >= 3.0) {
    umeyama_from_moments(tot, out);
    if (mode == 0) flags[view] = 0;
    return;
  }
  for (int i = 0; i < 13; ++i) out[i] = 0.f;
  out[0] = out[4] = out[8] = 1.f;
  out[12] = 1.f;
  if (mode == 0) flags[view] = 1;
}

// ------------------------------------------------------------------------------------------------- similarity apply
constexpr int APPLY_THREADS = 256;

__device__ __forceinline__ void apply_pt(const float* r, float x0, float x1, float x2, float& o0, float& o1, float& o2) {
  o0 = fmaf(r[12], fmaf(r[2], x2, fmaf(r[1], x1, r[0] * x0)), r[9]);
  o1 = fmaf(r[12], fmaf(r[5], x2, fmaf(r[4], x1, r[3] * x0)), r[10]);
  o2 = fmaf(r[12], fmaf(r[8], x2, fmaf(r[7], x1, r[6] * x0)), r[11]);
}

// kVec: n % 4 == 0 and 16-byte aligned bases - each thread moves 4 points as 3 float4
template <bool kVec>
__global__ void __launch_bounds__(APPLY_THREADS) similarity_apply_kernel(const float* __restrict__ x,
                                                                         const float* __restrict__ rts,
                                                                         float* __restrict__ out, int n) {
  __shared__ float r[13];
  const int view = blockIdx.y;
  if (threadIdx.x < 13) r[threadIdx.x] = rts[static_cast<size_t>(view) * 13 + threadIdx.x];
  __syncthreads();
  const size_t base = static_cast<size_t>(view) * n * 3;
  if (kVec) {
    const int g = blockIdx.x * APPLY_THREADS + threadIdx.x;  // group of 4 points
    if (g * 4 >= n) return;
    const float4* src = reinterpret_cast<const float4*>(x + base) + static_cast<size_t>(g) * 3;
    float4* dst = reinterpret_cast<float4*>(out + base) + static_cast<size_t>(g) * 3;
    const float4 a = __ldcs(src), b = __ldcs(src + 1), c = __ldcs(src + 2);
    float4 oa, ob, oc;
    apply_pt(r, a.x, a.y, a.z, oa.x, oa.y, oa.z);
    apply_pt(r, a.w, b.x, b.y, oa.w, ob.x, ob.y);
    apply_pt(r, b.z, b.w, c.x, ob.z, ob.w, oc.x);
    apply_pt(r, c.y, c.z, c.w, oc.y, oc.z, oc.w);
    __stcs(dst, oa);
    __stcs(dst + 1, ob);
    __stcs(dst + 2, oc);
  } else {
    const int i = blockIdx.x * APPLY_THREADS + threadIdx.x;
    if (i >= n) return;
    const float* p = x + base + static_cast<size_t>(i) * 3;
    float* o = out + base + static_cast<size_t>(i) * 3;
    float o0, o1, o2;
    apply_pt(r, p[0], p[1], p[2], o0, o1, o2);
    o[0] = o0;
    o[1] = o1;
    o[2] = o2;
  }
}

// ------------------------------------------------------------------------------------------------- Weiszfeld focal
constexpr int FOC_THREADS = 256;
constexpr int FOC_CHUNKS = 256;  // partial sums per view and iteration
constexpr int FOC_P = 3;         // numerator, denominator, selected points

// One IRLS iteration over all views: every block first re-derives the current focal of its view from the previous
// iteration's partial sums (prev == NULL: the closed-form L2 initialisation, unit weights), then reduces its chunk.
__global__ void __launch_bounds__(FOC_THREADS) weiszfeld_iter_kernel(
    const float* __restrict__ pts, const float* __restrict__ conf, const float* __restrict__ thr,
    const float* __restrict__ pp, int H, int W, const double* __restrict__ prev, double* __restrict__ next) {
  __shared__ double red[FOC_THREADS / 32][FOC_P];
  __shared__ float s_focal;
  const int view = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
  const int n = H * W;
  float focal = 0.f;
  if (prev) {
    double pn = 0.0, pd = 0.0;
    const double* pv = prev + static_cast<size_t>(view) * FOC_CHUNKS * FOC_P;
    for (int c = tid; c < FOC_CHUNKS; c += FOC_THREADS) {
      pn += pv[c * FOC_P];
      pd += pv[c * FOC_P + 1];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      pn += __shfl_down_sync(0xffffffffu, pn, o);
      pd += __shfl_down_sync(0xffffffffu, pd, o);
    }
    if ((tid & 31) == 0) {
      red[tid >> 5][0] = pn;
      red[tid >> 5][1] = pd;
    }
    __syncthreads();
    if (tid == 0) {
      double sn = 0.0, sd = 0.0;
      for (int wp = 0; wp < FOC_THREADS / 32; ++wp) {
        sn += red[wp][0];
        sd += red[wp][1];
      }
      s_focal = static_cast<float>(sn / sd);
    }
    __syncthreads();
    focal = s_focal;
  }
  const float cx = pp ? pp[2 * view] : 0.5f * static_cast<float>(W);
  const float cy = pp ? pp[2 * view + 1] : 0.5f * static_cast<float>(H);
  const size_t base = static_cast<size_t>(view) * n;
  const float* pv3 = pts + base * 3;
  const float* cv = (conf && thr) ? conf + base : nullptr;
  const float t = cv ? thr[view] : 0.f;
  const int per = (n + FOC_CHUNKS - 1) / FOC_CHUNKS;
  const int i0 = chunk * per, i1 = min(n, i0 + per);
  double num = 0.0, den = 0.0, cnt = 0.0;
  for (int i = i0 + tid; i < i1; i += FOC_THREADS) {
    if (cv && !(cv[i] >= t)) continue;
    const float x = pv3[3 * i], y = pv3[3 * i + 1], z = pv3[3 * i + 2];
    float xz = __fdiv_rn(x, z), yz = __fdiv_rn(y, z);
    if (!isfinite(xz)) xz = 0.f;   // nan_to_num(posinf=0, neginf=0), NaN -> 0
    if (!isfinite(yz)) yz = 0.f;
    const float u = static_cast<float>(i % W) - cx, v = static_cast<float>(i / W) - cy;
    const float dpx = __fadd_rn(__fmul_rn(xz, u), __fmul_rn(yz, v));
    const float dxx = __fadd_rn(__fmul_rn(xz, xz), __fmul_rn(yz, yz));
    float wgt = 1.f;
    if (prev) {
      const float du = u - focal * xz, dv = v - focal * yz;
      wgt = 1.f / fmaxf(sqrtf(du * du + dv * dv), 1e-8f);
    }
    num += static_cast<double>(wgt * dpx);
    den += static_cast<double>(wgt * dxx);
    cnt += 1.0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    num += __shfl_down_sync(0xffffffffu, num, o);
    den += __shfl_down_sync(0xffffffffu, den, o);
    cnt += __shfl_down_sync(0xffffffffu, cnt, o);
  }
  if ((tid & 31) == 0) {
    red[tid >> 5][0] = num;
    red[tid >> 5][1] = den;
    red[tid >> 5][2] = cnt;
  }
  __syncthreads();
  if (tid < FOC_P) {
    double s = 0.0;
#pragma unroll
    for (int wp = 0; wp < FOC_THREADS / 32; ++wp) s += red[wp][tid];
    next[(static_cast<size_t>(view) * FOC_CHUNKS + chunk) * FOC_P + tid] = s;
  }
}

__global__ void weiszfeld_final_kernel(const double* __restrict__ last, int views, int H, int W, float* __restrict__ focal) {
  const int view = blockIdx.x * blockDim.x + threadIdx.x;
  if (view >= views) return;
  double num = 0.0, den = 0.0, cnt = 0.0;
  const double* pv = last + static_cast<size_t>(view) * FOC_CHUNKS * FOC_P;
  for (int c = 0; c < FOC_CHUNKS; ++c) {
    num += pv[c * FOC_P];
    den += pv[c * FOC_P + 1];
    cnt += pv[c * FOC_P + 2];
  }
  float f;
  if (cnt == 0.0) {
    f = static_cast<float>(static_cast<double>(max(H, W)) / (2.0 * tan(M_PI / 6.0)));  // post_process.py:108
  } else {
    f = static_cast<float>(num / den);
    if (f < 0.f) f = 0.f;  // focal.clip(min=0 * focal_base, max=inf)
  }
  focal[view] = f;
}

}  // namespace

// ------------------------------------------------------------------------------------------------- launchers
cudaError_t launch_conf_quantile(const float* conf, int views, int n, float q, float* thr, cudaStream_t stream) {
  const int vec_ok = (n % 4 == 0) && (reinterpret_cast<uintptr_t>(conf) & 15) == 0;
  return launch<QC>(conf_quantile_kernel, static_cast<unsigned>(views) * QC, QT, 0, stream, false, conf, n, q, thr, vec_ok);
}

// partial sums [views][FIT_CHUNKS][MOM] fp64, then one int flag per view
size_t similarity_fit_workspace(int views) {
  const size_t flags = (static_cast<size_t>(views) * sizeof(int) + 7) & ~static_cast<size_t>(7);
  return static_cast<size_t>(views) * FIT_CHUNKS * MOM * sizeof(double) + flags;
}

cudaError_t launch_similarity_fit(const float* x, const float* y, const float* conf, const float* thr,
                                  const uint8_t* valid, int views, int n, float* rts, double* workspace,
                                  cudaStream_t stream) {
  int* flags = reinterpret_cast<int*>(workspace + static_cast<size_t>(views) * FIT_CHUNKS * MOM);
  const uintptr_t al = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(conf);
  const int vec_ok = (n % 4 == 0) && (al & 15) == 0 && (reinterpret_cast<uintptr_t>(valid) & 3) == 0;
  const int modes = (conf && thr) ? 2 : 1;  // without a confidence mask the first fallback is the same point set
  for (int mode = 0; mode < modes; ++mode) {
    cudaError_t e;
    if ((e = launch(similarity_moments_kernel, dim3(FIT_CHUNKS, views), FIT_THREADS, 0, stream, false, x, y, conf, thr,
                    valid, n, vec_ok, mode, flags, workspace)) != cudaSuccess)
      return e;
    if ((e = launch(similarity_solve_kernel, views, 64, 0, stream, false, workspace, rts, mode, flags)) != cudaSuccess)
      return e;
  }
  return cudaSuccess;
}

cudaError_t launch_similarity_apply(const float* x, const float* rts, float* out, int views, int n, cudaStream_t stream) {
  const bool vec = (n % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  const int items = vec ? n / 4 : n;
  return launch(vec ? similarity_apply_kernel<true> : similarity_apply_kernel<false>,
                dim3((items + APPLY_THREADS - 1) / APPLY_THREADS, views), APPLY_THREADS, 0, stream, false, x, rts, out, n);
}

size_t focal_workspace(int views) { return 2 * static_cast<size_t>(views) * FOC_CHUNKS * FOC_P * sizeof(double); }

cudaError_t launch_focal_weiszfeld(const float* pts, const float* conf, const float* thr, const float* pp, int views,
                                   int H, int W, int iters, float* focal, double* workspace, cudaStream_t stream) {
  const size_t half = static_cast<size_t>(views) * FOC_CHUNKS * FOC_P;
  double* buf[2] = {workspace, workspace + half};
  const dim3 grid(FOC_CHUNKS, views);
  for (int it = 0; it <= iters; ++it) {
    const cudaError_t e = launch(weiszfeld_iter_kernel, grid, FOC_THREADS, 0, stream, false, pts, conf, thr, pp, H, W,
                                 it ? buf[(it - 1) & 1] : nullptr, buf[it & 1]);
    if (e != cudaSuccess) return e;
  }
  return launch(weiszfeld_final_kernel, (views + 127) / 128, 128, 0, stream, false, buf[iters & 1], views, H, W, focal);
}

}  // namespace f3r
