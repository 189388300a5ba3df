// The viewer's scene (fast3r/viz/viser_visualizer.py): the frame preparation of start_visualization (:343-427) and the
// point export behind "Download PLY" (:168-254, :693-714), exact with respect to numpy / cv2 / scipy:
//   sky mask     u8 image -> OpenCV HSV -> colour boxes (scene_math.h) -> separable 7x7 dilate, erode, dilate ->
//                4-connected components by union-find -> the selection rule of detect_sky_mask
//   frame order  stable LSD radix sort of (frame << 32 | descending key of conf) per group of frames, then one gather
//                of points, u8 colours and not-sky values
//   visible      per-(frame, head) prefix and sky filter, tile counts, one exclusive scan, a write in frame order
//   PLY          15-byte little-endian records (3 x f32, 3 x u8)
//   extent       np.percentile(P, 20 / 80, axis=0) in float32: two order statistics per axis by a 32-bit radix select
//                and numpy's lerp
#include "f3r_kernels.h"
#include "scene_math.h"

namespace f3r {

namespace {

constexpr int ST = 256;       // threads of the pixel and element kernels
constexpr int VT = 2048;      // elements per tile of the visible-point compaction
constexpr int SCAN_T = 1024;

size_t al256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }

int blocks(long long n) { return static_cast<int>((n + ST - 1) / ST); }

// ------------------------------------------------------------------------------------------------- sky mask
struct SkyLayout {
  size_t m0, m1, lab, cnt, top, total;
};

SkyLayout sky_layout(int frames, int h, int w) {
  const size_t n = static_cast<size_t>(frames) * h * w;
  SkyLayout l;
  size_t o = 0;
  l.m0 = o; o += al256(n);
  l.m1 = o; o += al256(n);
  l.lab = o; o += al256(n * 4);
  l.cnt = o; o += al256(static_cast<size_t>(frames) * w * 4);
  l.top = o; o += al256(static_cast<size_t>(frames) * 4);
  l.total = o;
  return l;
}

// img [frames][3][h][w] in [-1, 1] -> m 1 where a colour box (or, in rows < upper, the upper-rows rule) holds
__global__ void sky_pixel_kernel(const float* __restrict__ img, int frames, int h, int w, int upper, uint8_t* __restrict__ m) {
  const long long hw = static_cast<long long>(h) * w;
  const long long i = blockIdx.x * static_cast<long long>(ST) + threadIdx.x;
  if (i >= frames * hw) return;
  const long long f = i / hw, p = i - f * hw;
  const float* s = img + 3 * f * hw + p;
  m[i] = scene_sky_pixel(scene_u8(s[0]), scene_u8(s[hw]), scene_u8(s[2 * hw]), p / w < upper);
}

// one 7-wide pass of a flat 7x7 dilate (max) or erode (min), along rows or along columns.  Windows are clipped to the
// image: with cv2's default border, out-of-image pixels never count, and a clipped rectangle is separable.
__global__ void sky_morph_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int frames, int h, int w,
                                 int along_cols, int dilate) {
  const long long hw = static_cast<long long>(h) * w;
  const long long i = blockIdx.x * static_cast<long long>(ST) + threadIdx.x;
  if (i >= frames * hw) return;
  const int p = static_cast<int>(i % hw);
  const int pos = along_cols ? p / w : p % w, n = along_cols ? h : w;
  const long long stride = along_cols ? w : 1;
  const int a = max(0, pos - 3) - pos, b = min(n - 1, pos + 3) - pos;
  uint8_t r = dilate ? 0 : 1;
  for (int j = a; j <= b; ++j) {
    const uint8_t v = in[i + j * stride];
    r = dilate ? (r | v) : (r & v);
  }
  out[i] = r;
}

// labels: every set pixel its own root (its index); clears the per-frame tables of the count pass
__global__ void sky_label_init_kernel(const uint8_t* __restrict__ m, int frames, int h, int w, int* __restrict__ lab,
                                      int* __restrict__ cnt, int* __restrict__ top, int* __restrict__ not_sky_count) {
  const long long hw = static_cast<long long>(h) * w;
  const long long i = blockIdx.x * static_cast<long long>(ST) + threadIdx.x;
  if (i >= frames * hw) return;
  const long long f = i / hw, p = i - f * hw;
  lab[i] = m[i] ? static_cast<int>(i) : -1;
  if (p < w) cnt[f * w + p] = 0;
  if (p == 0) {
    top[f] = 0;
    not_sky_count[f] = 0;
  }
}

// Union-find without locks (Playne & Hawick's scheme).  Every write to `lab` is an atomicMin that lowers an entry to
// an index of the same component, so a parent is never larger than its child and the root of each finished tree is
// the smallest index of its component: its first pixel in raster order.
// find with path compression: each node on the path is pointed (atomicMin) at the root found, an ancestor of all of
// them, so no link is lost whatever other threads write meanwhile
__device__ __forceinline__ int uf_find(int* lab, int x) {
  const volatile int* l = lab;
  int r = x, y;
  while ((y = l[r]) != r) r = y;
  while ((y = l[x]) > r) {
    atomicMin(&lab[x], r);
    x = y;
  }
  return r;
}

// links the roots of a and b, the larger under the smaller.  If root b was linked elsewhere (to `old`) in the meantime,
// the atomicMin may have replaced that link, so the loop goes on with `old`: its tree still has to join a's.
__device__ __forceinline__ void uf_union(int* lab, int a, int b) {
  while (true) {
    a = uf_find(lab, a);
    b = uf_find(lab, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(&lab[b], a);
    if (old == b) return;
    b = old;
  }
}

// 4-connectivity (scipy.ndimage.label's default structure): each set pixel unites with its left and upper neighbours
__global__ void sky_label_merge_kernel(const uint8_t* __restrict__ m, int frames, int h, int w, int* lab) {
  const long long hw = static_cast<long long>(h) * w;
  const long long i = blockIdx.x * static_cast<long long>(ST) + threadIdx.x;
  if (i >= frames * hw || !m[i]) return;
  const int p = static_cast<int>(i % hw);
  if (p % w && m[i - 1]) uf_union(lab, static_cast<int>(i), static_cast<int>(i - 1));
  if (p >= w && m[i - w]) uf_union(lab, static_cast<int>(i), static_cast<int>(i - w));
}

// every set pixel gets its root; pixels count towards their component when its root lies in row 0 (the component
// touches row 0 exactly then: the root is its first pixel); top[f] records whether any component touches row 0
__global__ void sky_label_count_kernel(int frames, int h, int w, int* lab, int* __restrict__ cnt, int* __restrict__ top) {
  const long long hw = static_cast<long long>(h) * w;
  const long long i = blockIdx.x * static_cast<long long>(ST) + threadIdx.x;
  if (i >= frames * hw || lab[i] < 0) return;
  const long long f = i / hw, p = i - f * hw;
  const int r = uf_find(lab, static_cast<int>(i));
  lab[i] = r;
  const long long rp = r - f * hw;
  if (rp < w) atomicAdd(&cnt[f * w + rp], 1);
  if (p < w) top[f] = 1;
}

// detect_sky_mask's selection: sky = the components that touch row 0 with more than H W 0.01 pixels (count >= min_sky);
// if no component touches row 0, the whole morphological mask.  Writes the not-sky int8 and counts it per frame.
__global__ void sky_select_kernel(int frames, int h, int w, const int* __restrict__ lab, const int* __restrict__ cnt,
                                  const int* __restrict__ top, int min_sky, int8_t* __restrict__ not_sky,
                                  int* __restrict__ not_sky_count) {
  const long long hw = static_cast<long long>(h) * w;
  const long long i = blockIdx.x * static_cast<long long>(ST) + threadIdx.x;
  const bool ok = i < frames * hw;
  const int f = ok ? static_cast<int>(i / hw) : -1;
  bool ns = false;
  if (ok) {
    const int r = lab[i];
    bool sky = r >= 0;
    if (sky && top[f]) {
      const long long rp = r - static_cast<long long>(f) * hw;
      sky = rp < w && cnt[static_cast<long long>(f) * w + rp] >= min_sky;
    }
    ns = !sky;
    not_sky[i] = ns ? 1 : 0;
  }
  const unsigned peers = __match_any_sync(0xffffffffu, f);
  const unsigned set = __ballot_sync(0xffffffffu, ns) & peers;
  if (ok && set && (__ffs(peers) - 1) == static_cast<int>(threadIdx.x & 31)) atomicAdd(&not_sky_count[f], __popc(set));
}

// ------------------------------------------------------------------------------------------------- frame order
struct SortLayout {
  size_t ka, kb, va, vb, hist, total;
};

SortLayout sort_layout(long long n) {
  SortLayout l;
  const size_t N = static_cast<size_t>(n);
  size_t o = 0;
  l.ka = o; o += al256(N * 8);
  l.kb = o; o += al256(N * 8);
  l.va = o; o += al256(N * 4);
  l.vb = o; o += al256(N * 4);
  l.hist = o; o += al256(radix_sort_hist_bytes(static_cast<int>(n)));
  l.total = o;
  return l;
}

__global__ void scene_key_kernel(const float* __restrict__ conf, const long long* __restrict__ off, int frames, int n,
                                 unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  const int i = blockIdx.x * ST + threadIdx.x;
  if (i >= n) return;
  int lo = 0, hi = frames - 1;  // the frame f with off[f] <= i < off[f + 1]
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= i) lo = mid;
    else hi = mid - 1;
  }
  keys[i] = (static_cast<unsigned long long>(lo) << 32) | scene_desc_key(conf[i]);
  vals[i] = i;
}

// slot j of the sorted group <- element vals[j]: its point, its u8 colour (planar image of its frame) and not-sky value;
// the first slot of each frame also writes conf.max() of the frame (NaN if the frame has a NaN: NaNs sort last)
__global__ void scene_gather_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ vals,
                                    const long long* __restrict__ off, int n, const float* __restrict__ pts,
                                    const float* __restrict__ img, const int8_t* __restrict__ not_sky,
                                    float* __restrict__ out_pts, uint8_t* __restrict__ out_rgb,
                                    int8_t* __restrict__ out_not_sky, float* __restrict__ max_conf) {
  const int j = blockIdx.x * ST + threadIdx.x;
  if (j >= n) return;
  const int s = vals[j];
  const int f = static_cast<int>(keys[j] >> 32);
  const long long o = off[f], hw = off[f + 1] - o, p = s - o;
  out_pts[3ll * j] = pts[3ll * s];
  out_pts[3ll * j + 1] = pts[3ll * s + 1];
  out_pts[3ll * j + 2] = pts[3ll * s + 2];
  const float* im = img + 3 * o + p;
  out_rgb[3ll * j] = scene_u8(im[0]);
  out_rgb[3ll * j + 1] = scene_u8(im[hw]);
  out_rgb[3ll * j + 2] = scene_u8(im[2 * hw]);
  out_not_sky[j] = not_sky[s];
  if (j == o) {
    const uint32_t last = static_cast<uint32_t>(keys[off[f + 1] - 1]);
    max_conf[f] = last == 0xffffffffu ? NAN : scene_desc_value(static_cast<uint32_t>(keys[j]));
  }
}

// ------------------------------------------------------------------------------------------------- visible points
// segment s: rows [start, start + len) of the global (head 0) or local (head 1) frame arrays; color < 0: the points'
// own RGB, else 0xRRGGBB for all of them
struct Seg {
  long long head, start, len, color;
};

__device__ __forceinline__ bool seg_keep(const Seg& g, const int8_t* ns_g, const int8_t* ns_l, int mask_sky, long long k) {
  return !mask_sky || (g.head ? ns_l : ns_g)[g.start + k] > 0;
}

__global__ void __launch_bounds__(ST) visible_count_kernel(const Seg* __restrict__ segs, int tiles,
                                                           const int8_t* __restrict__ ns_g, const int8_t* __restrict__ ns_l,
                                                           int mask_sky, unsigned long long* __restrict__ tile_cnt) {
  __shared__ unsigned ws[ST / 32];
  const Seg g = segs[blockIdx.y];
  const long long k0 = static_cast<long long>(blockIdx.x) * VT, k1 = min(g.len, k0 + VT);
  unsigned c = 0;
  for (long long k = k0 + threadIdx.x; k < k1; k += ST) c += seg_keep(g, ns_g, ns_l, mask_sky, k);
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned t = 0;
    for (int w = 0; w < ST / 32; ++w) t += ws[w];
    tile_cnt[static_cast<size_t>(blockIdx.y) * tiles + blockIdx.x] = t;
  }
}

// in-place exclusive scan of m counts (one block); total <- the sum
__global__ void __launch_bounds__(SCAN_T) scan_u64_kernel(unsigned long long* __restrict__ a, long long m,
                                                          unsigned long long* __restrict__ total) {
  __shared__ unsigned long long ws[SCAN_T / 32];
  const int tid = threadIdx.x;
  const long long per = (m + SCAN_T - 1) / SCAN_T;
  const long long i0 = min(m, tid * per), i1 = min(m, i0 + per);
  unsigned long long s = 0;
  for (long long i = i0; i < i1; ++i) s += a[i];
  unsigned long long x = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
    if ((tid & 31) >= o) x += y;
  }
  if ((tid & 31) == 31) ws[tid >> 5] = x;
  __syncthreads();
  if (tid < 32) {
    unsigned long long w = ws[tid];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, w, o);
      if (tid >= o) w += y;
    }
    ws[tid] = w;
  }
  __syncthreads();
  unsigned long long run = x - s + ((tid >> 5) ? ws[(tid >> 5) - 1] : 0ull);
  for (long long i = i0; i < i1; ++i) {
    const unsigned long long v = a[i];
    a[i] = run;
    run += v;
  }
  if (tid == SCAN_T - 1) *total = run;
}

__global__ void __launch_bounds__(ST) visible_write_kernel(const Seg* __restrict__ segs, int tiles,
                                                           const float* __restrict__ pts_g, const float* __restrict__ pts_l,
                                                           const uint8_t* __restrict__ rgb_g,
                                                           const uint8_t* __restrict__ rgb_l,
                                                           const int8_t* __restrict__ ns_g, const int8_t* __restrict__ ns_l,
                                                           int mask_sky, const unsigned long long* __restrict__ tile_off,
                                                           float* __restrict__ out_pts, uint8_t* __restrict__ out_rgb) {
  __shared__ unsigned wsum[ST / 32];
  const Seg g = segs[blockIdx.y];
  const long long k0 = static_cast<long long>(blockIdx.x) * VT, k1 = min(g.len, k0 + VT);
  if (k0 >= k1) return;
  const float* pts = g.head ? pts_l : pts_g;
  const uint8_t* rgb = g.head ? rgb_l : rgb_g;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long base = tile_off[static_cast<size_t>(blockIdx.y) * tiles + blockIdx.x];
  for (long long r = k0; r < k1; r += ST) {
    const long long k = r + threadIdx.x;
    const bool keep = k < k1 && seg_keep(g, ns_g, ns_l, mask_sky, k);
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) wsum[warp] = __popc(b);
    __syncthreads();
    unsigned before = 0, all = 0;
    for (int w = 0; w < ST / 32; ++w) {
      before += w < warp ? wsum[w] : 0u;
      all += wsum[w];
    }
    if (keep) {
      const unsigned long long o = base + before + __popc(b & ((1u << lane) - 1u));
      const long long src = g.start + k;
      out_pts[3 * o] = pts[3 * src];
      out_pts[3 * o + 1] = pts[3 * src + 1];
      out_pts[3 * o + 2] = pts[3 * src + 2];
      if (g.color < 0) {
        out_rgb[3 * o] = rgb[3 * src];
        out_rgb[3 * o + 1] = rgb[3 * src + 1];
        out_rgb[3 * o + 2] = rgb[3 * src + 2];
      } else {
        out_rgb[3 * o] = static_cast<uint8_t>(g.color >> 16);
        out_rgb[3 * o + 1] = static_cast<uint8_t>(g.color >> 8);
        out_rgb[3 * o + 2] = static_cast<uint8_t>(g.color);
      }
    }
    base += all;
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------- PLY records
__global__ void ply_pack_kernel(const float* __restrict__ pts, const uint8_t* __restrict__ rgb, long long n,
                                uint8_t* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(ST) + threadIdx.x;
  if (i >= n) return;
  uint8_t rec[15];
  memcpy(rec, pts + 3 * i, 12);  // little-endian float32 on the device, as numpy's "<f4" record field
  rec[12] = rgb[3 * i];
  rec[13] = rgb[3 * i + 1];
  rec[14] = rgb[3 * i + 2];
  uint8_t* o = out + 15 * i;
#pragma unroll
  for (int b = 0; b < 15; ++b) o[b] = rec[b];
}

// ------------------------------------------------------------------------------------------------- percentile
// Six radix selects at once: selection s = 3 j + a is order statistic rank[j] of axis a (j = 0, 1: the two
// percentiles).  Four 8-bit digit passes over the ascending 32-bit key, then the count <= the selected key and the
// smallest key above it give the next order statistic.
struct PctState {
  uint32_t prefix[6], k[6], cnt_le[6], min_gt[6], nan[3];
};

__global__ void pct_init_kernel(PctState* s, uint32_t* hist, long long k0, long long k1) {
  for (int b = threadIdx.x; b < 6 * 256; b += blockDim.x) hist[b] = 0;
  if (threadIdx.x < 6) {
    s->prefix[threadIdx.x] = 0;
    s->k[threadIdx.x] = static_cast<uint32_t>(threadIdx.x < 3 ? k0 : k1);
    s->cnt_le[threadIdx.x] = 0;
    s->min_gt[threadIdx.x] = 0xffffffffu;
  }
  if (threadIdx.x < 3) s->nan[threadIdx.x] = 0;
}

__global__ void __launch_bounds__(ST) pct_hist_kernel(const float* __restrict__ pts, long long n, PctState* s,
                                                      uint32_t* __restrict__ hist, int shift) {
  __shared__ uint32_t h[6 * 256];
  for (int b = threadIdx.x; b < 6 * 256; b += ST) h[b] = 0;
  __syncthreads();
  uint32_t prefix[6];
#pragma unroll
  for (int q = 0; q < 6; ++q) prefix[q] = s->prefix[q];
  const uint32_t mask = shift == 24 ? 0u : ~0u << (shift + 8);
  bool nan[3] = {false, false, false};
  const long long stride = static_cast<long long>(gridDim.x) * ST;
  const long long n_round = (n + stride - 1) / stride * stride;  // every lane of a warp runs every iteration
  for (long long i = blockIdx.x * static_cast<long long>(ST) + threadIdx.x; i < n_round; i += stride) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const bool in = i < n;
      const float x = in ? pts[3 * i + a] : 0.0f;
      nan[a] |= x != x;
      const uint32_t u = scene_asc_key(x);
#pragma unroll
      for (int j = 0; j < 2; ++j) {  // one shared atomic per distinct digit of the warp: the high digits pile up
        const bool ok = in && (u & mask) == prefix[3 * j + a];
        const uint32_t d = (u >> shift) & 255u;
        const unsigned act = __ballot_sync(0xffffffffu, ok);
        if (ok) {
          const unsigned peers = __match_any_sync(act, d);
          if ((__ffs(peers) - 1) == static_cast<int>(threadIdx.x & 31)) atomicAdd(&h[(3 * j + a) * 256 + d], __popc(peers));
        }
      }
    }
  }
  if (shift == 24)
    for (int a = 0; a < 3; ++a)
      if (nan[a]) s->nan[a] = 1;
  __syncthreads();
  for (int b = threadIdx.x; b < 6 * 256; b += ST)
    if (h[b]) atomicAdd(&hist[b], h[b]);
}

__global__ void pct_digit_kernel(PctState* s, uint32_t* hist, int shift) {
  const int q = threadIdx.x;
  if (q >= 6) return;
  uint32_t* h = hist + q * 256;
  uint32_t cum = 0;
  int d = 0;
  for (; d < 255; ++d) {
    if (cum + h[d] > s->k[q]) break;
    cum += h[d];
  }
  for (int b = 0; b < 256; ++b) h[b] = 0;
  s->prefix[q] |= static_cast<uint32_t>(d) << shift;
  s->k[q] -= cum;
}

__global__ void __launch_bounds__(ST) pct_succ_kernel(const float* __restrict__ pts, long long n, PctState* s) {
  uint32_t key[6], cnt[6], mn[6];
#pragma unroll
  for (int q = 0; q < 6; ++q) {
    key[q] = s->prefix[q];
    cnt[q] = 0;
    mn[q] = 0xffffffffu;
  }
  for (long long i = blockIdx.x * static_cast<long long>(ST) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * ST) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const uint32_t u = scene_asc_key(pts[3 * i + a]);  // a NaN key lies outside [-inf, +inf]: the result is NaN anyway
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int q = 3 * j + a;
        if (u <= key[q]) ++cnt[q];
        else mn[q] = min(mn[q], u);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < 6; ++q) {
    cnt[q] = __reduce_add_sync(0xffffffffu, cnt[q]);
    mn[q] = __reduce_min_sync(0xffffffffu, mn[q]);
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(&s->cnt_le[q], cnt[q]);
      atomicMin(&s->min_gt[q], mn[q]);
    }
  }
}

// numpy's _lerp in float32: a + (b - a) t, or b - (b - a) (1 - t) where t >= 0.5
__device__ __forceinline__ float np_lerp(float a, float b, float t) {
  const float d = __fsub_rn(b, a);
  return t >= 0.5f ? __fsub_rn(b, __fmul_rn(d, __fsub_rn(1.0f, t))) : __fadd_rn(a, __fmul_rn(d, t));
}

// out[0..2] = percentile j = 0 per axis, out[3..5] = percentile j = 1, out[6] = max over axes of out[3 + a] - out[a]
// (NaN where an axis holds a NaN, as np.percentile and np.max give)
__global__ void pct_final_kernel(const PctState* s, long long k0, long long k1, long long n, float g0, float g1,
                                 float* out) {
  if (threadIdx.x != 0) return;
  float ext = 0.0f;
  for (int a = 0; a < 3; ++a) {
    float v[2];
    for (int j = 0; j < 2; ++j) {
      const int q = 3 * j + a;
      const long long k = j ? k1 : k0;
      const float lo = scene_asc_value(s->prefix[q]);
      const float hi = (k + 1 >= n || s->cnt_le[q] > k + 1) ? lo : scene_asc_value(s->min_gt[q]);
      v[j] = s->nan[a] ? NAN : np_lerp(lo, hi, j ? g1 : g0);
      out[3 * j + a] = v[j];
    }
    const float e = __fsub_rn(v[1], v[0]);
    ext = a == 0 ? e : ((ext != ext || e != e) ? NAN : fmaxf(ext, e));
  }
  out[6] = ext;
}

}  // namespace

// ------------------------------------------------------------------------------------------------- launchers
size_t sky_mask_workspace(int frames, int h, int w) { return sky_layout(frames, h, w).total; }

cudaError_t launch_sky_mask(const float* img, int frames, int h, int w, int upper, int min_sky, int8_t* not_sky,
                            int* not_sky_count, void* workspace, cudaStream_t st) {
  const SkyLayout l = sky_layout(frames, h, w);
  uint8_t* b = static_cast<uint8_t*>(workspace);
  uint8_t* m[2] = {b + l.m0, b + l.m1};
  int* lab = reinterpret_cast<int*>(b + l.lab);
  int* cnt = reinterpret_cast<int*>(b + l.cnt);
  int* top = reinterpret_cast<int*>(b + l.top);
  const int g = blocks(static_cast<long long>(frames) * h * w);
  cudaError_t e;
  if ((e = launch(sky_pixel_kernel, g, ST, 0, st, false, img, frames, h, w, upper, m[0])) != cudaSuccess) return e;
  // dilate, then the open (erode, dilate); each as a row pass and a column pass; ends in m[0]
  const int dil[3] = {1, 0, 1};
  for (int pass = 0; pass < 6; ++pass)
    if ((e = launch(sky_morph_kernel, g, ST, 0, st, false, m[pass & 1], m[1 - (pass & 1)], frames, h, w, pass & 1,
                    dil[pass >> 1])) != cudaSuccess)
      return e;
  if ((e = launch(sky_label_init_kernel, g, ST, 0, st, false, m[0], frames, h, w, lab, cnt, top, not_sky_count)) !=
      cudaSuccess)
    return e;
  if ((e = launch(sky_label_merge_kernel, g, ST, 0, st, false, m[0], frames, h, w, lab)) != cudaSuccess) return e;
  if ((e = launch(sky_label_count_kernel, g, ST, 0, st, false, frames, h, w, lab, cnt, top)) != cudaSuccess) return e;
  return launch(sky_select_kernel, g, ST, 0, st, false, frames, h, w, lab, cnt, top, min_sky, not_sky, not_sky_count);
}

size_t scene_sort_workspace(long long n) { return sort_layout(n).total; }

cudaError_t launch_scene_sort(const float* conf, const float* pts, const float* img, const int8_t* not_sky,
                              const long long* off, int frames, int n, float* out_pts, uint8_t* out_rgb,
                              int8_t* out_not_sky, float* max_conf, void* workspace, cudaStream_t st) {
  const SortLayout l = sort_layout(n);
  uint8_t* b = static_cast<uint8_t*>(workspace);
  unsigned long long* k[2] = {reinterpret_cast<unsigned long long*>(b + l.ka),
                              reinterpret_cast<unsigned long long*>(b + l.kb)};
  int* v[2] = {reinterpret_cast<int*>(b + l.va), reinterpret_cast<int*>(b + l.vb)};
  uint32_t* hist = reinterpret_cast<uint32_t*>(b + l.hist);
  int fbits = 0;
  while ((1 << fbits) < frames) ++fbits;
  cudaError_t e;
  if ((e = launch(scene_key_kernel, blocks(n), ST, 0, st, false, conf, off, frames, n, k[0], v[0])) != cudaSuccess)
    return e;
  int in_b = 0;
  if ((e = launch_radix_sort(k, v, n, 32 + fbits, hist, &in_b, st)) != cudaSuccess) return e;
  return launch(scene_gather_kernel, blocks(n), ST, 0, st, false, k[in_b], v[in_b], off, n, pts, img, not_sky, out_pts,
                out_rgb, out_not_sky, max_conf);
}

int scene_visible_tiles(long long max_len) { return static_cast<int>((max_len + VT - 1) / VT); }

size_t scene_visible_workspace(int nseg, int tiles) {
  return al256(static_cast<size_t>(nseg) * 32) + al256(static_cast<size_t>(nseg) * tiles * 8);
}

cudaError_t launch_scene_visible(const long long* segs, int nseg, int tiles, const float* pts_g, const float* pts_l,
                                 const uint8_t* rgb_g, const uint8_t* rgb_l, const int8_t* ns_g, const int8_t* ns_l,
                                 int mask_sky, unsigned long long* total, float* out_pts, uint8_t* out_rgb,
                                 void* workspace, cudaStream_t st) {
  uint8_t* b = static_cast<uint8_t*>(workspace);
  const Seg* sg = reinterpret_cast<const Seg*>(segs);
  unsigned long long* tile = reinterpret_cast<unsigned long long*>(b + al256(static_cast<size_t>(nseg) * 32));
  const dim3 grid(tiles, nseg);
  if (!out_pts) {  // counting phase: tile counts, their exclusive scan and the total
    cudaError_t e;
    if ((e = launch(visible_count_kernel, grid, ST, 0, st, false, sg, tiles, ns_g, ns_l, mask_sky, tile)) != cudaSuccess)
      return e;
    return launch(scan_u64_kernel, 1, SCAN_T, 0, st, false, tile, static_cast<long long>(nseg) * tiles, total);
  }
  return launch(visible_write_kernel, grid, ST, 0, st, false, sg, tiles, pts_g, pts_l, rgb_g, rgb_l, ns_g, ns_l, mask_sky,
                tile, out_pts, out_rgb);
}

cudaError_t launch_ply_pack(const float* pts, const uint8_t* rgb, long long n, uint8_t* out, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  return launch(ply_pack_kernel, blocks(n), ST, 0, st, false, pts, rgb, n, out);
}

size_t percentile_workspace() { return al256(sizeof(PctState)) + al256(6 * 256 * 4); }

cudaError_t launch_extent_percentiles(const float* pts, long long n, long long k0, long long k1, float g0, float g1,
                                      float* out, void* workspace, cudaStream_t st) {
  PctState* s = static_cast<PctState*>(workspace);
  uint32_t* hist = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(workspace) + al256(sizeof(PctState)));
  const int g = static_cast<int>(min(1024ll, (n + ST - 1) / ST));
  cudaError_t e;
  if ((e = launch(pct_init_kernel, 1, ST, 0, st, false, s, hist, k0, k1)) != cudaSuccess) return e;
  for (int shift = 24; shift >= 0; shift -= 8) {
    if ((e = launch(pct_hist_kernel, g, ST, 0, st, false, pts, n, s, hist, shift)) != cudaSuccess) return e;
    if ((e = launch(pct_digit_kernel, 1, 32, 0, st, false, s, hist, shift)) != cudaSuccess) return e;
  }
  if ((e = launch(pct_succ_kernel, g, ST, 0, st, false, pts, n, s)) != cudaSuccess) return e;
  return launch(pct_final_kernel, 1, 32, 0, st, false, s, k0, k1, n, g0, g1, out);
}

}  // namespace f3r
