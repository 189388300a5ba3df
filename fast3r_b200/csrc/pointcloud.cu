// Reconstruction metrics (fast3r/eval/recon_metric.py and the normals of evaluate_reconstruction,
// fast3r/models/multiview_dust3r_module.py:551-735), exact with respect to scipy's cKDTree:
//   index build      bounding box -> 33-bit-per-axis Morton keys -> LSD radix sort -> buckets of PC_LEAF consecutive
//                    points with fp64 AABBs, parents = AABBs of PC_FAN consecutive children
//   nearest          exact 1-NN per query (queries in Morton order), depth-first with AABB pruning, fp64 distances
//                    rounded exactly as scipy rounds them
//   knn normals      k <= 32 nearest (the point itself included) -> fp64 covariance -> smallest eigenvector
//   reductions       fixed-order fp64 mean, exact median (64-bit radix select), count below a threshold, |dot|
// No library sort or reduction: every pass is a kernel here, and every result is independent of scheduling.
#include <math.h>

#include "f3r_kernels.h"
#include "pointcloud_math.h"

namespace f3r {

namespace {

constexpr int PC_LEAF = 32;   // points per bucket
constexpr int PC_FAN = 8;     // children per parent
constexpr int PC_MAX_LEVELS = 12;
constexpr int PC_STACK = 8 * PC_MAX_LEVELS;
constexpr int PC_LEVEL_SHIFT = 26;  // stack entry = level << 26 | node (n < 2^31 -> < 2^26 buckets)
constexpr int PC_THREADS = 128;

constexpr int ST = 256;           // radix sort: threads per tile
constexpr int SI = 16;            // keys per thread
constexpr int STILE = ST * SI;

size_t al256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }

// ------------------------------------------------------------------------------------------------- layout
struct Tree {
  int levels;
  int cnt[PC_MAX_LEVELS];        // nodes per level, level 0 = buckets
  long long off[PC_MAX_LEVELS];  // first node of each level
};

Tree make_tree(int n) {
  Tree t = {};
  int c = (n + PC_LEAF - 1) / PC_LEAF;
  long long off = 0;
  t.levels = 0;
  while (true) {
    t.cnt[t.levels] = c;
    t.off[t.levels] = off;
    off += c;
    ++t.levels;
    if (c <= 1) break;
    c = (c + PC_FAN - 1) / PC_FAN;
  }
  return t;
}

long long tree_nodes(const Tree& t) { return t.off[t.levels - 1] + t.cnt[t.levels - 1]; }

// Index layout (one caller-owned block): header | sorted Morton keys | sorted original indices | sorted fp64 points |
// node boxes | build scratch (second key/value buffers, low keys, tile histograms)
struct IndexLayout {
  size_t hdr, codes, perm, pts, nodes, keys_b, vals_b, lo, hist, total;
};

int sort_tiles(int n) { return (n + STILE - 1) / STILE; }

IndexLayout index_layout(int n) {
  IndexLayout l;
  const size_t N = static_cast<size_t>(n);
  const Tree t = make_tree(n);
  size_t o = 0;
  l.hdr = o; o += al256(16 * sizeof(double));
  l.codes = o; o += al256(N * 8);
  l.perm = o; o += al256(N * 4);
  l.pts = o; o += al256(N * 24);
  l.nodes = o; o += al256(static_cast<size_t>(tree_nodes(t)) * 48);
  l.keys_b = o; o += al256(N * 8);
  l.vals_b = o; o += al256(N * 4);
  l.lo = o; o += al256(N * 8);
  l.hist = o; o += al256(static_cast<size_t>(sort_tiles(n)) * 256 * 4 + 4096 * 4);
  l.total = o;
  return l;
}

struct QueryLayout {
  size_t keys_a, keys_b, vals_a, vals_b, hist, total;
};

QueryLayout query_layout(int nq) {
  QueryLayout l;
  const size_t N = static_cast<size_t>(nq);
  size_t o = 0;
  l.keys_a = o; o += al256(N * 8);
  l.keys_b = o; o += al256(N * 8);
  l.vals_a = o; o += al256(N * 4);
  l.vals_b = o; o += al256(N * 4);
  l.hist = o; o += al256(static_cast<size_t>(sort_tiles(nq)) * 256 * 4 + 4096 * 4);
  l.total = o;
  return l;
}

// header (fp64 words): [0..2] min key image, [3..5] max key image (as uint64), [6..8] origin, [9] 1 / extent
struct Header {
  unsigned long long kmin[3], kmax[3];
  double origin[3], inv_extent;
};

__device__ __forceinline__ void load_pt(const void* pts, int f64, long long i, double* p) {
  if (f64) {
    const double* s = static_cast<const double*>(pts) + 3 * i;
    p[0] = s[0]; p[1] = s[1]; p[2] = s[2];
  } else {
    const float* s = static_cast<const float*>(pts) + 3 * i;
    p[0] = s[0]; p[1] = s[1]; p[2] = s[2];
  }
}

// ------------------------------------------------------------------------------------------------- bounding box
__global__ void pc_bbox_init_kernel(Header* h) {
  if (threadIdx.x < 3) {
    h->kmin[threadIdx.x] = ~0ull;
    h->kmax[threadIdx.x] = 0ull;
  }
}

__global__ void pc_bbox_kernel(const void* pts, int f64, int n, Header* h) {
  unsigned long long mn[3] = {~0ull, ~0ull, ~0ull}, mx[3] = {0ull, 0ull, 0ull};
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    double p[3];
    load_pt(pts, f64, i, p);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const unsigned long long k = pc_dkey(p[a]);
      mn[a] = min(mn[a], k);
      mx[a] = max(mx[a], k);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = min(mn[a], __shfl_down_sync(0xffffffffu, mn[a], o));
      mx[a] = max(mx[a], __shfl_down_sync(0xffffffffu, mx[a], o));
    }
    if ((threadIdx.x & 31) == 0) {
      atomicMin(&h->kmin[a], mn[a]);
      atomicMax(&h->kmax[a], mx[a]);
    }
  }
}

__global__ void pc_bbox_finish_kernel(Header* h) {
  if (threadIdx.x != 0) return;
  double ext = 0.0;
  for (int a = 0; a < 3; ++a) {
    const double lo = pc_dkey_inv(h->kmin[a]), hi = pc_dkey_inv(h->kmax[a]);
    h->origin[a] = lo;
    ext = fmax(ext, hi - lo);
  }
  h->inv_extent = ext > 0.0 ? 1.0 / ext : 0.0;
}

// ------------------------------------------------------------------------------------------------- Morton keys
// mode 0 (index): hi keys to `hi`, lo keys to `keys`; mode 1 (queries): hi keys to `keys`
__global__ void pc_code_kernel(const void* pts, int f64, int n, const Header* h, unsigned long long* keys, int* vals,
                               unsigned long long* hi, int mode) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  double p[3];
  load_pt(pts, f64, i, p);
  uint64_t kh, kl;
  pc_morton(p, h->origin, h->inv_extent, &kh, &kl);
  if (mode == 0) {
    keys[i] = kl;
    hi[i] = kh;
  } else {
    keys[i] = kh;
  }
  vals[i] = static_cast<int>(i);
}

__global__ void pc_gather_keys_kernel(const unsigned long long* hi, const int* vals_in, unsigned long long* keys,
                                      int* vals_out, int n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int v = vals_in[i];
  keys[i] = hi[v];
  vals_out[i] = v;
}

// ------------------------------------------------------------------------------------------------- LSD radix sort
// One 8-bit digit per pass: tile histograms (digit-major), one exclusive scan over them, then a stable scatter that
// ranks each round of 256 keys with warp match + per-warp counts, so equal digits keep their input order.

// warp-collective: every thread of the warp must call it
__device__ __forceinline__ void hist_add(uint32_t* hist, bool ok, uint32_t d) {
  const unsigned act = __ballot_sync(0xffffffffu, ok);
  if (ok) {
    const unsigned peers = __match_any_sync(act, d);
    if ((__ffs(peers) - 1) == static_cast<int>(threadIdx.x & 31)) atomicAdd(&hist[d], static_cast<uint32_t>(__popc(peers)));
  }
}

__global__ void __launch_bounds__(ST) sort_hist_kernel(const unsigned long long* __restrict__ keys, int n, int shift,
                                                       uint32_t* __restrict__ hist, int tiles) {
  __shared__ uint32_t h[256];
  const int tid = threadIdx.x;
  h[tid] = 0;
  __syncthreads();
  const long long base = static_cast<long long>(blockIdx.x) * STILE;
#pragma unroll 4
  for (int r = 0; r < SI; ++r) {
    const long long i = base + r * ST + tid;
    const bool ok = i < n;
    const uint32_t d = ok ? static_cast<uint32_t>((keys[i] >> shift) & 255u) : 0u;
    hist_add(h, ok, d);
  }
  __syncthreads();
  hist[static_cast<size_t>(tid) * tiles + blockIdx.x] = h[tid];
}

constexpr int SCAN_T = 1024;

// in-place exclusive scan of m uint32 (one block)
__global__ void __launch_bounds__(SCAN_T) sort_scan_kernel(uint32_t* __restrict__ a, int m) {
  __shared__ uint32_t ws[SCAN_T / 32];
  const int tid = threadIdx.x;
  const int per = (m + SCAN_T - 1) / SCAN_T;
  const int i0 = min(m, tid * per), i1 = min(m, i0 + per);
  uint32_t s = 0;
  for (int i = i0; i < i1; ++i) s += a[i];
  // block exclusive scan of s
  uint32_t x = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if ((tid & 31) >= o) x += y;
  }
  if ((tid & 31) == 31) ws[tid >> 5] = x;
  __syncthreads();
  if (tid < 32) {
    uint32_t w = ws[tid];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, w, o);
      if (tid >= o) w += y;
    }
    ws[tid] = w;
  }
  __syncthreads();
  uint32_t run = x - s + ((tid >> 5) ? ws[(tid >> 5) - 1] : 0u);
  for (int i = i0; i < i1; ++i) {
    const uint32_t v = a[i];
    a[i] = run;
    run += v;
  }
}

__global__ void __launch_bounds__(ST) sort_scatter_kernel(const unsigned long long* __restrict__ kin,
                                                          const int* __restrict__ vin, unsigned long long* __restrict__ kout,
                                                          int* __restrict__ vout, int n, int shift,
                                                          const uint32_t* __restrict__ hist, int tiles) {
  __shared__ uint32_t base[256];
  __shared__ uint32_t wcnt[ST / 32][256];
  __shared__ uint32_t woff[ST / 32][256];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  base[tid] = hist[static_cast<size_t>(tid) * tiles + blockIdx.x];
#pragma unroll
  for (int w = 0; w < ST / 32; ++w) wcnt[w][tid] = 0;
  __syncthreads();
  const long long tile0 = static_cast<long long>(blockIdx.x) * STILE;
  for (int r = 0; r < SI; ++r) {
    const long long i = tile0 + r * ST + tid;
    const bool ok = i < n;
    unsigned long long k = 0;
    int v = 0;
    uint32_t d = 0, rank = 0;
    if (ok) {
      k = kin[i];
      v = vin[i];
      d = static_cast<uint32_t>((k >> shift) & 255u);
    }
    const unsigned act = __ballot_sync(0xffffffffu, ok);
    if (ok) {
      const unsigned peers = __match_any_sync(act, d);
      rank = __popc(peers & ((1u << lane) - 1u));
      if ((__ffs(peers) - 1) == lane) wcnt[warp][d] = __popc(peers);
    }
    __syncthreads();
    {
      uint32_t run = base[tid];
#pragma unroll
      for (int w = 0; w < ST / 32; ++w) {
        const uint32_t c = wcnt[w][tid];
        woff[w][tid] = run;
        run += c;
        wcnt[w][tid] = 0;
      }
      base[tid] = run;
    }
    __syncthreads();
    if (ok) {
      const uint32_t pos = woff[warp][d] + rank;
      kout[pos] = k;
      vout[pos] = v;
    }
  }
}

// sorts (keys, vals) by the low `bits` bits, ping-ponging between buffer 0 and 1; *in_b tells (in and out) where the
// data is
cudaError_t radix_sort(unsigned long long* k[2], int* v[2], int n, int bits, uint32_t* hist, int* in_b, cudaStream_t st) {
  const int tiles = sort_tiles(n);
  for (int shift = 0; shift < bits; shift += 8) {
    const int a = *in_b, b = 1 - a;
    cudaError_t e;
    if ((e = launch(sort_hist_kernel, tiles, ST, 0, st, false, k[a], n, shift, hist, tiles)) != cudaSuccess) return e;
    if ((e = launch(sort_scan_kernel, 1, SCAN_T, 0, st, false, hist, tiles * 256)) != cudaSuccess) return e;
    if ((e = launch(sort_scatter_kernel, tiles, ST, 0, st, false, k[a], v[a], k[b], v[b], n, shift, hist, tiles)) !=
        cudaSuccess)
      return e;
    *in_b = b;
  }
  return cudaSuccess;
}

// ------------------------------------------------------------------------------------------------- buckets and tree
__global__ void pc_gather_points_kernel(const void* pts, int f64, const int* __restrict__ perm, double* __restrict__ out,
                                        int n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  double p[3];
  load_pt(pts, f64, perm[i], p);
  out[3 * i] = p[0];
  out[3 * i + 1] = p[1];
  out[3 * i + 2] = p[2];
}

__global__ void pc_leaf_box_kernel(const double* __restrict__ pts, int n, double* __restrict__ box, int leaves) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= leaves) return;
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  const int i1 = min(n, (l + 1) * PC_LEAF);
  for (int i = l * PC_LEAF; i < i1; ++i)
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      lo[a] = fmin(lo[a], pts[3 * static_cast<size_t>(i) + a]);
      hi[a] = fmax(hi[a], pts[3 * static_cast<size_t>(i) + a]);
    }
  double* b = box + 6 * static_cast<size_t>(l);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    b[a] = lo[a];
    b[3 + a] = hi[a];
  }
}

__global__ void pc_parent_box_kernel(const double* __restrict__ child, int n_child, double* __restrict__ parent, int n_parent) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_parent) return;
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  const int c1 = min(n_child, (p + 1) * PC_FAN);
  for (int c = p * PC_FAN; c < c1; ++c)
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      lo[a] = fmin(lo[a], child[6 * static_cast<size_t>(c) + a]);
      hi[a] = fmax(hi[a], child[6 * static_cast<size_t>(c) + 3 + a]);
    }
  double* b = parent + 6 * static_cast<size_t>(p);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    b[a] = lo[a];
    b[3 + a] = hi[a];
  }
}

// ------------------------------------------------------------------------------------------------- traversal
struct IndexView {
  const unsigned long long* codes;  // sorted hi Morton keys
  const int* perm;                  // original index of each sorted point
  const double* pts;                // sorted points [n][3]
  const double* nodes;              // [nodes][6] = lo xyz, hi xyz
  const Header* hdr;
  int n;
  Tree tree;
};

IndexView index_view(const void* index, int n) {
  const IndexLayout l = index_layout(n);
  const uint8_t* b = static_cast<const uint8_t*>(index);
  IndexView v;
  v.hdr = reinterpret_cast<const Header*>(b + l.hdr);
  v.codes = reinterpret_cast<const unsigned long long*>(b + l.codes);
  v.perm = reinterpret_cast<const int*>(b + l.perm);
  v.pts = reinterpret_cast<const double*>(b + l.pts);
  v.nodes = reinterpret_cast<const double*>(b + l.nodes);
  v.n = n;
  v.tree = make_tree(n);
  return v;
}

// A lower bound on the real squared distance from q to any point of the box, with every operation rounded towards
// -inf.  A point p of the box has computed distance pc_dist2(q, p) >= real |q - p|^2 (1 - 5u) (u = 2^-53: one rounding
// per difference, square and sum), so a box whose bound times (1 - 2^-50), rounded down, is >= the current best holds
// no point that is strictly nearer than the best under scipy's arithmetic.
__device__ __forceinline__ double box_lb(const double* q, const double* box) {
  double s = 0.0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double g = fmax(0.0, fmax(__dsub_rd(box[a], q[a]), __dsub_rd(q[a], box[3 + a])));
    s = __dadd_rd(s, __dmul_rd(g, g));
  }
  return s;
}
__device__ __forceinline__ bool pruned(double lb, double best) { return __dmul_rd(lb, 1.0 - 0x1p-50) >= best; }

// Best-first-ordered depth-first search.  Visitor: `scan(bucket)` evaluates the points of a bucket, `bound()` returns
// the current pruning radius (squared, +inf while nothing bounds the search).
template <class Scan, class Bound>
__device__ __forceinline__ void traverse(const IndexView& ix, const double* q, int skip_leaf, Scan scan, Bound bound) {
  int st[PC_STACK];
  double sl[PC_STACK];
  int sp = 0;
  const int top = ix.tree.levels - 1;
  st[0] = top << PC_LEVEL_SHIFT;
  sl[0] = 0.0;
  sp = 1;
  while (sp > 0) {
    --sp;
    const int e = st[sp];
    if (pruned(sl[sp], bound())) continue;
    const int lvl = e >> PC_LEVEL_SHIFT, id = e & ((1 << PC_LEVEL_SHIFT) - 1);
    if (lvl == 0) {
      if (id != skip_leaf) scan(id);
      continue;
    }
    const int c0 = id * PC_FAN, c1 = min(c0 + PC_FAN, ix.tree.cnt[lvl - 1]);
    const double* cb = ix.nodes + 6 * ix.tree.off[lvl - 1];
    // children sorted by bound, the nearest pushed last so that it is popped first
    int ci[PC_FAN];
    double cl[PC_FAN];
    int m = 0;
    const double b = bound();
    for (int c = c0; c < c1; ++c) {
      const double lb = box_lb(q, cb + 6 * static_cast<size_t>(c));
      if (pruned(lb, b)) continue;
      int j = m++;
      while (j > 0 && cl[j - 1] < lb) {
        cl[j] = cl[j - 1];
        ci[j] = ci[j - 1];
        --j;
      }
      cl[j] = lb;
      ci[j] = ((lvl - 1) << PC_LEVEL_SHIFT) | c;
    }
    for (int j = 0; j < m; ++j) {
      st[sp] = ci[j];
      sl[sp] = cl[j];
      ++sp;
    }
  }
}

__device__ __forceinline__ int lower_bound(const unsigned long long* a, int n, unsigned long long key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(PC_THREADS) pc_nearest_kernel(IndexView ix, const void* query, int f64, int nq,
                                                                 const unsigned long long* __restrict__ qcodes,
                                                                 const int* __restrict__ qperm, double* __restrict__ dist,
                                                                 long long* __restrict__ idx) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nq) return;
  const int qi = qperm[t];
  double q[3];
  load_pt(query, f64, qi, q);
  int pos = lower_bound(ix.codes, ix.n, qcodes[t]);
  if (pos >= ix.n) pos = ix.n - 1;
  const int leaf0 = pos / PC_LEAF;
  double best = INFINITY;
  int bj = -1;
  auto scan = [&](int leaf) {
    const int i1 = min(ix.n, (leaf + 1) * PC_LEAF);
    for (int i = leaf * PC_LEAF; i < i1; ++i) {
      const double s = pc_dist2(q, ix.pts + 3 * static_cast<size_t>(i));
      if (s < best) {
        best = s;
        bj = i;
      }
    }
  };
  scan(leaf0);
  traverse(ix, q, leaf0, scan, [&]() { return best; });
  dist[qi] = bj >= 0 ? __dsqrt_rn(best) : INFINITY;  // a NaN coordinate matches nothing: scipy rejects such input
  idx[qi] = bj >= 0 ? ix.perm[bj] : ix.n;
}

__global__ void pc_fill_empty_kernel(int nq, int n_ref, double* dist, long long* idx) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= nq) return;
  dist[i] = INFINITY;
  idx[i] = n_ref;
}

// k nearest of every indexed point (itself included) in a bounded max-heap, then the normal of that neighbourhood
__global__ void __launch_bounds__(PC_THREADS) pc_knn_normals_kernel(IndexView ix, int k, double* __restrict__ normals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ix.n) return;
  double q[3] = {ix.pts[3 * static_cast<size_t>(i)], ix.pts[3 * static_cast<size_t>(i) + 1],
                 ix.pts[3 * static_cast<size_t>(i) + 2]};
  double hs[32];
  int hj[32];
  int m = 0;
  auto push = [&](double s, int j) {
    if (m < k) {  // sift up
      int c = m++;
      while (c > 0) {
        const int p = (c - 1) >> 1;
        if (hs[p] >= s) break;
        hs[c] = hs[p];
        hj[c] = hj[p];
        c = p;
      }
      hs[c] = s;
      hj[c] = j;
    } else if (s < hs[0]) {  // replace the farthest, sift down
      int c = 0;
      while (true) {
        int l = 2 * c + 1;
        if (l >= m) break;
        if (l + 1 < m && hs[l + 1] > hs[l]) ++l;
        if (hs[l] <= s) break;
        hs[c] = hs[l];
        hj[c] = hj[l];
        c = l;
      }
      hs[c] = s;
      hj[c] = j;
    }
  };
  auto scan = [&](int leaf) {
    const int i1 = min(ix.n, (leaf + 1) * PC_LEAF);
    for (int j = leaf * PC_LEAF; j < i1; ++j) push(pc_dist2(q, ix.pts + 3 * static_cast<size_t>(j)), j);
  };
  const int leaf0 = i / PC_LEAF;
  scan(leaf0);
  traverse(ix, q, leaf0, scan, [&]() { return m < k ? INFINITY : hs[0]; });
  double nrm[3];
  pc_neighbourhood_normal([&](int a) { return ix.pts + 3 * static_cast<size_t>(hj[a]); }, m, nrm);
  double* o = normals + 3 * static_cast<size_t>(ix.perm[i]);
  o[0] = nrm[0];
  o[1] = nrm[1];
  o[2] = nrm[2];
}

// ------------------------------------------------------------------------------------------------- reductions
constexpr int RED_BLOCKS = 256, RED_T = 256;

__global__ void __launch_bounds__(RED_T) f64_sum_kernel(const double* __restrict__ x, int n, double* __restrict__ part) {
  __shared__ double ws[RED_T / 32];
  double s = 0.0;
  for (long long i = blockIdx.x * static_cast<long long>(RED_T) + threadIdx.x; i < n; i += static_cast<long long>(RED_BLOCKS) * RED_T)
    s += x[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < RED_T / 32; ++w) t += ws[w];
    part[blockIdx.x] = t;
  }
}

__global__ void f64_mean_final_kernel(const double* __restrict__ part, int n, double* __restrict__ out) {
  if (threadIdx.x != 0) return;
  double t = 0.0;
  for (int b = 0; b < RED_BLOCKS; ++b) t += part[b];
  *out = n > 0 ? t / n : NAN;
}

// exact order statistic: 8 passes of an 8-bit radix select on the order-preserving 64-bit image.  pc_dkey puts a NaN
// above +inf (sign clear) or below -inf (sign set); numpy.median returns NaN if any element is NaN, so the first pass
// flags such keys and the result is NaN.
struct SelState {
  unsigned long long prefix, mask, min_gt;
  unsigned int k, cnt_le, nan;
};
constexpr unsigned long long KEY_PINF = 0xfff0000000000000ull;  // pc_dkey(+inf)
constexpr unsigned long long KEY_NINF = 0x000fffffffffffffull;  // pc_dkey(-inf)

__global__ void sel_init_kernel(SelState* s, uint32_t* hist, int k) {
  hist[threadIdx.x] = 0;
  if (threadIdx.x == 0) {
    s->prefix = 0;
    s->mask = 0;
    s->k = static_cast<unsigned>(k);
    s->min_gt = ~0ull;
    s->cnt_le = 0;
    s->nan = 0;
  }
}

__global__ void __launch_bounds__(RED_T) sel_hist_kernel(const double* __restrict__ x, int n, SelState* __restrict__ s,
                                                         uint32_t* __restrict__ hist, int shift) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const unsigned long long prefix = s->prefix, mask = s->mask;
  const long long stride = static_cast<long long>(gridDim.x) * RED_T;
  const long long n_round = (n + stride - 1) / stride * stride;  // every thread of a warp runs every iteration
  bool nan = false;
  for (long long i = blockIdx.x * static_cast<long long>(RED_T) + threadIdx.x; i < n_round; i += stride) {
    bool ok = i < n;
    unsigned long long u = ok ? pc_dkey(x[i]) : 0ull;
    nan |= ok && (u > KEY_PINF || u < KEY_NINF);
    ok = ok && (u & mask) == prefix;
    hist_add(h, ok, static_cast<uint32_t>((u >> shift) & 255u));
  }
  if (shift == 56 && __any_sync(0xffffffffu, nan) && (threadIdx.x & 31) == 0) s->nan = 1;
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], h[threadIdx.x]);
}

__global__ void sel_digit_kernel(SelState* s, uint32_t* hist, int shift) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = hist[threadIdx.x];
  hist[threadIdx.x] = 0;
  __syncthreads();
  if (threadIdx.x != 0) return;
  uint32_t cum = 0;
  int d = 0;
  for (; d < 255; ++d) {
    if (cum + h[d] > s->k) break;
    cum += h[d];
  }
  s->prefix |= static_cast<unsigned long long>(d) << shift;
  s->mask |= 255ull << shift;
  s->k -= cum;
}

__global__ void __launch_bounds__(RED_T) sel_succ_kernel(const double* __restrict__ x, int n, SelState* s) {
  const unsigned long long a = s->prefix;
  unsigned int cnt = 0;
  unsigned long long mn = ~0ull;
  for (long long i = blockIdx.x * static_cast<long long>(RED_T) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * RED_T) {
    const unsigned long long u = pc_dkey(x[i]);
    if (u <= a) ++cnt;
    else mn = min(mn, u);
  }
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_down_sync(0xffffffffu, cnt, o);
    mn = min(mn, __shfl_down_sync(0xffffffffu, mn, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&s->cnt_le, cnt);
    atomicMin(&s->min_gt, mn);
  }
}

// numpy.median: the middle order statistic, or the mean (a + b) / 2 of the two middle ones; NaN if any element is NaN
__global__ void sel_final_kernel(const SelState* s, int n, double* out) {
  if (threadIdx.x != 0) return;
  if (s->nan) {
    *out = NAN;
    return;
  }
  const double a = pc_dkey_inv(s->prefix);
  if (n & 1) {
    *out = a;
    return;
  }
  const double b = (static_cast<unsigned>(n / 2) < s->cnt_le) ? a : pc_dkey_inv(s->min_gt);
  *out = __ddiv_rn(__dadd_rn(a, b), 2.0);
}

__global__ void __launch_bounds__(RED_T) f64_count_below_kernel(const double* __restrict__ x, int n,
                                                                const double* __restrict__ th, unsigned long long* count) {
  const double t = *th;
  unsigned int c = 0;
  for (long long i = blockIdx.x * static_cast<long long>(RED_T) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * RED_T)
    c += x[i] < t;
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, static_cast<unsigned long long>(c));
}

__global__ void pc_count_nonfinite_kernel(const void* pts, int f64, long long count, unsigned int* out) {
  unsigned int c = 0;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < count;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const double v = f64 ? static_cast<const double*>(pts)[i] : static_cast<double>(static_cast<const float*>(pts)[i]);
    c += !isfinite(v);
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

// |a[ia] . b[ib]| with numpy's rounding: products, then (p0 + p1) + p2
__global__ void pc_abs_dot_kernel(const double* __restrict__ a, const long long* __restrict__ a_idx,
                                  const double* __restrict__ b, const long long* __restrict__ b_idx, int n,
                                  double* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const double* pa = a + 3 * (a_idx ? a_idx[i] : i);
  const double* pb = b + 3 * (b_idx ? b_idx[i] : i);
  const double s = __dadd_rn(__dadd_rn(__dmul_rn(pa[0], pb[0]), __dmul_rn(pa[1], pb[1])), __dmul_rn(pa[2], pb[2]));
  out[i] = fabs(s);
}

}  // namespace

// ------------------------------------------------------------------------------------------------- launchers
size_t pc_index_workspace(int n) { return index_layout(n).total; }
size_t pc_query_workspace(int nq) { return query_layout(nq).total; }
size_t f64_reduce_workspace() { return al256(sizeof(SelState)) + al256(256 * 4) + al256(RED_BLOCKS * 8); }

cudaError_t launch_pc_index_build(const void* pts, int f64, int n, void* index, cudaStream_t st) {
  const IndexLayout l = index_layout(n);
  uint8_t* b = static_cast<uint8_t*>(index);
  Header* h = reinterpret_cast<Header*>(b + l.hdr);
  unsigned long long* k[2] = {reinterpret_cast<unsigned long long*>(b + l.codes),
                              reinterpret_cast<unsigned long long*>(b + l.keys_b)};
  int* v[2] = {reinterpret_cast<int*>(b + l.perm), reinterpret_cast<int*>(b + l.vals_b)};
  unsigned long long* hi = reinterpret_cast<unsigned long long*>(b + l.lo);
  uint32_t* hist = reinterpret_cast<uint32_t*>(b + l.hist);
  const int g = (n + 255) / 256;
  cudaError_t e;
  if ((e = launch(pc_bbox_init_kernel, 1, 32, 0, st, false, h)) != cudaSuccess) return e;
  if ((e = launch(pc_bbox_kernel, min(g, 1024), 256, 0, st, false, pts, f64, n, h)) != cudaSuccess) return e;
  if ((e = launch(pc_bbox_finish_kernel, 1, 32, 0, st, false, h)) != cudaSuccess) return e;
  if ((e = launch(pc_code_kernel, g, 256, 0, st, false, pts, f64, n, h, k[0], v[0], hi, 0)) != cudaSuccess) return e;
  int in_b = 0;
  if ((e = radix_sort(k, v, n, 36, hist, &in_b, st)) != cudaSuccess) return e;  // low 12 bits per axis (5 passes)
  if ((e = launch(pc_gather_keys_kernel, g, 256, 0, st, false, hi, v[in_b], k[1 - in_b], v[1 - in_b], n)) != cudaSuccess)
    return e;
  in_b = 1 - in_b;
  if ((e = radix_sort(k, v, n, 63, hist, &in_b, st)) != cudaSuccess) return e;  // 63-bit code (8 passes)
  // 13 passes in all: the sorted keys and permutation end where the index keeps them (buffer 0)
  double* pts_s = reinterpret_cast<double*>(b + l.pts);
  if ((e = launch(pc_gather_points_kernel, g, 256, 0, st, false, pts, f64, v[0], pts_s, n)) != cudaSuccess) return e;
  const Tree t = make_tree(n);
  double* nodes = reinterpret_cast<double*>(b + l.nodes);
  if ((e = launch(pc_leaf_box_kernel, (t.cnt[0] + 127) / 128, 128, 0, st, false, pts_s, n, nodes, t.cnt[0])) != cudaSuccess)
    return e;
  for (int lv = 1; lv < t.levels; ++lv)
    if ((e = launch(pc_parent_box_kernel, (t.cnt[lv] + 127) / 128, 128, 0, st, false, nodes + 6 * t.off[lv - 1],
                    t.cnt[lv - 1], nodes + 6 * t.off[lv], t.cnt[lv])) != cudaSuccess)
      return e;
  return cudaSuccess;
}

cudaError_t launch_pc_nearest(const void* index, int n_ref, const void* query, int f64, int nq, double* dist,
                              long long* idx, void* workspace, cudaStream_t st) {
  if (n_ref == 0) return launch(pc_fill_empty_kernel, (nq + 255) / 256, 256, 0, st, false, nq, n_ref, dist, idx);
  const IndexView ix = index_view(index, n_ref);
  const QueryLayout l = query_layout(nq);
  uint8_t* w = static_cast<uint8_t*>(workspace);
  unsigned long long* k[2] = {reinterpret_cast<unsigned long long*>(w + l.keys_a),
                              reinterpret_cast<unsigned long long*>(w + l.keys_b)};
  int* v[2] = {reinterpret_cast<int*>(w + l.vals_a), reinterpret_cast<int*>(w + l.vals_b)};
  uint32_t* hist = reinterpret_cast<uint32_t*>(w + l.hist);
  cudaError_t e;
  if ((e = launch(pc_code_kernel, (nq + 255) / 256, 256, 0, st, false, query, f64, nq, ix.hdr, k[0], v[0], nullptr, 1)) !=
      cudaSuccess)
    return e;
  int in_b = 0;
  if ((e = radix_sort(k, v, nq, 63, hist, &in_b, st)) != cudaSuccess) return e;
  return launch(pc_nearest_kernel, (nq + PC_THREADS - 1) / PC_THREADS, PC_THREADS, 0, st, false, ix, query, f64, nq,
                k[in_b], v[in_b], dist, idx);
}

cudaError_t launch_pc_knn_normals(const void* index, int n, int k, double* normals, cudaStream_t st) {
  const IndexView ix = index_view(index, n);
  return launch(pc_knn_normals_kernel, (n + PC_THREADS - 1) / PC_THREADS, PC_THREADS, 0, st, false, ix, k, normals);
}

cudaError_t launch_pc_count_nonfinite(const void* pts, int f64, int n, unsigned int* count, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(count, 0, sizeof(unsigned int), st);
  if (e != cudaSuccess) return e;
  const long long c = 3ll * n;
  if (c == 0) return cudaSuccess;
  return launch(pc_count_nonfinite_kernel, static_cast<int>(min(1024ll, (c + 255) / 256)), 256, 0, st, false, pts, f64, c,
                count);
}

cudaError_t launch_pc_abs_dot(const double* a, const long long* a_idx, const double* b, const long long* b_idx, int n,
                              double* out, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  return launch(pc_abs_dot_kernel, (n + 255) / 256, 256, 0, st, false, a, a_idx, b, b_idx, n, out);
}

cudaError_t launch_f64_mean(const double* x, int n, double* out, void* workspace, cudaStream_t st) {
  double* part = reinterpret_cast<double*>(static_cast<uint8_t*>(workspace) + al256(sizeof(SelState)) + al256(256 * 4));
  const cudaError_t e = launch(f64_sum_kernel, RED_BLOCKS, RED_T, 0, st, false, x, n, part);
  if (e != cudaSuccess) return e;
  return launch(f64_mean_final_kernel, 1, 32, 0, st, false, part, n, out);
}

cudaError_t launch_f64_median(const double* x, int n, double* out, void* workspace, cudaStream_t st) {
  SelState* s = static_cast<SelState*>(workspace);
  uint32_t* hist = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(workspace) + al256(sizeof(SelState)));
  const int k = (n - 1) / 2;  // odd n: the middle; even n: the lower middle, its successor below
  const int g = min(1024, (n + RED_T - 1) / RED_T);
  cudaError_t e;
  if ((e = launch(sel_init_kernel, 1, 256, 0, st, false, s, hist, k)) != cudaSuccess) return e;
  for (int shift = 56; shift >= 0; shift -= 8) {
    if ((e = launch(sel_hist_kernel, g, RED_T, 0, st, false, x, n, s, hist, shift)) != cudaSuccess) return e;
    if ((e = launch(sel_digit_kernel, 1, 256, 0, st, false, s, hist, shift)) != cudaSuccess) return e;
  }
  if (!(n & 1) && (e = launch(sel_succ_kernel, g, RED_T, 0, st, false, x, n, s)) != cudaSuccess) return e;
  return launch(sel_final_kernel, 1, 32, 0, st, false, s, n, out);
}

cudaError_t launch_f64_count_below(const double* x, int n, const double* th, unsigned long long* count, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(count, 0, sizeof(unsigned long long), st);
  if (e != cudaSuccess || n == 0) return e;
  return launch(f64_count_below_kernel, min(1024, (n + RED_T - 1) / RED_T), RED_T, 0, st, false, x, n, th, count);
}

}  // namespace f3r
