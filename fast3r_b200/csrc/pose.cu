// Camera poses (fast_pnp, fast3r/dust3r/cloud_opt/init_im_poses.py:300-350): the per-point work of OpenCV's
// solvePnPRansac, the rest of which (sampling, EPnP hypotheses, bookkeeping, the SQPnP refit) runs on the host
// (fast3r_b200/poses.py):
//   pnp_gather   the masked points of every view and their pixel_grid coordinates, in numpy boolean-index order
//   pnp_score    inlier counts of a table of hypotheses: |pixel - projectPoints(point)|^2 <= thr^2 in OpenCV's
//                arithmetic (pose_math.h) over every point of the hypothesis' view
//   pnp_inliers  the inliers of one hypothesis per row of a table, compacted in index order (compressElems)
// Counts are integers and compactions are stable prefix sums, so every result is exact and independent of scheduling.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "f3r_kernels.h"
#include "pose_math.h"

namespace f3r {

namespace {

constexpr int CT = 256;        // threads per compaction CTA
constexpr int CPT = 4;         // consecutive elements per thread
constexpr int CB = CT * CPT;   // elements per compaction block
constexpr int ST = 256;        // threads per scoring CTA
constexpr int SPT = 4;         // points per thread of a scoring CTA (strided by ST)
constexpr int STILE = ST * SPT;
constexpr int SHB = 32;        // hypotheses per scoring chunk (one CTA row)
constexpr int SCAN_T = 1024;

enum { SEL_CONF = 0, SEL_MASK = 1, SEL_INLIER = 2 };

// threshold of squared error: findInliers' (float)(thresh * thresh)
float thr_sq(float thr) { return static_cast<float>(static_cast<double>(thr) * static_cast<double>(thr)); }

size_t al256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }

// One compaction "row": the inputs are elements [in_off, in_off + count) and the selected ones go to out_off on.
struct Row {
  long long in_off, out_off;
  int count, view;
};

struct CompactArgs {
  int mode;
  // gather (SEL_CONF / SEL_MASK): view v reads pts/conf/mask at v n and writes at v n
  const float* pts;
  const float* conf;
  const uint8_t* mask;
  int n, w;
  // inliers (SEL_INLIER): compacted points/pixels, one row and hypothesis per blockIdx.y
  const float* ipts;
  const float* ipix;
  const Row* rows;
  const f3r_pnp_hyp* hyps;
  float thr2;
  int* bcnt;  // [rows][nb] selected per block, scanned in place into block offsets
  int nb;
  float* out_pts;
  float* out_pix;
  int* counts;  // [rows]
};

__device__ __forceinline__ bool inlier(const f3r_pnp_hyp& h, const float* p, const float* q, float thr2) {
  float u, v;
  pnp_project(h.r, h.t, h.fx, h.fy, h.cx, h.cy, p[0], p[1], p[2], &u, &v);
  return pnp_error(q[0], q[1], u, v) <= thr2;
}

// selection flags of elements e0 .. e0 + CPT - 1 of row `row` (bit j = element e0 + j)
__device__ __forceinline__ unsigned select_bits(const CompactArgs& a, int row, int e0, int count) {
  unsigned bits = 0;
#pragma unroll
  for (int j = 0; j < CPT; ++j) {
    const int e = e0 + j;
    if (e >= count) break;
    bool s;
    if (a.mode == SEL_CONF) {
      s = a.conf[static_cast<size_t>(row) * a.n + e] > 1.0f;
    } else if (a.mode == SEL_MASK) {
      s = a.mask[static_cast<size_t>(row) * a.n + e] != 0;
    } else {
      const Row r = a.rows[row];
      s = inlier(a.hyps[row], a.ipts + 3 * (r.in_off + e), a.ipix + 2 * (r.in_off + e), a.thr2);
    }
    bits |= static_cast<unsigned>(s) << j;
  }
  return bits;
}

__device__ __forceinline__ int row_count(const CompactArgs& a, int row) {
  return a.mode == SEL_INLIER ? a.rows[row].count : a.n;
}

// exclusive prefix of `x` over the CTA (CT threads) and the CTA total
__device__ __forceinline__ int block_exclusive(int x, int* total) {
  __shared__ int warp_sum[CT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = x;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += y;
  }
  if (lane == 31) warp_sum[wid] = inc;
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int i = 0; i < CT / 32; ++i) {
    before += i < wid ? warp_sum[i] : 0;
    all += warp_sum[i];
  }
  *total = all;
  return before + inc - x;
}

__global__ void __launch_bounds__(CT) compact_count_kernel(CompactArgs a) {
  const int row = blockIdx.y, blk = blockIdx.x;
  if (blk >= a.nb) return;
  const int count = row_count(a, row);
  const unsigned bits = select_bits(a, row, blk * CB + threadIdx.x * CPT, count);
  int total;
  block_exclusive(__popc(bits), &total);
  if (threadIdx.x == 0) a.bcnt[static_cast<size_t>(row) * a.nb + blk] = total;
}

// per row: exclusive scan of the nb block counts in place, and the row total
__global__ void __launch_bounds__(SCAN_T) compact_scan_kernel(int* bcnt, int nb, int* counts) {
  __shared__ int warp_sum[SCAN_T / 32];
  int* c = bcnt + static_cast<size_t>(blockIdx.x) * nb;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int carry = 0;
  for (int base = 0; base < nb; base += SCAN_T) {
    const int i = base + threadIdx.x;
    const int x = i < nb ? c[i] : 0;
    int inc = x;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += y;
    }
    if (lane == 31) warp_sum[wid] = inc;
    __syncthreads();
    int before = 0, all = 0;
    for (int k = 0; k < SCAN_T / 32; ++k) {
      before += k < wid ? warp_sum[k] : 0;
      all += warp_sum[k];
    }
    if (i < nb) c[i] = carry + before + inc - x;
    carry += all;
    __syncthreads();  // warp_sum is rewritten by the next chunk
  }
  if (threadIdx.x == 0) counts[blockIdx.x] = carry;
}

__global__ void __launch_bounds__(CT) compact_scatter_kernel(CompactArgs a) {
  const int row = blockIdx.y, blk = blockIdx.x;
  if (blk >= a.nb) return;
  const int count = row_count(a, row);
  const int e0 = blk * CB + threadIdx.x * CPT;
  unsigned bits = select_bits(a, row, e0, count);
  int total;
  int pos = block_exclusive(__popc(bits), &total) + a.bcnt[static_cast<size_t>(row) * a.nb + blk];
  const long long out0 = a.mode == SEL_INLIER ? a.rows[row].out_off : static_cast<long long>(row) * a.n;
  const long long in0 = a.mode == SEL_INLIER ? a.rows[row].in_off : static_cast<long long>(row) * a.n;
  const float* src_pts = a.mode == SEL_INLIER ? a.ipts : a.pts;
  for (; bits; bits &= bits - 1) {
    const int e = e0 + __ffs(bits) - 1;
    const long long o = out0 + pos++;
    const long long i = in0 + e;
    a.out_pts[3 * o] = src_pts[3 * i];
    a.out_pts[3 * o + 1] = src_pts[3 * i + 1];
    a.out_pts[3 * o + 2] = src_pts[3 * i + 2];
    if (a.mode == SEL_INLIER) {
      a.out_pix[2 * o] = a.ipix[2 * i];
      a.out_pix[2 * o + 1] = a.ipix[2 * i + 1];
    } else {  // pixel_grid(H, W)[y, x] = (x, y)
      a.out_pix[2 * o] = static_cast<float>(e % a.w);
      a.out_pix[2 * o + 1] = static_cast<float>(e / a.w);
    }
  }
}

cudaError_t run_compaction(const CompactArgs& a, int rows, cudaStream_t st) {
  if (a.nb == 0) return cudaMemsetAsync(a.counts, 0, sizeof(int) * rows, st);
  cudaError_t e;
  const dim3 grid(a.nb, rows);
  if ((e = launch(compact_count_kernel, grid, CT, 0, st, false, a)) != cudaSuccess) return e;
  if ((e = launch(compact_scan_kernel, rows, SCAN_T, 0, st, false, a.bcnt, a.nb, a.counts)) != cudaSuccess) return e;
  return launch(compact_scatter_kernel, grid, CT, 0, st, false, a);
}

// ---------------------------------------------------------------------------------------------------------- scoring
struct Chunk {
  int row0, row1, view, tiles;
};

// CTA (tile, chunk): the chunk's hypotheses (all of one view) against STILE points of that view.  Points stay in
// registers for the whole chunk; each warp's count per hypothesis goes to shared memory, each CTA's to the output.
__global__ void __launch_bounds__(ST) pnp_score_kernel(const float* __restrict__ pts, const float* __restrict__ pix,
                                                       const Row* __restrict__ views, const f3r_pnp_hyp* __restrict__ hyps,
                                                       const Chunk* __restrict__ chunks, float thr2, int* __restrict__ counts) {
  __shared__ f3r_pnp_hyp sh[SHB];
  __shared__ int scnt[SHB];
  const Chunk ch = chunks[blockIdx.y];
  if (static_cast<int>(blockIdx.x) >= ch.tiles) return;
  const Row vw = views[ch.view];
  const int nh = ch.row1 - ch.row0;
  for (int i = threadIdx.x; i < nh * static_cast<int>(sizeof(f3r_pnp_hyp) / 8); i += ST)
    reinterpret_cast<double*>(sh)[i] = reinterpret_cast<const double*>(hyps + ch.row0)[i];
  if (threadIdx.x < SHB) scnt[threadIdx.x] = 0;
  float X[SPT], Y[SPT], Z[SPT], U[SPT], V[SPT];
  bool ok[SPT];
#pragma unroll
  for (int k = 0; k < SPT; ++k) {
    const int e = blockIdx.x * STILE + k * ST + threadIdx.x;
    ok[k] = e < vw.count;
    const long long i = vw.in_off + (ok[k] ? e : 0);
    X[k] = ok[k] ? pts[3 * i] : 0.f;
    Y[k] = ok[k] ? pts[3 * i + 1] : 0.f;
    Z[k] = ok[k] ? pts[3 * i + 2] : 0.f;
    U[k] = ok[k] ? pix[2 * i] : 0.f;
    V[k] = ok[k] ? pix[2 * i + 1] : 0.f;
  }
  __syncthreads();
  for (int h = 0; h < nh; ++h) {
    const f3r_pnp_hyp& hp = sh[h];
    int c = 0;
#pragma unroll
    for (int k = 0; k < SPT; ++k) {
      if (!ok[k]) continue;
      float u, v;
      pnp_project(hp.r, hp.t, hp.fx, hp.fy, hp.cx, hp.cy, X[k], Y[k], Z[k], &u, &v);
      c += pnp_error(U[k], V[k], u, v) <= thr2;
    }
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&scnt[h], c);
  }
  __syncthreads();
  if (static_cast<int>(threadIdx.x) < nh && scnt[threadIdx.x]) atomicAdd(&counts[ch.row0 + threadIdx.x], scnt[threadIdx.x]);
}

}  // namespace

size_t pnp_gather_workspace(int views, int n) { return sizeof(int) * static_cast<size_t>(views) * ((n + CB - 1) / CB); }

cudaError_t launch_pnp_gather(const float* pts, const float* conf, const uint8_t* mask, int views, int h, int w,
                              float* out_pts, float* out_pix, int* counts, void* workspace, cudaStream_t st) {
  CompactArgs a{};
  a.mode = mask ? SEL_MASK : SEL_CONF;
  a.pts = pts;
  a.conf = conf;
  a.mask = mask;
  a.n = h * w;
  a.w = w;
  a.bcnt = static_cast<int*>(workspace);
  a.nb = (a.n + CB - 1) / CB;
  a.out_pts = out_pts;
  a.out_pix = out_pix;
  a.counts = counts;
  return run_compaction(a, views, st);
}

size_t pnp_score_workspace(int views, int nh) {
  return al256(sizeof(Row) * views) + al256(sizeof(f3r_pnp_hyp) * static_cast<size_t>(nh)) +
         al256(sizeof(Chunk) * static_cast<size_t>(nh));
}

cudaError_t launch_pnp_score(const float* pts, const float* pix, const long long* offsets, const int* counts_in, int views,
                             const f3r_pnp_hyp* hyps, int nh, float thr, int* counts, void* workspace, cudaStream_t st) {
  // host tables: views, then the hypotheses, then the chunks (runs of at most SHB rows of one view)
  const size_t o_h = al256(sizeof(Row) * views), o_c = o_h + al256(sizeof(f3r_pnp_hyp) * static_cast<size_t>(nh));
  std::vector<char> host(o_c + sizeof(Chunk) * static_cast<size_t>(nh));
  Row* vt = reinterpret_cast<Row*>(host.data());
  for (int v = 0; v < views; ++v) vt[v] = Row{offsets[v], 0, counts_in[v], v};
  memcpy(host.data() + o_h, hyps, sizeof(f3r_pnp_hyp) * static_cast<size_t>(nh));
  Chunk* ch = reinterpret_cast<Chunk*>(host.data() + o_c);
  int nc = 0;
  for (int r = 0; r < nh;) {
    const int v = hyps[r].view;
    int r1 = r + 1;
    while (r1 < nh && r1 - r < SHB && hyps[r1].view == v) ++r1;
    ch[nc++] = Chunk{r, r1, v, (counts_in[v] + STILE - 1) / STILE};
    r = r1;
  }
  char* dev = static_cast<char*>(workspace);
  cudaError_t e;
  if ((e = cudaMemcpyAsync(dev, host.data(), o_c + sizeof(Chunk) * nc, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(counts, 0, sizeof(int) * static_cast<size_t>(nh), st)) != cudaSuccess) return e;
  const float thr2 = thr_sq(thr);
  for (int c0 = 0; c0 < nc; c0 += 65535) {  // grid.y limit: one launch per 65535 chunks
    const int c1 = c0 + 65535 < nc ? c0 + 65535 : nc;
    int tiles = 0;
    for (int c = c0; c < c1; ++c) tiles = ch[c].tiles > tiles ? ch[c].tiles : tiles;
    if (tiles == 0) continue;
    if ((e = launch(pnp_score_kernel, dim3(tiles, c1 - c0), ST, 0, st, false, pts, pix,
                    reinterpret_cast<const Row*>(dev), reinterpret_cast<const f3r_pnp_hyp*>(dev + o_h),
                    reinterpret_cast<const Chunk*>(dev + o_c) + c0, thr2, counts)) != cudaSuccess)
      return e;
  }
  return cudaSuccess;
}

size_t pnp_inliers_workspace(int nh, int max_count) {
  return al256(sizeof(Row) * static_cast<size_t>(nh)) + al256(sizeof(f3r_pnp_hyp) * static_cast<size_t>(nh)) +
         sizeof(int) * static_cast<size_t>(nh) * ((max_count + CB - 1) / CB);
}

cudaError_t launch_pnp_inliers(const float* pts, const float* pix, const long long* offsets, const int* counts_in,
                               const f3r_pnp_hyp* hyps, int nh, float thr, float* out_pts, float* out_pix, int* counts,
                               void* workspace, cudaStream_t st) {
  const size_t o_h = al256(sizeof(Row) * static_cast<size_t>(nh));
  const size_t o_b = o_h + al256(sizeof(f3r_pnp_hyp) * static_cast<size_t>(nh));
  std::vector<char> host(o_b);
  Row* rows = reinterpret_cast<Row*>(host.data());
  long long out = 0;
  int max_count = 0;
  for (int r = 0; r < nh; ++r) {  // row r's inliers start where row r - 1's candidates (all its view's points) end
    const int v = hyps[r].view;
    rows[r] = Row{offsets[v], out, counts_in[v], v};
    out += counts_in[v];
    max_count = counts_in[v] > max_count ? counts_in[v] : max_count;
  }
  memcpy(host.data() + o_h, hyps, sizeof(f3r_pnp_hyp) * static_cast<size_t>(nh));
  char* dev = static_cast<char*>(workspace);
  cudaError_t e;
  if ((e = cudaMemcpyAsync(dev, host.data(), o_b, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
  CompactArgs a{};
  a.mode = SEL_INLIER;
  a.ipts = pts;
  a.ipix = pix;
  a.rows = reinterpret_cast<const Row*>(dev);
  a.hyps = reinterpret_cast<const f3r_pnp_hyp*>(dev + o_h);
  a.thr2 = thr_sq(thr);
  a.bcnt = reinterpret_cast<int*>(dev + o_b);
  a.nb = (max_count + CB - 1) / CB;
  a.out_pts = out_pts;
  a.out_pix = out_pix;
  a.counts = counts;
  return run_compaction(a, nh, st);
}

}  // namespace f3r
