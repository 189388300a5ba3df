// Image ingest on the GPU (SURVEY.md §8 f3): the resize / crop / normalise arithmetic of the reference's load_images()
// (fast3r/dust3r/utils/image.py:68-159) on decoded 8-bit RGB images, bit-exact with the CPU path it replaces:
//   PIL.Image.resize(new_size, LANCZOS | BICUBIC)  ->  center crop  ->  torchvision ToTensor + Normalize(0.5, 0.5).
// The resize is Pillow's two-pass 8-bit resampler (third-party dependency of the reference, restated from its published
// algorithm, libImaging/Resample.c): per output coordinate a window of taps with double-precision weights normalised to 1
// and rounded to 22 fractional bits (host side, resample_coeffs below), integer accumulation from 1 << 21,
// (acc >> 22) clamped to 0..255; horizontal pass into an 8-bit intermediate image, then the vertical pass.
// HBM-bound byte/integer work: one read of the source image (36 MB for a 12-Mpixel photo), 8-bit intermediate, fp32
// output written once, coalesced, in the (3, H, W) layout the patch-embed im2col reads.
#include <cmath>

#include "common.cuh"
#include "f3r_kernels.h"

namespace f3r {

constexpr int ING_PREC = 32 - 8 - 2;
constexpr int ING_COLS = 64;  // output columns per block (horizontal pass)
constexpr int ING_ROWS = 8;   // rows per block

__device__ __forceinline__ uint8_t ing_clip8(int v) {
  v >>= ING_PREC;
  return static_cast<uint8_t>(min(max(v, 0), 255));
}

// ---- horizontal pass: src [h][w][3] u8 -> dst [h][ow][3] u8.  Block = 64 output columns x ING_ROWS_PER_BLOCK rows, walked
// 8 rows at a time; the taps of the 64 columns ([k][col], conflict-free) are staged in shared memory once per block, the
// source spans of 8 rows per step (4-byte aligned, coalesced word loads).
constexpr int ING_ROWS_PER_BLOCK = 32;
__global__ void __launch_bounds__(ING_COLS* ING_ROWS)
resize_h_kernel(const uint8_t* __restrict__ src, int h, int w, uint8_t* __restrict__ dst, int ow,
                const int32_t* __restrict__ bounds, const int32_t* __restrict__ kk, int ksize, int span_max) {
  extern __shared__ int32_t ing_smem[];
  int32_t* sk = ing_smem;                                                 // [ksize][ING_COLS]
  uint8_t* sp = reinterpret_cast<uint8_t*>(ing_smem + ksize * ING_COLS);  // [ING_ROWS][span_pad]
  const int c0 = blockIdx.x * ING_COLS, yb = blockIdx.y * ING_ROWS_PER_BLOCK;
  const int tx = threadIdx.x % ING_COLS, ty = threadIdx.x / ING_COLS;
  const int ncols = min(ING_COLS, ow - c0);
  const int x_lo = __ldg(bounds + 2 * c0);                               // first source pixel of the block
  const int last = c0 + ncols - 1;
  const int x_hi = __ldg(bounds + 2 * last) + __ldg(bounds + 2 * last + 1);  // one past the last source pixel
  const int span_pad = ((span_max * 3 + 3) & ~3) + 4;                    // (+4: room for the alignment shift)
  for (int i = threadIdx.x; i < ksize * ING_COLS; i += blockDim.x) {
    const int k = i / ING_COLS, c = i % ING_COLS;
    sk[i] = c < ncols ? __ldg(kk + static_cast<size_t>(c0 + c) * ksize + k) : 0;
  }
  const bool active = tx < ncols;
  const int xmin = active ? __ldg(bounds + 2 * (c0 + tx)) - x_lo : 0, n = active ? __ldg(bounds + 2 * (c0 + tx) + 1) : 0;
  for (int y0 = yb; y0 < min(yb + ING_ROWS_PER_BLOCK, h); y0 += ING_ROWS) {
    __syncthreads();  // taps staged / previous step's spans consumed
    for (int r = 0; r < ING_ROWS; ++r) {
      const int y = y0 + r;
      if (y >= h) break;
      // bytes [b0, b1) of the image, fetched as aligned 32-bit words [a0, a1)
      const size_t b0 = (static_cast<size_t>(y) * w + x_lo) * 3, b1 = (static_cast<size_t>(y) * w + x_hi) * 3;
      const size_t a0 = b0 & ~static_cast<size_t>(3);
      const size_t total = static_cast<size_t>(h) * w * 3;
      const int nwords = static_cast<int>((b1 - a0 + 3) >> 2);
      uint32_t* dstw = reinterpret_cast<uint32_t*>(sp + r * span_pad);
      for (int i = threadIdx.x; i < nwords; i += blockDim.x) {
        const size_t off = a0 + static_cast<size_t>(i) * 4;
        uint32_t v;
        if (off + 4 <= total) v = __ldg(reinterpret_cast<const uint32_t*>(src + off));
        else {  // last word of the image: assemble from bytes
          v = 0;
          for (int bidx = 0; bidx < 4 && off + bidx < total; ++bidx) v |= static_cast<uint32_t>(src[off + bidx]) << (8 * bidx);
        }
        dstw[i] = v;
      }
    }
    __syncthreads();
    const int y = y0 + ty;
    if (active && y < h) {
      const size_t b0 = (static_cast<size_t>(y) * w + x_lo) * 3;
      const uint8_t* px = sp + ty * span_pad + (b0 & 3) + xmin * 3;
      int a0 = 1 << (ING_PREC - 1), a1 = a0, a2 = a0;
      for (int t = 0; t < n; ++t) {
        const int kv = sk[t * ING_COLS + tx];
        a0 += static_cast<int>(px[3 * t + 0]) * kv;
        a1 += static_cast<int>(px[3 * t + 1]) * kv;
        a2 += static_cast<int>(px[3 * t + 2]) * kv;
      }
      uint8_t* o = dst + (static_cast<size_t>(y) * ow + c0 + tx) * 3;
      o[0] = ing_clip8(a0); o[1] = ing_clip8(a1); o[2] = ing_clip8(a2);
    }
  }
}

// ---- horizontal pass without shared memory, for geometries whose taps and spans exceed ING_SMEM_CAP (panoramas wider
// than ~32 000 px at size 512): one thread per output pixel reads its taps and source bytes straight from global memory.
// Same integer sums as resize_h_kernel, so the same bytes.
constexpr size_t ING_SMEM_CAP = 200 * 1024;
__global__ void __launch_bounds__(256)
resize_h_direct_kernel(const uint8_t* __restrict__ src, int h, int w, uint8_t* __restrict__ dst, int ow,
                       const int32_t* __restrict__ bounds, const int32_t* __restrict__ kk, int ksize) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= ow) return;
  const int xmin = __ldg(bounds + 2 * x), n = __ldg(bounds + 2 * x + 1);
  const int32_t* k = kk + static_cast<size_t>(x) * ksize;
  for (int y = blockIdx.y; y < h; y += gridDim.y) {  // grid.y is capped at 65535 rows
    const uint8_t* px = src + (static_cast<size_t>(y) * w + xmin) * 3;
    int a0 = 1 << (ING_PREC - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < n; ++t) {
      const int kv = __ldg(k + t);
      a0 += static_cast<int>(__ldg(px + 3 * t + 0)) * kv;
      a1 += static_cast<int>(__ldg(px + 3 * t + 1)) * kv;
      a2 += static_cast<int>(__ldg(px + 3 * t + 2)) * kv;
    }
    uint8_t* o = dst + (static_cast<size_t>(y) * ow + x) * 3;
    o[0] = ing_clip8(a0); o[1] = ing_clip8(a1); o[2] = ing_clip8(a2);
  }
}

// ---- vertical pass fused with the center crop and ToTensor + Normalize:
// mid [mh][mw][3] u8 (rows resampled to oh with the given taps, or used as they are when vk == nullptr)
//   -> out fp32 [3][ch][cw],  out = ((v / 255) - 0.5) / 0.5  in fp32 like torchvision.
__global__ void __launch_bounds__(256)
resize_v_crop_norm_kernel(const uint8_t* __restrict__ mid, int mw, const int32_t* __restrict__ vb,
                          const int32_t* __restrict__ vk, int vks, int left, int top, int cw, int ch,
                          float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  if (x >= cw) return;
  const int yy = y + top, xx = x + left;
  int v0, v1, v2;
  if (vk != nullptr) {
    const int ymin = __ldg(vb + 2 * yy), n = __ldg(vb + 2 * yy + 1);
    const int32_t* k = vk + static_cast<size_t>(yy) * vks;
    int a0 = 1 << (ING_PREC - 1), a1 = a0, a2 = a0;
    const uint8_t* p = mid + (static_cast<size_t>(ymin) * mw + xx) * 3;
    for (int t = 0; t < n; ++t, p += static_cast<size_t>(mw) * 3) {
      const int kv = __ldg(k + t);
      a0 += static_cast<int>(__ldg(p + 0)) * kv;
      a1 += static_cast<int>(__ldg(p + 1)) * kv;
      a2 += static_cast<int>(__ldg(p + 2)) * kv;
    }
    v0 = ing_clip8(a0); v1 = ing_clip8(a1); v2 = ing_clip8(a2);
  } else {
    const uint8_t* p = mid + (static_cast<size_t>(yy) * mw + xx) * 3;
    v0 = __ldg(p); v1 = __ldg(p + 1); v2 = __ldg(p + 2);
  }
  const size_t plane = static_cast<size_t>(ch) * cw, o = static_cast<size_t>(y) * cw + x;
  out[o] = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(v0), 255.0f), 0.5f), 0.5f);
  out[plane + o] = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(v1), 255.0f), 0.5f), 0.5f);
  out[2 * plane + o] = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(v2), 255.0f), 0.5f), 0.5f);
}

// dynamic shared memory of resize_h_kernel: taps [ksize][ING_COLS] + ING_ROWS source spans
static size_t ingest_h_smem(int hks, int h_span_max) {
  return static_cast<size_t>(hks) * ING_COLS * 4 + static_cast<size_t>(ING_ROWS) * (((h_span_max * 3 + 3) & ~3) + 4);
}

cudaError_t launch_ingest(const uint8_t* src, int h, int w, int oh, int ow, const int32_t* hb, const int32_t* hk, int hks,
                          int h_span_max, const int32_t* vb, const int32_t* vk, int vks, uint8_t* tmp, int left, int top,
                          int cw, int ch, float* out, cudaStream_t stream) {
  const uint8_t* mid = src;
  if (hk != nullptr) {
    const size_t smem = ingest_h_smem(hks, h_span_max);
    cudaError_t e;
    if (smem <= ING_SMEM_CAP) {
      dim3 grid((ow + ING_COLS - 1) / ING_COLS, (h + ING_ROWS_PER_BLOCK - 1) / ING_ROWS_PER_BLOCK);
      e = launch(resize_h_kernel, grid, ING_COLS * ING_ROWS, smem, stream, false, src, h, w, tmp, ow, hb, hk, hks,
                 h_span_max);
    } else {
      e = launch(resize_h_direct_kernel, dim3((ow + 255) / 256, h < 65535 ? h : 65535), 256, 0, stream, false, src, h, w,
                 tmp, ow, hb, hk, hks);
    }
    if (e != cudaSuccess) return e;
    mid = tmp;
  }
  dim3 grid((cw + 255) / 256, ch);
  (void)oh;
  return launch(resize_v_crop_norm_kernel, grid, 256, 0, stream, false, mid, ow, vb, vk, vks, left, top, cw, ch, out);
}

// ---------------------------------------------------------------- host: Pillow's coefficient tables
static double ing_sinc(double x) {
  if (x == 0.0) return 1.0;
  x = x * M_PI;
  return sin(x) / x;
}
static double ing_filter(int filter, double x) {
  if (filter == 1) {  // LANCZOS, support 3
    if (-3.0 <= x && x < 3.0) return ing_sinc(x) * ing_sinc(x / 3);
    return 0.0;
  }
  const double a = -0.5;  // BICUBIC, support 2
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}
int resample_ksize(int in_size, int out_size, int filter) {
  const double scale = static_cast<double>(in_size) / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  return static_cast<int>(ceil((filter == 1 ? 3.0 : 2.0) * filterscale)) * 2 + 1;
}
// bounds [out_size][2] = (first tap, tap count), kk [out_size][ksize] fixed-point weights; returns the widest source span
// (in pixels) covered by 64 consecutive outputs (shared-memory sizing of the horizontal pass)
int resample_coeffs(int in_size, int out_size, int filter, int32_t* bounds, int32_t* kk) {
  const double scale = static_cast<double>(in_size) / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = (filter == 1 ? 3.0 : 2.0) * filterscale;
  const int ksize = static_cast<int>(ceil(support)) * 2 + 1;
  double* k = new double[ksize];
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    const double ss = 1.0 / filterscale;
    double ww = 0.0;
    int xmin = static_cast<int>(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    for (int x = 0; x < xmax; ++x) {
      const double wv = ing_filter(filter, (x + xmin - center + 0.5) * ss);
      k[x] = wv;
      ww += wv;
    }
    for (int x = 0; x < ksize; ++x) {
      double v = 0.0;
      if (x < xmax) v = (ww != 0.0) ? k[x] / ww : k[x];
      kk[static_cast<size_t>(xx) * ksize + x] = v < 0 ? static_cast<int32_t>(-0.5 + v * (1 << ING_PREC))
                                                      : static_cast<int32_t>(0.5 + v * (1 << ING_PREC));
    }
    bounds[2 * xx] = xmin;
    bounds[2 * xx + 1] = xmax;
  }
  delete[] k;
  int span_max = 0;
  for (int c0 = 0; c0 < out_size; c0 += ING_COLS) {
    const int last = (c0 + ING_COLS < out_size ? c0 + ING_COLS : out_size) - 1;
    const int span = bounds[2 * last] + bounds[2 * last + 1] - bounds[2 * c0];
    if (span > span_max) span_max = span;
  }
  return span_max;
}

}  // namespace f3r
