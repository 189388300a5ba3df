// HBM-bound helper kernels: LayerNorm (fp32 residual stream -> 16-bit GEMM operand), patch im2col, strided
// 3x3 im2col, bilinear x2 upsample (align_corners=True), fp32 -> bf16 / fp16 cast.  All use 128-bit accesses.
// The 16-bit type is bf16 or, for the fp16 forward, fp16 (T = __half); the fp32 outputs serve the parity path.
#include <cstdlib>

#include "common.cuh"
#include "f3r_kernels.h"

namespace f3r {

int g_pdl = -1;
bool pdl_enabled() {
  if (g_pdl < 0) {
    const char* e = getenv("F3R_PDL");
    g_pdl = (e && e[0] == '0') ? 0 : 1;
  }
  return g_pdl == 1;
}
std::atomic<uint64_t> g_launch_count{0};

// ---------------------------------------------------------------- LayerNorm
// nn.LayerNorm over the last dim, biased variance, y = (x-mu)/sqrt(var+eps)*w+b.  One warp per row.
// eps 1e-6 for encoder blocks / enc_norm / dec_norm, 1e-5 for decoder blocks (fast3r/models/fast3r.py:509,683,700).
template <int VEC, typename T>  // dim = VEC * 128; T: the 16-bit output type
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        const float* __restrict__ b, void* __restrict__ out,
                                                        int out_f32, int rows, float eps) {
  pdl_wait();                // x is written by the preceding GEMM
  pdl_launch_dependents();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  constexpr int DIM = VEC * 128;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * DIM);
  float4 v[VEC];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    v[i] = xr[i * 32 + lane];
    sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mu = sum * (1.f / DIM);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const float a = v[i].x - mu, c = v[i].y - mu, d = v[i].z - mu, e = v[i].w - mu;
    sq += (a * a + c * c) + (d * d + e * e);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq * (1.f / DIM) + eps);
  const float4* w4 = reinterpret_cast<const float4*>(w);
  const float4* b4 = reinterpret_cast<const float4*>(b);
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const float4 ww = __ldg(w4 + i * 32 + lane), bb = __ldg(b4 + i * 32 + lane);
    const float y0 = (v[i].x - mu) * rstd * ww.x + bb.x, y1 = (v[i].y - mu) * rstd * ww.y + bb.y;
    const float y2 = (v[i].z - mu) * rstd * ww.z + bb.z, y3 = (v[i].w - mu) * rstd * ww.w + bb.w;
    if (out_f32) {
      reinterpret_cast<float4*>(static_cast<float*>(out) + static_cast<size_t>(row) * DIM)[i * 32 + lane] =
          make_float4(y0, y1, y2, y3);
    } else {
      uint2 o;
      o.x = Half16<T>::pack(y0, y1);
      o.y = Half16<T>::pack(y2, y3);
      reinterpret_cast<uint2*>(static_cast<T*>(out) + static_cast<size_t>(row) * DIM)[i * 32 + lane] = o;
    }
  }
}

template <typename T>
static cudaError_t launch_layernorm_t(const float* x, const float* w, const float* b, void* out, int out_f32, int rows,
                                      int dim, float eps, cudaStream_t stream) {
  decltype(&layernorm_kernel<1, T>) kernel;
  switch (dim) {
    case 128: kernel = layernorm_kernel<1, T>; break;
    case 256: kernel = layernorm_kernel<2, T>; break;
    case 384: kernel = layernorm_kernel<3, T>; break;
    case 512: kernel = layernorm_kernel<4, T>; break;
    case 768: kernel = layernorm_kernel<6, T>; break;
    case 1024: kernel = layernorm_kernel<8, T>; break;
    default: return cudaErrorInvalidValue;
  }
  return launch(kernel, (rows + 7) / 8, 256, 0, stream, true, x, w, b, out, out_f32, rows, eps);
}
cudaError_t launch_layernorm(const float* x, const float* w, const float* b, void* out, int out_type, int rows,
                             int dim, float eps, cudaStream_t stream) {
  if (out_type != ELT_BF16 && out_type != ELT_F32 && out_type != ELT_F16) return cudaErrorInvalidValue;
  if (rows <= 0) return cudaSuccess;
  if (out_type == ELT_F16) return launch_layernorm_t<__half>(x, w, b, out, 0, rows, dim, eps, stream);
  return launch_layernorm_t<__nv_bfloat16>(x, w, b, out, out_type == ELT_F32, rows, dim, eps, stream);
}

// ---------------------------------------------------------------- patch im2col
// img fp32 (n,3,H,W) -> OutT [n*(H/p)*(W/p), 3*p*p], k = c*p*p + ky*p + kx (Conv2d weight flattening,
// fast3r/croco/models/blocks.py:412-414), token order y*gw + x (patch_embed.py:30-33).  p == 16.  OutT: float,
// __nv_bfloat16 or __half.
template <typename OutT>
__global__ void __launch_bounds__(256) im2col_patch_kernel(const float* __restrict__ img, void* __restrict__ out_,
                                                           int n, int H, int W) {
  const int gh = H / 16, gw = W / 16;
  const size_t total = static_cast<size_t>(n) * gh * gw * 96;  // 768 / 8 vectors per token
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int vec = idx % 96;
    const size_t tok = idx / 96;
    const int c = vec / 32, ky = (vec % 32) / 2, kx0 = (vec % 2) * 8;
    const int gx = tok % gw, gy = (tok / gw) % gh;
    const size_t im = tok / (static_cast<size_t>(gw) * gh);
    const float4* src = reinterpret_cast<const float4*>(
        img + ((im * 3 + c) * H + gy * 16 + ky) * static_cast<size_t>(W) + gx * 16 + kx0);
    const float4 a = __ldg(src), b = __ldg(src + 1);
    if constexpr (std::is_same<OutT, float>::value) {  // parity mode: the GEMM operand is hi/lo-split later
      float4* out = static_cast<float4*>(out_);
      out[2 * idx] = a; out[2 * idx + 1] = b;
    } else {
      uint4 o;
      using H = Half16<OutT>;
      o.x = H::pack(a.x, a.y); o.y = H::pack(a.z, a.w);
      o.z = H::pack(b.x, b.y); o.w = H::pack(b.z, b.w);
      static_cast<uint4*>(out_)[idx] = o;
    }
  }
}
cudaError_t launch_im2col_patch(const float* img, void* out, int out_type, int n, int H, int W, int patch,
                                cudaStream_t stream) {
  if (patch != 16 || H % 16 || W % 16) return cudaErrorInvalidValue;
  if (out_type != ELT_BF16 && out_type != ELT_F32 && out_type != ELT_F16) return cudaErrorInvalidValue;
  const size_t total = static_cast<size_t>(n) * (H / 16) * (W / 16) * 96;
  if (total == 0) return cudaSuccess;
  const int grid = static_cast<int>(total / 256 + 1 < 132 * 16 ? total / 256 + 1 : 132 * 16);
  auto kernel = out_type == ELT_F32   ? im2col_patch_kernel<float>
                : out_type == ELT_F16 ? im2col_patch_kernel<__half>
                                      : im2col_patch_kernel<__nv_bfloat16>;
  return launch(kernel, grid, 256, 0, stream, false, img, out, n, H, W);
}

// ---------------------------------------------------------------- 3x3 stride-2 pad-1 im2col (NHWC, 16-bit)
// (copies 16-byte groups of 8 elements without looking at them: the same kernel serves bf16 and fp16)
// out [n*Ho*Wo, 9*C], k = tap*C + c, tap = ky*3+kx  (act_postprocess.3.1, fast3r/croco/models/dpt_block.py:471-478)
__global__ void __launch_bounds__(256) im2col3x3s2_kernel(const uint4* __restrict__ in, uint4* __restrict__ out,
                                                          int n, int H, int W, int C8, int Ho, int Wo) {
  const size_t total = static_cast<size_t>(n) * Ho * Wo * 9 * C8;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = idx % C8;
    const int tap = (idx / C8) % 9;
    const size_t pix = idx / (static_cast<size_t>(C8) * 9);
    const int ox = pix % Wo, oy = (pix / Wo) % Ho;
    const size_t im = pix / (static_cast<size_t>(Wo) * Ho);
    const int iy = oy * 2 - 1 + tap / 3, ix = ox * 2 - 1 + tap % 3;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(in + ((im * H + iy) * W + ix) * C8 + c);
    out[idx] = v;
  }
}
cudaError_t launch_im2col3x3s2(const void* in, void* out, int n, int H, int W, int C, int Ho, int Wo,
                               cudaStream_t stream) {
  if (C % 8) return cudaErrorInvalidValue;
  const size_t total = static_cast<size_t>(n) * Ho * Wo * 9 * (C / 8);
  if (total == 0) return cudaSuccess;
  const int grid = static_cast<int>(total / 256 + 1 < 132 * 16 ? total / 256 + 1 : 132 * 16);
  return launch(im2col3x3s2_kernel, grid, 256, 0, stream, false, static_cast<const uint4*>(in), static_cast<uint4*>(out), n,
                H, W, C / 8, Ho, Wo);
}

// ---------------------------------------------------------------- bilinear x2, align_corners=True (NHWC, 16-bit T)
// F.interpolate(scale_factor=2, mode="bilinear", align_corners=True) (fast3r/croco/models/dpt_block.py:234-247,
// 374): src = dst * (in-1)/(full-1), full = 2*in; only the top-left Ho x Wo window of the full output is produced
// (Ho < full implements the crop of refinenet4's output, fast3r/dust3r/heads/dpt_head.py:69-71).
constexpr int UPS_ROWS = 8;
template <typename T>
__global__ void __launch_bounds__(256) upsample2x_kernel(const uint4* __restrict__ in, uint4* __restrict__ out,
                                                         int H, int W, int C8, int c8_shift, int Ho, int Wo, float sy,
                                                         float sx) {
  // blockIdx.z = image, blockIdx.y = group of UPS_ROWS output rows, x covers (ox, 8-channel group) of a row.  A block
  // walks UPS_ROWS consecutive output rows of the same columns: they interpolate between the same 2-3 input rows, so every
  // input pixel is fetched from L2 once per block and served from L1 afterwards (one-row blocks read each input 4x from
  // L2, which capped the kernel at a third of the HBM rate - profiles/r02_ncu_kernel_families.txt).
  const size_t im = blockIdx.z;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Wo * C8) return;
  const int c = t & (C8 - 1), ox = t >> c8_shift;
  const float fx = sx * ox;
  const int x0 = static_cast<int>(fx);
  const int x1 = min(x0 + 1, W - 1);
  const float lx = fx - x0;
#pragma unroll 1
  for (int oy = blockIdx.y * UPS_ROWS; oy < min((static_cast<int>(blockIdx.y) + 1) * UPS_ROWS, Ho); ++oy) {
  const float fy = sy * oy;
  const int y0 = static_cast<int>(fy);
  const int y1 = min(y0 + 1, H - 1);
  const float ly = fy - y0;
  const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
  const uint4* base = in + im * H * W * C8 + c;
  const uint4 a = __ldg(base + (static_cast<size_t>(y0) * W + x0) * C8);
  const uint4 b = __ldg(base + (static_cast<size_t>(y0) * W + x1) * C8);
  const uint4 d = __ldg(base + (static_cast<size_t>(y1) * W + x0) * C8);
  const uint4 e = __ldg(base + (static_cast<size_t>(y1) * W + x1) * C8);
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
  const uint32_t dw[4] = {d.x, d.y, d.z, d.w}, ew[4] = {e.x, e.y, e.z, e.w};
  uint32_t ow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    using H = Half16<T>;
    const float lo = w00 * H::lo(aw[i]) + w01 * H::lo(bw[i]) + w10 * H::lo(dw[i]) + w11 * H::lo(ew[i]);
    const float hi = w00 * H::hi(aw[i]) + w01 * H::hi(bw[i]) + w10 * H::hi(dw[i]) + w11 * H::hi(ew[i]);
    ow[i] = H::pack(lo, hi);
  }
  out[((im * Ho + oy) * Wo + ox) * C8 + c] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
  }
}
// fp32 NHWC variant (parity mode): one float4 (4 channels) per thread
__global__ void __launch_bounds__(256) upsample2x_f32_kernel(const float4* __restrict__ in, float4* __restrict__ out,
                                                             int H, int W, int C4, int c4_shift, int Ho, int Wo, float sy,
                                                             float sx) {
  const int oy = blockIdx.y;
  const size_t im = blockIdx.z;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Wo * C4) return;
  const int c = t & (C4 - 1), ox = t >> c4_shift;
  const float fy = sy * oy, fx = sx * ox;
  const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
  const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
  const float ly = fy - y0, lx = fx - x0;
  const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
  const float4* base = in + im * H * W * C4 + c;
  const float4 a = __ldg(base + (static_cast<size_t>(y0) * W + x0) * C4);
  const float4 b = __ldg(base + (static_cast<size_t>(y0) * W + x1) * C4);
  const float4 d = __ldg(base + (static_cast<size_t>(y1) * W + x0) * C4);
  const float4 e = __ldg(base + (static_cast<size_t>(y1) * W + x1) * C4);
  float4 o;
  o.x = w00 * a.x + w01 * b.x + w10 * d.x + w11 * e.x;
  o.y = w00 * a.y + w01 * b.y + w10 * d.y + w11 * e.y;
  o.z = w00 * a.z + w01 * b.z + w10 * d.z + w11 * e.z;
  o.w = w00 * a.w + w01 * b.w + w10 * d.w + w11 * e.w;
  out[((im * Ho + oy) * Wo + ox) * C4 + c] = o;
}
cudaError_t launch_upsample2x(const void* in, void* out, int elt, int n, int H, int W, int C, int Ho, int Wo, int Hfull,
                              int Wfull, cudaStream_t stream) {
  if (C % 8 || Hfull < 2 || Wfull < 2) return cudaErrorInvalidValue;
  if (elt != ELT_BF16 && elt != ELT_F32 && elt != ELT_F16) return cudaErrorInvalidValue;
  if (elt == ELT_F32) {
    const int C4 = C / 4;
    int shift = 0;
    while ((1 << shift) < C4) ++shift;
    if ((1 << shift) != C4) return cudaErrorInvalidValue;
    if (n <= 0 || Ho <= 0 || Wo <= 0) return cudaSuccess;
    if (n > 65535 || Ho > 65535) return cudaErrorInvalidValue;
    const float sy = static_cast<float>(H - 1) / static_cast<float>(Hfull - 1);
    const float sx = static_cast<float>(W - 1) / static_cast<float>(Wfull - 1);
    dim3 grid((Wo * C4 + 255) / 256, Ho, n);
    return launch(upsample2x_f32_kernel, grid, 256, 0, stream, false, static_cast<const float4*>(in),
                  static_cast<float4*>(out), H, W, C4, shift, Ho, Wo, sy, sx);
  }
  const int C8 = C / 8;
  int shift = 0;
  while ((1 << shift) < C8) ++shift;
  if ((1 << shift) != C8) return cudaErrorInvalidValue;  // channel count / 8 must be a power of two
  if (n <= 0 || Ho <= 0 || Wo <= 0) return cudaSuccess;
  if (n > 65535 || Ho > 65535) return cudaErrorInvalidValue;
  const float sy = static_cast<float>(H - 1) / static_cast<float>(Hfull - 1);
  const float sx = static_cast<float>(W - 1) / static_cast<float>(Wfull - 1);
  dim3 grid((Wo * C8 + 255) / 256, (Ho + UPS_ROWS - 1) / UPS_ROWS, n);
  return launch(elt == ELT_F16 ? upsample2x_kernel<__half> : upsample2x_kernel<__nv_bfloat16>, grid, 256, 0, stream, false,
                static_cast<const uint4*>(in), static_cast<uint4*>(out), H, W, C8, shift, Ho, Wo, sy, sx);
}

// ---------------------------------------------------------------- fp32 -> bf16 / fp16 (T)
template <typename T>
__global__ void __launch_bounds__(256) cast_kernel(const float4* __restrict__ in, uint2* __restrict__ out, size_t n4) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 v = __ldg(in + i);
    out[i] = make_uint2(Half16<T>::pack(v.x, v.y), Half16<T>::pack(v.z, v.w));
  }
}
template <typename T>
static cudaError_t launch_cast(const float* in, void* out, size_t n, cudaStream_t stream) {
  if (n % 4) return cudaErrorInvalidValue;
  if (n == 0) return cudaSuccess;
  const size_t n4 = n / 4;
  const int grid = static_cast<int>(n4 / 256 + 1 < 132 * 16 ? n4 / 256 + 1 : 132 * 16);
  return launch(cast_kernel<T>, grid, 256, 0, stream, false, reinterpret_cast<const float4*>(in),
                static_cast<uint2*>(out), n4);
}
cudaError_t launch_cast_bf16(const float* in, void* out, size_t n, cudaStream_t stream) {
  return launch_cast<__nv_bfloat16>(in, out, n, stream);
}
cudaError_t launch_cast_f16(const float* in, void* out, size_t n, cudaStream_t stream) {
  return launch_cast<__half>(in, out, n, stream);
}

}  // namespace f3r
