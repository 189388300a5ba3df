// Parity-mode attention (head_dim 64): softmax(scale * Q K^T) V with fp32-level accuracy on the bf16 tensor pipe.
// (fast3r/croco/models/blocks.py:135-194 run WITHOUT autocast, i.e. the reference's fp32 path,
//  fast3r/dust3r/inference_multiview.py:41-49 dtype="32".)
//
// Every fp32 operand x is carried as a pair of bf16 numbers x = hi + lo (hi = bf16(x), lo = bf16(x - hi), 16 mantissa
// bits together) and every product is evaluated as hi*hi + lo*hi + hi*lo in the fp32 accumulator (the lo*lo term,
// 2^-18 relative, is dropped):
//   S = Q K^T : the head dimension is "concatenated" to 192: Q' = [Qhi | Qlo | Qhi], K' = [Khi | Khi | Klo]
//               (written by attn_split_kernel below) -> 12 k-steps of one 128x128x16 SS MMA chain instead of 4;
//   O += P V  : P is split in the softmax registers into Phi / Plo (two packed-bf16 register A operands), V arrives
//               as [Vhi | Vlo]; three wgmma chains Phi*Vhi + Plo*Vhi + Phi*Vlo accumulate into the same O registers.
// Softmax statistics, the row sum (of the un-split fp32 p) and the output are fp32.  One CTA = 128 query rows of one
// (batch, head), 64 per consumer warpgroup; K'/V' blocks of 128 keys stream through a 2-stage TMA ring.  This kernel
// trades speed for accuracy (3x the MMAs); the bf16 kernel in attention.cu is the fast path.
#include "common.cuh"
#include "f3r_kernels.h"

namespace f3r {

constexpr int X3_THREADS = 384;  // warpgroup 0: TMA producer; warpgroups 1, 2: 64 query rows each
constexpr int X3_STAGES = 2;
constexpr int X3_TILE = 128 * 64 * 2;  // 16 KB: 128 rows x 64 bf16, 128B-swizzled
constexpr int X3_SMEM_BYTES = (3 + X3_STAGES * 5) * X3_TILE + 1024 + 256;

__global__ void __launch_bounds__(X3_THREADS, 1)
attention_x3_kernel(const __grid_constant__ CUtensorMap tmap_q3, const __grid_constant__ CUtensorMap tmap_k3,
                    const __grid_constant__ CUtensorMap tmap_v2, const __grid_constant__ AttnArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;                                  // 3 sub-tiles
  uint8_t* smem_k = smem + 3 * X3_TILE;                    // X3_STAGES x 3 sub-tiles
  uint8_t* smem_v = smem_k + X3_STAGES * 3 * X3_TILE;      // X3_STAGES x 2 sub-tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_v + X3_STAGES * 2 * X3_TILE);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;
  uint64_t* k_empty = k_full + X3_STAGES;
  uint64_t* v_full = k_empty + X3_STAGES;
  uint64_t* v_empty = v_full + X3_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qt = blockIdx.x % p.q_tiles;
  const int bh = blockIdx.x / p.q_tiles;
  const int h = bh % p.heads;
  const int b = bh / p.heads;
  const int nkv = (p.skv + 127) / 128;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q3);
    tma_prefetch_desc(&tmap_k3);
    tma_prefetch_desc(&tmap_v2);
    mbar_init(q_full, 1);
    for (int s = 0; s < X3_STAGES; ++s) {
      mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], 2);
      mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      // ===================== TMA producer =====================
      mbar_arrive_expect_tx(q_full, 3 * X3_TILE);
      for (int s = 0; s < 3; ++s) tma_load_3d(smem_q + s * X3_TILE, &tmap_q3, q_full, h * 192 + s * 64, qt * 128, b);
      int stage = 0; uint32_t phase = 0;
      for (int j = 0; j < nkv; ++j) {
        mbar_wait_relaxed(&k_empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&k_full[stage], 3 * X3_TILE);
        for (int s = 0; s < 3; ++s)
          tma_load_3d(smem_k + (stage * 3 + s) * X3_TILE, &tmap_k3, &k_full[stage], h * 192 + s * 64, j * 128, b);
        mbar_wait_relaxed(&v_empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&v_full[stage], 2 * X3_TILE);
        for (int s = 0; s < 2; ++s)
          tma_load_3d(smem_v + (stage * 2 + s) * X3_TILE, &tmap_v2, &v_full[stage], h * 128 + s * 64, j * 128, b);
        if (++stage == X3_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ===================== consumer warpgroups (fragment layout: see common.cuh) =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cg = (warp - 4) >> 2;
    const int wg_tid = threadIdx.x & 127;
    const int rw = cg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    const float sl2 = p.scale_log2;
    float m_used[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    mbar_wait(q_full, 0);
    for (int j = 0; j < nkv; ++j) {
      const int st = j % X3_STAGES;
      const uint32_t ph = (j / X3_STAGES) & 1;
      float s[64];
      mbar_wait(&k_full[st], ph);
      wgmma_fence();
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const uint64_t qd = make_smem_desc_sw128(smem_u32(smem_q + t * X3_TILE + cg * 64 * 128));
        const uint64_t kd = make_smem_desc_sw128(smem_u32(smem_k + (st * 3 + t) * X3_TILE));
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss_n128<0>(s, qd + 2 * k, kd + 2 * k, (t | k) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      if (wg_tid == 0) mbar_arrive(&k_empty[st]);
      if (j == nkv - 1) {
        const int valid = p.skv - j * 128;
        if (valid < 128) {
#pragma unroll
          for (int i = 0; i < 64; ++i)
            if (8 * (i >> 2) + cq + (i & 1) >= valid) s[i] = -INFINITY;
        }
      }
      float nm[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float mx = fmaxf(s[2 * hh], s[2 * hh + 1]);
#pragma unroll
        for (int jn = 1; jn < 16; ++jn) mx = fmaxf(mx, fmaxf(s[4 * jn + 2 * hh], s[4 * jn + 2 * hh + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        if ((mx - m_used[hh]) * sl2 > 8.f) {  // lazy reference move (first block: -inf reference => true)
          const float alpha = exp2f((m_used[hh] - mx) * sl2);
          m_used[hh] = mx;
          l[hh] *= alpha;
#pragma unroll
          for (int jn = 0; jn < 8; ++jn) { o[4 * jn + 2 * hh] *= alpha; o[4 * jn + 2 * hh + 1] *= alpha; }
        }
        nm[hh] = -m_used[hh] * sl2;
      }
      uint32_t phi[8][4], plo[8][4];
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int i = 8 * kk + 2 * r, hh = r & 1;
          const float e0 = exp2f(fmaf(s[i], sl2, nm[hh])), e1 = exp2f(fmaf(s[i + 1], sl2, nm[hh]));
          l[hh] += e0 + e1;
          const uint32_t h2 = pack_bf16(e0, e1);
          phi[kk][r] = h2;
          plo[kk][r] = pack_bf16(e0 - bf16_lo(h2), e1 - bf16_hi(h2));
        }
      }
      mbar_wait(&v_full[st], ph);
      const uint64_t vhi = make_smem_desc_sw128(smem_u32(smem_v + (st * 2 + 0) * X3_TILE));
      const uint64_t vlo = make_smem_desc_sw128(smem_u32(smem_v + (st * 2 + 1) * X3_TILE));
      fence_regs(o);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) wgmma_rs_n64<1>(o, phi[kk], vhi + 128 * kk, 1u);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) wgmma_rs_n64<1>(o, plo[kk], vhi + 128 * kk, 1u);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) wgmma_rs_n64<1>(o, phi[kk], vlo + 128 * kk, 1u);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(o);
      if (wg_tid == 0) mbar_arrive(&v_empty[st]);
    }
    // ---- epilogue: O / l -> fp32 global
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
      l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
      const int q = qt * 128 + rw + 8 * hh;
      if (q >= p.sq) continue;
      const float inv = 1.f / l[hh];
      float* dst = static_cast<float*>(p.out) + (static_cast<size_t>(b) * p.sq + q) * p.ldo + h * 64 + cq;
#pragma unroll
      for (int jn = 0; jn < 8; ++jn)
        *reinterpret_cast<float2*>(dst + 8 * jn) = make_float2(o[4 * jn + 2 * hh] * inv, o[4 * jn + 2 * hh + 1] * inv);
      if (p.lse != nullptr && (lane & 3) == 0)
        p.lse[(static_cast<size_t>(b) * p.heads + h) * p.sq + q] = m_used[hh] * sl2 * 0.69314718056f + logf(l[hh]);
    }
  }
}

cudaError_t launch_attention_x3(const CUtensorMap& tq3, const CUtensorMap& tk3, const CUtensorMap& tv2,
                                const AttnArgs& a, cudaStream_t stream) {
  return launch(attention_x3_kernel, a.batch * a.heads * a.q_tiles, X3_THREADS, X3_SMEM_BYTES, stream, false, tq3, tk3, tv2,
                a);
}

// ---------------------------------------------------------------- operand preparation
// fp32 q [rows, heads*64], kv [rows, 2*heads*64] (K | V)  ->  bf16 q3 [rows, heads*192] = per head [Qhi | Qlo | Qhi],
// k3 [rows, heads*192] = per head [Khi | Khi | Klo], v2 [rows, heads*128] = per head [Vhi | Vlo].
__device__ __forceinline__ void split4(const float4 v, uint2& hi, uint2& lo) {
  hi.x = pack_bf16(v.x, v.y); hi.y = pack_bf16(v.z, v.w);
  lo.x = pack_bf16(v.x - bf16_lo(hi.x), v.y - bf16_hi(hi.x));
  lo.y = pack_bf16(v.z - bf16_lo(hi.y), v.w - bf16_hi(hi.y));
}
__global__ void __launch_bounds__(256) attn_split_kernel(const float4* __restrict__ q, int ldq4, const float4* __restrict__ kv,
                                                         int ldkv4, uint2* __restrict__ q3, uint2* __restrict__ k3,
                                                         uint2* __restrict__ v2, size_t rows_q, size_t rows_kv, int heads) {
  const int d4 = heads * 16;  // float4 vectors per row of one of q / k / v
  const size_t nq = rows_q * d4, nk = rows_kv * d4;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < nq + 2 * nk;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    uint2 hi, lo;
    if (idx < nq) {
      const size_t r = idx / d4; const int c = idx % d4, hh = c / 16, e = c % 16;
      split4(__ldg(q + r * ldq4 + c), hi, lo);
      uint2* o = q3 + (r * heads + hh) * 48 + e;
      o[0] = hi; o[16] = lo; o[32] = hi;
    } else if (idx < nq + nk) {
      const size_t i = idx - nq, r = i / d4; const int c = i % d4, hh = c / 16, e = c % 16;
      split4(__ldg(kv + r * ldkv4 + c), hi, lo);
      uint2* o = k3 + (r * heads + hh) * 48 + e;
      o[0] = hi; o[16] = hi; o[32] = lo;
    } else {
      const size_t i = idx - nq - nk, r = i / d4; const int c = i % d4, hh = c / 16, e = c % 16;
      split4(__ldg(kv + r * ldkv4 + d4 + c), hi, lo);
      uint2* o = v2 + (r * heads + hh) * 32 + e;
      o[0] = hi; o[16] = lo;
    }
  }
}
cudaError_t launch_attn_split(const float* q, int ldq, const float* kv, int ldkv, void* q3, void* k3, void* v2,
                              size_t rows_q, size_t rows_kv, int heads, cudaStream_t stream) {
  if (ldq % 4 || ldkv % 4) return cudaErrorInvalidValue;
  const size_t total = (rows_q + 2 * rows_kv) * heads * 16;
  if (total == 0) return cudaSuccess;
  const int grid = static_cast<int>(total / 256 + 1 < 132 * 16 ? total / 256 + 1 : 132 * 16);
  return launch(attn_split_kernel, grid, 256, 0, stream, false, reinterpret_cast<const float4*>(q), ldq / 4,
                reinterpret_cast<const float4*>(kv), ldkv / 4, static_cast<uint2*>(q3), static_cast<uint2*>(k3),
                static_cast<uint2*>(v2), rows_q, rows_kv, heads);
}

// ---------------------------------------------------------------- GEMM operand split
// fp32 x [rows, K] -> bf16 [rows, 3K] = [hi | lo | hi] (optionally of relu(x)); the matching weight layout is
// [Whi | Whi | Wlo] along K, so the ordinary bf16 GEMM over 3K accumulates hi*hi + lo*hi + hi*lo in fp32.
__global__ void __launch_bounds__(256) split3_kernel(const float4* __restrict__ in, uint2* __restrict__ out, size_t rows,
                                                     int k4, int relu) {
  const size_t total = rows * k4;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t r = idx / k4; const int c = idx % k4;
    float4 v = __ldg(in + idx);
    if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    uint2 hi, lo;
    split4(v, hi, lo);
    uint2* o = out + r * 3 * k4 + c;
    o[0] = hi; o[k4] = lo; o[2 * k4] = hi;
  }
}
cudaError_t launch_split3(const float* in, void* out, size_t rows, int k, int relu, cudaStream_t stream) {
  if (k % 4) return cudaErrorInvalidValue;
  const size_t total = rows * (k / 4);
  if (total == 0) return cudaSuccess;
  const int grid = static_cast<int>(total / 256 + 1 < 132 * 16 ? total / 256 + 1 : 132 * 16);
  return launch(split3_kernel, grid, 256, 0, stream, false, reinterpret_cast<const float4*>(in), static_cast<uint2*>(out),
                rows, k / 4, relu);
}

// dst += src (fp32; second residual operand of the DPT fusion blocks in parity mode)
__global__ void __launch_bounds__(256) add_f32_kernel(float4* __restrict__ dst, const float4* __restrict__ src, size_t n4) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float4 a = dst[i];
    const float4 b = __ldg(src + i);
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    dst[i] = a;
  }
}
cudaError_t launch_add_f32(float* dst, const float* src, size_t n, cudaStream_t stream) {
  if (n % 4) return cudaErrorInvalidValue;
  if (n == 0) return cudaSuccess;
  const size_t n4 = n / 4;
  const int grid = static_cast<int>(n4 / 256 + 1 < 132 * 16 ? n4 / 256 + 1 : 132 * 16);
  return launch(add_f32_kernel, grid, 256, 0, stream, false, reinterpret_cast<float4*>(dst),
                reinterpret_cast<const float4*>(src), n4);
}

}  // namespace f3r
