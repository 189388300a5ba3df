// Persistent warp-specialised wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
//   out[m, n] = epilogue( sum_{tap, k} A[pixel(m) + shift(tap), k] * Wt[n, tap, k] )
//
// A is a channels-last 16-bit activation (bf16, or fp16 with T = __half) viewed as (C, W, H, NB) and fetched by 4-D
// TMA boxes of 128 pixels x 64 channels (out-of-bounds pixels/channels are zero-filled by TMA, which gives the
// 3x3 zero padding and the K / N tails for free).  A plain linear layer is the 1-tap case with
// W = rows.  One producer thread issues TMA into a multi-stage smem ring; two consumer warpgroups each
// own 64 rows of the 128-row tile and accumulate in registers with wgmma (m64 x BLOCK_N x k16).
//
// Covers (reference file:line in DESIGN.md): nn.Linear qkv/proj/fc1/fc2/decoder_embed
// (fast3r/croco/models/blocks.py:94-97,125-128; fast3r/models/fast3r.py:673), patch-embed conv as
// im2col GEMM (blocks.py:412), DPT 1x1 / 3x3 / transposed convs (fast3r/croco/models/dpt_block.py).
#include "common.cuh"
#include "f3r_kernels.h"

namespace f3r {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int GEMM_THREADS = 384;  // warpgroup 0: warp 0 TMA, warps 1-3 idle; warpgroups 1, 2: wgmma + epilogue
constexpr int XCH_STRIDE = 68;     // fp32 row stride of the fragment -> row exchange tile (64 rows x 64 columns)

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int kStages = (BLOCK_N == 256) ? 3 : 4;
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kXchBytes = 64 * XCH_STRIDE * 4;  // per consumer warpgroup
  static constexpr int kSmemBytes =
      kStages * kStageBytes + 1024 /*align*/ + 1024 /*barriers*/ + 8 * 4096 /*epilogue staging*/ + 2 * kXchBytes;
};

// Epilogue data movement.  A thread owns one accumulator ROW (after the fragment exchange), but row-per-thread global
// accesses touch 32 different cache lines per instruction.  Every 32x32 fp32 chunk is therefore transposed through a
// per-warp 4 KB shared-memory tile (16-byte chunks XOR-swizzled by row, conflict-free both ways) and all global
// traffic (residual reads, stores) is issued in the "transposed" mapping: lane l handles 4 consecutive columns
// (16 B fp32 / 8 B bf16) of row 4*i + l/8, i = 0..7, so one warp instruction covers 4 full 128-byte row segments.
struct ResChunk {
  uint4 r0[8];  // res0 piece i: 4 fp32 (uint4) or 4 16-bit values (.x,.y)
  uint2 r1[8];  // res1 piece i: 4 16-bit values
};

__device__ __forceinline__ size_t out_offset(const GemmArgs& p, int m, int col0, int img, int py, int px) {
  if (p.epi == EPI_CONVT) {
    const int ij = col0 / p.ct_cout, o0 = col0 % p.ct_cout, k = p.ct_k;
    const int oy = py * k + ij / k, ox = px * k + ij % k;
    return ((static_cast<size_t>(img) * p.H * k + oy) * (p.W * k) + ox) * p.ct_cout + o0;
  }
  return static_cast<size_t>(m) * p.ldo + col0;
}

// off_row / ok_row: output offset and validity of THIS lane's accumulator row; piece i needs the values of row 4*i + lane/8
__device__ __forceinline__ void prefetch_res(const GemmArgs& p, ResChunk& rc, size_t off_row, bool ok_row, int lane) {
  if (p.res0 == nullptr && p.res1 == nullptr) return;
  const unsigned okmask = __ballot_sync(0xffffffffu, ok_row);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rr = 4 * i + (lane >> 3);
    const size_t off = __shfl_sync(0xffffffffu, off_row, rr) + (lane & 7) * 4;
    if (!((okmask >> rr) & 1)) continue;
    if (p.res0 != nullptr) {
      if (p.res0_f32) rc.r0[i] = *reinterpret_cast<const uint4*>(static_cast<const float*>(p.res0) + off);
      else {
        const uint2 t = *reinterpret_cast<const uint2*>(static_cast<const uint16_t*>(p.res0) + off);
        rc.r0[i].x = t.x; rc.r0[i].y = t.y;
      }
    }
    if (p.res1 != nullptr) rc.r1[i] = *reinterpret_cast<const uint2*>(static_cast<const uint16_t*>(p.res1) + off);
  }
}

// exact-erf GELU (nn.GELU(), fast3r/croco/models/blocks.py:83) with erf from Abramowitz-Stegun 7.1.26
// (|abs err| <= 1.5e-7, far below the bf16 rounding of the stored activation): 12 FMA-pipe ops + 2 MUFU (rcp, ex2).
__device__ __forceinline__ void gelu_fast(float& x) {
  const float z = __fmul_rn(fabsf(x), 0.70710678118654752440f);
  const float u = fmaf(z, 0.3275911f, 1.0f);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(u));
  float q = fmaf(t, 1.061405429f, -1.453152027f);
  q = fmaf(q, t, 1.421413741f);
  q = fmaf(q, t, -0.284496736f);
  q = fmaf(q, t, 0.254829592f);
  q = __fmul_rn(q, t);
  const float a = __fmul_rn(__fmul_rn(z, z), -1.4426950408889634f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(a));
  const float r = copysignf(fmaf(q, -e, 1.0f), x);  // erf(|z|) = 1 - poly * exp(-z^2)
  const float h = __fmul_rn(x, 0.5f);
  x = fmaf(h, r, h);                                 // 0.5 x (1 + erf)
}
// Row-domain part: bias, RoPE, image-index embedding, or the FINAL 128->4 dot product.  Returns false if the chunk is
// fully consumed here (FINAL).
__device__ __forceinline__ bool epilogue_rows(const GemmArgs& p, float (&v)[32], int m, int col0, bool row_ok,
                                              float (&fin)[4], bool add_bias, const float* w4s) {
  if (p.bias != nullptr && add_bias) {
    const float4* b4 = reinterpret_cast<const float4*>(p.bias + (p.epi == EPI_CONVT ? (col0 % p.ct_cout) : col0));
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float4 b = __ldg(b4 + i);
      v[4 * i + 0] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
    }
  }
  if (p.epi == EPI_ROPE && col0 < p.rope_cols && row_ok) {
    // RoPE2D (fast3r/croco/models/pos_embed.py:141-183): 32-wide half-head, pair (j, j+16), angle pos*base^(-j/16)
    const int t = m % p.tok_per_img;
    const int pos = ((col0 >> 5) & 1) ? (t % p.grid_w) : (t / p.grid_w);
    const float4* c4 = reinterpret_cast<const float4*>(p.rope_cos + pos * 16);
    const float4* s4 = reinterpret_cast<const float4*>(p.rope_sin + pos * 16);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float4 c = __ldg(c4 + i), s = __ldg(s4 + i);
      float cc[4] = {c.x, c.y, c.z, c.w}, ss[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * i + e;
        const float a = v[j], b = v[j + 16];
        v[j] = a * cc[e] - b * ss[e];
        v[j + 16] = b * cc[e] + a * ss[e];
      }
    }
  }
  if (p.epi == EPI_IDXEMB && row_ok) {
    // + image_idx_emb[id(view of token)]  (fast3r/models/fast3r.py:785-799)
    const int id = __ldg(p.emb_ids + (p.tok_per_img > 0 ? m / p.tok_per_img : m));  // per-image or per-row ids
    const float4* e4 = reinterpret_cast<const float4*>(p.emb_table + static_cast<size_t>(id) * p.N + col0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float4 e = __ldg(e4 + i);
      v[4 * i + 0] += e.x; v[4 * i + 1] += e.y; v[4 * i + 2] += e.z; v[4 * i + 3] += e.w;
    }
  }
  if (p.epi == EPI_FINAL) {
    // ReLU -> conv1x1 (BLOCK_N -> 4), accumulated across the column chunks of this row.  The 4 x N weights sit in shared
    // memory (all lanes read the same address: one broadcast 16-byte load per 4 weights instead of 4 global loads).
    if (row_ok) {
#pragma unroll
      for (int o = 0; o < 4; ++o) {
        const float4* w = reinterpret_cast<const float4*>(w4s + o * p.N + col0);
        float acc = fin[o];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 ww = w[i];
          acc = fmaf(fmaxf(v[4 * i + 0], 0.f), ww.x, acc);
          acc = fmaf(fmaxf(v[4 * i + 1], 0.f), ww.y, acc);
          acc = fmaf(fmaxf(v[4 * i + 2], 0.f), ww.z, acc);
          acc = fmaf(fmaxf(v[4 * i + 3], 0.f), ww.w, acc);
        }
        fin[o] = acc;
      }
    }
    return false;
  }
  return true;
}

// Transposed part: stage the 32x32 chunk, then residual adds / activation / stores with coalesced accesses.  T: the
// 16-bit element type of res0 / res1 / out0 / out1 when they are not fp32.
template <typename T>
__device__ __forceinline__ void epilogue_store(const GemmArgs& p, const float (&v)[32], const ResChunk& rc, uint8_t* stage,
                                               int lane, int m, int col0, size_t off_row, bool ok_row) {
  using H = Half16<T>;
  // write own row: 16-byte chunk j of row r lives at r*128 + ((j ^ (r & 7)) << 4)
#pragma unroll
  for (int j = 0; j < 8; ++j)
    *reinterpret_cast<float4*>(stage + lane * 128 + ((j ^ (lane & 7)) << 4)) =
        make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
  __syncwarp();
  const unsigned okmask = __ballot_sync(0xffffffffu, ok_row);
  const int cj = lane & 7;
  const bool to_b = p.split_col > 0 && col0 >= p.split_col;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rr = 4 * i + (lane >> 3);
    const size_t off = __shfl_sync(0xffffffffu, off_row, rr) + cj * 4;
    const int mrow = __shfl_sync(0xffffffffu, m, rr);
    if (!((okmask >> rr) & 1)) continue;
    const float4 a = *reinterpret_cast<const float4*>(stage + rr * 128 + ((cj ^ (rr & 7)) << 4));
    float x0 = a.x, x1 = a.y, x2 = a.z, x3 = a.w;
    if (p.res0 != nullptr) {
      if (p.res0_f32) {
        x0 += __uint_as_float(rc.r0[i].x); x1 += __uint_as_float(rc.r0[i].y);
        x2 += __uint_as_float(rc.r0[i].z); x3 += __uint_as_float(rc.r0[i].w);
      } else {
        x0 += H::lo(rc.r0[i].x); x1 += H::hi(rc.r0[i].x); x2 += H::lo(rc.r0[i].y); x3 += H::hi(rc.r0[i].y);
      }
    }
    if (p.res1 != nullptr) {
      x0 += H::lo(rc.r1[i].x); x1 += H::hi(rc.r1[i].x); x2 += H::lo(rc.r1[i].y); x3 += H::hi(rc.r1[i].y);
    }
    if (p.out1 != nullptr) {  // relu(v) in 16 bits: operand of the next 3x3 conv of a residual unit
      uint2 o;
      o.x = H::pack(fmaxf(x0, 0.f), fmaxf(x1, 0.f));
      o.y = H::pack(fmaxf(x2, 0.f), fmaxf(x3, 0.f));
      *reinterpret_cast<uint2*>(static_cast<T*>(p.out1) + off) = o;
    }
    if (p.out0 == nullptr) continue;
    if (p.act == ACT_RELU) {
      x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); x2 = fmaxf(x2, 0.f); x3 = fmaxf(x3, 0.f);
    } else if (p.act == ACT_GELU) {
      gelu_fast(x0); gelu_fast(x1); gelu_fast(x2); gelu_fast(x3);
    }
    void* base = p.out0;
    size_t o = off;
    if (to_b) {  // q | kv column split
      base = p.out0b;
      o = static_cast<size_t>(mrow) * p.ldo_b + (col0 - p.split_col) + cj * 4;
    }
    if (p.out0_f32) {
      *reinterpret_cast<float4*>(static_cast<float*>(base) + o) = make_float4(x0, x1, x2, x3);
    } else {
      uint2 q;
      q.x = H::pack(x0, x1);
      q.y = H::pack(x2, x3);
      *reinterpret_cast<uint2*>(static_cast<T*>(base) + o) = q;
    }
  }
  __syncwarp();  // staging tile is rewritten by the next chunk
}

// TMA epilogue (hot path: plain stores and the in-place fp32 residual update).  The thread that owns accumulator
// row r writes its 32 activated values into the warp's staging tile in the tensor map's swizzled layout (conflict-free
// 16-byte stores), then one lane hands the whole 32x32 tile to the TMA unit: a store, or for x += f(x) an fp32
// reduce-add executed by the memory system (the residual is never read by the SM).  Out-of-range rows / columns are
// clipped by the tensor map.
template <typename T>
__device__ __forceinline__ void epilogue_tma(const GemmArgs& p, float (&v)[32], uint8_t* stage, int lane,
                                             const CUtensorMap* map, bool reduce, int c_col, int c_x, int c_y, int c_img) {
  if (p.act == ACT_RELU) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.f);
  } else if (p.act == ACT_GELU) {
#pragma unroll
    for (int i = 0; i < 32; ++i) gelu_fast(v[i]);
  }
  if (lane == 0) tma_store_wait_read();  // the previous tile of this warp has left the staging buffer
  __syncwarp();
  if (p.out0_f32) {  // 128-byte rows, SWIZZLE_128B: chunk j of row r at r*128 + ((j ^ (r & 7)) << 4)
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<float4*>(stage + lane * 128 + ((j ^ (lane & 7)) << 4)) =
          make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
  } else {           // 64-byte rows, SWIZZLE_64B: chunk j of row r at r*64 + ((j ^ ((r >> 1) & 3)) << 4)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint4 q;
      q.x = Half16<T>::pack(v[8 * j + 0], v[8 * j + 1]);
      q.y = Half16<T>::pack(v[8 * j + 2], v[8 * j + 3]);
      q.z = Half16<T>::pack(v[8 * j + 4], v[8 * j + 5]);
      q.w = Half16<T>::pack(v[8 * j + 6], v[8 * j + 7]);
      *reinterpret_cast<uint4*>(stage + lane * 64 + ((j ^ ((lane >> 1) & 3)) << 4)) = q;
    }
  }
  fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the TMA (async proxy)
  __syncwarp();
  if (lane == 0) {
    if (reduce) tma_reduce_add_4d(map, stage, c_col, c_x, c_y, c_img);
    else tma_store_4d(map, stage, c_col, c_x, c_y, c_img);
    tma_store_commit();
  }
}

// T: the 16-bit type of A, the weights and the 16-bit outputs / residuals (__nv_bfloat16 or __half)
template <int BLOCK_N, typename T>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_o0, const __grid_constant__ CUtensorMap tmap_o0b,
            const __grid_constant__ GemmArgs p) {
  using Cfg = GemmCfg<BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kABytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;
  uint8_t* stage_base = smem + Cfg::kStages * Cfg::kStageBytes + 1024;  // 8 x 4 KB, 1024-aligned
  float* fin_smem = reinterpret_cast<float*>(stage_base);  // [128][4] (FINAL mode does not stage)
  float* w4_smem = reinterpret_cast<float*>(stage_base + 4096);  // FINAL: [4][N <= 256] copy of the 1x1 conv weights
  float* xch_base = reinterpret_cast<float*>(stage_base + 8 * 4096);  // [2][64][XCH_STRIDE]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    fence_barrier_init();
  }
  if (p.epi == EPI_FINAL)
    for (int i = threadIdx.x; i < 4 * p.N; i += GEMM_THREADS) w4_smem[i] = __ldg(p.w4 + i);
  __syncthreads();
  pdl_wait();                // operands / residual are produced by the preceding kernels: no global access above this line
  pdl_launch_dependents();   // except the 1x1-conv weights of FINAL and the tensor-map prefetch (parameters, not activations)

  // split-K (only with the fp32 reduce-add epilogue, x += A W^T: partial sums of the K slices are added by the memory
  // system): work item = (tile, K slice); used when there are fewer tiles than SMs (small M in sequence-parallel runs)
  const int num_out_tiles = p.num_m_tiles * p.num_n_tiles;
  const int num_tiles = num_out_tiles * p.k_split;
  const int k_chunks = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int k_iters = p.taps * k_chunks;

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");   // 128 x 40 + 256 x 232 <= 64K registers
    if (warp == 0 && lane == 0) {
      // ===================== TMA producer =====================
      int stage = 0; uint32_t phase = 0;
      for (int item = blockIdx.x; item < num_tiles; item += gridDim.x) {
        const int tile = item % num_out_tiles, ks = item / num_out_tiles;
        const int it0 = ks * k_iters / p.k_split, it1 = (ks + 1) * k_iters / p.k_split;
        const int mt = tile / p.num_n_tiles, nt = tile % p.num_n_tiles;
        const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, img = mt / (p.tiles_x * p.tiles_y);
        const int x0 = tx * p.bw, y0 = ty * p.bh, n0 = nt * BLOCK_N;
        for (int it = it0; it < it1; ++it) {
          const int tap = it / k_chunks, kc = it % k_chunks;
          int dy = 0, dx = 0;
          if (p.taps == 9) { dy = tap / 3 - 1; dx = tap % 3 - 1; }
          mbar_wait_relaxed(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_4d(smem_a + stage * Cfg::kABytes, &tmap_a, &full_bar[stage], kc * BLOCK_K, x0 + dx, y0 + dy, img);
          tma_load_3d(smem_b + stage * Cfg::kBBytes, &tmap_b, &full_bar[stage], kc * BLOCK_K, tap, n0);
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumer warpgroups: wgmma main loop, then the epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cg = (warp - 4) >> 2;          // consumer warpgroup: tile rows [64 cg, 64 cg + 64)
    const int wg_warp = warp & 3;            // warp inside the warpgroup
    const int wg_tid = threadIdx.x & 127;
    // epilogue mapping after the exchange: warp (wg_warp) takes rows 32 (wg_warp & 1) .. +32 of the warpgroup's 64 and
    // the even (half 0) or odd (half 1) 32-column chunk of every 64-column pair
    const int half = wg_warp >> 1;
    const int r_loc = (wg_warp & 1) * 32 + lane;
    const int r = cg * 64 + r_loc;           // row inside the 128-row tile
    float* xch = xch_base + cg * 64 * XCH_STRIDE;
    uint8_t* stage_buf = stage_base + (warp - 4) * 4096;
    const int bar_id = 1 + cg;               // named barrier of this warpgroup (0 is __syncthreads)
    constexpr int kAcc = BLOCK_N / 2;
    int stage = 0; uint32_t phase = 0;
    for (int item = blockIdx.x; item < num_tiles; item += gridDim.x) {
      const int tile = item % num_out_tiles, ks = item / num_out_tiles;
      const int it0 = ks * k_iters / p.k_split, it1 = (ks + 1) * k_iters / p.k_split;
      const bool add_bias = ks == 0;  // K slice 0 carries the bias
      float acc[kAcc];
#pragma unroll
      for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int it = it0; it < it1; ++it) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t a_desc = make_smem_desc_sw128(smem_u32(smem_a + stage * Cfg::kABytes + cg * 64 * 128));
        const uint64_t b_desc = make_smem_desc_sw128(smem_u32(smem_b + stage * Cfg::kBBytes));
        fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k) {
          // advance 16 elements = 32 B along K inside the 128 B swizzle row: +2 in the (addr >> 4) field
          if constexpr (BLOCK_N == 256) wgmma_ss_n256<0, T>(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
          else wgmma_ss_n128<0, T>(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the MMAs of the previous stage have read their operands: release that stage
        fence_regs(acc);
        if (prev >= 0 && wg_tid == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0 && wg_tid == 0) mbar_arrive(&empty_bar[prev]);

      const int mt = tile / p.num_n_tiles, nt = tile % p.num_n_tiles;
      const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, img = mt / (p.tiles_x * p.tiles_y);
      const int px = tx * p.bw + r % p.bw, py = ty * p.bh + r / p.bw;
      const bool row_ok = (px < p.W) && (py < p.H) && (mt < p.num_m_tiles);
      const int m = (img * p.H + py) * p.W + px;
      const int n_valid = min(BLOCK_N / 32, (p.N - nt * BLOCK_N + 31) / 32);
      float fin[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int cp = 0; cp < BLOCK_N / 64; ++cp) {
        // fragments of columns [64 cp, 64 cp + 64) -> exchange tile -> one row-chunk per thread
        asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");  // previous reads of the exchange tile are done
        {
          const int fr = wg_warp * 16 + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int jj = cp * 8 + j;
            *reinterpret_cast<float2*>(xch + fr * XCH_STRIDE + 8 * j + fc) = make_float2(acc[4 * jj], acc[4 * jj + 1]);
            *reinterpret_cast<float2*>(xch + (fr + 8) * XCH_STRIDE + 8 * j + fc) =
                make_float2(acc[4 * jj + 2], acc[4 * jj + 3]);
          }
        }
        asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
        const int c = 2 * cp + half;
        if (c >= n_valid) continue;
        const int col0 = nt * BLOCK_N + c * 32;
        float v[32];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 t = *reinterpret_cast<const float4*>(xch + r_loc * XCH_STRIDE + half * 32 + 4 * i);
          v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
        }
        if (epilogue_rows(p, v, m, col0, row_ok, fin, add_bias, w4_smem) && !(p.debug & 1)) {
          if (p.tma_epi) {
            const bool to_b = p.split_col > 0 && col0 >= p.split_col;
            const int r0 = cg * 64 + (wg_warp & 1) * 32;  // first tile row of this warp
            epilogue_tma<T>(p, v, stage_buf, lane, to_b ? &tmap_o0b : &tmap_o0, p.tma_epi == 2,
                         to_b ? col0 - p.split_col : col0, tx * p.bw + (r0 & (p.bw - 1)), ty * p.bh + (r0 >> p.bw_log2),
                         mt < p.num_m_tiles ? img : p.NB);
          } else {
            const size_t off = out_offset(p, m, col0, img, py, px);
            ResChunk rc;
            prefetch_res(p, rc, off, row_ok, lane);
            epilogue_store<T>(p, v, rc, stage_buf, lane, m, col0, off, row_ok);
          }
        }
      }
      if (p.epi == EPI_FINAL) {
        // combine the two half-row partial dot products, then postprocess
        // (fast3r/dust3r/heads/postprocess.py:16-64): pts = xyz/|xyz| * expm1(|xyz|), conf = 1+exp(c)
        float* slot = fin_smem + r * 4;
        if (half == 1) { slot[0] = fin[0]; slot[1] = fin[1]; slot[2] = fin[2]; slot[3] = fin[3]; }
        asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
        if (half == 0 && row_ok) {
          const float x = fin[0] + slot[0] + __ldg(p.b4 + 0), y = fin[1] + slot[1] + __ldg(p.b4 + 1);
          const float z = fin[2] + slot[2] + __ldg(p.b4 + 2), c = fin[3] + slot[3] + __ldg(p.b4 + 3);
          const float d = sqrtf(x * x + y * y + z * z);
          const float sc = expm1f(d) / fmaxf(d, 1e-8f);
          float* pt = p.pts + static_cast<size_t>(m) * 3;
          pt[0] = x * sc; pt[1] = y * sc; pt[2] = z * sc;
          p.conf[m] = 1.f + expf(c);
        }
      }
    }
    if (p.tma_epi && lane == 0) tma_store_wait_all();  // bulk stores of this warp are complete before the CTA retires
  }
}

template <int BLOCK_N, typename T>
static cudaError_t launch_gemm_t(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to0,
                                 const CUtensorMap& to0b, const GemmArgs& a, int num_sms, cudaStream_t stream) {
  const int items = a.num_m_tiles * a.num_n_tiles * a.k_split;
  return launch(gemm_kernel<BLOCK_N, T>, items < num_sms ? items : num_sms, GEMM_THREADS, GemmCfg<BLOCK_N>::kSmemBytes,
                stream, true, ta, tb, to0, to0b, a);
}

cudaError_t launch_gemm(int block_n, int f16, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to0,
                        const CUtensorMap& to0b, const GemmArgs& a, int num_sms, cudaStream_t stream) {
  if (f16) {
    if (block_n == 256) return launch_gemm_t<256, __half>(ta, tb, to0, to0b, a, num_sms, stream);
    return launch_gemm_t<128, __half>(ta, tb, to0, to0b, a, num_sms, stream);
  }
  if (block_n == 256) return launch_gemm_t<256, __nv_bfloat16>(ta, tb, to0, to0b, a, num_sms, stream);
  return launch_gemm_t<128, __nv_bfloat16>(ta, tb, to0, to0b, a, num_sms, stream);
}

}  // namespace f3r
