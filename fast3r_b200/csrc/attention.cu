// FlashAttention-style forward for head_dim 64 on sm_90a: softmax(scale * Q K^T) V, non-causal, no mask
// (fast3r/croco/models/blocks.py:135-194; encoder: batch = views, S = P; fusion decoder: batch = B, S = N*P).
//
// One CTA owns ATT_Q_TILE = 192 query rows of one (batch, head) and streams all keys of its range in blocks of 128.
// Warpgroup 0 is the TMA producer (Q once, K/V blocks into a 128B-swizzled smem ring); warpgroups 1, 2 and 3 each own
// 64 query rows, so every K/V byte brought in from L2 serves 192 rows: S = Q K^T is a wgmma with both operands in shared
// memory (S stays in registers), P is packed to bf16 in registers and used directly as the register A operand of
// O += P V (V consumed MN-major from shared memory, no transpose).  Every consumer warpgroup runs the whole key loop
// and releases every stage, also when all its rows lie past sq (the producer waits for three releases per stage); only
// its stores are masked.
// Softmax is exact online softmax in fp32 (exp2 domain) with lazy O rescaling: the running reference max is only
// moved when the row max grows by more than 2^8.
//
// At head dim 64 the tensor pipe (256 MMA FLOP per score) and the MUFU ex2 (one per score) need the same time, so the
// consumers overlap them (the intra-warpgroup pipelining of FlashAttention-3): S_{j+1} = Q K_{j+1}^T and O += P_j V_j
// are issued back to back, the softmax of S_{j+1} runs while the PV is still on the tensor core, and only then is O
// rescaled and P_{j+1} packed.  The consumer warpgroups are not ordered against each other: a named-barrier
// ping-pong (one warpgroup issues its GEMMs while the other is in its softmax) measured 2-4 % slower on top of this
// with two consumer warpgroups.
// The arithmetic (ex2 inputs, order of the l and O updates, lazy-rescale decisions) is that of a loop that finishes one
// key block before it starts the next, so the overlap does not change a bit of the result.
// fp16 (attention_kernel<..., __half>, the f3r_attention*_f16 entry points): Q, K, V, P and O are fp16 instead of bf16,
// with the same tiles, pipeline and fp32 softmax; P is packed with cvt.rn.f16x2.f32.
// Segment mode (attention_kernel<true, T>, f3r_attention_segments): block-diagonal attention over the segments of one packed
// sequence, each segment with the arithmetic of a launch over it alone.
#include "common.cuh"
#include "f3r_kernels.h"

namespace f3r {

constexpr int ATT_CONSUMERS = ATT_Q_TILE / 64;          // consumer warpgroups, 64 query rows each
constexpr int ATT_THREADS = 128 * (1 + ATT_CONSUMERS);   // + the producer warpgroup
constexpr int ATT_STAGES = 3;
constexpr int ATT_TILE_BYTES = 128 * 64 * 2;             // 16 KB: one K or V block, 128 keys x 64 bf16
constexpr int ATT_Q_BYTES = ATT_Q_TILE * 64 * 2;         // 24 KB
constexpr int ATT_SMEM_BYTES = ATT_Q_BYTES + 2 * ATT_STAGES * ATT_TILE_BYTES + 1024 + 256;
static_assert(ATT_Q_TILE == 192, "the register split below (setmaxnreg 24 / 160) is sized for three consumer warpgroups");
static_assert(ATT_Q_BYTES % 1024 == 0, "the K/V ring after Q must stay 1024-byte aligned (128B swizzle atoms)");

F3R_DEVICE float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// S (64 rows x 128 keys of this warpgroup) = Q K^T, four k16 steps; committed as one wgmma group
template <typename T>
F3R_DEVICE void att_issue_s(float (&s)[64], uint64_t qd, const uint8_t* smem_k_stage) {
  const uint64_t kd = make_smem_desc_sw128(smem_u32(smem_k_stage));
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_ss_n128<0, T>(s, qd + 2 * k, kd + 2 * k, k > 0 ? 1u : 0u);
  wgmma_commit();
}

// O += P V, eight k16 steps of 16 keys (16 smem rows = 2048 B of V); committed as one wgmma group
template <typename T>
F3R_DEVICE void att_issue_pv(float (&o)[32], const uint32_t (&pa)[8][4], const uint8_t* smem_v_stage) {
  const uint64_t vd = make_smem_desc_sw128(smem_u32(smem_v_stage));
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) wgmma_rs_n64<1, T>(o, pa[kk], vd + 128 * kk, 1u);
  wgmma_commit();
}

// Online softmax of one key block, in place: s becomes exp2(S sl2 - m sl2).  Keys >= valid are masked.  Updates the
// reference max and the row sums; the O rescale it decides (resc / alpha per row half) is applied by the caller once
// no PV that accumulates into O is in flight.
F3R_DEVICE void att_softmax(float (&s)[64], int valid, int cq, float sl2, float (&m_used)[2], float (&l)[2],
                            bool (&resc)[2], float (&alpha)[2]) {
  if (valid < 128) {
#pragma unroll
    for (int i = 0; i < 64; ++i)
      if (8 * (i >> 2) + cq + (i & 1) >= valid) s[i] = -INFINITY;
  }
  float nm[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float mx = fmaxf(s[2 * hh], s[2 * hh + 1]);
#pragma unroll
    for (int jn = 1; jn < 16; ++jn) mx = fmaxf(mx, fmaxf(s[4 * jn + 2 * hh], s[4 * jn + 2 * hh + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    // lazy rescale: move the reference only if the max grew by more than 8 (log2 domain)
    resc[hh] = (mx - m_used[hh]) * sl2 > 8.f;  // (-inf reference => true)
    if (resc[hh]) {
      alpha[hh] = ex2_approx((m_used[hh] - mx) * sl2);  // exp2(-inf) = 0 on the first block
      m_used[hh] = mx;
      l[hh] *= alpha[hh];
    }
    nm[hh] = -m_used[hh] * sl2;
  }
  // k-step kk of the PV covers key columns [16 kk, 16 kk + 16): s[8 kk + 2 r + {0, 1}], row half r & 1
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = 8 * kk + 2 * r, hh = r & 1;
      const float e0 = ex2_approx(fmaf(s[i], sl2, nm[hh])), e1 = ex2_approx(fmaf(s[i + 1], sl2, nm[hh]));
      l[hh] += e0 + e1;
      s[i] = e0;
      s[i + 1] = e1;
    }
  }
}

// After the last PV that read pa has landed: O *= alpha where the softmax moved the reference, then P -> 16-bit A
// fragments
template <typename T>
F3R_DEVICE void att_rescale_pack(float (&o)[32], uint32_t (&pa)[8][4], const float (&s)[64], const bool (&resc)[2],
                                 const float (&alpha)[2]) {
#pragma unroll
  for (int hh = 0; hh < 2; ++hh)
    if (resc[hh]) {
#pragma unroll
      for (int jn = 0; jn < 8; ++jn) { o[4 * jn + 2 * hh] *= alpha[hh]; o[4 * jn + 2 * hh + 1] *= alpha[hh]; }
    }
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) pa[kk][r] = Half16<T>::pack(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
}

// Segment mode: finds the segment of work item `item`.  Items are numbered segment by segment, heads * n_split per query
// tile of the segment; the warp scans the segments' query-tile counts 32 at a time.  Returns false past the last item
// (the grid is sized by an upper bound of the tile count).  local: the item's index inside its segment.
F3R_DEVICE bool att_find_segment(const AttnArgs& p, int item, int& s0, int& len, int& local) {
  const int lane = threadIdx.x & 31;
  const int per_tile = p.heads * p.n_split;
  const int tile = item / per_tile;  // query tile of the item, counted over all segments
  int base = 0;                      // query tiles of the segments before this step's first
  for (int c = 0; c < p.n_seg; c += 32) {
    const int i = c + lane;
    const int t = i < p.n_seg ? (max(__ldg(p.seg_off + i + 1) - __ldg(p.seg_off + i), 0) + ATT_Q_TILE - 1) / ATT_Q_TILE : 0;
    int incl = t;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += y;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, base + incl > tile);
    if (hit) {
      const int l = __ffs(hit) - 1;
      const int before = base + __shfl_sync(0xffffffffu, incl - t, l);
      s0 = __ldg(p.seg_off + c + l);
      len = __ldg(p.seg_off + c + l + 1) - s0;  // > 0: the segment has a query tile
      local = item - before * per_tile;
      return true;
    }
    base += __shfl_sync(0xffffffffu, incl, 31);
  }
  return false;
}

// kSeg = false: p.batch independent sequences of p.sq queries / p.skv keys.
// kSeg = true: one packed sequence of p.sq rows cut into p.n_seg segments (p.seg_off); each segment attends to its own
// rows only, with key blocks that start at its first row, so its rows get exactly the arithmetic of a kSeg = false launch
// over that segment alone.  A segment with fewer key blocks than p.n_split uses one slice per key block and fills the
// slots of its other slices with neutral partials (O = 0, LSE = -inf: merge weight 0).
// T: the type of Q, K, V and O (__nv_bfloat16 or __half).
template <bool kSeg, typename T>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_kv,
                 const __grid_constant__ AttnArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;                                   // ATT_Q_TILE rows
  uint8_t* smem_k = smem + ATT_Q_BYTES;                     // ATT_STAGES tiles
  uint8_t* smem_v = smem_k + ATT_STAGES * ATT_TILE_BYTES;   // ATT_STAGES tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_v + ATT_STAGES * ATT_TILE_BYTES);
  uint64_t* q_full = bars;                       // 1
  uint64_t* k_full = bars + 1;                   // ATT_STAGES
  uint64_t* k_empty = k_full + ATT_STAGES;
  uint64_t* v_full = k_empty + ATT_STAGES;
  uint64_t* v_empty = v_full + ATT_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // work item = (unit = (batch or segment, head, query tile of ATT_Q_TILE rows), split = slice of the key blocks of the
  // unit's key range).  sq / skv: queries / keys of the unit; s0: its first row in the packed sequence (segment mode)
  int split, qt, h, b, sq, skv, n_split, s0 = 0, kv_row0 = p.kv_row0;
  if constexpr (!kSeg) {
    const int unit = blockIdx.x / p.n_split;
    split = blockIdx.x % p.n_split;
    qt = unit % p.q_tiles;
    const int bh = unit / p.q_tiles;
    h = bh % p.heads;
    b = bh / p.heads;
    sq = p.sq; skv = p.skv; n_split = p.n_split;
  }
  const int dmodel = p.heads * 64;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_kv);
    mbar_init(q_full, 1);
    for (int s = 0; s < ATT_STAGES; ++s) {
      mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], ATT_CONSUMERS);  // released by every consumer warpgroup
      mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], ATT_CONSUMERS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                // q / kv come from the preceding QKV GEMM: no global access above this line
  pdl_launch_dependents();

  if constexpr (kSeg) {
    int local;
    if (!att_find_segment(p, blockIdx.x, s0, sq, local)) return;
    skv = sq;
    kv_row0 = s0;
    b = 0;
    split = local % p.n_split;
    const int unit = local / p.n_split;
    const int q_tiles = (sq + ATT_Q_TILE - 1) / ATT_Q_TILE;
    qt = unit % q_tiles;
    h = unit / q_tiles;
    n_split = min(p.n_split, (skv + 127) / 128);
    if (split >= n_split) {
      // no key block left for this slice (only with part_o, host-checked): a neutral partial for the merge
      const size_t slot = static_cast<size_t>(p.part_base + split);
      const int q0 = s0 + qt * ATT_Q_TILE, rows = min(ATT_Q_TILE, sq - qt * ATT_Q_TILE);
      for (int i = threadIdx.x; i < rows * 16; i += ATT_THREADS)
        *reinterpret_cast<float4*>(p.part_o + (slot * p.sq + q0 + (i >> 4)) * dmodel + h * 64 + 4 * (i & 15)) =
            make_float4(0.f, 0.f, 0.f, 0.f);
      for (int i = threadIdx.x; i < rows; i += ATT_THREADS)
        p.part_lse[(slot * p.heads + h) * p.sq + q0 + i] = -INFINITY;
      return;
    }
  }
  const int nkv_all = (skv + 127) / 128;
  const int j0 = static_cast<int>(static_cast<long long>(split) * nkv_all / n_split);  // first key block of this CTA
  const int nkv = static_cast<int>(static_cast<long long>(split + 1) * nkv_all / n_split) - j0;  // (>= 1, host-checked)

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");   // 128 x 24 + 384 x 160 <= 64K registers
    if (warp == 0 && lane == 0) {
      // ===================== TMA producer =====================
      // (Q rows past sq are zero-filled by the TMA unit and still count towards the transaction bytes)
      mbar_arrive_expect_tx(q_full, ATT_Q_BYTES);
      // (segment mode: the Q rows past the segment are the next segment's; they are computed and never stored)
      tma_load_3d(smem_q, &tmap_q, q_full, h * 64, s0 + qt * ATT_Q_TILE, b);
      int stage = 0; uint32_t phase = 0;
      for (int j = 0; j < nkv; ++j) {
        mbar_wait_relaxed(&k_empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&k_full[stage], ATT_TILE_BYTES);
        tma_load_3d(smem_k + stage * ATT_TILE_BYTES, &tmap_kv, &k_full[stage], h * 64, kv_row0 + (j0 + j) * 128, b);
        mbar_wait_relaxed(&v_empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&v_full[stage], ATT_TILE_BYTES);
        tma_load_3d(smem_v + stage * ATT_TILE_BYTES, &tmap_kv, &v_full[stage], dmodel + h * 64,
                    kv_row0 + (j0 + j) * 128, b);
        if (++stage == ATT_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ===================== consumer warpgroups: 64 query rows each =====================
    // accumulator fragments (common.cuh): this thread holds rows rw + 8 hh (hh = 0, 1) and, in every 8-column group jn,
    // the columns 8 jn + 2 (lane % 4) + {0, 1}
    asm volatile("setmaxnreg.inc.sync.aligned.u32 160;");
    const int cg = (warp - 4) >> 2;
    const int wg_tid = threadIdx.x & 127;
    const int rw = cg * 64 + (warp & 3) * 16 + (lane >> 2);  // first of the thread's two rows in the query tile
    const int cq = 2 * (lane & 3);
    const float sl2 = p.scale_log2;
    float m_used[2] = {-INFINITY, -INFINITY};  // raw-score reference max the exponentials are taken against
    float l[2] = {0.f, 0.f};                   // this thread's partial row sums (its 32 of the 128 columns)
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float s[64];         // S of the block in softmax, then its exponentials until they are packed
    uint32_t pa[8][4];   // P of the block whose PV is in flight (16-bit A fragments)
    bool resc[2];        // O rescale decided by the latest softmax ...
    float alpha[2];      // ... and its factor
    const uint64_t qd = make_smem_desc_sw128(smem_u32(smem_q + cg * 64 * 128));
    // keys valid in key block j of this CTA: only the last block of the launch's key range is partial
    auto valid_keys = [&](int j) { return j0 + j == nkv_all - 1 ? skv - (j0 + j) * 128 : 128; };
    mbar_wait(q_full, 0);

    // block 0: S_0 and its softmax
    mbar_wait(&k_full[0], 0);
    wgmma_fence();
    att_issue_s<T>(s, qd, smem_k);
    wgmma_wait<0>();
    fence_regs(s);
    if (wg_tid == 0) mbar_arrive(&k_empty[0]);
    att_softmax(s, valid_keys(0), cq, sl2, m_used, l, resc, alpha);

    // steady state: on entry the softmax of S_j is done and PV_{j-1} may be in flight.  S_{j+1} and PV_j go out
    // together and the softmax of S_{j+1} runs under PV_j.  The wait for PV_j sits at the top of the next trip, behind
    // the mbarrier polls: the instruction scheduler hoists a wgmma wait above independent math in the same basic block,
    // which would put the softmax back behind the PV.
    for (int j = 0; j + 1 < nkv; ++j) {
      const int sk = (j + 1) % ATT_STAGES, sv = j % ATT_STAGES;
      mbar_wait(&k_full[sk], ((j + 1) / ATT_STAGES) & 1);
      mbar_wait(&v_full[sv], (j / ATT_STAGES) & 1);
      wgmma_wait<0>();  // PV_{j-1} has landed: O may be rescaled and the P registers rewritten
      fence_regs(o);
      if (j > 0 && wg_tid == 0) mbar_arrive(&v_empty[(j - 1) % ATT_STAGES]);
      att_rescale_pack<T>(o, pa, s, resc, alpha);
      wgmma_fence();
      att_issue_s<T>(s, qd, smem_k + sk * ATT_TILE_BYTES);
      att_issue_pv<T>(o, pa, smem_v + sv * ATT_TILE_BYTES);
      wgmma_wait<1>();  // S_{j+1} has landed (groups complete in order)
      fence_regs(s);
      if (wg_tid == 0) mbar_arrive(&k_empty[sk]);
      att_softmax(s, valid_keys(j + 1), cq, sl2, m_used, l, resc, alpha);
    }

    // last block: PV only
    {
      const int sv = (nkv - 1) % ATT_STAGES;
      mbar_wait(&v_full[sv], ((nkv - 1) / ATT_STAGES) & 1);
      if constexpr (kSeg) {
        // The V rows past the segment's end belong to the next segment.  Their scores are masked, but P = 0 times a NaN
        // or Inf in V would still reach O, so they enter the PV product as zeros, as the TMA zero fill gives a single-
        // segment launch.  A 128B-swizzled row stays within its own 128 bytes, so whole rows are zeroed.
        const int valid = valid_keys(nkv - 1);
        if (valid < 128) {
          uint4* v4 = reinterpret_cast<uint4*>(smem_v + sv * ATT_TILE_BYTES + valid * 128);
          for (int i = threadIdx.x - 128; i < (128 - valid) * 8; i += 128 * ATT_CONSUMERS) v4[i] = make_uint4(0, 0, 0, 0);
          fence_proxy_async_smem();  // generic-proxy stores before the wgmma (async proxy) reads
          asm volatile("bar.sync 1, %0;" ::"n"(128 * ATT_CONSUMERS) : "memory");  // all consumer warpgroups
        }
      }
      wgmma_wait<0>();
      fence_regs(o);
      if (nkv > 1 && wg_tid == 0) mbar_arrive(&v_empty[(nkv - 2) % ATT_STAGES]);
      att_rescale_pack<T>(o, pa, s, resc, alpha);
      wgmma_fence();
      att_issue_pv<T>(o, pa, smem_v + sv * ATT_TILE_BYTES);
      wgmma_wait<0>();
      fence_regs(o);
      if (wg_tid == 0) mbar_arrive(&v_empty[sv]);
    }

    // ---- epilogue: O / l -> global
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
      l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int q = qt * ATT_Q_TILE + rw + 8 * hh;
      if (q >= sq) continue;
      const int qs = kSeg ? s0 + q : q;  // row in the per-batch sequence of p.sq rows
      if (kSeg && qs >= p.sq) continue;  // (segment offsets past the buffer)
      const float inv = 1.f / l[hh];
      const float lse = m_used[hh] * sl2 * 0.69314718056f + logf(l[hh]);
      if (p.part_o != nullptr) {
        // partial result of this key slice: normalised fp32 O and its log-sum-exp; f3r_attention_merge combines slices
        const size_t slot = static_cast<size_t>(p.part_base + split);
        float* dstf = p.part_o + (slot * p.batch * p.sq + static_cast<size_t>(b) * p.sq + qs) * dmodel + h * 64 + cq;
#pragma unroll
        for (int jn = 0; jn < 8; ++jn)
          *reinterpret_cast<float2*>(dstf + 8 * jn) = make_float2(o[4 * jn + 2 * hh] * inv, o[4 * jn + 2 * hh + 1] * inv);
        if ((lane & 3) == 0) p.part_lse[(slot * p.batch * p.heads + static_cast<size_t>(b) * p.heads + h) * p.sq + qs] = lse;
      } else {
        T* dst = static_cast<T*>(p.out) + (static_cast<size_t>(b) * p.sq + qs) * p.ldo + h * 64 + cq;
#pragma unroll
        for (int jn = 0; jn < 8; ++jn)
          *reinterpret_cast<uint32_t*>(dst + 8 * jn) =
              Half16<T>::pack(o[4 * jn + 2 * hh] * inv, o[4 * jn + 2 * hh + 1] * inv);
        if (p.lse != nullptr && (lane & 3) == 0) p.lse[(static_cast<size_t>(b) * p.heads + h) * p.sq + qs] = lse;
      }
    }
  }
}

cudaError_t launch_attention(const CUtensorMap& tq, const CUtensorMap& tkv, const AttnArgs& a, int f16,
                             cudaStream_t stream) {
  return launch(f16 ? attention_kernel<false, __half> : attention_kernel<false, __nv_bfloat16>,
                a.batch * a.heads * a.q_tiles * a.n_split, ATT_THREADS, ATT_SMEM_BYTES, stream, true, tq, tkv, a);
}

cudaError_t launch_attention_segments(const CUtensorMap& tq, const CUtensorMap& tkv, const AttnArgs& a, int max_tiles,
                                      int f16, cudaStream_t stream) {
  return launch(f16 ? attention_kernel<true, __half> : attention_kernel<true, __nv_bfloat16>,
                a.heads * a.n_split * max_tiles, ATT_THREADS, ATT_SMEM_BYTES, stream, true, tq, tkv, a);
}

// ---------------------------------------------------------------- merge of key-slice partials
// out[row, h*64 + d] = sum_p w_p O_p[row, h, d] / sum_p w_p,  w_p = exp(lse_p - max_p lse_p): the exact softmax over the
// union of the slices (each O_p is normalised over its own slice).  8 threads per (row, head), 8 columns each.  T: the
// type of out (__nv_bfloat16 or __half).
template <typename T>
__global__ void __launch_bounds__(256) attention_merge_kernel(const float* __restrict__ part_o,
                                                              const float* __restrict__ part_lse, int n_parts, int batch,
                                                              int heads, int sq, T* __restrict__ out, int ldo) {
  pdl_wait();                // the partials come from the preceding attention launches
  pdl_launch_dependents();
  const size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t rows = static_cast<size_t>(batch) * sq;
  if (idx >= rows * heads * 8) return;
  const int g = idx & 7;
  const int h = (idx >> 3) % heads;
  const size_t m = (idx >> 3) / heads;  // row = b * sq + q
  const int b = static_cast<int>(m / sq), q = static_cast<int>(m % sq);
  const int dm = heads * 64;
  const size_t lse_i = (static_cast<size_t>(b) * heads + h) * sq + q, lse_stride = static_cast<size_t>(batch) * heads * sq;
  float mx = -INFINITY;
  for (int p = 0; p < n_parts; ++p) mx = fmaxf(mx, __ldg(part_lse + p * lse_stride + lse_i));
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float wsum = 0.f;
  for (int p = 0; p < n_parts; ++p) {
    const float w = __expf(__ldg(part_lse + p * lse_stride + lse_i) - mx);
    wsum += w;
    const float4* src = reinterpret_cast<const float4*>(part_o + (p * rows + m) * dm + h * 64 + g * 8);
    const float4 a = __ldg(src), c = __ldg(src + 1);
    acc[0] += w * a.x; acc[1] += w * a.y; acc[2] += w * a.z; acc[3] += w * a.w;
    acc[4] += w * c.x; acc[5] += w * c.y; acc[6] += w * c.z; acc[7] += w * c.w;
  }
  const float inv = 1.f / wsum;
  uint4 o;
  using H = Half16<T>;
  o.x = H::pack(acc[0] * inv, acc[1] * inv); o.y = H::pack(acc[2] * inv, acc[3] * inv);
  o.z = H::pack(acc[4] * inv, acc[5] * inv); o.w = H::pack(acc[6] * inv, acc[7] * inv);
  *reinterpret_cast<uint4*>(out + m * ldo + h * 64 + g * 8) = o;
}
cudaError_t launch_attention_merge(const float* part_o, const float* part_lse, int n_parts, int batch, int heads, int sq,
                                   void* out, int ldo, int f16, cudaStream_t stream) {
  const size_t total = static_cast<size_t>(batch) * sq * heads * 8;
  if (total == 0) return cudaSuccess;
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  if (f16)
    return launch(attention_merge_kernel<__half>, grid, 256, 0, stream, true, part_o, part_lse, n_parts, batch, heads, sq,
                  static_cast<__half*>(out), ldo);
  return launch(attention_merge_kernel<__nv_bfloat16>, grid, 256, 0, stream, true, part_o, part_lse, n_parts, batch,
                heads, sq, static_cast<__nv_bfloat16*>(out), ldo);
}

}  // namespace f3r
