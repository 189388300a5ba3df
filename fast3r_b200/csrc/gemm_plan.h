// Launch plan of f3r_gemm: the pixel tile, BLOCK_N, the epilogue and the K split chosen for one descriptor.  Host-only
// and free of CUDA, so that tests/gemm_plan_host.cpp compiles the same rule with g++ and the test suite can tell which
// code path of gemm_kernel a call reaches.
#pragma once
#include "../../include/fast3r_b200.h"

namespace f3r {

struct GemmPlan {
  int bw, bh, bw_log2;      // pixel tile bw x bh = 128 rows, bw a power of two
  int sbx_log2;             // TMA-store box = (32 ch, sbx, 32/sbx) pixels, sbx = min(bw, 32)
  int tiles_x, tiles_y, num_m_tiles;
  int block_n, num_n_tiles;
  int tma_epi;              // 0: generic epilogue, 1: TMA store of out0(/out0b), 2: TMA reduce-add into fp32 out0
  int k_split;              // K slices per output tile (> 1 only with tma_epi == 2)
};

// d: a descriptor that passed f3r_gemm's argument checks.  num_sms: SMs of the device.  allow_tma_epi /
// allow_k_split: the F3R_GEMM_TMA_EPI / F3R_GEMM_KSPLIT preferences (1 = the default: allowed).
inline GemmPlan gemm_plan(const f3r_gemm_desc& d, int num_sms, int allow_tma_epi, int allow_k_split) {
  GemmPlan p;
  // pixel tile (bw x bh = 128) minimising the number of tiles
  int best_bw = 128;
  long best_tiles = -1;
  for (int bw = 128; bw >= 1; bw >>= 1) {
    const int bh = 128 / bw;
    const long tiles = static_cast<long>((d.w + bw - 1) / bw) * ((d.h + bh - 1) / bh);
    if (best_tiles < 0 || tiles < best_tiles) { best_tiles = tiles; best_bw = bw; }
  }
  p.bw = best_bw; p.bh = 128 / best_bw;
  p.bw_log2 = 0;
  while ((1 << p.bw_log2) < p.bw) ++p.bw_log2;
  p.sbx_log2 = p.bw_log2 < 5 ? p.bw_log2 : 5;
  p.tiles_x = (d.w + p.bw - 1) / p.bw; p.tiles_y = (d.h + p.bh - 1) / p.bh;
  p.num_m_tiles = p.tiles_x * p.tiles_y * d.nb;
  p.block_n = 128;
  if (d.epi != F3R_EPI_FINAL && d.n > 128) {
    const long tiles256 = static_cast<long>(p.num_m_tiles) * ((d.n + 255) / 256);
    if (tiles256 >= num_sms) p.block_n = 256;
  }
  p.num_n_tiles = (d.n + p.block_n - 1) / p.block_n;
  // TMA epilogue for the hot cases: plain stores, and the in-place fp32 residual update as a reduce-add.  The reduce-add
  // adds the epilogue's value to out0 (and with a K split, each slice adds its own), so it only implements
  // out0 = res0 + v when v is linear in the accumulator and is added once: no activation (act(res0 + v) is not
  // res0 + act(v)) and no image-index embedding (it would be added once per K slice).  Everything else takes the
  // generic epilogue, which reads res0 and writes out0 at the same offset in the same lane, so aliasing is safe there.
  p.tma_epi = 0;
  const bool plain = (d.epi == F3R_EPI_STORE || d.epi == F3R_EPI_ROPE || d.epi == F3R_EPI_IDXEMB) && d.out0 &&
                     !d.out1 && !d.res1;
  if (allow_tma_epi && plain && !d.res0) p.tma_epi = 1;
  else if (allow_tma_epi && plain && d.res0 == d.out0 && d.res0_f32 && d.out0_f32 && !d.split_col &&
           d.act == F3R_ACT_NONE && d.epi != F3R_EPI_IDXEMB)
    p.tma_epi = 2;
  p.k_split = 1;
  if (p.tma_epi == 2 && d.taps == 1 && allow_k_split) {
    // x += A W^T with fewer output tiles than SMs: cut K into slices, each CTA reduce-adds its partial sum
    const long slots = num_sms;
    const long items = static_cast<long>(p.num_m_tiles) * p.num_n_tiles;
    const int k_iters = (d.k + 63) / 64;
    double best = 1e30;
    for (int s = 1; s <= 4 && (s == 1 || k_iters / s >= 16); ++s) {  // (short K: the reduce-add epilogue dominates, slicing loses)
      const double cost = static_cast<double>((items * s + slots - 1) / slots) / s * (1.0 + 0.03 * (s - 1));
      if (cost < best - 1e-9) { best = cost; p.k_split = s; }
    }
  }
  return p;
}

}  // namespace f3r
