// Host build of the launch-plan rule of f3r_gemm (fast3r_b200/csrc/gemm_plan.h), so that the tests compute the plan a
// descriptor reaches with the library's own code.  Compiled by tests/gemm_plans.py with g++.
#include "gemm_plan.h"

// out: bw, bh, bw_log2, sbx_log2, tiles_x, tiles_y, num_m_tiles, block_n, num_n_tiles, tma_epi, k_split
extern "C" void f3r_test_gemm_plan(const f3r_gemm_desc* d, int num_sms, int allow_tma_epi, int allow_k_split, int* out) {
  const f3r::GemmPlan p = f3r::gemm_plan(*d, num_sms, allow_tma_epi, allow_k_split);
  const int v[11] = {p.bw, p.bh, p.bw_log2, p.sbx_log2, p.tiles_x, p.tiles_y, p.num_m_tiles, p.block_n, p.num_n_tiles,
                     p.tma_epi, p.k_split};
  for (int i = 0; i < 11; ++i) out[i] = v[i];
}

extern "C" unsigned long f3r_test_gemm_desc_size(void) { return sizeof(f3r_gemm_desc); }
