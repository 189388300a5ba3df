// Internal launch interfaces between capi.cu and the kernel translation units.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <utility>

#include "../../include/fast3r_b200.h"

namespace f3r {

// 1: launch the hot-chain kernels with programmatic stream serialization (PDL); F3R_PDL=0 / f3r_set_option("pdl", 0) disable
extern int g_pdl;
bool pdl_enabled();
// kernels launched by launch() so far (f3r_launch_count)
extern std::atomic<uint64_t> g_launch_count;

// Every kernel of the library is launched here, so g_launch_count counts exactly the launches that were enqueued.
// pdl: programmatic stream serialization (if pdl_enabled()), for the kernels that execute griddepcontrol.
// kCluster > 1: thread-block clusters of kCluster CTAs along x.  Dynamic shared memory above 48 KB is opted into on
// every launch: the attribute is per device and one process may drive several GPUs.
template <int kCluster = 1, typename... Params, typename... Args>
cudaError_t launch(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                   Args&&... args) {
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
  }
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = attr;
  if (kCluster > 1) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeClusterDimension;
    attr[cfg.numAttrs].val.clusterDim.x = kCluster;
    attr[cfg.numAttrs].val.clusterDim.y = 1;
    attr[cfg.numAttrs].val.clusterDim.z = 1;
    ++cfg.numAttrs;
  }
  if (pdl && pdl_enabled()) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[cfg.numAttrs].val.programmaticStreamSerializationAllowed = 1;
    ++cfg.numAttrs;
  }
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  if (e != cudaSuccess) {
    cudaGetLastError();  // the error is returned here; do not leave it behind for the caller's next CUDA error check
    return e;
  }
  ++g_launch_count;
  return e;
}

enum { EPI_STORE = 0, EPI_ROPE = 1, EPI_IDXEMB = 2, EPI_CONVT = 3, EPI_FINAL = 4 };
enum { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2 };

struct GemmArgs {
  int M, N, K, taps;
  int W, H, NB, bw, bh, tiles_x, tiles_y;
  int bw_log2;  // bw is a power of two
  int num_m_tiles, num_n_tiles;
  int epi, act, out0_f32, res0_f32;
  int ldo;               // row stride (elements) of out0 / out1 / res0 / res1
  int split_col, ldo_b;  // columns >= split_col go to out0b (row stride ldo_b); 0 = no split
  int tok_per_img, grid_w, rope_cols;  // EPI_ROPE / EPI_IDXEMB
  int ct_k, ct_cout;                   // EPI_CONVT
  int tma_epi;                         // 0: generic epilogue, 1: TMA store of out0(/out0b), 2: TMA reduce-add into fp32 out0
  int sbx_log2;                        // TMA-store box = (32 ch, sbx, 32/sbx) pixels, sbx = min(bw, 32)
  int k_split;                         // K slices per output tile (>1 only with tma_epi == 2: partial sums reduce-added)
  int debug;                           // F3R_GEMM_DEBUG bitmask (1: no epilogue stores) - timing experiments only
  const float* bias;
  const void* res0;
  const void* res1;
  void* out0;
  void* out0b;
  void* out1;
  const float* rope_cos;
  const float* rope_sin;
  const float* emb_table;
  const int* emb_ids;
  const float* w4;
  const float* b4;
  float* pts;
  float* conf;
};

// f16: A, the weights and every 16-bit output / residual are fp16 instead of bf16
cudaError_t launch_gemm(int block_n, int f16, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to0,
                        const CUtensorMap& to0b, const GemmArgs& a, int num_sms, cudaStream_t stream);

// query rows per CTA of attention_kernel: three consumer warpgroups of 64 rows (ops.ATT_Q_TILE on the Python side)
constexpr int ATT_Q_TILE = 192;

struct AttnArgs {
  int batch, heads, sq, skv;  // per-batch query / key lengths
  int q_tiles;                // ceil(sq / ATT_Q_TILE) (attention_x3: ceil(sq / 128))
  float scale_log2;           // softmax scale * log2(e)
  int ldo;                    // row stride of out (elements)
  void* out;                  // 16-bit [batch*sq, ldo] (bf16, or fp16 with f16), head h at columns h*64
  float* lse;                 // optional fp32 [batch, heads, sq] log-sum-exp (natural log)
  // key range of this launch inside the kv buffer: rows [kv_row0, kv_row0 + skv) of every batch
  int kv_row0;
  // key-slice partials: the key blocks are cut into n_split slices (one CTA each per query tile); with part_o != NULL
  // slice s writes its normalised fp32 output / LSE into slot part_base + s (merged by launch_attention_merge)
  int n_split;
  int part_base;
  float* part_o;              // fp32 [slots, batch*sq, heads*64]
  float* part_lse;            // fp32 [slots, batch, heads, sq]
  // segment mode (launch_attention_segments): batch = 1, sq = skv = all rows; segment s is rows
  // [seg_off[s], seg_off[s+1]) and attends to its own rows only
  const int* seg_off;         // device int32 [n_seg + 1]
  int n_seg;
};
// f16: q, kv and out are fp16 instead of bf16
cudaError_t launch_attention_merge(const float* part_o, const float* part_lse, int n_parts, int batch, int heads, int sq,
                                   void* out, int ldo, int f16, cudaStream_t stream);
cudaError_t launch_attention(const CUtensorMap& tq, const CUtensorMap& tkv, const AttnArgs& a, int f16,
                             cudaStream_t stream);
// segment mode: grid of heads * n_split * max_tiles CTAs, max_tiles >= the total query tiles of all segments
cudaError_t launch_attention_segments(const CUtensorMap& tq, const CUtensorMap& tkv, const AttnArgs& a, int max_tiles,
                                      int f16, cudaStream_t stream);

// parity mode (attention_x3.cu): hi/lo-split bf16 operands, fp32 out (AttnArgs.out is float*)
cudaError_t launch_attention_x3(const CUtensorMap& tq3, const CUtensorMap& tk3, const CUtensorMap& tv2,
                                const AttnArgs& a, cudaStream_t stream);
cudaError_t launch_attn_split(const float* q, int ldq, const float* kv, int ldkv, void* q3, void* k3, void* v2,
                              size_t rows_q, size_t rows_kv, int heads, cudaStream_t stream);
cudaError_t launch_split3(const float* in, void* out, size_t rows, int k, int relu, cudaStream_t stream);
cudaError_t launch_add_f32(float* dst, const float* src, size_t n, cudaStream_t stream);

// element-type codes of f3r_layernorm / f3r_im2col_patch / f3r_upsample2x
enum { ELT_BF16 = 0, ELT_F32 = 1, ELT_F16 = 2 };
cudaError_t launch_layernorm(const float* x, const float* w, const float* b, void* out, int out_type, int rows,
                             int dim, float eps, cudaStream_t stream);
cudaError_t launch_im2col_patch(const float* img, void* out, int out_type, int n, int H, int W, int patch,
                                cudaStream_t stream);
cudaError_t launch_im2col3x3s2(const void* in, void* out, int n, int H, int W, int C, int Ho, int Wo,
                               cudaStream_t stream);
cudaError_t launch_upsample2x(const void* in, void* out, int elt, int n, int H, int W, int C, int Ho, int Wo,
                              int Hfull, int Wfull, cudaStream_t stream);
cudaError_t launch_cast_bf16(const float* in, void* out, size_t n, cudaStream_t stream);
cudaError_t launch_cast_f16(const float* in, void* out, size_t n, cudaStream_t stream);

// baseline JPEG decode (jpeg.cu); both return nullptr or the reason of the failure
const char* jpeg_probe(const uint8_t* data, size_t size, f3r_jpeg_info* info);
const char* launch_jpeg_decode(const uint8_t* data, size_t size, const uint8_t* data_dev, int orientation, int rotate_cw90,
                               int left, int top, int out_w, int out_h, uint8_t* out, int32_t* status, void* workspace,
                               size_t workspace_bytes, cudaStream_t stream);

// image ingest (ingest.cu)
int resample_ksize(int in_size, int out_size, int filter);
int resample_coeffs(int in_size, int out_size, int filter, int32_t* bounds, int32_t* kk);
cudaError_t launch_ingest(const uint8_t* src, int h, int w, int oh, int ow, const int32_t* hb, const int32_t* hk, int hks,
                          int h_span_max, const int32_t* vb, const int32_t* vk, int vks, uint8_t* tmp, int left, int top,
                          int cw, int ch, float* out, cudaStream_t stream);

// geometry tail (geometry.cu)
cudaError_t launch_conf_quantile(const float* conf, int views, int n, float q, float* thr, cudaStream_t stream);
size_t similarity_fit_workspace(int views);
cudaError_t launch_similarity_fit(const float* x, const float* y, const float* conf, const float* thr,
                                  const uint8_t* valid, int views, int n, float* rts, double* workspace,
                                  cudaStream_t stream);
cudaError_t launch_similarity_apply(const float* x, const float* rts, float* out, int views, int n, cudaStream_t stream);
size_t focal_workspace(int views);
cudaError_t launch_focal_weiszfeld(const float* pts, const float* conf, const float* thr, const float* pp, int views,
                                   int H, int W, int iters, float* focal, double* workspace, cudaStream_t stream);

// reconstruction metrics (pointcloud.cu)
size_t pc_index_workspace(int n);
size_t pc_query_workspace(int nq);
size_t f64_reduce_workspace();
cudaError_t launch_pc_index_build(const void* pts, int f64, int n, void* index, cudaStream_t stream);
cudaError_t launch_pc_nearest(const void* index, int n_ref, const void* query, int f64, int nq, double* dist,
                              long long* idx, void* workspace, cudaStream_t stream);
cudaError_t launch_pc_knn_normals(const void* index, int n, int k, double* normals, cudaStream_t stream);
cudaError_t launch_pc_count_nonfinite(const void* pts, int f64, int n, unsigned int* count, cudaStream_t stream);
cudaError_t launch_pc_abs_dot(const double* a, const long long* a_idx, const double* b, const long long* b_idx, int n,
                              double* out, cudaStream_t stream);
cudaError_t launch_f64_mean(const double* x, int n, double* out, void* workspace, cudaStream_t stream);
cudaError_t launch_f64_median(const double* x, int n, double* out, void* workspace, cudaStream_t stream);
cudaError_t launch_f64_count_below(const double* x, int n, const double* th, unsigned long long* count,
                                   cudaStream_t stream);
// the stable LSD radix sort of the index build: (keys, vals) by the low `bits` bits of the keys, ping-ponging between
// buffer 0 and 1; *in_b tells (in and out) where the data is; hist: radix_sort_hist_bytes(n) bytes
size_t radix_sort_hist_bytes(int n);
cudaError_t launch_radix_sort(unsigned long long* keys[2], int* vals[2], int n, int bits, uint32_t* hist, int* in_b,
                              cudaStream_t stream);

// camera poses (pose.cu); offsets, counts_in and hyps are host arrays
size_t pnp_gather_workspace(int views, int n);
cudaError_t launch_pnp_gather(const float* pts, const float* conf, const uint8_t* mask, int views, int h, int w,
                              float* out_pts, float* out_pix, int* counts, void* workspace, cudaStream_t stream);
size_t pnp_score_workspace(int views, int nh);
cudaError_t launch_pnp_score(const float* pts, const float* pix, const long long* offsets, const int* counts_in, int views,
                             const f3r_pnp_hyp* hyps, int nh, float thr, int* counts, void* workspace, cudaStream_t stream);
size_t pnp_inliers_workspace(int nh, int max_count);
cudaError_t launch_pnp_inliers(const float* pts, const float* pix, const long long* offsets, const int* counts_in,
                               const f3r_pnp_hyp* hyps, int nh, float thr, float* out_pts, float* out_pix, int* counts,
                               void* workspace, cudaStream_t stream);

// camera-pose metric (pose_metric.cu); counts: [items][PM_COUNTS] (F3R_PM_* of include/fast3r_b200.h)
constexpr int PM_FLAGS = F3R_PM_HIST;
constexpr int PM_MAX_BINS = F3R_PM_MAX_BINS;
constexpr int PM_COUNTS = F3R_PM_COUNTS;
size_t pose_metric_workspace(int f64, int items, int views);
cudaError_t launch_pose_metric(int f64, const void* pred, const void* gt, int items, int views, int hmax, void* r_out,
                               void* t_out, unsigned long long* counts, void* workspace, cudaStream_t stream);
cudaError_t launch_pose_metric_counts(int f64, const void* r, const void* t, long long n, int hmax,
                                      unsigned long long* counts, cudaStream_t stream);

// validation criterion (val_loss.cu); out: [views][items][5] (val_loss_math.h vl::TERM_SUMS)
size_t val_loss_workspace(int views, int items, int n);
cudaError_t launch_val_loss(const float* gt, const uint8_t* valid, const float* pr, const float* pr_local,
                            const float* conf, const float* conf_local, const float* poses, int views, int items,
                            int n, float alpha, bool log1p, bool gt_scale, bool local_scale_consistent, bool has_local,
                            double* out, void* workspace, cudaStream_t stream);

// ground-truth views (views.cu); params on the device, max_pixels = the largest out_w * out_h
cudaError_t launch_view_geometry(const f3r_view_param* params, int count, int max_pixels, float* out_pts,
                                 uint8_t* out_valid, float* out_depth, cudaStream_t st);

// viewer scene (scene.cu)
size_t sky_mask_workspace(int frames, int h, int w);
cudaError_t launch_sky_mask(const float* img, int frames, int h, int w, int upper, int min_sky, int8_t* not_sky,
                            int* not_sky_count, void* workspace, cudaStream_t stream);
size_t scene_sort_workspace(long long n);
cudaError_t launch_scene_sort(const float* conf, const float* pts, const float* img, const int8_t* not_sky,
                              const long long* off, int frames, int n, float* out_pts, uint8_t* out_rgb,
                              int8_t* out_not_sky, float* max_conf, void* workspace, cudaStream_t stream);
int scene_visible_tiles(long long max_len);
size_t scene_visible_workspace(int nseg, int tiles);
cudaError_t launch_scene_visible(const long long* segs, int nseg, int tiles, const float* pts_g, const float* pts_l,
                                 const uint8_t* rgb_g, const uint8_t* rgb_l, const int8_t* ns_g, const int8_t* ns_l,
                                 int mask_sky, unsigned long long* total, float* out_pts, uint8_t* out_rgb,
                                 void* workspace, cudaStream_t stream);
cudaError_t launch_ply_pack(const float* pts, const uint8_t* rgb, long long n, uint8_t* out, cudaStream_t stream);
size_t percentile_workspace();
cudaError_t launch_extent_percentiles(const float* pts, long long n, long long k0, long long k1, float g0, float g1,
                                      float* out, void* workspace, cudaStream_t stream);

}  // namespace f3r
