/* fast3r_b200 — C ABI of the H100-native (sm_90a) Fast3R forward-pass kernels (libfast3r_b200.so).
 *
 * Drop-in boundary for the single-forward-pass hot path of facebookresearch/fast3r
 * (CroCo encoder -> fusion decoder -> DPT heads).  The reference's only native precedent is the
 * `curope` torch extension (fast3r/croco/models/curope/curope.cpp:54-59, kernels.cu:84-108): free functions
 * over caller-owned device buffers, default/current stream, no ownership transfer, errors reported to Python
 * as RuntimeError.  This ABI keeps those conventions but is torch-free: plain pointers, sizes and a
 * cudaStream_t (passed as void*).  Every entry point
 *   - works on caller-owned DEVICE pointers (16-byte aligned), never allocates or synchronises,
 *   - enqueues on the given stream and returns 0 on success, non-zero on error (text via f3r_last_error()),
 *   - is reentrant per thread (one Python thread per GPU/process, like the reference).
 *
 * Layout conventions: activations are row-major "channels-last": a token / pixel is a row; bf16 unless noted.  The
 * fp16 forward uses the same entry points with fp16 in place of every bf16 tensor (f3r_gemm_desc.f16, the element-type
 * code 2 of f3r_layernorm / f3r_im2col_patch / f3r_upsample2x, the *_f16 attention entry points, f3r_cast_f16).
 * Weights are bf16 [N_out, taps, K_in] (K contiguous); nn.Linear.weight (out,in) is already that with taps=1;
 * nn.Conv2d.weight (out,in,kh,kw) must be permuted to (out, kh*kw, in); ConvTranspose2d (in,out,k,k) to
 * ((i*k+j)*out + o, in).
 */
#ifndef FAST3R_B200_H
#define FAST3R_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define F3R_ABI_VERSION 3

/* epilogue kinds of f3r_gemm */
enum { F3R_EPI_STORE = 0, F3R_EPI_ROPE = 1, F3R_EPI_IDXEMB = 2, F3R_EPI_CONVT = 3, F3R_EPI_FINAL = 4 };
enum { F3R_ACT_NONE = 0, F3R_ACT_RELU = 1, F3R_ACT_GELU = 2 };

/* One fused GEMM / implicit-GEMM convolution:
 *   acc[m, n] = sum_{tap, k} A[pixel(m) + shift(tap), k] * Wt[n, tap, k]          (fp32 accumulation in registers)
 *   v = acc + bias[n] (+ RoPE2D | + idx-embedding row) (+ res0[m,n]) (+ res1[m,n])
 *   out1[m,n] = bf16(relu(v))   (optional);   out0[m,n] = act(v) as bf16 or fp32 (optional)
 * With f16 = 1 every 16-bit tensor of the call (a, wt, and res0 / res1 / out0 / out0b / out1 where not fp32) is fp16
 * instead of bf16; the products and the epilogue are the same, in fp32. 
 * Replaces: nn.Linear qkv/proj/fc1/fc2 (fast3r/croco/models/blocks.py:94-97,125-128), decoder_embed + image-index
 * embedding add (fast3r/models/fast3r.py:782-799), RoPE2D on q,k (fast3r/croco/models/pos_embed.py:162-183),
 * patch-embed conv (blocks.py:412-414), every Conv2d/ConvTranspose2d of the DPT head
 * (fast3r/croco/models/dpt_block.py:42-77,105-123,187-195,367-381,416-481) and, with F3R_EPI_FINAL, the last
 * ReLU + conv1x1 + postprocess (dpt_block.py:378-381, fast3r/dust3r/heads/postprocess.py:16-64). */
typedef struct f3r_gemm_desc {
  const void* a;       /* bf16 activation, viewed as (nb, h, w, c) with pixel stride a_ld elements            */
  const void* wt;      /* bf16 weights [n, taps, k]                                                            */
  int32_t n, k, taps;  /* taps: 1 (linear / 1x1) or 9 (3x3, stride 1, zero pad 1)                              */
  int32_t w, h, nb;    /* spatial extent of A; a linear layer over M rows is (w=M, h=1, nb=1)                  */
  int32_t a_ld;        /* elements between consecutive pixels of A (>= k)                                      */
  int32_t epi, act;
  int32_t out0_f32, res0_f32;
  int32_t ldo;         /* row stride (elements) of out0 / out1 / res0 / res1                                   */
  int32_t split_col, ldo_b; /* columns >= split_col of out0 go to out0b (row stride ldo_b); 0 disables         */
  int32_t tok_per_img, grid_w, rope_cols; /* ROPE: tokens per image, patch-grid width, #leading columns rotated;
                                             IDXEMB: tok_per_img tokens share emb_ids[m / tok_per_img];
                                             tok_per_img == 0: one id per row, emb_ids[m]                     */
  int32_t ct_k, ct_cout;                  /* CONVT: kernel==stride k, out channels; n == k*k*ct_cout           */
  int32_t f16;                            /* 0: the 16-bit tensors are bf16; 1: they are fp16                  */
  const float* bias;   /* [n] (CONVT: [ct_cout]) or NULL                                                       */
  const void* res0;    /* fp32 or bf16 [M, ldo] or NULL (may alias out0: in-place residual stream update)      */
  const void* res1;    /* bf16 [M, ldo] or NULL                                                                */
  void* out0;
  void* out0b;
  void* out1;
  const float* rope_cos; /* [max_pos, 16] cos(pos * base^(-j/16))                                              */
  const float* rope_sin;
  const float* emb_table; /* fp32 [1000, n]                                                                    */
  const int32_t* emb_ids; /* int32 [M / tok_per_img] (or [M] when tok_per_img == 0)                            */
  const float* w4;     /* FINAL: fp32 [4, n] 1x1 conv weight, b4 fp32 [4]                                      */
  const float* b4;
  float* pts;          /* FINAL: fp32 [M, 3]                                                                   */
  float* conf;         /* FINAL: fp32 [M]                                                                      */
} f3r_gemm_desc;

const char* f3r_last_error(void);
int f3r_abi_version(void);
/* sizeof(f3r_gemm_desc) as compiled into the library (binding-side struct layout guard). */
size_t f3r_gemm_desc_size(void);
/* Number of kernels launched through this library by the calling process so far. */
uint64_t f3r_launch_count(void);

/* Tuning knobs for A/B measurements (process-wide).  The only option is "pdl" = 1 / 0: launch the GEMM / attention /
 * LayerNorm chain with programmatic dependent launch (successor prologues overlap predecessor tails; default 1, env
 * F3R_PDL=0 disables).  Any other name is an error. */
int f3r_set_option(const char* name, int32_t value);

int f3r_gemm(const f3r_gemm_desc* d, void* stream);

/* softmax(scale * Q K^T) V per (batch, head), head_dim 64, non-causal (blocks.py:135-194).
 * q: bf16 [batch, sq, ldq] (head h at columns h*64); kv: bf16 [batch, skv, ldkv] with K of head h at columns
 * h*64 and V at columns heads*64 + h*64; out: bf16 [batch, sq, ldo].  lse (optional): fp32 [batch, heads, sq]. */
int f3r_attention(const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out, int32_t ldo, float* lse,
                  int32_t batch, int32_t heads, int32_t sq, int32_t skv, float scale, void* stream);

/* Key-slice form of f3r_attention, for (a) filling the SMs when batch*heads*ceil(sq/192) is small and (b) attending
 * to key ranges as they arrive over NVLink (sequence-parallel decoder, fast3r_b200/parallel.py): attends the queries to
 * the keys [kv_row0, kv_row0 + skv) of a kv buffer of kv_rows_total rows per batch (rows outside that range are never
 * read, so they may hold anything, NaN included), cut into n_split slices (one CTA each
 * per query tile of ATT_Q_TILE = 192 rows, csrc/f3r_kernels.h); slice s writes its softmax-normalised fp32 output into
 * part_o[part_base + s] (layout [slot, batch*sq, heads*64]) and its log-sum-exp into part_lse[part_base + s]
 * ([slot, batch, heads, sq]).
 * f3r_attention_merge combines n_parts slots into the exact softmax over the union of their keys (bf16 out). */
int f3r_attention_partial(const void* q, int32_t ldq, const void* kv, int32_t ldkv, int32_t kv_rows_total,
                          int32_t kv_row0, int32_t skv, int32_t n_split, float* part_o, float* part_lse,
                          int32_t part_base, int32_t batch, int32_t heads, int32_t sq, float scale, void* stream);
/* Block-diagonal form of f3r_attention, for several independent sequences packed into one (Fast3R.forward_many): q bf16
 * [rows, ldq], kv bf16 [rows, ldkv] ([K | V] as in f3r_attention), out bf16 [rows, ldo].  seg_off: device int32
 * [n_seg + 1], non-decreasing, seg_off[0] = 0 and seg_off[n_seg] = rows; the rows [seg_off[s], seg_off[s+1]) of
 * segment s attend to those rows only, and every row gets exactly what f3r_attention (batch 1) over its segment alone
 * computes.  Rows of other segments never reach a segment's result, NaN or Inf included.  One launch for all segments.
 * n_split > 1: key slices as in f3r_attention_partial; slice s writes slot s of part_o (fp32 [n_split, rows, heads*64])
 * and part_lse (fp32 [n_split, heads, rows]) and out is not written: f3r_attention_merge (batch 1, sq = rows,
 * n_parts = n_split) gives the result.  A segment of fewer than n_split key blocks uses one slice per block and writes
 * neutral partials (0, -inf) into its other slots, so it matches f3r_attention_partial with that many slices. */
int f3r_attention_segments(const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out, int32_t ldo,
                           const int32_t* seg_off, int32_t n_seg, int32_t rows, int32_t heads, float scale,
                           int32_t n_split, float* part_o, float* part_lse, void* stream);
int f3r_attention_merge(const float* part_o, const float* part_lse, int32_t n_parts, void* out, int32_t ldo,
                        int32_t batch, int32_t heads, int32_t sq, void* stream);
/* fp16 forms of the four attention entry points above: the same arguments and contracts, with fp16 q / kv / out in place
 * of bf16 (P is rounded to fp16 for the PV product; statistics, partials and LSE stay fp32). */
int f3r_attention_f16(const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out, int32_t ldo, float* lse,
                      int32_t batch, int32_t heads, int32_t sq, int32_t skv, float scale, void* stream);
int f3r_attention_partial_f16(const void* q, int32_t ldq, const void* kv, int32_t ldkv, int32_t kv_rows_total,
                              int32_t kv_row0, int32_t skv, int32_t n_split, float* part_o, float* part_lse,
                              int32_t part_base, int32_t batch, int32_t heads, int32_t sq, float scale, void* stream);
int f3r_attention_segments_f16(const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out, int32_t ldo,
                               const int32_t* seg_off, int32_t n_seg, int32_t rows, int32_t heads, float scale,
                               int32_t n_split, float* part_o, float* part_lse, void* stream);
int f3r_attention_merge_f16(const float* part_o, const float* part_lse, int32_t n_parts, void* out, int32_t ldo,
                            int32_t batch, int32_t heads, int32_t sq, void* stream);

/* Element-type codes of the out_f32 / f32 arguments below: 0 = bf16, 1 = fp32, 2 = fp16. */
/* nn.LayerNorm over the last dim of fp32 x [rows, dim] -> bf16 (or fp32 / fp16) out  (blocks.py:219,228; fast3r.py:558,805) */
int f3r_layernorm(const float* x, const float* w, const float* b, void* out, int32_t out_f32, int32_t rows,
                  int32_t dim, float eps, void* stream);
/* fp32 image batch (n,3,H,W) -> bf16 (or, by out_f32's code, fp32 / fp16) [n*(H/16)*(W/16), 768] patch rows
 * (im2col of blocks.py:412 Conv2d k=s=16) */
int f3r_im2col_patch(const float* img, void* out, int32_t out_f32, int32_t n, int32_t h, int32_t w, void* stream);
/* bf16 NHWC (n,h,w,c) -> bf16 [n*ho*wo, 9*c] for the 3x3 stride-2 pad-1 conv (dpt_block.py:471-478); a pure copy of
 * 16-bit elements, so fp16 in gives fp16 out */
int f3r_im2col3x3s2(const void* in, void* out, int32_t n, int32_t h, int32_t w, int32_t c, int32_t ho, int32_t wo,
                    void* stream);
/* bilinear x2 align_corners=True on NHWC in and out of the type coded by f32 (bf16, fp32 or fp16); writes the top-left (ho, wo) window of the (2h, 2w)
 * result (dpt_block.py:234-247,374; crop of dpt_head.py:69-71) */
int f3r_upsample2x(const void* in, void* out, int32_t f32, int32_t n, int32_t h, int32_t w, int32_t c, int32_t ho,
                   int32_t wo, void* stream);
/* fp32 -> bf16, count multiple of 4 */
int f3r_cast_bf16(const float* in, void* out, size_t count, void* stream);
/* fp32 -> fp16 (round to nearest even), count multiple of 4 */
int f3r_cast_f16(const float* in, void* out, size_t count, void* stream);

/* ---- image ingest (SURVEY §8 f3): PIL.Image.resize(LANCZOS | BICUBIC) + center crop + ToTensor + Normalize(0.5, 0.5) of
 * load_images() (fast3r/dust3r/utils/image.py:68-159) on a decoded 8-bit RGB image, bit-exact with Pillow's 8-bit
 * resampler.  filter: 0 = BICUBIC, 1 = LANCZOS.  f3r_resample_coeffs (HOST function, no CUDA call) fills the tap tables of
 * one dimension: bounds [out_size][2] = (first tap, count), kk [out_size][f3r_resample_ksize()] fixed-point weights, and
 * returns the widest source span of 64 consecutive outputs (h_span_max below; < 0 on error).  f3r_ingest_rgb8 takes DEVICE
 * copies of the tables (NULL for a dimension that keeps its size), a device scratch tmp [h][ow][3] (when ow != w) and
 * writes the crop box (left, top, cw, ch) of the resized image as fp32 [3][ch][cw] in [-1, 1].  src must be 4-byte
 * aligned (refused before any CUDA call otherwise). */
int f3r_resample_ksize(int32_t in_size, int32_t out_size, int32_t filter);
int f3r_resample_coeffs(int32_t in_size, int32_t out_size, int32_t filter, int32_t* bounds, int32_t* kk);
int f3r_ingest_rgb8(const uint8_t* src, int32_t h, int32_t w, int32_t oh, int32_t ow, const int32_t* hb, const int32_t* hk,
                    int32_t hks, int32_t h_span_max, const int32_t* vb, const int32_t* vk, int32_t vks, uint8_t* tmp,
                    int32_t left, int32_t top, int32_t cw, int32_t ch, float* out, void* stream);

/* ---- baseline JPEG decode, bit-exact with Pillow's (libjpeg-turbo: accurate integer IDCT, fancy upsampling, JCS_RGB
 * output).  The GPU decodes Huffman-coded 8-bit sequential JPEGs (SOF0, SOF1) with one component or three YCbCr
 * components at 4:4:4, 4:2:2 or 4:2:0, with or without restart markers; the caller keeps every other file on its host
 * decoder.
 * f3r_jpeg_probe (HOST function, no CUDA call) parses the `size` bytes at `data` and fills *info: status
 * F3R_JPEG_SUPPORTED, F3R_JPEG_UNSUPPORTED or F3R_JPEG_MALFORMED (the reason in f3r_last_error()), the image size and,
 * when supported, the scan layout and the device workspace f3r_jpeg_decode needs.  Returns non-zero only for bad
 * arguments.
 * f3r_jpeg_decode parses the same host bytes again (header only) and decodes the DEVICE copy data_dev of those bytes into
 * out, uint8 [out_h][out_w][3] RGB: the decoded image after ImageOps.exif_transpose for `orientation` (1..8; anything
 * else is 1), then rotate(-90, expand=True) when rotate_cw90 != 0, then the crop box (left, top, out_w, out_h).
 * workspace: info.workspace_bytes, 256-byte aligned.  The stream is decoded asynchronously: *status_dev (a device
 * int32) becomes 0, or a combination of the F3R_JPEG_ERR_* bits when the entropy-coded data is inconsistent (the image in
 * out is then undefined; the file should be decoded on the host instead). */
enum { F3R_JPEG_SUPPORTED = 0, F3R_JPEG_UNSUPPORTED = 1, F3R_JPEG_MALFORMED = 2 };
enum { F3R_JPEG_ERR_SYNC = 1, F3R_JPEG_ERR_CODE = 2, F3R_JPEG_ERR_COUNT = 4, F3R_JPEG_ERR_TRUNC = 8 };
typedef struct f3r_jpeg_info {
  int32_t status;
  int32_t width, height, components;
  int32_t h_samp, v_samp;            /* luma sampling factors (chroma is 1x1)                                        */
  int32_t restart_interval, segments; /* MCUs per restart interval (0: none), entropy-coded segments                  */
  size_t scan_offset, scan_bytes;    /* the entropy-coded data: bytes [scan_offset, scan_offset + scan_bytes)        */
  size_t workspace_bytes;
} f3r_jpeg_info;
int f3r_jpeg_probe(const uint8_t* data, size_t size, f3r_jpeg_info* info);
int f3r_jpeg_decode(const uint8_t* data, size_t size, const uint8_t* data_dev, int32_t orientation, int32_t rotate_cw90,
                    int32_t left, int32_t top, int32_t out_w, int32_t out_h, uint8_t* out, int32_t* status_dev,
                    void* workspace, size_t workspace_bytes, void* stream);

/* ---- geometry tail (SURVEY §8 f2, first slice): what every caller runs on the forward's outputs before poses.
 * A "view" below is one (view, batch item) pointmap of n = H*W pixels; all arrays are DEVICE pointers, fp32, view-major.
 *
 * f3r_conf_quantile: thr[v] = torch.quantile(conf[v].reshape(-1), q) (linear interpolation, fp32 like ATen) - the
 *   confidence threshold of align_local_pts3d_to_global (fast3r/models/multiview_dust3r_module.py:477) and of
 *   estimate_focal (:1093).  Exact: radix select on the float bit patterns.  A view holding a NaN (either sign) gives
 *   NaN, as torch.quantile does, so conf >= thr then selects nothing.
 * f3r_similarity_fit: per view the least-squares similarity (R, t, s), y ~ s R x + t, over the pixels with
 *   conf >= thr & valid; fewer than 3 such pixels -> over valid only; still fewer -> identity (:480-515, where the fit is
 *   roma.rigid_points_registration(x, y, compute_scaling=True)).  conf/thr and valid may be NULL (no such mask).
 *   rts [views][13] = R row-major (9), t (3), s.  workspace: f3r_similarity_fit_workspace(views) bytes, 8-byte aligned.
 * f3r_similarity_apply: out = s (x R^T) + t on all n pixels of every view (:517-521).  out may alias x.
 * f3r_focal_weiszfeld: focal[v] = argmin_f sum |pixel - pp - f (x, y)/z| by `iters` IRLS steps from the L2 closed form,
 *   over the pixels with conf >= thr (conf/thr NULL: all pixels), clipped to [0, inf); no selected pixel -> max(H, W) /
 *   (2 tan 30 deg).  iters = 100 with a mask reproduces estimate_focal_knowing_depth_and_confidence_mask(weiszfeld)
 *   (fast3r/dust3r/post_process.py:82-142), iters = 10 without one estimate_focal_knowing_depth(weiszfeld) (:19-79).
 *   pts [views][H][W][3]; pp [views][2] or NULL (= (W/2, H/2)).  workspace: f3r_focal_workspace(views) bytes. */
int f3r_conf_quantile(const float* conf, int32_t views, int32_t n, float q, float* thr, void* stream);
size_t f3r_similarity_fit_workspace(int32_t views);
int f3r_similarity_fit(const float* x, const float* y, const float* conf, const float* thr, const uint8_t* valid,
                       int32_t views, int32_t n, float* rts, void* workspace, size_t workspace_bytes, void* stream);
int f3r_similarity_apply(const float* x, const float* rts, float* out, int32_t views, int32_t n, void* stream);
size_t f3r_focal_workspace(int32_t views);
int f3r_focal_weiszfeld(const float* pts, const float* conf, const float* thr, const float* pp, int32_t views, int32_t h,
                        int32_t w, int32_t iters, float* focal, void* workspace, size_t workspace_bytes, void* stream);

/* ---- parity mode: the reference's fp32 path (inference_multiview.py:41-49, dtype="32": no autocast) on the bf16
 * tensor pipe.  Every fp32 operand x is carried as hi + lo (two bf16), every product as hi*hi + lo*hi + hi*lo with
 * fp32 accumulation.  For f3r_gemm this is the ordinary kernel over a 3x longer K: A' = f3r_split3(A) = [hi|lo|hi],
 * weights packed by the caller as [Whi | Whi | Wlo] along K (per tap); all outputs fp32 (out0_f32). */

/* fp32 in [rows, k] -> bf16 out [rows, 3k] = [hi | lo | hi] of x (relu != 0: of max(x, 0)) */
int f3r_split3(const float* in, void* out, size_t rows, int32_t k, int32_t relu, void* stream);
/* dst[i] += src[i], fp32, count multiple of 4 (second residual operand of dpt_block.py:241 in parity mode) */
int f3r_add_f32(float* dst, const float* src, size_t count, void* stream);
/* Same contract as f3r_attention with fp32 q / kv / out (blocks.py:135-194 without autocast).  workspace: caller-owned
 * device scratch of at least f3r_attention_x3_workspace() bytes, 256-byte aligned (holds the split operands). */
size_t f3r_attention_x3_workspace(int32_t batch, int32_t heads, int32_t sq, int32_t skv);
int f3r_attention_x3(const float* q, int32_t ldq, const float* kv, int32_t ldkv, float* out, int32_t ldo, float* lse,
                     void* workspace, size_t workspace_bytes, int32_t batch, int32_t heads, int32_t sq, int32_t skv,
                     float scale, void* stream);

/* ---- reconstruction metrics: accuracy / completion / completion_ratio of fast3r/eval/recon_metric.py:14-49 and the
 * normals of evaluate_reconstruction (fast3r/models/multiview_dust3r_module.py:551-735), exact with respect to scipy's
 * cKDTree.  Point clouds are DEVICE arrays [n][3] of fp32 (f64 == 0) or fp64 (f64 != 0), converted exactly to fp64.
 * Coordinates must be finite (check with the non-finite count first): a non-finite point never faults, but it makes
 * the search exhaustive and its results are unspecified.
 *
 * Spatial index over a reference cloud of n >= 1 points, built into a caller-owned block of
 *   f3r_pc_index_workspace(n) bytes, 256-byte aligned: Morton order (radix sort), buckets of 32 consecutive points with
 *   fp64 bounding boxes, parents of 8 consecutive children.  The block also holds the build's scratch; it stays valid
 *   until the caller reuses it.
 * Nearest: for each of nq query points the exact nearest reference point under scipy's arithmetic,
 *   dist (fp64) = sqrt((dx*dx + dy*dy) + dz*dz) and idx (int64, original index; any one of equidistant points).
 *   n_ref == 0 (index may be NULL): dist = +inf, idx = n_ref, as scipy.  workspace: f3r_pc_query_workspace(nq) bytes,
 *   256-byte aligned (the queries are processed in Morton order).
 * kNN normals of the indexed cloud itself: per point the unit eigenvector of the smallest eigenvalue of the fp64
 *   covariance of its k <= 32 nearest points, the point included (Open3D's EstimateNormals with KDTreeSearchParamKNN);
 *   fewer than 3 points: (0, 0, 1).  The sign is unspecified.  normals fp64 [n][3], original order.
 * Non-finite count: *count (device uint32) = number of non-finite coordinates of the n points.
 * Absolute dot: out[i] = |a[ia] . b[ib]| (ia = a_idx[i], or i when a_idx is NULL; int64 indices), rounded as numpy's
 *   np.abs(np.sum(a * b, axis=-1)).
 * fp64 reductions over x[0..n): mean in a fixed order (not numpy's pairwise order: equal to a few ulp), median exactly
 *   as numpy.median (radix select on the bit patterns; the mean of the two middle values for even n), and the count
 *   of x < *th (th a device fp64 scalar) into *count (device uint64).  workspace: f3r_f64_reduce_workspace() bytes,
 *   256-byte aligned. */
size_t f3r_pc_index_workspace(int32_t n);
int f3r_pc_index_build(const void* pts, int32_t f64, int32_t n, void* index, size_t index_bytes, void* stream);
size_t f3r_pc_query_workspace(int32_t nq);
int f3r_pc_nearest(const void* index, size_t index_bytes, int32_t n_ref, const void* query, int32_t f64, int32_t nq,
                   double* dist, int64_t* idx, void* workspace, size_t workspace_bytes, void* stream);
int f3r_pc_knn_normals(const void* index, size_t index_bytes, int32_t n, int32_t k, double* normals, void* stream);
int f3r_pc_count_nonfinite(const void* pts, int32_t f64, int32_t n, uint32_t* count, void* stream);
int f3r_pc_abs_dot(const double* a, const int64_t* a_idx, const double* b, const int64_t* b_idx, int32_t n, double* out,
                   void* stream);
size_t f3r_f64_reduce_workspace(void);
int f3r_f64_mean(const double* x, int32_t n, double* out, void* workspace, size_t workspace_bytes, void* stream);
int f3r_f64_median(const double* x, int32_t n, double* out, void* workspace, size_t workspace_bytes, void* stream);
int f3r_f64_count_below(const double* x, int32_t n, const double* th, uint64_t* count, void* stream);

/* ---- camera poses: the per-point work of cv2.solvePnPRansac(..., flags=SOLVEPNP_SQPNP) as fast_pnp calls it
 * (fast3r/dust3r/cloud_opt/init_im_poses.py:300-350), exact with respect to OpenCV's classic RANSAC.  The host draws
 * the samples, solves the EPnP hypotheses, keeps the books and refits (fast3r_b200/poses.py).
 *
 * f3r_pnp_gather: per view v of n = h w pixels, the pixels with conf > 1 (conf given, mask NULL) or mask != 0 (mask
 *   given, conf NULL) in raster order, as numpy's boolean indexing orders them: out_pts [views][n][3] gets the points,
 *   out_pix [views][n][2] their pixel_grid coordinates (x, y), both from slot v n on; counts [views] (int32) how many.
 *   workspace: f3r_pnp_gather_workspace(views, h, w) bytes, 4-byte aligned.
 * f3r_pnp_score: counts[r] = the number of points of view hyps[r].view whose error under hypothesis r is
 *   <= (float)(thr * thr): OpenCV's projectPoints with zero distortion in double, stored as float, then the float
 *   |pixel - projection|^2 (fast3r_b200/csrc/pose_math.h).  Points and pixels are DEVICE arrays (pts [.][3], pix [.][2]);
 *   view v is [offsets[v], offsets[v] + view_counts[v]) of them.  offsets, view_counts and hyps are HOST arrays.  Rows
 *   of one view that follow each other share their reads of the points.  workspace: f3r_pnp_score_workspace(views, nh)
 *   bytes, 256-byte aligned.
 * f3r_pnp_inliers: for every row r the points and pixels of view hyps[r].view that are inliers of hypothesis r (the
 *   rule of f3r_pnp_score), in index order, into out_pts / out_pix from slot sum_{s<r} view_counts[hyps[s].view] on;
 *   out_counts [nh] (int32, device) how many.  workspace: f3r_pnp_inliers_workspace(nh, max view_counts) bytes, 256-byte
 *   aligned. */
typedef struct f3r_pnp_hyp {
  double r[9];                /* rotation, row-major: cv2.Rodrigues of the hypothesis' rvec */
  double t[3];
  double fx, fy, cx, cy;      /* the camera matrix as double */
  int32_t view, reserved;
} f3r_pnp_hyp;
size_t f3r_pnp_gather_workspace(int32_t views, int32_t h, int32_t w);
int f3r_pnp_gather(const float* pts, const float* conf, const uint8_t* mask, int32_t views, int32_t h, int32_t w,
                   float* out_pts, float* out_pix, int32_t* counts, void* workspace, size_t workspace_bytes, void* stream);
size_t f3r_pnp_score_workspace(int32_t views, int32_t nh);
int f3r_pnp_score(const float* pts, const float* pix, const int64_t* offsets, const int32_t* view_counts, int32_t views,
                  const f3r_pnp_hyp* hyps, int32_t nh, float thr, int32_t* counts, void* workspace, size_t workspace_bytes,
                  void* stream);
size_t f3r_pnp_inliers_workspace(int32_t nh, int32_t max_count);
int f3r_pnp_inliers(const float* pts, const float* pix, const int64_t* offsets, const int32_t* view_counts, int32_t views,
                    const f3r_pnp_hyp* hyps, int32_t nh, float thr, float* out_pts, float* out_pix, int32_t* out_counts,
                    void* workspace, size_t workspace_bytes, void* stream);

/* ---- camera-pose metric: the relative-pose errors of all view pairs behind evaluate_camera_poses' RRA / RTA / mAA
 * (fast3r/eval/cam_pose_metric.py camera_to_rel_deg / calculate_auc with fast3r/utils/so3_utils.py), in the
 * reference's CPU arithmetic (fast3r_b200/csrc/pose_metric_math.h); the host forms the means (fast3r_b200/cam_pose_metric.py).
 *
 * f3r_pose_metric: pred and gt [items][views][4][4] (row-major cam-to-world, float32 or float64 by f64; DEVICE), pairs
 *   (i, j), i < j, in torch.combinations order, P = views (views - 1) / 2 per item.  Per pair: the rotation angle of
 *   R_gt R_pred^T and the translation angle of the relative poses inv(pose_i) pose_j, in degrees.  r_out / t_out
 *   [items][P] (same type; both NULL or both given) receive them.  counts [items][F3R_PM_COUNTS] (int64) receive: [0..2]
 *   pairs with rotation angle < 5, 15, 30; [3..5] translation angle < 5, 15, 30; [6] pairs whose trace is outside
 *   [-1 - 1e-4, 3 + 1e-4] (NaN is not); [7] pairs counted (= P); [F3R_PM_HIST + b] torch.histc(max(r, t),
 *   bins = hist_max + 1, min = 0, max = hist_max) bin b.  1 <= hist_max < F3R_PM_MAX_BINS; 2 <= views <= 65536;
 *   1 <= items <= 65535, items * views < 2^31.  workspace: f3r_pose_metric_workspace(f64, items, views) bytes, 8-byte aligned.
 * f3r_pose_metric_counts: the counts of one item ([6] = 0) from given angles r, t [n] (DEVICE). */
#define F3R_PM_HIST 8
#define F3R_PM_MAX_BINS 64
#define F3R_PM_COUNTS (F3R_PM_HIST + F3R_PM_MAX_BINS)
size_t f3r_pose_metric_workspace(int32_t f64, int32_t items, int32_t views);
int f3r_pose_metric(int32_t f64, const void* pred, const void* gt, int32_t items, int32_t views, int32_t hist_max,
                    void* r_out, void* t_out, int64_t* counts, void* workspace, size_t workspace_bytes, void* stream);
int f3r_pose_metric_counts(int32_t f64, const void* r, const void* t, size_t n, int32_t hist_max, int64_t* counts,
                           void* stream);

/* ---- validation criterion: ConfLossMultiviewV2(Regr3DMultiviewV4(L21Loss())) of fast3r/dust3r/losses.py:570-848,
 * forward only (fast3r_b200/csrc/val_loss.cu); the host forms the means, the loss and the details
 * (fast3r_b200/losses.py).
 *
 * f3r_val_loss: every map is stacked [views][items][n] (DEVICE): gt [.][3] (pts3d), valid (uint8 0/1), pr [.][3]
 *   (pts3d_in_other_view), conf, and with has_local pr_local [.][3] (pts3d_local) and conf_local (else NULL); poses
 *   [views][items][4][4] (camera_pose, float32, row-major).  Ground truth goes to view 0's frame (global term) and to its
 *   own view's frame (local term) through inverses formed in double.  Norm factors: the mean of ||p|| (log1p ||p|| with
 *   log1p) over the valid pixels where it is not NaN, clipped below at 1e-8 - per item over all views for the global
 *   term, per (view, item) for the local term, or the global ones with local_scale_consistent; with gt_scale the ground
 *   truth keeps its scale.  out [views][items][5] (float64, DEVICE) receives per (view, item), over the valid pixels:
 *   [0] sum of d = ||pr / f_pr - gt / f_gt|| and [1] sum of d c - alpha log c of the global term, [2] and [3] the same
 *   of the local term (0 without has_local), [4] the number of valid pixels.  alpha > 0; views, items, n >= 1 and
 *   views * items * n < 2^31.  workspace: f3r_val_loss_workspace(views, items, n) bytes, 8-byte aligned.  Two calls
 *   on the same inputs give the same bits. */
size_t f3r_val_loss_workspace(int32_t views, int32_t items, int32_t n);
int f3r_val_loss(const float* gt, const uint8_t* valid, const float* pr, const float* pr_local, const float* conf,
                 const float* conf_local, const float* poses, int32_t views, int32_t items, int32_t n, float alpha,
                 int32_t log1p, int32_t gt_scale, int32_t local_scale_consistent, int32_t has_local, double* out,
                 void* workspace, size_t workspace_bytes, void* stream);

/* ---- viewer scene: the frame preparation and the point export of the reference's viewer
 * (fast3r/viz/viser_visualizer.py:24-72, :168-254, :343-427), exact with respect to numpy / cv2 / scipy.  The host
 * groups the frames, applies the viewer's settings and writes the PLY header (fast3r_b200/scene.py).
 *
 * f3r_sky_mask: detect_sky_mask of `frames` images of one shape, img [frames][3][h][w] (fp32 in [-1, 1]): u8
 *   ((x + 1) * 127.5, truncated), OpenCV's 8-bit RGB -> HSV, the three inRange boxes, S < 50 and V > 150 in rows
 *   < upper_rows (= int(h * 0.4)), a 7x7 dilate then a 7x7 open, 4-connected components; sky = the components touching
 *   row 0 of >= min_sky (= floor(h w 0.01) + 1) pixels, or the whole mask if none touches row 0.  not_sky [frames][h][w]
 *   (int8 0/1) and not_sky_count [frames] (int32).  workspace: f3r_sky_mask_workspace(frames, h, w) bytes, 256-byte
 *   aligned.
 * f3r_scene_sort: one group of frames, frame f = elements [offsets[f], offsets[f + 1]) (offsets: DEVICE int64
 *   [frames + 1], offsets[0] = 0, offsets[frames] = n): each frame in the order of np.argsort(-conf, kind="stable")
 *   (descending, -0.0 == +0.0, NaN last, ties by index).  Slot j of that order gets the point (pts [n][3]), the u8
 *   colour of the pixel (img: frame f's planar [3][hw] image at 3 offsets[f]) and its not-sky value into out_pts
 *   [n][3], out_rgb [n][3], out_not_sky [n]; max_conf [frames] gets conf.max() of each frame (NaN if it holds a NaN).
 *   workspace: f3r_scene_sort_workspace(n) bytes, 256-byte aligned.
 * f3r_scene_visible: segments segs [nseg][4] (DEVICE int64: head 0 = global / 1 = local, first row, row count <=
 *   max_len, colour -1 = the rows' own RGB or 0xRRGGBB) of the frame arrays pts_* [.][3], rgb_* [.][3], not_sky_*;
 *   with mask_sky only rows of not_sky > 0.  Two calls on one workspace: with total (DEVICE uint64) the count of kept
 *   rows; then with out_pts [total][3] and out_rgb [total][3] the kept rows, segment after segment in row order.
 *   workspace: f3r_scene_visible_workspace(nseg, max_len) bytes, 256-byte aligned.
 * f3r_ply_pack: out [n][15] = the binary_little_endian PLY records of the points (3 x float32, 3 x uint8).
 * f3r_extent_percentiles: out[7] = np.percentile(pts, 20 and 80, axis=0) for pts [n][3] (float32, method "linear") as
 *   out[0..2] and out[3..5], and out[6] = max over axes of out[3 + a] - out[a].  The host gives each percentile's lower
 *   rank k0 / k1 and float32 weight g0 / g1 as numpy forms them; a column holding a NaN gives NaN.  workspace:
 *   f3r_extent_percentiles_workspace() bytes, 256-byte aligned. */
size_t f3r_sky_mask_workspace(int32_t frames, int32_t h, int32_t w);
int f3r_sky_mask(const float* img, int32_t frames, int32_t h, int32_t w, int32_t upper_rows, int32_t min_sky,
                 int8_t* not_sky, int32_t* not_sky_count, void* workspace, size_t workspace_bytes, void* stream);
size_t f3r_scene_sort_workspace(int32_t n);
int f3r_scene_sort(const float* conf, const float* pts, const float* img, const int8_t* not_sky, const int64_t* offsets,
                   int32_t frames, int32_t n, float* out_pts, uint8_t* out_rgb, int8_t* out_not_sky, float* max_conf,
                   void* workspace, size_t workspace_bytes, void* stream);
size_t f3r_scene_visible_workspace(int32_t nseg, size_t max_len);
int f3r_scene_visible(const int64_t* segs, int32_t nseg, size_t max_len, const float* pts_g, const float* pts_l,
                      const uint8_t* rgb_g, const uint8_t* rgb_l, const int8_t* not_sky_g, const int8_t* not_sky_l,
                      int32_t mask_sky, uint64_t* total, float* out_pts, uint8_t* out_rgb, void* workspace,
                      size_t workspace_bytes, void* stream);
int f3r_ply_pack(const float* pts, const uint8_t* rgb, size_t n, uint8_t* out, void* stream);
size_t f3r_extent_percentiles_workspace(void);
int f3r_extent_percentiles(const float* pts, size_t n, size_t k0, size_t k1, float g0, float g1, float* out,
                           void* workspace, size_t workspace_bytes, void* stream);

/* ---- ground-truth views: the depth half of the datasets' principal-point crop, rescale and crop
 * (fast3r/dust3r/datasets/base/base_stereo_view_dataset.py:165-221), the unprojection to world points
 * (fast3r/dust3r/utils/geometry.py:186-243), the validity mask and the landscape transpose (:78-142, :243-261).  The host
 * plans the geometry and runs the image half through f3r_ingest_rgb8 (fast3r_b200/views.py).
 *
 * One f3r_view_param per (view, item).  The depth map depth [src_h][src_w] (DEVICE, float32) is cropped to the box
 * (crop_x, crop_y, crop_w, crop_h), resized to (rs_w, rs_h) with cv2's INTER_NEAREST rule and cropped to (box_x, box_y,
 * out_w, out_h).  Pixel (u, v) of that crop at depth z has the camera point ((u - k[2]) z / k[0], (v - k[3]) z / k[1], z)
 * (in float64, rounded to float32) and the world point pose[0..11] = [R | t] (row-major) applied in float32; it is
 * valid when z > 0 and the world point is finite (a NaN pose makes every pixel invalid).  Pixel i of the view's outputs
 * is element out_offset + i of out_pts [.][3], out_valid (uint8 0/1) and out_depth; the outputs are stored row-major as
 * [out_h][out_w], or transposed as [out_w][out_h] when transpose = 1. */
typedef struct f3r_view_param {
  const float* depth;
  int64_t out_offset;
  int32_t src_w, src_h;
  int32_t crop_x, crop_y, crop_w, crop_h;
  int32_t rs_w, rs_h;
  int32_t box_x, box_y, out_w, out_h;
  int32_t transpose, reserved;
  float k[4];     /* fu, fv, cu, cv of the final intrinsics */
  float pose[12]; /* cam2world rows [R | t] */
} f3r_view_param;

/* f3r_view_geometry: params (HOST) is checked before any CUDA call - every box inside its image, depth 4-byte
 * aligned, every view's outputs inside [0, out_pixels), out_pixels and every source below 2^31 pixels, 1 <= count <=
 * 65535 - and params_dev holds the same count records on the DEVICE, which the kernel reads.  One launch. */
int f3r_view_geometry(const f3r_view_param* params, const f3r_view_param* params_dev, int32_t count, float* out_pts,
                      uint8_t* out_valid, float* out_depth, size_t out_pixels, void* stream);

#ifdef __cplusplus
}
#endif
#endif
