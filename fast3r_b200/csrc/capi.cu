// extern "C" boundary of libfast3r_b200.so (see include/fast3r_b200.h).  Builds the TMA descriptors
// (cuTensorMapEncodeTiled through cudaGetDriverEntryPoint, so libcuda is not a link-time dependency),
// validates arguments and enqueues the kernels on the caller's stream.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../include/fast3r_b200.h"
#include "f3r_kernels.h"
#include "gemm_plan.h"

namespace {

thread_local char g_err[512] = "";

int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
int check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  return fail("%s: %s", what, cudaGetErrorString(e));
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// Tensor map with zero OOB fill.  dims[0] is the contiguous dimension.  Defaults: bf16, 128B swizzle (MMA operands).
int make_tmap(CUtensorMap* m, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
              const uint32_t* box, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
              CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail("cuTensorMapEncodeTiled not available (no CUDA driver?)");
  cuuint64_t gd[5];
  cuuint64_t gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i < rank - 1; ++i) gs[i] = strides_bytes[i];
  if (reinterpret_cast<uintptr_t>(ptr) & 15) return fail("tensor map base not 16-byte aligned");
  for (int i = 0; i < rank - 1; ++i)
    if (gs[i] % 16) return fail("tensor map stride %d (%llu B) not a multiple of 16", i, (unsigned long long)gs[i]);
  CUresult r = enc(m, dtype, rank, const_cast<void*>(ptr), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed with CUresult %d", static_cast<int>(r));
  return 0;
}

int num_sms() {
  static int cache[64] = {0};  // per device: one process may drive several GPUs
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  int& n = cache[dev & 63];
  if (n) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  return n;
}

}  // namespace

extern "C" {

const char* f3r_last_error(void) { return g_err; }
int f3r_abi_version(void) { return F3R_ABI_VERSION; }
size_t f3r_gemm_desc_size(void) { return sizeof(f3r_gemm_desc); }
uint64_t f3r_launch_count(void) { return f3r::g_launch_count.load(); }

int f3r_set_option(const char* name, int32_t value) {
  if (!name) return fail("f3r_set_option: null name");
  if (!strcmp(name, "pdl")) {
    if (value != 0 && value != 1) return fail("f3r_set_option: pdl must be 0 or 1");
    f3r::g_pdl = value;
    return 0;
  }
  return fail("f3r_set_option: unknown option '%s'", name);
}

int f3r_gemm(const f3r_gemm_desc* d, void* stream) {
  if (!d || !d->a || !d->wt) return fail("f3r_gemm: null operand");
  if (d->n <= 0 || d->k <= 0 || d->w <= 0 || d->h <= 0 || d->nb <= 0) return fail("f3r_gemm: bad shape");
  if (d->n % 32) return fail("f3r_gemm: n=%d must be a multiple of 32", d->n);
  if (d->k % 8 || d->a_ld % 8) return fail("f3r_gemm: k=%d and a_ld=%d must be multiples of 8", d->k, d->a_ld);
  if (d->taps != 1 && d->taps != 9) return fail("f3r_gemm: taps must be 1 or 9");
  if (d->epi == F3R_EPI_FINAL && d->n != 128) return fail("f3r_gemm: FINAL epilogue needs n == 128");
  if (d->epi == F3R_EPI_CONVT && (d->ct_k <= 0 || d->ct_cout % 32 || d->n != d->ct_k * d->ct_k * d->ct_cout))
    return fail("f3r_gemm: bad CONVT geometry");
  if (d->epi == F3R_EPI_ROPE && (!d->rope_cos || !d->rope_sin || d->tok_per_img <= 0 || d->grid_w <= 0))
    return fail("f3r_gemm: bad ROPE arguments");
  if (d->epi == F3R_EPI_IDXEMB && (!d->emb_table || !d->emb_ids || d->tok_per_img < 0))
    return fail("f3r_gemm: bad IDXEMB arguments");
  if (d->f16 != 0 && d->f16 != 1) return fail("f3r_gemm: f16=%d must be 0 or 1", d->f16);

  static int dbg = -1, tma_pref = -1, ksplit_pref = -1;
  if (dbg < 0) { const char* e = getenv("F3R_GEMM_DEBUG"); dbg = e ? atoi(e) : 0; }
  if (tma_pref < 0) { const char* e = getenv("F3R_GEMM_TMA_EPI"); tma_pref = (e && e[0] == '0') ? 0 : 1; }
  // F3R_GEMM_KSPLIT=1 disables the K slicing (A/B measurements)
  if (ksplit_pref < 0) { const char* e = getenv("F3R_GEMM_KSPLIT"); ksplit_pref = (e && e[0] == '1') ? 1 : 0; }
  const f3r::GemmPlan plan = f3r::gemm_plan(*d, num_sms(), tma_pref, ksplit_pref != 1);
  const int block_n = plan.block_n;

  f3r::GemmArgs a;
  memset(&a, 0, sizeof(a));
  a.M = d->w * d->h * d->nb; a.N = d->n; a.K = d->k; a.taps = d->taps;
  a.W = d->w; a.H = d->h; a.NB = d->nb;
  a.bw = plan.bw; a.bh = plan.bh; a.bw_log2 = plan.bw_log2; a.sbx_log2 = plan.sbx_log2;
  a.tiles_x = plan.tiles_x; a.tiles_y = plan.tiles_y; a.num_m_tiles = plan.num_m_tiles;
  a.num_n_tiles = plan.num_n_tiles;
  a.tma_epi = plan.tma_epi; a.k_split = plan.k_split;
  a.debug = dbg;
  a.epi = d->epi; a.act = d->act; a.out0_f32 = d->out0_f32; a.res0_f32 = d->res0_f32;
  a.ldo = d->ldo > 0 ? d->ldo : d->n;
  a.split_col = d->split_col; a.ldo_b = d->ldo_b;
  a.tok_per_img = d->tok_per_img; a.grid_w = d->grid_w; a.rope_cols = d->rope_cols;
  a.ct_k = d->ct_k; a.ct_cout = d->ct_cout;
  a.bias = d->bias; a.res0 = d->res0; a.res1 = d->res1;
  a.out0 = d->out0; a.out0b = d->out0b; a.out1 = d->out1;
  a.rope_cos = d->rope_cos; a.rope_sin = d->rope_sin;
  a.emb_table = d->emb_table; a.emb_ids = d->emb_ids;
  a.w4 = d->w4; a.b4 = d->b4; a.pts = d->pts; a.conf = d->conf;
  if (a.split_col && (a.split_col % 32 || !a.out0b)) return fail("f3r_gemm: bad column split");

  // the 16-bit operands and outputs: bf16, or fp16 with d->f16
  const CUtensorMapDataType t16 = d->f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap ta, tb;
  {
    const uint64_t ld = static_cast<uint64_t>(d->a_ld) * 2;
    const uint64_t dims[4] = {static_cast<uint64_t>(d->k), static_cast<uint64_t>(d->w),
                              static_cast<uint64_t>(d->h), static_cast<uint64_t>(d->nb)};
    const uint64_t str[3] = {ld, ld * d->w, ld * d->w * d->h};
    const uint32_t box[4] = {64, static_cast<uint32_t>(a.bw), static_cast<uint32_t>(a.bh), 1};
    if (make_tmap(&ta, d->a, 4, dims, str, box, t16)) return 1;
  }
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(d->k), static_cast<uint64_t>(d->taps),
                              static_cast<uint64_t>(d->n)};
    const uint64_t str[2] = {static_cast<uint64_t>(d->k) * 2, static_cast<uint64_t>(d->k) * 2 * d->taps};
    const uint32_t box[3] = {64, 1, static_cast<uint32_t>(block_n)};
    if (make_tmap(&tb, d->wt, 3, dims, str, box, t16)) return 1;
  }
  // output tensor maps of the TMA epilogue (plan.tma_epi: plain stores, or the in-place fp32 residual reduce-add)
  CUtensorMap to0, to0b;
  memset(&to0, 0, sizeof(to0));
  memset(&to0b, 0, sizeof(to0b));
  if (a.tma_epi) {
    const uint64_t es = d->out0_f32 ? 4 : 2;
    const CUtensorMapDataType dt = d->out0_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : t16;
    const CUtensorMapSwizzle sw = d->out0_f32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    const uint32_t sbx = 1u << a.sbx_log2;
    const uint32_t box[4] = {32, sbx, 32 / sbx, 1};
    const uint64_t ncols0 = a.split_col ? a.split_col : d->n;
    {
      const uint64_t ld = static_cast<uint64_t>(a.ldo) * es;
      const uint64_t dims[4] = {ncols0, static_cast<uint64_t>(d->w), static_cast<uint64_t>(d->h),
                                static_cast<uint64_t>(d->nb)};
      const uint64_t str[3] = {ld, ld * d->w, ld * d->w * d->h};
      if (make_tmap(&to0, d->out0, 4, dims, str, box, dt, sw)) return 1;
    }
    if (a.split_col) {
      const uint64_t ld = static_cast<uint64_t>(a.ldo_b) * es;
      const uint64_t dims[4] = {static_cast<uint64_t>(d->n - a.split_col), static_cast<uint64_t>(d->w),
                                static_cast<uint64_t>(d->h), static_cast<uint64_t>(d->nb)};
      const uint64_t str[3] = {ld, ld * d->w, ld * d->w * d->h};
      if (make_tmap(&to0b, d->out0b, 4, dims, str, box, dt, sw)) return 1;
    }
  }
  return check(f3r::launch_gemm(block_n, d->f16, ta, tb, to0, to0b, a, num_sms(), static_cast<cudaStream_t>(stream)),
               "f3r_gemm");
}

// f16: q, kv and out are fp16 (the *_f16 entry points) instead of bf16
static int attention_impl(const char* what, int f16, const void* q, int32_t ldq, const void* kv, int32_t ldkv,
                          int32_t kv_rows_total, int32_t kv_row0, void* out, int32_t ldo, float* lse, float* part_o,
                          float* part_lse, int32_t part_base, int32_t n_split, int32_t batch, int32_t heads, int32_t sq,
                          int32_t skv, float scale, void* stream) {
  const CUtensorMapDataType t16 = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  if (!q || !kv) return fail("%s: null operand", what);
  if (batch <= 0 || heads <= 0 || sq <= 0 || skv <= 0) return fail("%s: bad shape", what);
  if (ldq % 8 || ldkv % 8 || ldq < heads * 64 || ldkv < 2 * heads * 64) return fail("%s: bad leading dimensions", what);
  if (kv_row0 < 0 || kv_row0 + skv > kv_rows_total) return fail("%s: key range outside the kv buffer", what);
  if (n_split < 1 || n_split > (skv + 127) / 128) return fail("%s: n_split=%d must be in [1, #key blocks]", what, n_split);
  CUtensorMap tq, tkv;
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * 64, static_cast<uint64_t>(sq),
                              static_cast<uint64_t>(batch)};
    const uint64_t str[2] = {static_cast<uint64_t>(ldq) * 2, static_cast<uint64_t>(ldq) * 2 * sq};
    const uint32_t box[3] = {64, f3r::ATT_Q_TILE, 1};
    if (make_tmap(&tq, q, 3, dims, str, box, t16)) return 1;
  }
  {
    // the map ends where the key range ends (the batch stride stays kv_rows_total rows): the last key block of the range
    // is a full 128-row load, and the rows past the range come back zero-filled, never as whatever follows in the
    // buffer.  Their scores are masked, but their V rows enter the PV product with P = 0, and 0 * NaN would be NaN.
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * 128, static_cast<uint64_t>(kv_row0 + skv),
                              static_cast<uint64_t>(batch)};
    const uint64_t str[2] = {static_cast<uint64_t>(ldkv) * 2, static_cast<uint64_t>(ldkv) * 2 * kv_rows_total};
    const uint32_t box[3] = {64, 128, 1};
    if (make_tmap(&tkv, kv, 3, dims, str, box, t16)) return 1;
  }
  f3r::AttnArgs a;
  memset(&a, 0, sizeof(a));
  a.batch = batch; a.heads = heads; a.sq = sq; a.skv = skv;
  a.q_tiles = (sq + f3r::ATT_Q_TILE - 1) / f3r::ATT_Q_TILE;
  a.scale_log2 = scale * 1.4426950408889634f;
  a.ldo = ldo; a.out = out; a.lse = lse;
  a.kv_row0 = kv_row0; a.n_split = n_split; a.part_base = part_base; a.part_o = part_o; a.part_lse = part_lse;
  return check(f3r::launch_attention(tq, tkv, a, f16, static_cast<cudaStream_t>(stream)), what);
}

static int attention_full(const char* what, int f16, const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out,
                          int32_t ldo, float* lse, int32_t batch, int32_t heads, int32_t sq, int32_t skv, float scale,
                          void* stream) {
  if (!out) return fail("%s: null operand", what);
  if (ldo % 8 || ldo < heads * 64) return fail("%s: bad leading dimensions", what);
  return attention_impl(what, f16, q, ldq, kv, ldkv, skv, 0, out, ldo, lse, nullptr, nullptr, 0, 1, batch, heads, sq, skv,
                        scale, stream);
}

static int attention_partial(const char* what, int f16, const void* q, int32_t ldq, const void* kv, int32_t ldkv,
                             int32_t kv_rows_total, int32_t kv_row0, int32_t skv, int32_t n_split, float* part_o,
                             float* part_lse, int32_t part_base, int32_t batch, int32_t heads, int32_t sq, float scale,
                             void* stream) {
  if (!part_o || !part_lse || part_base < 0) return fail("%s: bad partial buffers", what);
  return attention_impl(what, f16, q, ldq, kv, ldkv, kv_rows_total, kv_row0, nullptr, 0, nullptr, part_o, part_lse,
                        part_base, n_split, batch, heads, sq, skv, scale, stream);
}

static int attention_segments(const char* what, int f16, const void* q, int32_t ldq, const void* kv, int32_t ldkv,
                              void* out, int32_t ldo, const int32_t* seg_off, int32_t n_seg, int32_t rows, int32_t heads,
                              float scale, int32_t n_split, float* part_o, float* part_lse, void* stream) {
  const CUtensorMapDataType t16 = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  if (!q || !kv || !seg_off) return fail("%s: null operand", what);
  if (reinterpret_cast<uintptr_t>(seg_off) & 3) return fail("%s: seg_off not 4-byte aligned", what);
  if (n_seg <= 0 || rows <= 0 || heads <= 0) return fail("%s: bad shape", what);
  if (ldq % 8 || ldkv % 8 || ldq < heads * 64 || ldkv < 2 * heads * 64) return fail("%s: bad leading dimensions", what);
  if (n_split < 1 || n_split > (rows + 127) / 128) return fail("%s: n_split=%d must be in [1, #key blocks]", what, n_split);
  if (!part_o != !part_lse) return fail("%s: part_o and part_lse must be given together", what);
  if (!part_o) {
    if (n_split != 1) return fail("%s: n_split > 1 writes key-slice partials: part_o / part_lse needed", what);
    if (!out) return fail("%s: null operand", what);
    if (ldo % 8 || ldo < heads * 64) return fail("%s: bad leading dimensions", what);
  }
  // sum over segments of ceil(len / ATT_Q_TILE) <= (rows + (ATT_Q_TILE - 1) * n_seg) / ATT_Q_TILE; the CTAs past the
  // last work item exit at once
  const long long max_tiles = (rows + static_cast<long long>(f3r::ATT_Q_TILE - 1) * n_seg) / f3r::ATT_Q_TILE;
  if (max_tiles * heads * n_split > 0x7fffffffLL) return fail("%s: too many work items", what);
  CUtensorMap tq, tkv;
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * 64, static_cast<uint64_t>(rows), 1};
    const uint64_t str[2] = {static_cast<uint64_t>(ldq) * 2, static_cast<uint64_t>(ldq) * 2 * rows};
    const uint32_t box[3] = {64, f3r::ATT_Q_TILE, 1};
    if (make_tmap(&tq, q, 3, dims, str, box, t16)) return 1;
  }
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * 128, static_cast<uint64_t>(rows), 1};
    const uint64_t str[2] = {static_cast<uint64_t>(ldkv) * 2, static_cast<uint64_t>(ldkv) * 2 * rows};
    const uint32_t box[3] = {64, 128, 1};
    if (make_tmap(&tkv, kv, 3, dims, str, box, t16)) return 1;
  }
  f3r::AttnArgs a;
  memset(&a, 0, sizeof(a));
  a.batch = 1; a.heads = heads; a.sq = rows; a.skv = rows;
  a.scale_log2 = scale * 1.4426950408889634f;
  a.ldo = ldo; a.out = out;
  a.n_split = n_split; a.part_o = part_o; a.part_lse = part_lse;
  a.seg_off = seg_off; a.n_seg = n_seg;
  return check(f3r::launch_attention_segments(tq, tkv, a, static_cast<int>(max_tiles), f16,
                                              static_cast<cudaStream_t>(stream)),
               what);
}

static int attention_merge(const char* what, int f16, const float* part_o, const float* part_lse, int32_t n_parts,
                           void* out, int32_t ldo, int32_t batch, int32_t heads, int32_t sq, void* stream) {
  if (!part_o || !part_lse || !out || n_parts < 1) return fail("%s: bad arguments", what);
  if (ldo % 8 || ldo < heads * 64) return fail("%s: bad leading dimension", what);
  return check(f3r::launch_attention_merge(part_o, part_lse, n_parts, batch, heads, sq, out, ldo, f16,
                                           static_cast<cudaStream_t>(stream)), what);
}

int f3r_attention(const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out, int32_t ldo, float* lse,
                  int32_t batch, int32_t heads, int32_t sq, int32_t skv, float scale, void* stream) {
  return attention_full("f3r_attention", 0, q, ldq, kv, ldkv, out, ldo, lse, batch, heads, sq, skv, scale, stream);
}

int f3r_attention_partial(const void* q, int32_t ldq, const void* kv, int32_t ldkv, int32_t kv_rows_total,
                          int32_t kv_row0, int32_t skv, int32_t n_split, float* part_o, float* part_lse,
                          int32_t part_base, int32_t batch, int32_t heads, int32_t sq, float scale, void* stream) {
  return attention_partial("f3r_attention_partial", 0, q, ldq, kv, ldkv, kv_rows_total, kv_row0, skv, n_split, part_o,
                           part_lse, part_base, batch, heads, sq, scale, stream);
}

int f3r_attention_segments(const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out, int32_t ldo,
                           const int32_t* seg_off, int32_t n_seg, int32_t rows, int32_t heads, float scale,
                           int32_t n_split, float* part_o, float* part_lse, void* stream) {
  return attention_segments("f3r_attention_segments", 0, q, ldq, kv, ldkv, out, ldo, seg_off, n_seg, rows, heads, scale,
                            n_split, part_o, part_lse, stream);
}

int f3r_attention_merge(const float* part_o, const float* part_lse, int32_t n_parts, void* out, int32_t ldo,
                        int32_t batch, int32_t heads, int32_t sq, void* stream) {
  return attention_merge("f3r_attention_merge", 0, part_o, part_lse, n_parts, out, ldo, batch, heads, sq, stream);
}

int f3r_attention_f16(const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out, int32_t ldo, float* lse,
                      int32_t batch, int32_t heads, int32_t sq, int32_t skv, float scale, void* stream) {
  return attention_full("f3r_attention_f16", 1, q, ldq, kv, ldkv, out, ldo, lse, batch, heads, sq, skv, scale, stream);
}

int f3r_attention_partial_f16(const void* q, int32_t ldq, const void* kv, int32_t ldkv, int32_t kv_rows_total,
                              int32_t kv_row0, int32_t skv, int32_t n_split, float* part_o, float* part_lse,
                              int32_t part_base, int32_t batch, int32_t heads, int32_t sq, float scale, void* stream) {
  return attention_partial("f3r_attention_partial_f16", 1, q, ldq, kv, ldkv, kv_rows_total, kv_row0, skv, n_split, part_o,
                           part_lse, part_base, batch, heads, sq, scale, stream);
}

int f3r_attention_segments_f16(const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out, int32_t ldo,
                               const int32_t* seg_off, int32_t n_seg, int32_t rows, int32_t heads, float scale,
                               int32_t n_split, float* part_o, float* part_lse, void* stream) {
  return attention_segments("f3r_attention_segments_f16", 1, q, ldq, kv, ldkv, out, ldo, seg_off, n_seg, rows, heads,
                            scale, n_split, part_o, part_lse, stream);
}

int f3r_attention_merge_f16(const float* part_o, const float* part_lse, int32_t n_parts, void* out, int32_t ldo,
                            int32_t batch, int32_t heads, int32_t sq, void* stream) {
  return attention_merge("f3r_attention_merge_f16", 1, part_o, part_lse, n_parts, out, ldo, batch, heads, sq, stream);
}

static bool bad_elt(int32_t elt) { return elt != f3r::ELT_BF16 && elt != f3r::ELT_F32 && elt != f3r::ELT_F16; }

int f3r_layernorm(const float* x, const float* w, const float* b, void* out, int32_t out_f32, int32_t rows,
                  int32_t dim, float eps, void* stream) {
  if (!x || !w || !b || !out) return fail("f3r_layernorm: null operand");
  if (bad_elt(out_f32)) return fail("f3r_layernorm: out_f32=%d must be 0 (bf16), 1 (fp32) or 2 (fp16)", out_f32);
  return check(f3r::launch_layernorm(x, w, b, out, out_f32, rows, dim, eps, static_cast<cudaStream_t>(stream)),
               "f3r_layernorm (dim must be one of 128,256,384,512,768,1024)");
}

int f3r_im2col_patch(const float* img, void* out, int32_t out_f32, int32_t n, int32_t h, int32_t w, void* stream) {
  if (!img || !out) return fail("f3r_im2col_patch: null operand");
  if (bad_elt(out_f32)) return fail("f3r_im2col_patch: out_f32=%d must be 0 (bf16), 1 (fp32) or 2 (fp16)", out_f32);
  return check(f3r::launch_im2col_patch(img, out, out_f32, n, h, w, 16, static_cast<cudaStream_t>(stream)),
               "f3r_im2col_patch");
}

int f3r_im2col3x3s2(const void* in, void* out, int32_t n, int32_t h, int32_t w, int32_t c, int32_t ho, int32_t wo,
                    void* stream) {
  if (!in || !out) return fail("f3r_im2col3x3s2: null operand");
  return check(f3r::launch_im2col3x3s2(in, out, n, h, w, c, ho, wo, static_cast<cudaStream_t>(stream)),
               "f3r_im2col3x3s2");
}

int f3r_upsample2x(const void* in, void* out, int32_t f32, int32_t n, int32_t h, int32_t w, int32_t c, int32_t ho,
                   int32_t wo, void* stream) {
  if (!in || !out) return fail("f3r_upsample2x: null operand");
  if (bad_elt(f32)) return fail("f3r_upsample2x: f32=%d must be 0 (bf16), 1 (fp32) or 2 (fp16)", f32);
  if (ho > 2 * h || wo > 2 * w) return fail("f3r_upsample2x: window larger than the x2 output");
  return check(f3r::launch_upsample2x(in, out, f32, n, h, w, c, ho, wo, 2 * h, 2 * w,
                                      static_cast<cudaStream_t>(stream)),
               "f3r_upsample2x");
}

int f3r_split3(const float* in, void* out, size_t rows, int32_t k, int32_t relu, void* stream) {
  if (!in || !out) return fail("f3r_split3: null operand");
  if (k <= 0 || k % 8) return fail("f3r_split3: k=%d must be a positive multiple of 8", k);
  return check(f3r::launch_split3(in, out, rows, k, relu, static_cast<cudaStream_t>(stream)), "f3r_split3");
}

int f3r_add_f32(float* dst, const float* src, size_t count, void* stream) {
  if (!dst || !src) return fail("f3r_add_f32: null operand");
  return check(f3r::launch_add_f32(dst, src, count, static_cast<cudaStream_t>(stream)), "f3r_add_f32");
}

size_t f3r_attention_x3_workspace(int32_t batch, int32_t heads, int32_t sq, int32_t skv) {
  // q3 [batch*sq, heads*192] + k3 [batch*skv, heads*192] + v2 [batch*skv, heads*128] bf16, each 256-byte aligned
  auto al = [](size_t b) { return (b + 255) & ~static_cast<size_t>(255); };
  return al(static_cast<size_t>(batch) * sq * heads * 192 * 2) + al(static_cast<size_t>(batch) * skv * heads * 192 * 2) +
         al(static_cast<size_t>(batch) * skv * heads * 128 * 2);
}

int f3r_attention_x3(const float* q, int32_t ldq, const float* kv, int32_t ldkv, float* out, int32_t ldo, float* lse,
                     void* workspace, size_t workspace_bytes, int32_t batch, int32_t heads, int32_t sq, int32_t skv,
                     float scale, void* stream) {
  if (!q || !kv || !out || !workspace) return fail("f3r_attention_x3: null operand");
  if (batch <= 0 || heads <= 0 || sq <= 0 || skv <= 0) return fail("f3r_attention_x3: bad shape");
  if (ldq % 4 || ldkv % 4 || ldo % 4 || ldq < heads * 64 || ldkv < 2 * heads * 64 || ldo < heads * 64)
    return fail("f3r_attention_x3: bad leading dimensions");
  if (workspace_bytes < f3r_attention_x3_workspace(batch, heads, sq, skv))
    return fail("f3r_attention_x3: workspace too small (%zu < %zu bytes)", workspace_bytes,
                f3r_attention_x3_workspace(batch, heads, sq, skv));
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("f3r_attention_x3: workspace not 256-byte aligned");
  auto al = [](size_t b) { return (b + 255) & ~static_cast<size_t>(255); };
  uint8_t* w = static_cast<uint8_t*>(workspace);
  void* q3 = w;
  void* k3 = w + al(static_cast<size_t>(batch) * sq * heads * 192 * 2);
  void* v2 = static_cast<uint8_t*>(k3) + al(static_cast<size_t>(batch) * skv * heads * 192 * 2);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (check(f3r::launch_attn_split(q, ldq, kv, ldkv, q3, k3, v2, static_cast<size_t>(batch) * sq,
                                   static_cast<size_t>(batch) * skv, heads, st), "f3r_attention_x3 (split)"))
    return 1;
  CUtensorMap tq3, tk3, tv2;
  const uint32_t box[3] = {64, 128, 1};
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * 192, static_cast<uint64_t>(sq), static_cast<uint64_t>(batch)};
    const uint64_t str[2] = {static_cast<uint64_t>(heads) * 192 * 2, static_cast<uint64_t>(heads) * 192 * 2 * sq};
    if (make_tmap(&tq3, q3, 3, dims, str, box)) return 1;
  }
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * 192, static_cast<uint64_t>(skv), static_cast<uint64_t>(batch)};
    const uint64_t str[2] = {static_cast<uint64_t>(heads) * 192 * 2, static_cast<uint64_t>(heads) * 192 * 2 * skv};
    if (make_tmap(&tk3, k3, 3, dims, str, box)) return 1;
  }
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * 128, static_cast<uint64_t>(skv), static_cast<uint64_t>(batch)};
    const uint64_t str[2] = {static_cast<uint64_t>(heads) * 128 * 2, static_cast<uint64_t>(heads) * 128 * 2 * skv};
    if (make_tmap(&tv2, v2, 3, dims, str, box)) return 1;
  }
  f3r::AttnArgs a;
  memset(&a, 0, sizeof(a));
  a.batch = batch; a.heads = heads; a.sq = sq; a.skv = skv;
  a.q_tiles = (sq + 127) / 128;
  a.scale_log2 = scale * 1.4426950408889634f;
  a.ldo = ldo; a.out = out; a.lse = lse;
  return check(f3r::launch_attention_x3(tq3, tk3, tv2, a, st), "f3r_attention_x3");
}

int f3r_resample_ksize(int32_t in_size, int32_t out_size, int32_t filter) {
  if (in_size <= 0 || out_size <= 0 || (filter != 0 && filter != 1)) return -1;
  return f3r::resample_ksize(in_size, out_size, filter);
}

int f3r_resample_coeffs(int32_t in_size, int32_t out_size, int32_t filter, int32_t* bounds, int32_t* kk) {
  if (in_size <= 0 || out_size <= 0 || (filter != 0 && filter != 1) || !bounds || !kk) {
    fail("f3r_resample_coeffs: bad arguments");
    return -1;
  }
  return f3r::resample_coeffs(in_size, out_size, filter, bounds, kk);
}

int f3r_ingest_rgb8(const uint8_t* src, int32_t h, int32_t w, int32_t oh, int32_t ow, const int32_t* hb, const int32_t* hk,
                    int32_t hks, int32_t h_span_max, const int32_t* vb, const int32_t* vk, int32_t vks, uint8_t* tmp,
                    int32_t left, int32_t top, int32_t cw, int32_t ch, float* out, void* stream) {
  if (!src || !out) return fail("f3r_ingest_rgb8: null operand");
  // the horizontal pass loads the source as 32-bit words counted from src (checked before the shape)
  if (reinterpret_cast<uintptr_t>(src) & 3) return fail("f3r_ingest_rgb8: src not 4-byte aligned");
  if (h <= 0 || w <= 0 || oh <= 0 || ow <= 0 || cw <= 0 || ch <= 0) return fail("f3r_ingest_rgb8: bad shape");
  if (left < 0 || top < 0 || left + cw > ow || top + ch > oh) return fail("f3r_ingest_rgb8: crop box outside the resized image");
  if ((ow != w) != (hk != nullptr) || (oh != h) != (vk != nullptr))
    return fail("f3r_ingest_rgb8: tap tables must be given exactly for the resized dimensions");
  if (hk && (!hb || !tmp || hks <= 0 || h_span_max <= 0)) return fail("f3r_ingest_rgb8: incomplete horizontal pass arguments");
  if (vk && (!vb || vks <= 0)) return fail("f3r_ingest_rgb8: incomplete vertical pass arguments");
  return check(f3r::launch_ingest(src, h, w, oh, ow, hb, hk, hks, h_span_max, vb, vk, vks, tmp, left, top, cw, ch, out,
                                  static_cast<cudaStream_t>(stream)), "f3r_ingest_rgb8");
}

int f3r_jpeg_probe(const uint8_t* data, size_t size, f3r_jpeg_info* info) {
  if (!info || (!data && size)) return fail("f3r_jpeg_probe: null operand");
  const char* why = f3r::jpeg_probe(data, size, info);
  if (info->status != F3R_JPEG_SUPPORTED) fail("f3r_jpeg_probe: %s", why ? why : "");
  return 0;
}

int f3r_jpeg_decode(const uint8_t* data, size_t size, const uint8_t* data_dev, int32_t orientation, int32_t rotate_cw90,
                    int32_t left, int32_t top, int32_t out_w, int32_t out_h, uint8_t* out, int32_t* status_dev,
                    void* workspace, size_t workspace_bytes, void* stream) {
  if (!data || !data_dev || !out || !status_dev || !workspace) return fail("f3r_jpeg_decode: null operand");
  const char* err = f3r::launch_jpeg_decode(data, size, data_dev, orientation, rotate_cw90, left, top, out_w, out_h, out,
                                            status_dev, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
  return err ? fail("f3r_jpeg_decode: %s", err) : 0;
}

// ---------------------------------------------------------------- geometry tail
int f3r_conf_quantile(const float* conf, int32_t views, int32_t n, float q, float* thr, void* stream) {
  if (!conf || !thr) return fail("f3r_conf_quantile: null operand");
  if (views <= 0 || n <= 0 || n > (1 << 24)) return fail("f3r_conf_quantile: bad shape (n must be in [1, 2^24]: ranks are fp32)");
  if (!(q >= 0.f && q <= 1.f)) return fail("f3r_conf_quantile: q must be in [0, 1]");
  return check(f3r::launch_conf_quantile(conf, views, n, q, thr, static_cast<cudaStream_t>(stream)), "f3r_conf_quantile");
}

size_t f3r_similarity_fit_workspace(int32_t views) { return views > 0 ? f3r::similarity_fit_workspace(views) : 0; }

int f3r_similarity_fit(const float* x, const float* y, const float* conf, const float* thr, const uint8_t* valid,
                       int32_t views, int32_t n, float* rts, void* workspace, size_t workspace_bytes, void* stream) {
  if (!x || !y || !rts || !workspace) return fail("f3r_similarity_fit: null operand");
  if (views <= 0 || views > 65535 || n <= 0 || n > (1 << 29)) return fail("f3r_similarity_fit: bad shape");
  if ((conf != nullptr) != (thr != nullptr)) return fail("f3r_similarity_fit: conf and thr must be given together");
  if (workspace_bytes < f3r::similarity_fit_workspace(views)) return fail("f3r_similarity_fit: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 7) return fail("f3r_similarity_fit: workspace not 8-byte aligned");
  return check(f3r::launch_similarity_fit(x, y, conf, thr, valid, views, n, rts, static_cast<double*>(workspace),
                                          static_cast<cudaStream_t>(stream)), "f3r_similarity_fit");
}

int f3r_similarity_apply(const float* x, const float* rts, float* out, int32_t views, int32_t n, void* stream) {
  if (!x || !rts || !out) return fail("f3r_similarity_apply: null operand");
  if (views <= 0 || views > 65535 || n <= 0 || n > (1 << 29)) return fail("f3r_similarity_apply: bad shape");
  return check(f3r::launch_similarity_apply(x, rts, out, views, n, static_cast<cudaStream_t>(stream)), "f3r_similarity_apply");
}

size_t f3r_focal_workspace(int32_t views) { return views > 0 ? f3r::focal_workspace(views) : 0; }

int f3r_focal_weiszfeld(const float* pts, const float* conf, const float* thr, const float* pp, int32_t views, int32_t h,
                        int32_t w, int32_t iters, float* focal, void* workspace, size_t workspace_bytes, void* stream) {
  if (!pts || !focal || !workspace) return fail("f3r_focal_weiszfeld: null operand");
  if (views <= 0 || views > 65535 || h <= 0 || w <= 0 || static_cast<int64_t>(h) * w > (1 << 29))
    return fail("f3r_focal_weiszfeld: bad shape");
  if (iters < 0 || iters > 10000) return fail("f3r_focal_weiszfeld: bad iteration count");
  if ((conf != nullptr) != (thr != nullptr)) return fail("f3r_focal_weiszfeld: conf and thr must be given together");
  if (workspace_bytes < f3r::focal_workspace(views)) return fail("f3r_focal_weiszfeld: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 7) return fail("f3r_focal_weiszfeld: workspace not 8-byte aligned");
  return check(f3r::launch_focal_weiszfeld(pts, conf, thr, pp, views, h, w, iters, focal, static_cast<double*>(workspace),
                                           static_cast<cudaStream_t>(stream)), "f3r_focal_weiszfeld");
}

// ---------------------------------------------------------------- reconstruction metrics
size_t f3r_pc_index_workspace(int32_t n) { return n > 0 ? f3r::pc_index_workspace(n) : 0; }

int f3r_pc_index_build(const void* pts, int32_t f64, int32_t n, void* index, size_t index_bytes, void* stream) {
  if (!pts || !index) return fail("f3r_pc_index_build: null operand");
  if (n <= 0) return fail("f3r_pc_index_build: bad size n=%d (must be >= 1)", n);
  if (index_bytes < f3r::pc_index_workspace(n)) return fail("f3r_pc_index_build: index block too small");
  if (reinterpret_cast<uintptr_t>(index) & 255) return fail("f3r_pc_index_build: index block not 256-byte aligned");
  return check(f3r::launch_pc_index_build(pts, f64 != 0, n, index, static_cast<cudaStream_t>(stream)), "f3r_pc_index_build");
}

size_t f3r_pc_query_workspace(int32_t nq) { return nq > 0 ? f3r::pc_query_workspace(nq) : 0; }

int f3r_pc_nearest(const void* index, size_t index_bytes, int32_t n_ref, const void* query, int32_t f64, int32_t nq,
                   double* dist, int64_t* idx, void* workspace, size_t workspace_bytes, void* stream) {
  if (!query || !dist || !idx) return fail("f3r_pc_nearest: null operand");
  if (n_ref < 0 || nq <= 0) return fail("f3r_pc_nearest: bad sizes n_ref=%d nq=%d", n_ref, nq);
  if (n_ref > 0) {
    if (!index || !workspace) return fail("f3r_pc_nearest: null operand");
    if (index_bytes < f3r::pc_index_workspace(n_ref)) return fail("f3r_pc_nearest: index block too small");
    if (workspace_bytes < f3r::pc_query_workspace(nq)) return fail("f3r_pc_nearest: workspace too small");
    if ((reinterpret_cast<uintptr_t>(index) | reinterpret_cast<uintptr_t>(workspace)) & 255)
      return fail("f3r_pc_nearest: index or workspace not 256-byte aligned");
  }
  return check(f3r::launch_pc_nearest(index, n_ref, query, f64 != 0, nq, dist, reinterpret_cast<long long*>(idx), workspace,
                                       static_cast<cudaStream_t>(stream)), "f3r_pc_nearest");
}

int f3r_pc_knn_normals(const void* index, size_t index_bytes, int32_t n, int32_t k, double* normals, void* stream) {
  if (!index || !normals) return fail("f3r_pc_knn_normals: null operand");
  if (n <= 0) return fail("f3r_pc_knn_normals: bad size n=%d", n);
  if (k < 1 || k > 32) return fail("f3r_pc_knn_normals: k=%d must be in [1, 32]", k);
  if (index_bytes < f3r::pc_index_workspace(n)) return fail("f3r_pc_knn_normals: index block too small");
  if (reinterpret_cast<uintptr_t>(index) & 255) return fail("f3r_pc_knn_normals: index block not 256-byte aligned");
  return check(f3r::launch_pc_knn_normals(index, n, k, normals, static_cast<cudaStream_t>(stream)), "f3r_pc_knn_normals");
}

int f3r_pc_count_nonfinite(const void* pts, int32_t f64, int32_t n, uint32_t* count, void* stream) {
  if (!count || (!pts && n)) return fail("f3r_pc_count_nonfinite: null operand");
  if (n < 0) return fail("f3r_pc_count_nonfinite: bad size n=%d", n);
  return check(f3r::launch_pc_count_nonfinite(pts, f64 != 0, n, count, static_cast<cudaStream_t>(stream)),
               "f3r_pc_count_nonfinite");
}

int f3r_pc_abs_dot(const double* a, const int64_t* a_idx, const double* b, const int64_t* b_idx, int32_t n, double* out,
                   void* stream) {
  if (!a || !b || !out) return fail("f3r_pc_abs_dot: null operand");
  if (n < 0) return fail("f3r_pc_abs_dot: bad size n=%d", n);
  return check(f3r::launch_pc_abs_dot(a, reinterpret_cast<const long long*>(a_idx), b,
                                      reinterpret_cast<const long long*>(b_idx), n, out, static_cast<cudaStream_t>(stream)),
               "f3r_pc_abs_dot");
}

size_t f3r_f64_reduce_workspace(void) { return f3r::f64_reduce_workspace(); }

static int reduce_args(const char* what, const double* x, int32_t n, const double* out, const void* workspace,
                       size_t workspace_bytes) {
  if (!x || !out || !workspace) return fail("%s: null operand", what);
  if (n <= 0) return fail("%s: bad size n=%d (must be >= 1)", what, n);
  if (workspace_bytes < f3r::f64_reduce_workspace()) return fail("%s: workspace too small", what);
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("%s: workspace not 256-byte aligned", what);
  return 0;
}

int f3r_f64_mean(const double* x, int32_t n, double* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (reduce_args("f3r_f64_mean", x, n, out, workspace, workspace_bytes)) return 1;
  return check(f3r::launch_f64_mean(x, n, out, workspace, static_cast<cudaStream_t>(stream)), "f3r_f64_mean");
}

int f3r_f64_median(const double* x, int32_t n, double* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (reduce_args("f3r_f64_median", x, n, out, workspace, workspace_bytes)) return 1;
  return check(f3r::launch_f64_median(x, n, out, workspace, static_cast<cudaStream_t>(stream)), "f3r_f64_median");
}

int f3r_f64_count_below(const double* x, int32_t n, const double* th, uint64_t* count, void* stream) {
  if (!th || !count || (!x && n)) return fail("f3r_f64_count_below: null operand");
  if (n < 0) return fail("f3r_f64_count_below: bad size n=%d", n);
  return check(f3r::launch_f64_count_below(x, n, th, reinterpret_cast<unsigned long long*>(count),
                                           static_cast<cudaStream_t>(stream)), "f3r_f64_count_below");
}

// ---------------------------------------------------------------- camera poses
size_t f3r_pnp_gather_workspace(int32_t views, int32_t h, int32_t w) {
  return views > 0 && h > 0 && w > 0 && static_cast<long long>(h) * w <= (1 << 30)
             ? f3r::pnp_gather_workspace(views, h * w) : 0;
}

int f3r_pnp_gather(const float* pts, const float* conf, const uint8_t* mask, int32_t views, int32_t h, int32_t w,
                   float* out_pts, float* out_pix, int32_t* counts, void* workspace, size_t workspace_bytes, void* stream) {
  if (!pts || !out_pts || !out_pix || !counts || !workspace) return fail("f3r_pnp_gather: null operand");
  if ((conf != nullptr) == (mask != nullptr)) return fail("f3r_pnp_gather: give exactly one of conf and mask");
  if (views <= 0 || views > 65535 || h <= 0 || w <= 0 || static_cast<long long>(h) * w > (1 << 30))
    return fail("f3r_pnp_gather: bad shape views=%d h=%d w=%d", views, h, w);
  if (workspace_bytes < f3r::pnp_gather_workspace(views, h * w)) return fail("f3r_pnp_gather: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 3) return fail("f3r_pnp_gather: workspace not 4-byte aligned");
  return check(f3r::launch_pnp_gather(pts, conf, mask, views, h, w, out_pts, out_pix, counts, workspace,
                                      static_cast<cudaStream_t>(stream)), "f3r_pnp_gather");
}

// the host tables of f3r_pnp_score / f3r_pnp_inliers; returns the largest view count or -1 (after fail()) if invalid
static int pnp_tables(const char* what, const int64_t* offsets, const int32_t* view_counts, int32_t views,
                      const f3r_pnp_hyp* hyps, int32_t nh, float thr) {
  if (!offsets || !view_counts || !hyps) return fail("%s: null table", what), -1;
  if (views <= 0 || nh <= 0) return fail("%s: bad sizes views=%d nh=%d", what, views, nh), -1;
  if (!(thr >= 0.f && thr <= 3.4028234663852886e38f)) return fail("%s: threshold %g is not finite and >= 0", what, thr), -1;
  int max_count = 0;
  for (int v = 0; v < views; ++v) {
    if (view_counts[v] < 0 || offsets[v] < 0) return fail("%s: view %d has offset %lld and count %d", what, v,
                                                            static_cast<long long>(offsets[v]), view_counts[v]), -1;
    max_count = view_counts[v] > max_count ? view_counts[v] : max_count;
  }
  for (int r = 0; r < nh; ++r)
    if (hyps[r].view < 0 || hyps[r].view >= views)
      return fail("%s: hypothesis %d names view %d of %d", what, r, hyps[r].view, views), -1;
  return max_count;
}

size_t f3r_pnp_score_workspace(int32_t views, int32_t nh) {
  return views > 0 && nh > 0 ? f3r::pnp_score_workspace(views, nh) : 0;
}

int f3r_pnp_score(const float* pts, const float* pix, const int64_t* offsets, const int32_t* view_counts, int32_t views,
                  const f3r_pnp_hyp* hyps, int32_t nh, float thr, int32_t* counts, void* workspace, size_t workspace_bytes,
                  void* stream) {
  if (!pts || !pix || !counts || !workspace) return fail("f3r_pnp_score: null operand");
  if (pnp_tables("f3r_pnp_score", offsets, view_counts, views, hyps, nh, thr) < 0) return 1;
  if (workspace_bytes < f3r::pnp_score_workspace(views, nh)) return fail("f3r_pnp_score: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("f3r_pnp_score: workspace not 256-byte aligned");
  return check(f3r::launch_pnp_score(pts, pix, reinterpret_cast<const long long*>(offsets), view_counts, views, hyps, nh,
                                     thr, counts, workspace, static_cast<cudaStream_t>(stream)), "f3r_pnp_score");
}

size_t f3r_pnp_inliers_workspace(int32_t nh, int32_t max_count) {
  return nh > 0 && max_count >= 0 ? f3r::pnp_inliers_workspace(nh, max_count) : 0;
}

int f3r_pnp_inliers(const float* pts, const float* pix, const int64_t* offsets, const int32_t* view_counts, int32_t views,
                    const f3r_pnp_hyp* hyps, int32_t nh, float thr, float* out_pts, float* out_pix, int32_t* out_counts,
                    void* workspace, size_t workspace_bytes, void* stream) {
  if (!pts || !pix || !out_pts || !out_pix || !out_counts || !workspace) return fail("f3r_pnp_inliers: null operand");
  const int max_count = pnp_tables("f3r_pnp_inliers", offsets, view_counts, views, hyps, nh, thr);
  if (max_count < 0) return 1;
  if (nh > 65535) return fail("f3r_pnp_inliers: %d rows (at most 65535)", nh);
  if (workspace_bytes < f3r::pnp_inliers_workspace(nh, max_count)) return fail("f3r_pnp_inliers: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("f3r_pnp_inliers: workspace not 256-byte aligned");
  return check(f3r::launch_pnp_inliers(pts, pix, reinterpret_cast<const long long*>(offsets), view_counts, hyps, nh, thr,
                                       out_pts, out_pix, out_counts, workspace, static_cast<cudaStream_t>(stream)),
               "f3r_pnp_inliers");
}

// ---------------------------------------------------------------- camera-pose metric
static bool pose_metric_shape_ok(int32_t items, int32_t views) {
  return items >= 1 && items <= 65535 && views >= 2 && views <= 65536 &&
         static_cast<long long>(items) * views < (1ll << 31);
}

size_t f3r_pose_metric_workspace(int32_t f64, int32_t items, int32_t views) {
  return pose_metric_shape_ok(items, views) ? f3r::pose_metric_workspace(f64 != 0, items, views) : 0;
}

int f3r_pose_metric(int32_t f64, const void* pred, const void* gt, int32_t items, int32_t views, int32_t hist_max,
                    void* r_out, void* t_out, int64_t* counts, void* workspace, size_t workspace_bytes, void* stream) {
  if (!pred || !gt || !counts || !workspace) return fail("f3r_pose_metric: null operand");
  if ((r_out != nullptr) != (t_out != nullptr)) return fail("f3r_pose_metric: give both of r_out and t_out or neither");
  if (!pose_metric_shape_ok(items, views)) return fail("f3r_pose_metric: bad shape items=%d views=%d", items, views);
  if (hist_max < 1 || hist_max >= F3R_PM_MAX_BINS) return fail("f3r_pose_metric: hist_max %d not in [1, %d)", hist_max,
                                                               F3R_PM_MAX_BINS);
  if (workspace_bytes < f3r::pose_metric_workspace(f64 != 0, items, views))
    return fail("f3r_pose_metric: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 7) return fail("f3r_pose_metric: workspace not 8-byte aligned");
  return check(f3r::launch_pose_metric(f64 != 0, pred, gt, items, views, hist_max, r_out, t_out,
                                       reinterpret_cast<unsigned long long*>(counts), workspace,
                                       static_cast<cudaStream_t>(stream)), "f3r_pose_metric");
}

int f3r_pose_metric_counts(int32_t f64, const void* r, const void* t, size_t n, int32_t hist_max, int64_t* counts,
                           void* stream) {
  if (!counts || (n && (!r || !t))) return fail("f3r_pose_metric_counts: null operand");
  if (n > (1ull << 40)) return fail("f3r_pose_metric_counts: %zu angles (at most 2^40)", n);
  if (hist_max < 1 || hist_max >= F3R_PM_MAX_BINS) return fail("f3r_pose_metric_counts: hist_max %d not in [1, %d)",
                                                               hist_max, F3R_PM_MAX_BINS);
  return check(f3r::launch_pose_metric_counts(f64 != 0, r, t, static_cast<long long>(n), hist_max,
                                              reinterpret_cast<unsigned long long*>(counts),
                                              static_cast<cudaStream_t>(stream)), "f3r_pose_metric_counts");
}

// ---------------------------------------------------------------- validation criterion
static bool val_loss_shape_ok(int32_t views, int32_t items, int32_t n) {
  return views >= 1 && items >= 1 && n >= 1 && static_cast<long long>(views) * items * n < (1ll << 31);
}

size_t f3r_val_loss_workspace(int32_t views, int32_t items, int32_t n) {
  return val_loss_shape_ok(views, items, n) ? f3r::val_loss_workspace(views, items, n) : 0;
}

int f3r_val_loss(const float* gt, const uint8_t* valid, const float* pr, const float* pr_local, const float* conf,
                 const float* conf_local, const float* poses, int32_t views, int32_t items, int32_t n, float alpha,
                 int32_t log1p, int32_t gt_scale, int32_t local_scale_consistent, int32_t has_local, double* out,
                 void* workspace, size_t workspace_bytes, void* stream) {
  if (!gt || !valid || !pr || !conf || !poses || !out || !workspace) return fail("f3r_val_loss: null operand");
  if (has_local && (!pr_local || !conf_local)) return fail("f3r_val_loss: has_local needs pr_local and conf_local");
  if (!val_loss_shape_ok(views, items, n))
    return fail("f3r_val_loss: bad shape views=%d items=%d n=%d (views * items * n must be below 2^31)", views, items, n);
  if (!(alpha > 0.f) || !std::isfinite(alpha)) return fail("f3r_val_loss: alpha must be positive and finite");
  if (workspace_bytes < f3r::val_loss_workspace(views, items, n)) return fail("f3r_val_loss: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 7) return fail("f3r_val_loss: workspace not 8-byte aligned");
  return check(f3r::launch_val_loss(gt, valid, pr, pr_local, conf, conf_local, poses, views, items, n, alpha, log1p != 0,
                                    gt_scale != 0, local_scale_consistent != 0, has_local != 0, out, workspace,
                                    static_cast<cudaStream_t>(stream)), "f3r_val_loss");
}

// ---------------------------------------------------------------- viewer scene
static bool sky_shape_ok(int32_t frames, int32_t h, int32_t w) {
  return frames > 0 && h > 0 && w > 0 && static_cast<long long>(frames) * h * w < (1ll << 31);
}

size_t f3r_sky_mask_workspace(int32_t frames, int32_t h, int32_t w) {
  return sky_shape_ok(frames, h, w) ? f3r::sky_mask_workspace(frames, h, w) : 0;
}

int f3r_sky_mask(const float* img, int32_t frames, int32_t h, int32_t w, int32_t upper_rows, int32_t min_sky,
                 int8_t* not_sky, int32_t* not_sky_count, void* workspace, size_t workspace_bytes, void* stream) {
  if (!img || !not_sky || !not_sky_count || !workspace) return fail("f3r_sky_mask: null operand");
  if (!sky_shape_ok(frames, h, w)) return fail("f3r_sky_mask: bad shape frames=%d h=%d w=%d", frames, h, w);
  if (workspace_bytes < f3r::sky_mask_workspace(frames, h, w)) return fail("f3r_sky_mask: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("f3r_sky_mask: workspace not 256-byte aligned");
  return check(f3r::launch_sky_mask(img, frames, h, w, upper_rows, min_sky, not_sky, not_sky_count, workspace,
                                    static_cast<cudaStream_t>(stream)), "f3r_sky_mask");
}

size_t f3r_scene_sort_workspace(int32_t n) { return n > 0 ? f3r::scene_sort_workspace(n) : 0; }

int f3r_scene_sort(const float* conf, const float* pts, const float* img, const int8_t* not_sky, const int64_t* offsets,
                   int32_t frames, int32_t n, float* out_pts, uint8_t* out_rgb, int8_t* out_not_sky, float* max_conf,
                   void* workspace, size_t workspace_bytes, void* stream) {
  if (!conf || !pts || !img || !not_sky || !offsets || !out_pts || !out_rgb || !out_not_sky || !max_conf || !workspace)
    return fail("f3r_scene_sort: null operand");
  if (frames <= 0 || frames > (1 << 24) || n <= 0) return fail("f3r_scene_sort: bad sizes frames=%d n=%d", frames, n);
  if (workspace_bytes < f3r::scene_sort_workspace(n)) return fail("f3r_scene_sort: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("f3r_scene_sort: workspace not 256-byte aligned");
  return check(f3r::launch_scene_sort(conf, pts, img, not_sky, reinterpret_cast<const long long*>(offsets), frames, n,
                                      out_pts, out_rgb, out_not_sky, max_conf, workspace,
                                      static_cast<cudaStream_t>(stream)), "f3r_scene_sort");
}

static bool visible_sizes_ok(int32_t nseg, size_t max_len) {
  return nseg > 0 && nseg <= 65535 && max_len > 0 && max_len < (1ull << 40);
}

size_t f3r_scene_visible_workspace(int32_t nseg, size_t max_len) {
  return visible_sizes_ok(nseg, max_len) ? f3r::scene_visible_workspace(nseg, f3r::scene_visible_tiles(max_len)) : 0;
}

int f3r_scene_visible(const int64_t* segs, int32_t nseg, size_t max_len, const float* pts_g, const float* pts_l,
                      const uint8_t* rgb_g, const uint8_t* rgb_l, const int8_t* not_sky_g, const int8_t* not_sky_l,
                      int32_t mask_sky, uint64_t* total, float* out_pts, uint8_t* out_rgb, void* workspace,
                      size_t workspace_bytes, void* stream) {
  if (!segs || !pts_g || !pts_l || !rgb_g || !rgb_l || !not_sky_g || !not_sky_l || !workspace)
    return fail("f3r_scene_visible: null operand");
  if ((total != nullptr) == (out_pts != nullptr) || (out_pts != nullptr) != (out_rgb != nullptr))
    return fail("f3r_scene_visible: give total (counting) or out_pts and out_rgb (writing)");
  if (!visible_sizes_ok(nseg, max_len)) return fail("f3r_scene_visible: bad sizes nseg=%d", nseg);
  const int tiles = f3r::scene_visible_tiles(max_len);
  if (tiles > (1 << 30)) return fail("f3r_scene_visible: segments too long");
  if (workspace_bytes < f3r::scene_visible_workspace(nseg, tiles)) return fail("f3r_scene_visible: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("f3r_scene_visible: workspace not 256-byte aligned");
  return check(f3r::launch_scene_visible(reinterpret_cast<const long long*>(segs), nseg, tiles, pts_g, pts_l, rgb_g,
                                         rgb_l, not_sky_g, not_sky_l, mask_sky,
                                         reinterpret_cast<unsigned long long*>(total), out_pts, out_rgb, workspace,
                                         static_cast<cudaStream_t>(stream)), "f3r_scene_visible");
}

int f3r_ply_pack(const float* pts, const uint8_t* rgb, size_t n, uint8_t* out, void* stream) {
  if (n && (!pts || !rgb || !out)) return fail("f3r_ply_pack: null operand");
  return check(f3r::launch_ply_pack(pts, rgb, static_cast<long long>(n), out, static_cast<cudaStream_t>(stream)),
               "f3r_ply_pack");
}

size_t f3r_extent_percentiles_workspace(void) { return f3r::percentile_workspace(); }

int f3r_extent_percentiles(const float* pts, size_t n, size_t k0, size_t k1, float g0, float g1, float* out,
                           void* workspace, size_t workspace_bytes, void* stream) {
  if (!pts || !out || !workspace) return fail("f3r_extent_percentiles: null operand");
  if (n == 0 || n >= (1ull << 32) || k0 >= n || k1 >= n) return fail("f3r_extent_percentiles: bad ranks");
  if (workspace_bytes < f3r::percentile_workspace()) return fail("f3r_extent_percentiles: workspace too small");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("f3r_extent_percentiles: workspace not 256-byte aligned");
  return check(f3r::launch_extent_percentiles(pts, static_cast<long long>(n), static_cast<long long>(k0),
                                              static_cast<long long>(k1), g0, g1, out, workspace,
                                              static_cast<cudaStream_t>(stream)), "f3r_extent_percentiles");
}

int f3r_cast_bf16(const float* in, void* out, size_t count, void* stream) {
  if (!in || !out) return fail("f3r_cast_bf16: null operand");
  return check(f3r::launch_cast_bf16(in, out, count, static_cast<cudaStream_t>(stream)), "f3r_cast_bf16");
}

int f3r_cast_f16(const float* in, void* out, size_t count, void* stream) {
  if (!in || !out) return fail("f3r_cast_f16: null operand");
  return check(f3r::launch_cast_f16(in, out, count, static_cast<cudaStream_t>(stream)), "f3r_cast_f16");
}

}  // extern "C"
