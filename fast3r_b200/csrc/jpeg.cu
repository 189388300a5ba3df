// Baseline JPEG decode on the GPU, bit-exact with Pillow (libjpeg-turbo): Huffman-coded 8-bit sequential JPEGs (SOF0 /
// SOF1), grayscale or YCbCr at 4:4:4, 4:2:2 or 4:2:0, any restart interval and any Huffman tables.  The header is parsed
// on the host (jpeg_parse.h); the compressed bytes are decoded on the device in five stages:
//   1. unstuff / split   remove FF00 stuffing, fill bytes and RSTn markers (3 launches: count, scan, write), recording
//                        where each restart segment starts in the unstuffed stream;
//   2. sync              self-synchronising parallel Huffman decode (Weissenberger & Schmidt, ICPP 2018): the stream is
//                        cut into SUB_BITS-bit subsequences, one thread each.  A thread decodes from a start state (bit
//                        position, block of the MCU, coefficient index) until it passes the end of its subsequence and
//                        hands its end state to the next thread.  Starting states are guesses at first; the rounds
//                        iterate to the fixed point (block-local iterations in shared memory, then grid-wide rounds),
//                        which is the exact sequential decode because thread 0 starts at the true state.  Every
//                        restart marker is a known state, so the decoder resets there;
//   3. scan + write      a prefix sum of the per-subsequence block counts and DC-difference sums (segmented at restart
//                        markers) gives every thread its first block index and DC predictors; a second decode pass
//                        writes the coefficients in natural order and checks every segment's block count;
//   4. IDCT              dequantise + libjpeg's accurate integer IDCT (jpeg_math.h), one thread per 8x8 block;
//   5. colour            fancy chroma upsampling + YCbCr -> RGB, stored through the orientation / rotation / crop index
//                        map as the (h, w, 3) uint8 image the resize reads.
// A stream the device cannot decode consistently ends with a non-zero status word, never a fault: every index the
// entropy decoder derives is bounds-checked.
#include <cstring>
#include <new>

#include "../../include/fast3r_b200.h"
#include "common.cuh"
#include "f3r_kernels.h"
#include "jpeg_math.h"
#include "jpeg_parse.h"

namespace f3r {

using jpeg::HuffTable;

namespace {

constexpr int SUB_BITS = 1024;       // bits per subsequence (one thread)
constexpr int SYNC_THREADS = 128;    // subsequences per sync CTA (block-local iterations)
constexpr int MAX_ROUNDS = 12;       // grid-wide sync rounds before the stream is reported unsynchronisable
constexpr int UNSTUFF_THREADS = 256, UNSTUFF_BYTES = 16, UNSTUFF_CHUNK = UNSTUFF_THREADS * UNSTUFF_BYTES;
constexpr int SCAN_THREADS = 1024;
constexpr uint32_t ST_END = 255, ST_ERR = 254;

__constant__ uint8_t c_natural[64] = F3R_JPEG_NATURAL;

struct DevTables {
  HuffTable dc[2], ac[2];
  uint16_t qt[3][64];
};
static_assert(sizeof(DevTables) % 16 == 0, "DevTables is copied as uint4");

struct Rec {  // per subsequence: blocks completed and DC differences summed since its start or its last restart
  int32_t reset, seg, cnt, dc[3];
};

struct Params {
  const uint8_t* scan;
  uint32_t scan_bytes;
  int32_t ncomp, width, height, hs, vs;
  int32_t bpm, mcux, mcus, ri, nseg;
  int32_t mcu_comp[6], mcu_dx[6], mcu_dy[6];
  int32_t comp_h[3], comp_v[3], td[3], ta[3];
  int32_t bw[3], bh[3];
  uint32_t coef_off[3];  // in blocks
  size_t plane_off[3];   // in bytes
  uint32_t total_blocks, nsub_max;
  // workspace
  const DevTables* tab;
  uint8_t* stream;       // unstuffed bytes (+ slack)
  uint32_t* chunk;       // [nchunks][2] kept bytes / RST markers, then their exclusive prefix
  uint32_t* seg_start;   // [nseg + 1] first byte of each segment in `stream`
  uint32_t* hdr;         // [0] unstuffed bytes, [1] error flags, [2] end of stream reached, [3..] sync changed flags
  uint64_t* st[2];       // [nsub_max + 1] start states, ping-pong
  Rec* rec;              // [nsub_max]
  Rec* pre;              // [nsub_max] exclusive prefix of rec
  int16_t* coef;         // [total_blocks][64] natural order
  uint8_t* planes;
};

__host__ __device__ __forceinline__ uint64_t pack(uint32_t p, uint32_t blk, uint32_t z) {
  return (static_cast<uint64_t>(p) << 16) | (blk << 8) | z;
}
__device__ __forceinline__ uint32_t st_p(uint64_t s) { return static_cast<uint32_t>(s >> 16); }
__device__ __forceinline__ uint32_t st_blk(uint64_t s) { return static_cast<uint32_t>(s >> 8) & 255; }
__device__ __forceinline__ uint32_t st_z(uint64_t s) { return static_cast<uint32_t>(s) & 255; }

__device__ __forceinline__ uint32_t ld_be32(const uint8_t* s, uint32_t word) {
  return __byte_perm(__ldg(reinterpret_cast<const uint32_t*>(s) + word), 0, 0x0123);
}
// 32 bits of the unstuffed stream starting at bit p, MSB first
__device__ __forceinline__ uint32_t peek(const uint8_t* s, uint32_t p) {
  const uint32_t w = p >> 5;
  return __funnelshift_l(ld_be32(s, w + 1), ld_be32(s, w), p & 31);
}

__device__ __forceinline__ int huff(const HuffTable& t, uint32_t v, int& len) {
  const uint32_t e = t.lut[v >> (32 - jpeg::kLutBits)];
  if (e) {
    len = static_cast<int>(e >> 8);
    return static_cast<int>(e & 255);
  }
  for (int l = jpeg::kLutBits + 1; l <= 16; ++l) {
    const int32_t code = static_cast<int32_t>(v >> (32 - l));
    if (code <= t.maxcode[l]) {
      len = l;
      return t.vals[(t.valoff[l] + code) & 255];
    }
  }
  return -1;
}

__device__ __forceinline__ int extend(uint32_t v, int s) {
  return static_cast<int>(v) < (1 << (s - 1)) ? static_cast<int>(v) - (1 << s) + 1 : static_cast<int>(v);
}

__device__ __forceinline__ void load_tables(const DevTables* g, DevTables* s) {
  const uint4* src = reinterpret_cast<const uint4*>(g);
  uint4* dst = reinterpret_cast<uint4*>(s);
  for (int i = threadIdx.x; i < static_cast<int>(sizeof(DevTables) / 16); i += blockDim.x) dst[i] = __ldg(src + i);
  __syncthreads();
}

__device__ __forceinline__ int find_seg(const Params& P, uint32_t p) {
  int lo = 0, hi = P.nseg - 1;  // largest seg with seg_start[seg] * 8 <= p
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (P.seg_start[mid] * 8u <= p) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// Decodes from state s until the first code boundary at or past `stop` (or the end of the stream).  `blocks` / `dc`
// carry the running block index and DC predictors (sync pass: relative to the start, or to the last restart; write
// pass: absolute).  Returns the end state.
template <bool WRITE>
__device__ uint64_t run(const Params& P, const DevTables& T, uint64_t s, uint32_t stop, int& blocks, int dc[3], Rec* r) {
  uint32_t p = st_p(s), blk = st_blk(s), z = st_z(s);
  if (blk == ST_END) return s;
  int seg = find_seg(P, p);
  uint32_t seg_end = P.seg_start[seg + 1] * 8u;
  const uint32_t total_bits = P.hdr[0] * 8u;
  if (p > seg_end || blk >= static_cast<uint32_t>(P.bpm) || z > 63) return pack(p, ST_ERR, 0);
  int16_t* cur = nullptr;
  while (true) {
    const uint32_t rem = seg_end - p;
    if (rem < 8 && (rem == 0 || (peek(P.stream, p) >> (32 - rem)) == (1u << rem) - 1u)) {  // restart segment done
      if (WRITE) {
        const int expect = static_cast<int>(min(static_cast<long long>(seg + 1) * P.ri, static_cast<long long>(P.mcus))) * P.bpm;
        if (blk != 0 || z != 0 || blocks != expect) atomicOr(P.hdr + 1, F3R_JPEG_ERR_COUNT);
      }
      if (++seg >= P.nseg) {
        if (WRITE) P.hdr[2] = 1;
        return pack(total_bits, ST_END, 0);
      }
      p = P.seg_start[seg] * 8u;
      seg_end = P.seg_start[seg + 1] * 8u;
      blk = 0;
      z = 0;
      blocks = seg * P.ri * P.bpm;
      dc[0] = dc[1] = dc[2] = 0;
      if (!WRITE) { r->reset = 1; r->seg = seg; }
      continue;
    }
    if (p >= stop) break;
    const uint32_t v = peek(P.stream, p);
    const int c = P.mcu_comp[blk];
    int len;
    if (z == 0) {
      const int sz = huff(T.dc[P.td[c]], v, len);
      if (sz < 0 || sz > 15) return pack(p, ST_ERR, 0);
      dc[c] += sz ? extend((v << len) >> (32 - sz), sz) : 0;
      p += len + sz;
      if (WRITE) {
        if (blocks < 0 || static_cast<uint32_t>(blocks) >= P.total_blocks) return pack(p, ST_ERR, 0);
        const int mcu = blocks / P.bpm;
        int bx, by;
        if (P.ncomp == 1) { bx = mcu % P.mcux; by = mcu / P.mcux; }
        else {
          bx = (mcu % P.mcux) * P.comp_h[c] + P.mcu_dx[blk];
          by = (mcu / P.mcux) * P.comp_v[c] + P.mcu_dy[blk];
        }
        cur = P.coef + (static_cast<size_t>(P.coef_off[c]) + static_cast<size_t>(by) * P.bw[c] + bx) * 64;
        cur[0] = static_cast<int16_t>(dc[c]);
      }
      z = 1;
    } else {
      const int rs = huff(T.ac[P.ta[c]], v, len);
      if (rs < 0) return pack(p, ST_ERR, 0);
      const int run_len = rs >> 4, sz = rs & 15;
      if (sz == 0) {
        z = run_len == 15 ? z + 16 : 64;
      } else {
        z += run_len;
        if (z > 63) return pack(p, ST_ERR, 0);
        if (WRITE) {
          if (cur == nullptr) {  // this thread started inside the block
            if (blocks < 0 || static_cast<uint32_t>(blocks) >= P.total_blocks) return pack(p, ST_ERR, 0);
            const int mcu = blocks / P.bpm;
            int bx, by;
            if (P.ncomp == 1) { bx = mcu % P.mcux; by = mcu / P.mcux; }
            else {
              bx = (mcu % P.mcux) * P.comp_h[c] + P.mcu_dx[blk];
              by = (mcu / P.mcux) * P.comp_v[c] + P.mcu_dy[blk];
            }
            cur = P.coef + (static_cast<size_t>(P.coef_off[c]) + static_cast<size_t>(by) * P.bw[c] + bx) * 64;
          }
          cur[c_natural[z]] = static_cast<int16_t>(extend((v << len) >> (32 - sz), sz));
        }
        ++z;
      }
      p += len + sz;
      if (z >= 64) {
        ++blocks;
        blk = blk + 1 == static_cast<uint32_t>(P.bpm) ? 0 : blk + 1;
        z = 0;
        cur = nullptr;
      }
    }
    if (p > seg_end) return pack(p, ST_ERR, 0);
  }
  return pack(p, blk, z);
}

// ---------------------------------------------------------------- stage 1: unstuff / split
__device__ __forceinline__ void unstuff_flags(const Params& P, uint32_t i, uint32_t& keep, uint32_t& rst) {
  const uint32_t b = P.scan[i];
  const uint32_t prev = i > 0 ? P.scan[i - 1] : 0;
  const uint32_t next = i + 1 < P.scan_bytes ? P.scan[i + 1] : 0;
  if (b == 0xFF) { keep = next == 0x00; rst = 0; }
  else if (prev == 0xFF) { keep = 0; rst = b >= 0xD0 && b <= 0xD7; }  // stuffed zero or RSTn code
  else { keep = 1; rst = 0; }
}

__global__ void __launch_bounds__(UNSTUFF_THREADS) jpeg_unstuff_count_kernel(Params P) {
  const uint32_t i0 = blockIdx.x * UNSTUFF_CHUNK + threadIdx.x * UNSTUFF_BYTES;
  uint32_t kept = 0, rsts = 0;
  for (uint32_t i = i0; i < min(i0 + UNSTUFF_BYTES, P.scan_bytes); ++i) {
    uint32_t k, r;
    unstuff_flags(P, i, k, r);
    kept += k;
    rsts += r;
  }
  __shared__ uint32_t sk[UNSTUFF_THREADS / 32], sr[UNSTUFF_THREADS / 32];
  for (int o = 16; o; o >>= 1) {
    kept += __shfl_xor_sync(0xffffffffu, kept, o);
    rsts += __shfl_xor_sync(0xffffffffu, rsts, o);
  }
  if ((threadIdx.x & 31) == 0) { sk[threadIdx.x >> 5] = kept; sr[threadIdx.x >> 5] = rsts; }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t a = 0, b = 0;
    for (int w = 0; w < UNSTUFF_THREADS / 32; ++w) { a += sk[w]; b += sr[w]; }
    P.chunk[2 * blockIdx.x] = a;
    P.chunk[2 * blockIdx.x + 1] = b;
  }
}

// Exclusive prefix of the chunk counts (one CTA), segment bounds 0 and total, and the Rec-scan helper below.
__global__ void __launch_bounds__(SCAN_THREADS) jpeg_chunk_scan_kernel(Params P, uint32_t nchunks) {
  __shared__ uint2 buf[SCAN_THREADS];
  const uint32_t per = (nchunks + SCAN_THREADS - 1) / SCAN_THREADS;
  const uint32_t a = threadIdx.x * per, b = min(a + per, nchunks);
  uint2 agg = make_uint2(0, 0);
  for (uint32_t i = a; i < b; ++i) { agg.x += P.chunk[2 * i]; agg.y += P.chunk[2 * i + 1]; }
  buf[threadIdx.x] = agg;
  __syncthreads();
  for (int off = 1; off < SCAN_THREADS; off <<= 1) {
    uint2 v = buf[threadIdx.x];
    if (static_cast<int>(threadIdx.x) >= off) { v.x += buf[threadIdx.x - off].x; v.y += buf[threadIdx.x - off].y; }
    __syncthreads();
    buf[threadIdx.x] = v;
    __syncthreads();
  }
  uint2 run = threadIdx.x ? buf[threadIdx.x - 1] : make_uint2(0, 0);
  for (uint32_t i = a; i < b; ++i) {
    const uint32_t k = P.chunk[2 * i], r = P.chunk[2 * i + 1];
    P.chunk[2 * i] = run.x;
    P.chunk[2 * i + 1] = run.y;
    run.x += k;
    run.y += r;
  }
  if (threadIdx.x == SCAN_THREADS - 1) {
    const uint2 tot = buf[SCAN_THREADS - 1];
    P.hdr[0] = tot.x;
    P.seg_start[0] = 0;
    P.seg_start[P.nseg] = tot.x;
    if (tot.y != static_cast<uint32_t>(P.nseg - 1)) atomicOr(P.hdr + 1, F3R_JPEG_ERR_COUNT);
  }
}

__global__ void __launch_bounds__(UNSTUFF_THREADS) jpeg_unstuff_write_kernel(Params P) {
  const uint32_t i0 = blockIdx.x * UNSTUFF_CHUNK + threadIdx.x * UNSTUFF_BYTES;
  const uint32_t i1 = min(i0 + UNSTUFF_BYTES, P.scan_bytes);
  uint32_t kept = 0, rsts = 0;
  for (uint32_t i = i0; i < i1; ++i) {
    uint32_t k, r;
    unstuff_flags(P, i, k, r);
    kept += k;
    rsts += r;
  }
  // block-exclusive prefix of (kept, rsts)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t ik = kept, ir = rsts;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t tk = __shfl_up_sync(0xffffffffu, ik, o), tr = __shfl_up_sync(0xffffffffu, ir, o);
    if (lane >= o) { ik += tk; ir += tr; }
  }
  __shared__ uint32_t wk[UNSTUFF_THREADS / 32], wr[UNSTUFF_THREADS / 32];
  if (lane == 31) { wk[warp] = ik; wr[warp] = ir; }
  __syncthreads();
  uint32_t bk = P.chunk[2 * blockIdx.x], br = P.chunk[2 * blockIdx.x + 1];
  for (int w = 0; w < warp; ++w) { bk += wk[w]; br += wr[w]; }
  uint32_t o = bk + ik - kept, r = br + ir - rsts;
  for (uint32_t i = i0; i < i1; ++i) {
    uint32_t k, rr;
    unstuff_flags(P, i, k, rr);
    if (k) P.stream[o++] = P.scan[i];
    if (rr) {
      if (r + 1 < static_cast<uint32_t>(P.nseg)) P.seg_start[r + 1] = o;
      ++r;
    }
  }
}

// ---------------------------------------------------------------- stage 2: sync
__global__ void jpeg_sync_init_kernel(Params P) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > P.nsub_max) return;
  P.st[0][i] = pack(i * static_cast<uint32_t>(SUB_BITS), 0, 0);
  if (i == 0) P.st[1][0] = pack(0, 0, 0);
}

__global__ void __launch_bounds__(SYNC_THREADS) jpeg_sync_kernel(Params P, int round) {
  uint32_t* changed = P.hdr + 3;
  if (round > 0 && changed[round - 1] == 0) return;  // converged in an earlier round
  __shared__ DevTables T;
  __shared__ uint64_t s_out[SYNC_THREADS];
  load_tables(P.tab, &T);
  const uint64_t* in = P.st[round & 1];
  uint64_t* out = P.st[(round + 1) & 1];
  const uint32_t nsub = (P.hdr[0] * 8u + SUB_BITS - 1) / SUB_BITS;
  const uint32_t i = blockIdx.x * SYNC_THREADS + threadIdx.x;
  const bool active = i < nsub;
  const uint64_t guess = pack(i * static_cast<uint32_t>(SUB_BITS), 0, 0);
  uint64_t s = active ? in[i] : 0;
  if (st_blk(s) == ST_ERR) s = guess;
  uint64_t e = 0;
  Rec r;
  bool dirty = true;  // re-decode only when the start state moved
  for (int it = 0; it <= SYNC_THREADS; ++it) {  // thread t's input is final after t iterations
    if (active && dirty) {
      r = Rec{0, 0, 0, {0, 0, 0}};
      int blocks = 0, dc[3] = {0, 0, 0};
      e = run<false>(P, T, s, (i + 1) * static_cast<uint32_t>(SUB_BITS), blocks, dc, &r);
      r.cnt = blocks;
      r.dc[0] = dc[0]; r.dc[1] = dc[1]; r.dc[2] = dc[2];
    }
    s_out[threadIdx.x] = e;
    __syncthreads();
    uint64_t ns = s;
    if (threadIdx.x > 0 && active) {
      ns = s_out[threadIdx.x - 1];
      if (st_blk(ns) == ST_ERR) ns = guess;
    }
    dirty = ns != s;
    if (!__syncthreads_or(dirty)) break;
    s = ns;
  }
  if (active) {
    out[i + 1] = e;
    P.rec[i] = r;
    if (e != in[i + 1]) changed[round] = 1;
  }
}

// ---------------------------------------------------------------- stage 3: scan + write
__device__ __forceinline__ Rec rec_op(const Rec& a, const Rec& b) {
  if (b.reset) return b;
  return Rec{a.reset, a.seg, a.cnt + b.cnt, {a.dc[0] + b.dc[0], a.dc[1] + b.dc[1], a.dc[2] + b.dc[2]}};
}

__global__ void __launch_bounds__(SCAN_THREADS) jpeg_rec_scan_kernel(Params P) {
  __shared__ Rec buf[SCAN_THREADS];
  const uint32_t n = (P.hdr[0] * 8u + SUB_BITS - 1) / SUB_BITS;
  const uint32_t per = (n + SCAN_THREADS - 1) / SCAN_THREADS;
  const uint32_t a = threadIdx.x * per, b = min(a + per, n);
  Rec agg{0, 0, 0, {0, 0, 0}};
  for (uint32_t i = a; i < b; ++i) agg = rec_op(agg, P.rec[i]);
  buf[threadIdx.x] = agg;
  __syncthreads();
  for (int off = 1; off < SCAN_THREADS; off <<= 1) {
    Rec v = buf[threadIdx.x];
    if (static_cast<int>(threadIdx.x) >= off) v = rec_op(buf[threadIdx.x - off], v);
    __syncthreads();
    buf[threadIdx.x] = v;
    __syncthreads();
  }
  Rec run = threadIdx.x ? buf[threadIdx.x - 1] : Rec{0, 0, 0, {0, 0, 0}};
  for (uint32_t i = a; i < b; ++i) {
    const Rec x = P.rec[i];
    P.pre[i] = run;
    run = rec_op(run, x);
  }
}

__global__ void __launch_bounds__(SYNC_THREADS) jpeg_write_kernel(Params P) {
  __shared__ DevTables T;
  load_tables(P.tab, &T);
  const uint32_t nsub = (P.hdr[0] * 8u + SUB_BITS - 1) / SUB_BITS;
  const uint32_t i = blockIdx.x * SYNC_THREADS + threadIdx.x;
  if (i >= nsub) return;
  const uint64_t s = P.st[0][i];
  if (st_blk(s) == ST_ERR) { atomicOr(P.hdr + 1, F3R_JPEG_ERR_CODE); return; }
  const Rec pre = P.pre[i];
  int blocks = pre.cnt, dc[3] = {pre.dc[0], pre.dc[1], pre.dc[2]};
  const uint64_t e = run<true>(P, T, s, (i + 1) * static_cast<uint32_t>(SUB_BITS), blocks, dc, nullptr);
  if (st_blk(e) == ST_ERR) atomicOr(P.hdr + 1, F3R_JPEG_ERR_CODE);
  else if (e != P.st[0][i + 1]) atomicOr(P.hdr + 1, F3R_JPEG_ERR_SYNC);
}

// ---------------------------------------------------------------- stage 4: IDCT
__global__ void __launch_bounds__(128) jpeg_idct_kernel(Params P) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= P.total_blocks) return;
  const int c = (P.ncomp == 3 && b >= P.coef_off[2]) ? 2 : (P.ncomp == 3 && b >= P.coef_off[1]) ? 1 : 0;
  const uint32_t lb = b - P.coef_off[c];
  const uint32_t by = lb / P.bw[c], bx = lb - by * P.bw[c];
  __align__(16) int16_t blk[64];
  const uint4* src = reinterpret_cast<const uint4*>(P.coef + static_cast<size_t>(b) * 64);
#pragma unroll
  for (int k = 0; k < 8; ++k) reinterpret_cast<uint4*>(blk)[k] = __ldg(src + k);
  __align__(16) uint16_t q[64];
#pragma unroll
  for (int k = 0; k < 8; ++k) reinterpret_cast<uint4*>(q)[k] = __ldg(reinterpret_cast<const uint4*>(P.tab->qt[c]) + k);
  const int stride = P.bw[c] * 8;
  uint8_t* out = P.planes + P.plane_off[c] + static_cast<size_t>(by) * 8 * stride + bx * 8;
  __align__(8) uint8_t px[64];
  jpeg::idct_islow(blk, q, px, 8);
#pragma unroll
  for (int r = 0; r < 8; ++r) *reinterpret_cast<uint2*>(out + static_cast<size_t>(r) * stride) = reinterpret_cast<uint2*>(px)[r];
}

// ---------------------------------------------------------------- stage 5: upsample + colour + oriented store
struct Map { int32_t m[6]; };

__global__ void __launch_bounds__(256) jpeg_color_kernel(Params P, Map M, int out_w, int out_h, uint8_t* __restrict__ out) {
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
  if (ox >= out_w) return;
  const int x = M.m[0] * ox + M.m[1] * oy + M.m[2], y = M.m[3] * ox + M.m[4] * oy + M.m[5];
  const uint8_t* Yp = P.planes + P.plane_off[0];
  const int Y = __ldg(Yp + static_cast<size_t>(y) * (P.bw[0] * 8) + x);
  uint8_t* o = out + (static_cast<size_t>(oy) * out_w + ox) * 3;
  if (P.ncomp == 1) {
    o[0] = o[1] = o[2] = static_cast<uint8_t>(Y);
    return;
  }
  const int dw = (P.width + P.hs - 1) / P.hs, dh = (P.height + P.vs - 1) / P.vs;
  const int cb = jpeg::upsample(P.planes + P.plane_off[1], P.bw[1] * 8, dw, dh, P.hs, P.vs, x, y);
  const int cr = jpeg::upsample(P.planes + P.plane_off[2], P.bw[2] * 8, dw, dh, P.hs, P.vs, x, y);
  uint8_t rgb[3];
  jpeg::ycc_to_rgb(Y, cb, cr, rgb);
  o[0] = rgb[0]; o[1] = rgb[1]; o[2] = rgb[2];
}

__global__ void jpeg_finish_kernel(Params P, int32_t* status) {
  uint32_t s = P.hdr[1];
  if (P.hdr[3 + MAX_ROUNDS - 1]) s |= F3R_JPEG_ERR_SYNC;
  if (!P.hdr[2]) s |= F3R_JPEG_ERR_TRUNC;
  *status = static_cast<int32_t>(s);
}

// ---------------------------------------------------------------- host side
struct Layout {
  size_t tab, stream, chunk, seg, hdr, st0, st1, rec, pre, coef, planes, total;
  uint32_t nchunks, nsub_max, total_blocks;
  uint32_t coef_off[3];
  size_t plane_off[3];
  int32_t bw[3], bh[3];
};

size_t align256(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

void layout(const jpeg::Header& h, Layout* L) {
  L->nchunks = static_cast<uint32_t>((h.scan_bytes + UNSTUFF_CHUNK - 1) / UNSTUFF_CHUNK);
  L->nsub_max = static_cast<uint32_t>((h.scan_bytes * 8 + SUB_BITS - 1) / SUB_BITS);
  uint32_t blocks = 0;
  size_t plane = 0;
  for (int c = 0; c < 3; ++c) {
    L->bw[c] = L->bh[c] = 0;
    L->coef_off[c] = blocks;
    L->plane_off[c] = plane;
    if (c >= h.ncomp) continue;
    L->bw[c] = h.mcux * h.comp_h[c];
    L->bh[c] = h.mcuy * h.comp_v[c];
    blocks += static_cast<uint32_t>(L->bw[c]) * L->bh[c];
    plane += static_cast<size_t>(L->bw[c]) * L->bh[c] * 64;
  }
  L->total_blocks = blocks;
  size_t o = 0;
  L->tab = o;    o = align256(o + sizeof(DevTables));
  L->stream = o; o = align256(o + h.scan_bytes + 16);
  L->chunk = o;  o = align256(o + static_cast<size_t>(L->nchunks + 1) * 8);
  L->seg = o;    o = align256(o + (static_cast<size_t>(h.segments) + 1) * 4);
  L->hdr = o;    o = align256(o + (3 + MAX_ROUNDS) * 4);
  L->st0 = o;    o = align256(o + (static_cast<size_t>(L->nsub_max) + 2) * 8);
  L->st1 = o;    o = align256(o + (static_cast<size_t>(L->nsub_max) + 2) * 8);
  L->rec = o;    o = align256(o + static_cast<size_t>(L->nsub_max + 1) * sizeof(Rec));
  L->pre = o;    o = align256(o + static_cast<size_t>(L->nsub_max + 1) * sizeof(Rec));
  L->coef = o;   o = align256(o + static_cast<size_t>(blocks) * 128);
  L->planes = o; o = align256(o + plane);
  L->total = o;
}

struct HeaderBox {  // the parsed header is ~6 KB: keep it off the caller's stack
  jpeg::Header h;
};

}  // namespace

const char* jpeg_probe(const uint8_t* data, size_t size, f3r_jpeg_info* info) {
  HeaderBox* b = new (std::nothrow) HeaderBox;
  if (!b) return "out of host memory";
  const int st = jpeg::parse(data, size, &b->h);
  const jpeg::Header& h = b->h;
  memset(info, 0, sizeof(*info));
  info->status = st;
  info->width = h.width;
  info->height = h.height;
  info->components = h.ncomp;
  if (st == jpeg::kSupported) {
    info->h_samp = h.hmax;
    info->v_samp = h.vmax;
    info->restart_interval = h.restart_interval;
    info->segments = h.segments;
    info->scan_offset = h.scan_offset;
    info->scan_bytes = h.scan_bytes;
    Layout L;
    layout(h, &L);
    info->workspace_bytes = L.total;
  }
  const char* why = h.why;
  delete b;
  return why;
}

const char* launch_jpeg_decode(const uint8_t* data, size_t size, const uint8_t* data_dev, int orientation, int rotate_cw90,
                               int left, int top, int out_w, int out_h, uint8_t* out, int32_t* status, void* workspace,
                               size_t workspace_bytes, cudaStream_t stream) {
  HeaderBox* b = new (std::nothrow) HeaderBox;
  if (!b) return "out of host memory";
  struct Free { HeaderBox* b; ~Free() { delete b; } } guard{b};
  const jpeg::Header& h = b->h;
  if (jpeg::parse(data, size, &b->h) != jpeg::kSupported) return "not a JPEG the GPU decodes (probe it first)";
  Layout L;
  layout(h, &L);
  if (workspace_bytes < L.total) return "workspace too small";
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return "workspace not 256-byte aligned";
  const int w1 = (orientation >= 5 && orientation <= 8) ? h.height : h.width;
  const int h1 = (orientation >= 5 && orientation <= 8) ? h.width : h.height;
  const int w2 = rotate_cw90 ? h1 : w1, h2 = rotate_cw90 ? w1 : h1;
  if (left < 0 || top < 0 || out_w <= 0 || out_h <= 0 || left + out_w > w2 || top + out_h > h2)
    return "crop box outside the oriented image";
  if (h.scan_bytes >= (1u << 28)) return "scan too large";
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  DevTables* tab = new (std::nothrow) DevTables;
  if (!tab) return "out of host memory";
  for (int i = 0; i < 2; ++i) { tab->dc[i] = h.dc[i]; tab->ac[i] = h.ac[i]; }
  for (int c = 0; c < 3; ++c) memcpy(tab->qt[c], h.qt[c < h.ncomp ? h.comp_tq[c] : 0], 128);
  // pageable source: the copy is staged before cudaMemcpyAsync returns, so the host buffer can go right after
  cudaError_t e = cudaMemcpyAsync(ws + L.tab, tab, sizeof(DevTables), cudaMemcpyHostToDevice, stream);
  delete tab;
  if (e != cudaSuccess) return cudaGetErrorString(e);
  Params P;
  memset(&P, 0, sizeof(P));
  P.scan = data_dev + h.scan_offset;
  P.scan_bytes = static_cast<uint32_t>(h.scan_bytes);
  P.ncomp = h.ncomp; P.width = h.width; P.height = h.height; P.hs = h.hmax; P.vs = h.vmax;
  P.bpm = h.blocks_per_mcu; P.mcux = h.mcux; P.mcus = h.mcux * h.mcuy;
  P.ri = h.restart_interval ? h.restart_interval : P.mcus;
  P.nseg = h.segments;
  for (int k = 0; k < 6; ++k) { P.mcu_comp[k] = h.mcu_comp[k]; P.mcu_dx[k] = h.mcu_dx[k]; P.mcu_dy[k] = h.mcu_dy[k]; }
  for (int c = 0; c < 3; ++c) {
    P.comp_h[c] = h.comp_h[c]; P.comp_v[c] = h.comp_v[c]; P.td[c] = h.comp_td[c]; P.ta[c] = h.comp_ta[c];
    P.bw[c] = L.bw[c]; P.bh[c] = L.bh[c]; P.coef_off[c] = L.coef_off[c]; P.plane_off[c] = L.plane_off[c];
  }
  P.total_blocks = L.total_blocks;
  P.nsub_max = L.nsub_max;
  P.tab = reinterpret_cast<const DevTables*>(ws + L.tab);
  P.stream = ws + L.stream;
  P.chunk = reinterpret_cast<uint32_t*>(ws + L.chunk);
  P.seg_start = reinterpret_cast<uint32_t*>(ws + L.seg);
  P.hdr = reinterpret_cast<uint32_t*>(ws + L.hdr);
  P.st[0] = reinterpret_cast<uint64_t*>(ws + L.st0);
  P.st[1] = reinterpret_cast<uint64_t*>(ws + L.st1);
  P.rec = reinterpret_cast<Rec*>(ws + L.rec);
  P.pre = reinterpret_cast<Rec*>(ws + L.pre);
  P.coef = reinterpret_cast<int16_t*>(ws + L.coef);
  P.planes = ws + L.planes;
  if ((e = cudaMemsetAsync(P.hdr, 0, (3 + MAX_ROUNDS) * 4, stream)) != cudaSuccess) return cudaGetErrorString(e);
  if ((e = cudaMemsetAsync(P.coef, 0, static_cast<size_t>(L.total_blocks) * 128, stream)) != cudaSuccess)
    return cudaGetErrorString(e);
  const uint32_t nchunks = L.nchunks > 0 ? L.nchunks : 1;
  const uint32_t sync_ctas = (L.nsub_max + SYNC_THREADS - 1) / SYNC_THREADS > 0 ? (L.nsub_max + SYNC_THREADS - 1) / SYNC_THREADS : 1;
  Map M;
  jpeg::orient_map(h.width, h.height, orientation, rotate_cw90, left, top, M.m);
  if ((e = launch(jpeg_unstuff_count_kernel, nchunks, UNSTUFF_THREADS, 0, stream, false, P)) != cudaSuccess ||
      (e = launch(jpeg_chunk_scan_kernel, 1, SCAN_THREADS, 0, stream, false, P, L.nchunks)) != cudaSuccess ||
      (e = launch(jpeg_unstuff_write_kernel, nchunks, UNSTUFF_THREADS, 0, stream, false, P)) != cudaSuccess ||
      (e = launch(jpeg_sync_init_kernel, (L.nsub_max + 2 + 255) / 256, 256, 0, stream, false, P)) != cudaSuccess)
    return cudaGetErrorString(e);
  for (int r = 0; r < MAX_ROUNDS; ++r)
    if ((e = launch(jpeg_sync_kernel, sync_ctas, SYNC_THREADS, 0, stream, false, P, r)) != cudaSuccess)
      return cudaGetErrorString(e);
  if ((e = launch(jpeg_rec_scan_kernel, 1, SCAN_THREADS, 0, stream, false, P)) != cudaSuccess ||
      (e = launch(jpeg_write_kernel, sync_ctas, SYNC_THREADS, 0, stream, false, P)) != cudaSuccess ||
      (e = launch(jpeg_idct_kernel, (L.total_blocks + 127) / 128, 128, 0, stream, false, P)) != cudaSuccess ||
      (e = launch(jpeg_color_kernel, dim3((out_w + 255) / 256, out_h), 256, 0, stream, false, P, M, out_w, out_h,
                  out)) != cudaSuccess ||
      (e = launch(jpeg_finish_kernel, 1, 1, 0, stream, false, P, status)) != cudaSuccess)
    return cudaGetErrorString(e);
  return nullptr;
}

}  // namespace f3r
