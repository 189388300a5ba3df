// Host/device per-sample arithmetic of the baseline JPEG decoder (jpeg.cu): dequantisation + libjpeg's accurate integer
// inverse DCT, libjpeg-turbo's "fancy" chroma upsampling, its fixed-point YCbCr -> RGB conversion, and the index map of
// EXIF orientation + 90-degree rotation + crop.  Restated from the published IJG / libjpeg-turbo algorithms (jidctint.c,
// jdsample.c, jdcolor.c) so that the output is bit-exact with what Pillow gets from libjpeg-turbo.  Kept in a header that
// also compiles as plain C++ so the CPU suite runs exactly this code against Pillow (tests/jpeg_host_decoder.cpp).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define F3R_JHD __host__ __device__ __forceinline__
#else
#define F3R_JHD inline
#endif

namespace f3r {
namespace jpeg {

// zigzag position -> natural (row-major) index (host table; the kernels keep a copy in constant memory)
#define F3R_JPEG_NATURAL                                                                                              \
  {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, \
   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63}
constexpr uint8_t kNatural[64] = F3R_JPEG_NATURAL;

F3R_JHD int clamp_i(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// ---- jidctint.c (JDCT_ISLOW): 13-bit constants, PASS1_BITS = 2, DESCALE = round-half-up arithmetic shift.
// The pass-1 results are saturated to 16 bits and the final samples to 0..255, as the x86 SIMD version Pillow runs does
// (packssdw / packsswb); for the coefficients a real encoder writes neither saturation is ever reached.
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr int32_t F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                  F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

// One 1-D 8-point IDCT of in[0..7] (stride-free), outputs before descaling in out[0..7] = (tmp + round) >> shift.
F3R_JHD void idct_1d(const int32_t* in, int32_t* out, int shift) {
  int32_t z2 = in[2], z3 = in[6];
  int32_t z1 = (z2 + z3) * F0541;
  const int32_t t2 = z1 - z3 * F1847, t3 = z1 + z2 * F0765;
  z2 = in[0];
  z3 = in[4];
  const int32_t t0 = (z2 + z3) * (1 << kConstBits), t1 = (z2 - z3) * (1 << kConstBits);
  const int32_t e10 = t0 + t3, e13 = t0 - t3, e11 = t1 + t2, e12 = t1 - t2;
  int32_t o0 = in[7], o1 = in[5], o2 = in[3], o3 = in[1];
  z1 = o0 + o3;
  z2 = o1 + o2;
  z3 = o0 + o2;
  int32_t z4 = o1 + o3;
  const int32_t z5 = (z3 + z4) * F1175;
  o0 *= F0298;
  o1 *= F2053;
  o2 *= F3072;
  o3 *= F1501;
  z1 *= -F0899;
  z2 *= -F2562;
  z3 = z3 * -F1961 + z5;
  z4 = z4 * -F0390 + z5;
  o0 += z1 + z3;
  o1 += z2 + z4;
  o2 += z2 + z3;
  o3 += z1 + z4;
  const int32_t rnd = 1 << (shift - 1);
  out[0] = (e10 + o3 + rnd) >> shift;
  out[7] = (e10 - o3 + rnd) >> shift;
  out[1] = (e11 + o2 + rnd) >> shift;
  out[6] = (e11 - o2 + rnd) >> shift;
  out[2] = (e12 + o1 + rnd) >> shift;
  out[5] = (e12 - o1 + rnd) >> shift;
  out[3] = (e13 + o0 + rnd) >> shift;
  out[4] = (e13 - o0 + rnd) >> shift;
}

// coef: 64 quantised coefficients in natural order, q: the quantisation table in natural order.
// Writes the 8x8 samples to out[r * stride + c].
F3R_JHD void idct_islow(const int16_t* coef, const uint16_t* q, uint8_t* out, int stride) {
  int32_t ws[64];
  int32_t col[8], res[8];
  for (int c = 0; c < 8; ++c) {  // pass 1: columns
    for (int r = 0; r < 8; ++r) col[r] = static_cast<int32_t>(coef[r * 8 + c]) * static_cast<int32_t>(q[r * 8 + c]);
    idct_1d(col, res, kConstBits - kPass1Bits);
    for (int r = 0; r < 8; ++r) ws[r * 8 + c] = clamp_i(res[r], -32768, 32767);
  }
  for (int r = 0; r < 8; ++r) {  // pass 2: rows
    idct_1d(ws + r * 8, res, kConstBits + kPass1Bits + 3);
    for (int c = 0; c < 8; ++c) out[r * stride + c] = static_cast<uint8_t>(clamp_i(res[c] + 128, 0, 255));
  }
}

// ---- jdsample.c: chroma sample at full-resolution (x, y) of a plane p (row stride `stride`) holding the dw x dh
// downsampled samples.  hs / vs: horizontal / vertical upsampling factor (1 or 2).  libjpeg-turbo upsamples with the
// triangle filter ("fancy") only when the downsampled width exceeds 2, otherwise by replication; edges replicate.
F3R_JHD int upsample(const uint8_t* p, int stride, int dw, int dh, int hs, int vs, int x, int y) {
  if (hs == 1 && vs == 1) return p[y * stride + x];
  const int j = x >> 1, i = vs == 2 ? y >> 1 : y;
  if (dw <= 2) return p[i * stride + j];
  const int jn = (x & 1) ? (j + 1 < dw ? j + 1 : j) : (j > 0 ? j - 1 : 0);
  if (vs == 1) {  // h2v1: 3/4 nearer + 1/4 further, biases 1 (even) / 2 (odd)
    return (3 * p[i * stride + j] + p[i * stride + jn] + ((x & 1) ? 2 : 1)) >> 2;
  }
  // h2v2: vertical triangle into column sums, then horizontal; biases 8 (even) / 7 (odd)
  const int in = (y & 1) ? (i + 1 < dh ? i + 1 : i) : (i > 0 ? i - 1 : 0);
  const int cs = 3 * p[i * stride + j] + p[in * stride + j];
  const int csn = 3 * p[i * stride + jn] + p[in * stride + jn];
  return (3 * cs + csn + ((x & 1) ? 7 : 8)) >> 4;
}

// ---- jdcolor.c: YCbCr -> RGB with 16-bit fixed-point tables (computed inline; identical integers)
constexpr int kScaleBits = 16;
constexpr int32_t kHalf = 1 << (kScaleBits - 1);
constexpr int32_t FCrR = 91881, FCbB = 116130, FCrG = 46802, FCbG = 22554;  // FIX(1.40200), FIX(1.77200), FIX(0.71414), FIX(0.34414)

F3R_JHD void ycc_to_rgb(int y, int cb, int cr, uint8_t* rgb) {
  const int32_t xb = cb - 128, xr = cr - 128;
  const int r = y + ((FCrR * xr + kHalf) >> kScaleBits);
  const int g = y + ((-FCbG * xb + kHalf - FCrG * xr) >> kScaleBits);
  const int b = y + ((FCbB * xb + kHalf) >> kScaleBits);
  rgb[0] = static_cast<uint8_t>(clamp_i(r, 0, 255));
  rgb[1] = static_cast<uint8_t>(clamp_i(g, 0, 255));
  rgb[2] = static_cast<uint8_t>(clamp_i(b, 0, 255));
}

// ---- index map of load_images' lossless PIL steps on a decoded w x h image: ImageOps.exif_transpose (orientation
// 1..8), optionally rotate(-90, expand=True), then crop at (left, top).  Output pixel (ox, oy) reads source pixel
// (m[0] ox + m[1] oy + m[2], m[3] ox + m[4] oy + m[5]).
F3R_JHD void orient_map(int w, int h, int orientation, int rotate_cw90, int left, int top, int32_t m[6]) {
  // (x1, y1) in the transposed image -> source: x0 = a x1 + b y1 + c, y0 = d x1 + e y1 + f
  int32_t a = 1, b = 0, c = 0, d = 0, e = 1, f = 0;
  switch (orientation) {
    case 2: a = -1; c = w - 1; break;                                 // FLIP_LEFT_RIGHT
    case 3: a = -1; c = w - 1; e = -1; f = h - 1; break;              // ROTATE_180
    case 4: e = -1; f = h - 1; break;                                 // FLIP_TOP_BOTTOM
    case 5: a = 0; b = 1; d = 1; e = 0; break;                        // TRANSPOSE
    case 6: a = 0; b = 1; d = -1; e = 0; f = h - 1; break;            // ROTATE_270
    case 7: a = 0; b = -1; c = w - 1; d = -1; e = 0; f = h - 1; break; // TRANSVERSE
    case 8: a = 0; b = -1; c = w - 1; d = 1; e = 0; break;            // ROTATE_90
    default: break;
  }
  const int h1 = (orientation >= 5 && orientation <= 8) ? w : h;
  // rotate(-90, expand=True) = ROTATE_270: (x2, y2) -> (x1, y1) = (y2, h1 - 1 - x2)
  int32_t ra = 1, rb = 0, rc = 0, rd = 0, re = 1, rf = 0;
  if (rotate_cw90) { ra = 0; rb = 1; rd = -1; re = 0; rf = h1 - 1; }
  // compose: source = T(R(x2, y2)), with (x2, y2) = (ox + left, oy + top)
  const int32_t A = a * ra + b * rd, B = a * rb + b * re, Cc = a * rc + b * rf + c;
  const int32_t D = d * ra + e * rd, E = d * rb + e * re, F = d * rc + e * rf + f;
  m[0] = A; m[1] = B; m[2] = A * left + B * top + Cc;
  m[3] = D; m[4] = E; m[5] = D * left + E * top + F;
}

}  // namespace jpeg
}  // namespace f3r
