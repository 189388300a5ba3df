// Host-side JPEG header parser of the GPU decoder (jpeg.cu) and of the test-only sequential decoder
// (tests/jpeg_host_decoder.cpp).  Reads SOI / DQT / DHT / SOF / DRI / APP0 / APP14 / SOS, walks the entropy-coded segment to
// EOI (checking the RSTn sequence) and classifies the stream as one the GPU decodes, one it does not (Pillow keeps it) or
// a malformed one.  Plain C++, no CUDA.
#pragma once
#include <stdint.h>
#include <string.h>

#include "jpeg_math.h"

namespace f3r {
namespace jpeg {

enum { kSupported = 0, kUnsupported = 1, kMalformed = 2 };

// Canonical Huffman table: lookahead LUT for codes of <= kLutBits bits (entry = symbol | length << 8, 0 = longer code),
// maxcode / valoff per length for the rest, symbols in code order.
constexpr int kLutBits = 9;
struct HuffTable {
  uint16_t lut[1 << kLutBits];
  int32_t maxcode[18];  // largest code of each length (-1: none); maxcode[17] = sentinel
  int32_t valoff[18];   // symbol index of the first code of each length minus that code
  uint8_t vals[256];
};

struct Header {
  int status;
  int width, height, ncomp;
  int hmax, vmax;
  int comp_h[3], comp_v[3], comp_tq[3], comp_td[3], comp_ta[3];
  int restart_interval;
  int mcux, mcuy, blocks_per_mcu;
  int mcu_comp[6], mcu_dx[6], mcu_dy[6];  // per block of an MCU: component and position inside the MCU
  int segments;                           // restart segments (RST markers + 1)
  size_t scan_offset, scan_bytes;         // entropy-coded data between the SOS header and EOI
  uint16_t qt[4][64];                     // natural order
  bool qt_set[4];
  HuffTable dc[2], ac[2];
  bool dc_set[2], ac_set[2];
  const char* why;                        // reason for kUnsupported / kMalformed
};

inline bool build_huff(const uint8_t* counts, const uint8_t* vals, int nvals, HuffTable* t) {
  memset(t->lut, 0, sizeof(t->lut));
  memcpy(t->vals, vals, nvals);
  int32_t code = 0, k = 0;
  for (int len = 1; len <= 16; ++len) {
    t->valoff[len] = k - code;
    for (int i = 0; i < counts[len - 1]; ++i, ++k, ++code) {
      if (len <= kLutBits) {
        const int shift = kLutBits - len;
        for (int j = 0; j < (1 << shift); ++j) t->lut[(code << shift) | j] = static_cast<uint16_t>(vals[k] | (len << 8));
      }
    }
    t->maxcode[len] = counts[len - 1] ? code - 1 : -1;
    // over-subscribed, or a code of all ones: libjpeg (jpeg_make_d_derived_tbl) rejects code >= 2^len after each length
    if (code >= (1 << len)) return false;
    code <<= 1;
  }
  t->maxcode[0] = -1;
  t->maxcode[17] = 0x7fffffff;
  t->valoff[0] = t->valoff[17] = 0;
  return true;
}

inline int finish(Header* h, int status, const char* why) {
  h->status = status;
  h->why = why;
  return status;
}

// Parses the whole stream.  Fills `h` and returns h->status.
inline int parse(const uint8_t* d, size_t n, Header* h) {
  memset(h, 0, sizeof(*h));
  if (n < 2 || d[0] != 0xFF || d[1] != 0xD8) return finish(h, kUnsupported, "not a JPEG (no SOI)");
  size_t p = 2;
  bool sof = false, jfif = false, adobe = false;
  int adobe_transform = -1;
  int comp_id[3] = {0, 0, 0};
  while (true) {
    while (p < n && d[p] != 0xFF) ++p;  // libjpeg skips garbage between markers
    while (p < n && d[p] == 0xFF) ++p;  // fill bytes
    if (p >= n) return finish(h, kMalformed, "truncated before the scan");
    const int m = d[p++];
    if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;  // parameterless
    if (m == 0xD9) return finish(h, kMalformed, "EOI before the scan");
    if (p + 2 > n) return finish(h, kMalformed, "truncated marker");
    const size_t len = (static_cast<size_t>(d[p]) << 8) | d[p + 1];
    if (len < 2 || p + len > n) return finish(h, kMalformed, "truncated marker segment");
    const uint8_t* s = d + p + 2;
    const size_t sl = len - 2;
    switch (m) {
      case 0xC0: case 0xC1: {  // baseline / extended sequential Huffman
        if (sof) return finish(h, kMalformed, "two SOF markers");
        sof = true;
        if (sl < 6) return finish(h, kMalformed, "short SOF");
        if (s[0] != 8) return finish(h, kUnsupported, "sample precision is not 8 bits");
        h->height = (s[1] << 8) | s[2];
        h->width = (s[3] << 8) | s[4];
        h->ncomp = s[5];
        if (h->height == 0) return finish(h, kUnsupported, "height defined by DNL");
        if (h->width == 0) return finish(h, kMalformed, "zero width");
        if (h->ncomp != 1 && h->ncomp != 3) return finish(h, kUnsupported, "component count is not 1 or 3");
        if (sl < 6 + 3 * static_cast<size_t>(h->ncomp)) return finish(h, kMalformed, "short SOF");
        for (int c = 0; c < h->ncomp; ++c) {
          comp_id[c] = s[6 + 3 * c];
          h->comp_h[c] = s[7 + 3 * c] >> 4;
          h->comp_v[c] = s[7 + 3 * c] & 15;
          h->comp_tq[c] = s[8 + 3 * c];
          if (h->comp_h[c] < 1 || h->comp_h[c] > 4 || h->comp_v[c] < 1 || h->comp_v[c] > 4 || h->comp_tq[c] > 3)
            return finish(h, kMalformed, "bad component parameters");
        }
        break;
      }
      case 0xC2: case 0xC3: case 0xC5: case 0xC6: case 0xC7: case 0xC9: case 0xCA: case 0xCB: case 0xCD: case 0xCE:
      case 0xCF:
        return finish(h, kUnsupported, "progressive, lossless, hierarchical or arithmetic-coded JPEG");
      case 0xCC: return finish(h, kUnsupported, "arithmetic coding conditioning");
      case 0xDB: {  // DQT
        size_t q = 0;
        while (q < sl) {
          const int pq = s[q] >> 4, tq = s[q] & 15;
          if (tq > 3 || pq > 1) return finish(h, kMalformed, "bad DQT");
          if (q + 1 + 64 * (pq + 1) > sl) return finish(h, kMalformed, "short DQT");
          for (int k = 0; k < 64; ++k)
            h->qt[tq][kNatural[k]] = pq ? static_cast<uint16_t>((s[q + 1 + 2 * k] << 8) | s[q + 2 + 2 * k]) : s[q + 1 + k];
          h->qt_set[tq] = true;
          q += 1 + 64 * (pq + 1);
        }
        break;
      }
      case 0xC4: {  // DHT
        size_t q = 0;
        while (q < sl) {
          if (q + 17 > sl) return finish(h, kMalformed, "short DHT");
          const int tc = s[q] >> 4, th = s[q] & 15;
          int total = 0;
          for (int i = 0; i < 16; ++i) total += s[q + 1 + i];
          if (tc > 1 || total > 256 || q + 17 + total > sl) return finish(h, kMalformed, "bad DHT");
          if (th > 1) return finish(h, kUnsupported, "Huffman table slot above 1");
          // libjpeg rejects a DC table with a symbol above 15 whether or not the scan codes it
          for (int i = 0; i < total && tc == 0; ++i)
            if (s[q + 17 + i] > 15) return finish(h, kMalformed, "DC Huffman symbol above 15");
          HuffTable* t = tc ? &h->ac[th] : &h->dc[th];
          if (!build_huff(s + q + 1, s + q + 17, total, t)) return finish(h, kMalformed, "bad Huffman table");
          (tc ? h->ac_set : h->dc_set)[th] = true;
          q += 17 + total;
        }
        break;
      }
      case 0xDD:  // DRI
        if (sl < 2) return finish(h, kMalformed, "short DRI");
        h->restart_interval = (s[0] << 8) | s[1];
        break;
      case 0xE0:
        if (sl >= 5 && !memcmp(s, "JFIF\0", 5)) jfif = true;
        break;
      case 0xEE:
        if (sl >= 12 && !memcmp(s, "Adobe", 5)) { adobe = true; adobe_transform = s[11]; }
        break;
      case 0xDA: {  // SOS
        if (!sof) return finish(h, kMalformed, "SOS before SOF");
        if (sl < 1) return finish(h, kMalformed, "short SOS");
        const int ns = s[0];
        if (ns != h->ncomp) return finish(h, kUnsupported, "scan does not interleave every component");
        if (sl < 4 + 2 * static_cast<size_t>(ns)) return finish(h, kMalformed, "short SOS");
        for (int i = 0; i < ns; ++i) {
          const int cid = s[1 + 2 * i];
          if (cid != comp_id[i]) return finish(h, kUnsupported, "scan component order differs from the frame");
          h->comp_td[i] = s[2 + 2 * i] >> 4;
          h->comp_ta[i] = s[2 + 2 * i] & 15;
          if (h->comp_td[i] > 1 || h->comp_ta[i] > 1) return finish(h, kUnsupported, "Huffman table slot above 1");
          if (!h->dc_set[h->comp_td[i]] || !h->ac_set[h->comp_ta[i]] || !h->qt_set[h->comp_tq[i]])
            return finish(h, kMalformed, "missing table");
        }
        const uint8_t ss = s[1 + 2 * ns], se = s[2 + 2 * ns], a = s[3 + 2 * ns];
        if (ss != 0 || se != 63 || a != 0) return finish(h, kMalformed, "bad spectral selection for a sequential scan");
        // colour space as libjpeg infers it (jdapimin.c); only YCbCr is decoded here
        if (h->ncomp == 3) {
          bool ycc = true;
          if (jfif) ycc = true;
          else if (adobe) ycc = adobe_transform != 0;
          else if (comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B') ycc = false;
          if (!ycc) return finish(h, kUnsupported, "RGB (untransformed) colour space");
          if (h->comp_h[1] != 1 || h->comp_v[1] != 1 || h->comp_h[2] != 1 || h->comp_v[2] != 1)
            return finish(h, kUnsupported, "chroma sampling factors are not 1x1");
          const int hv = h->comp_h[0] * 10 + h->comp_v[0];
          if (hv != 11 && hv != 21 && hv != 22) return finish(h, kUnsupported, "sampling is not 4:4:4, 4:2:2 or 4:2:0");
          h->hmax = h->comp_h[0];
          h->vmax = h->comp_v[0];
          h->mcux = (h->width + 8 * h->hmax - 1) / (8 * h->hmax);
          h->mcuy = (h->height + 8 * h->vmax - 1) / (8 * h->vmax);
          int k = 0;
          for (int c = 0; c < 3; ++c)
            for (int dy = 0; dy < h->comp_v[c]; ++dy)
              for (int dx = 0; dx < h->comp_h[c]; ++dx) { h->mcu_comp[k] = c; h->mcu_dx[k] = dx; h->mcu_dy[k] = dy; ++k; }
          h->blocks_per_mcu = k;
        } else {  // one component: non-interleaved, one block per MCU whatever its sampling factors
          h->hmax = h->vmax = 1;
          h->comp_h[0] = h->comp_v[0] = 1;
          h->mcux = (h->width + 7) / 8;
          h->mcuy = (h->height + 7) / 8;
          h->blocks_per_mcu = 1;
          h->mcu_comp[0] = h->mcu_dx[0] = h->mcu_dy[0] = 0;
        }
        // entropy-coded segment: up to EOI; only stuffed zeros, fill bytes and RST0..7 in sequence may follow an FF
        const size_t start = p + len;
        size_t q = start;
        int rst = 0;
        while (true) {
          const void* f = q < n ? memchr(d + q, 0xFF, n - q) : nullptr;
          if (!f) return finish(h, kMalformed, "truncated scan (no EOI)");
          q = static_cast<const uint8_t*>(f) - d;
          size_t r = q + 1;
          while (r < n && d[r] == 0xFF) ++r;
          if (r >= n) return finish(h, kMalformed, "truncated scan (no EOI)");
          const int c = d[r];
          if (c == 0x00) { q = r + 1; continue; }
          if (c >= 0xD0 && c <= 0xD7) {
            if (c != 0xD0 + (rst & 7)) return finish(h, kMalformed, "restart markers out of sequence");
            ++rst;
            q = r + 1;
            continue;
          }
          if (c == 0xD9) { h->scan_offset = start; h->scan_bytes = q - start; break; }
          return finish(h, kUnsupported, "marker inside or after the scan (DNL or a second scan)");
        }
        const long long mcus = static_cast<long long>(h->mcux) * h->mcuy;
        if (h->restart_interval == 0 ? rst != 0 : rst != (mcus + h->restart_interval - 1) / h->restart_interval - 1)
          return finish(h, kMalformed, "restart marker count does not match the restart interval");
        h->segments = rst + 1;
        if (static_cast<unsigned long long>(mcus) * h->blocks_per_mcu > (1ull << 26))
          return finish(h, kUnsupported, "image too large");
        return finish(h, kSupported, "");
      }
      default:
        break;
    }
    p += len;
  }
}

}  // namespace jpeg
}  // namespace f3r
