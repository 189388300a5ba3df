// Test-only sequential baseline JPEG decoder: the header parser (fast3r_b200/csrc/jpeg_parse.h) and the per-sample math
// of the GPU decoder (fast3r_b200/csrc/jpeg_math.h) with a plain one-bit-at-a-time Huffman decoder around them, so the CPU
// suite can check that math bit-exactly against Pillow.  Compiled by tests/test_jpeg_cpu.py with g++.
#include <stdlib.h>
#include <vector>

#include "jpeg_parse.h"

using namespace f3r::jpeg;

namespace {

struct Bits {
  std::vector<uint8_t> buf;  // unstuffed bytes of one restart segment
  size_t pos = 0;            // bit position
  int get() {
    if ((pos >> 3) >= buf.size()) return -1;
    const int b = (buf[pos >> 3] >> (7 - (pos & 7))) & 1;
    ++pos;
    return b;
  }
  int receive(int s) {
    int v = 0;
    for (int i = 0; i < s; ++i) {
      const int b = get();
      if (b < 0) return -100000;
      v = (v << 1) | b;
    }
    return v;
  }
};

int decode_symbol(Bits& bs, const HuffTable& t) {
  int code = 0;
  for (int len = 1; len <= 16; ++len) {
    const int b = bs.get();
    if (b < 0) return -1;
    code = (code << 1) | b;
    if (t.maxcode[len] >= 0 && code <= t.maxcode[len]) return t.vals[t.valoff[len] + code];
  }
  return -1;
}

int extend(int v, int s) { return s == 0 ? 0 : (v < (1 << (s - 1)) ? v - (1 << s) + 1 : v); }

}  // namespace

// status of the parser (kSupported / kUnsupported / kMalformed); dims = (width, height, components)
extern "C" int f3r_test_jpeg_parse(const uint8_t* d, size_t n, int32_t* dims) {
  Header* h = static_cast<Header*>(malloc(sizeof(Header)));
  const int st = parse(d, n, h);
  dims[0] = h->width;
  dims[1] = h->height;
  dims[2] = h->ncomp;
  free(h);
  return st;
}

// Decodes a supported stream to RGB (height, width, 3).  Returns 0, or non-zero on an entropy-coding error.
extern "C" int f3r_test_jpeg_decode(const uint8_t* d, size_t n, uint8_t* rgb) {
  Header* hp = static_cast<Header*>(malloc(sizeof(Header)));
  Header& h = *hp;
  if (parse(d, n, &h) != kSupported) { free(hp); return 1; }
  // split the scan into unstuffed restart segments
  std::vector<Bits> segs(1);
  const uint8_t* s = d + h.scan_offset;
  for (size_t i = 0; i < h.scan_bytes; ++i) {
    if (s[i] != 0xFF) { segs.back().buf.push_back(s[i]); continue; }
    size_t r = i + 1;
    while (s[r] == 0xFF) ++r;
    if (s[r] == 0x00) { segs.back().buf.push_back(0xFF); i = r; continue; }
    segs.emplace_back();  // RSTn
    i = r;
  }
  std::vector<int> bw(3), bh(3);
  std::vector<std::vector<int16_t>> coef(3);
  for (int c = 0; c < h.ncomp; ++c) {
    bw[c] = h.mcux * h.comp_h[c];
    bh[c] = h.mcuy * h.comp_v[c];
    if (h.ncomp == 1) { bw[c] = h.mcux; bh[c] = h.mcuy; }
    coef[c].assign(static_cast<size_t>(bw[c]) * bh[c] * 64, 0);
  }
  const int mcus = h.mcux * h.mcuy;
  const int ri = h.restart_interval ? h.restart_interval : mcus;
  int err = 0;
  for (int mcu = 0; mcu < mcus && !err; ++mcu) {
    Bits& bs = segs[mcu / ri];
    static thread_local int pred[3];
    if (mcu % ri == 0) pred[0] = pred[1] = pred[2] = 0;
    const int mx = mcu % h.mcux, my = mcu / h.mcux;
    for (int k = 0; k < h.blocks_per_mcu && !err; ++k) {
      const int c = h.mcu_comp[k];
      int16_t* blk = &coef[c][(static_cast<size_t>(my * h.comp_v[c] + h.mcu_dy[k]) * bw[c] + mx * h.comp_h[c] + h.mcu_dx[k]) * 64];
      int sz = decode_symbol(bs, h.dc[h.comp_td[c]]);
      if (sz < 0 || sz > 11) { err = 2; break; }
      pred[c] += extend(bs.receive(sz), sz);
      blk[0] = static_cast<int16_t>(pred[c]);
      for (int z = 1; z < 64;) {
        const int rs = decode_symbol(bs, h.ac[h.comp_ta[c]]);
        if (rs < 0) { err = 3; break; }
        const int r = rs >> 4, ss = rs & 15;
        if (ss == 0) {
          if (r != 15) break;
          z += 16;
          continue;
        }
        z += r;
        if (z > 63) { err = 4; break; }
        blk[kNatural[z]] = static_cast<int16_t>(extend(bs.receive(ss), ss));
        ++z;
      }
    }
  }
  if (err) { free(hp); return err; }
  std::vector<std::vector<uint8_t>> plane(3);
  for (int c = 0; c < h.ncomp; ++c) {
    const int stride = bw[c] * 8;
    plane[c].assign(static_cast<size_t>(stride) * bh[c] * 8, 0);
    for (int by = 0; by < bh[c]; ++by)
      for (int bx = 0; bx < bw[c]; ++bx)
        idct_islow(&coef[c][(static_cast<size_t>(by) * bw[c] + bx) * 64], h.qt[h.comp_tq[c]],
                   &plane[c][static_cast<size_t>(by) * 8 * stride + bx * 8], stride);
  }
  const int hs = h.hmax, vs = h.vmax;
  const int dw = (h.width + hs - 1) / hs, dh = (h.height + vs - 1) / vs;
  for (int y = 0; y < h.height; ++y)
    for (int x = 0; x < h.width; ++x) {
      uint8_t* o = rgb + (static_cast<size_t>(y) * h.width + x) * 3;
      const int Y = plane[0][static_cast<size_t>(y) * bw[0] * 8 + x];
      if (h.ncomp == 1) { o[0] = o[1] = o[2] = static_cast<uint8_t>(Y); continue; }
      const int cb = upsample(plane[1].data(), bw[1] * 8, dw, dh, hs, vs, x, y);
      const int cr = upsample(plane[2].data(), bw[2] * 8, dw, dh, hs, vs, x, y);
      ycc_to_rgb(Y, cb, cr, o);
    }
  free(hp);
  return 0;
}

extern "C" void f3r_test_jpeg_orient_map(int w, int h, int orientation, int rotate, int left, int top, int32_t* m) {
  orient_map(w, h, orientation, rotate, left, top, m);
}
