// Per-point arithmetic of the reconstruction metrics (pointcloud.cu): the squared distance whose rounding matches
// scipy's cKDTree, the 63-bit Morton codes of the spatial index, and the normal of a k-neighbourhood.  Kept in a header
// that also compiles as plain C++ (with -ffp-contract=off) so the CPU suite checks exactly this code against scipy and
// numpy (tests/pointcloud_math_host.cpp).
#pragma once
#include <math.h>
#include <stdint.h>

#include "geometry_math.h"

namespace f3r {

#if defined(__CUDA_ARCH__)
F3R_HD inline double pc_mul(double a, double b) { return __dmul_rn(a, b); }
F3R_HD inline double pc_add(double a, double b) { return __dadd_rn(a, b); }
F3R_HD inline double pc_sub(double a, double b) { return __dsub_rn(a, b); }
#else
F3R_HD inline double pc_mul(double a, double b) { return a * b; }
F3R_HD inline double pc_add(double a, double b) { return a + b; }
F3R_HD inline double pc_sub(double a, double b) { return a - b; }
#endif

// cKDTree's squared Euclidean distance: fp64 differences, (dx*dx + dy*dy) + dz*dz, no fused multiply-add.  The distance
// it reports is sqrt() of this value, and sqrt is monotone, so the nearest point under this value is scipy's.
F3R_HD inline double pc_dist2(const double* q, const double* p) {
  const double dx = pc_sub(q[0], p[0]), dy = pc_sub(q[1], p[1]), dz = pc_sub(q[2], p[2]);
  return pc_add(pc_add(pc_mul(dx, dx), pc_mul(dy, dy)), pc_mul(dz, dz));
}

// spreads the low 21 bits of v to every third bit (bit i -> bit 3i)
F3R_HD inline uint64_t pc_spread3(uint64_t v) {
  v &= 0x1fffffull;
  v = (v | (v << 32)) & 0x1f00000000ffffull;
  v = (v | (v << 16)) & 0x1f0000ff0000ffull;
  v = (v | (v << 8)) & 0x100f00f00f00f00full;
  v = (v | (v << 4)) & 0x10c30c30c30c30c3ull;
  v = (v | (v << 2)) & 0x1249249249249249ull;
  return v;
}

// Morton codes of a point inside the cube [origin, origin + 1/inv_extent]^3 at 33 bits per axis, split in two keys:
// hi interleaves the top 21 bits of each axis (the 63-bit code), lo the next 12 (36 bits).  Sorting by (hi, lo) orders
// points along the 33-bit curve, so points that share a 63-bit cell (a tight cluster next to far outliers) still come
// out spatially ordered.  Coordinates outside the cube (queries) are clamped to it; a NaN maps to cell 0.
F3R_HD inline void pc_morton(const double* p, const double* origin, double inv_extent, uint64_t* hi, uint64_t* lo) {
  uint64_t h = 0, l = 0;
  const double cells = 8589934592.0;  // 2^33
  for (int a = 0; a < 3; ++a) {
    const double t = (p[a] - origin[a]) * inv_extent * cells;
    uint64_t c = 0;
    if (t >= cells - 1.0) c = (1ull << 33) - 1;
    else if (t > 0.0) c = static_cast<uint64_t>(t);
    h |= pc_spread3(c >> 12) << (2 - a);
    l |= pc_spread3(c & 0xfffull) << (2 - a);
  }
  *hi = h;
  *lo = l;
}

// unit eigenvector of the smallest eigenvalue of a symmetric 3x3 (Jacobi, geometry_math.h)
F3R_HD inline void pc_normal_from_cov(double cov[3][3], double* n) {
  double v[3][3], lam[3];
  jacobi_eig3(cov, v, lam);  // eigenvalues descending: the last column belongs to the smallest
  const double l = sqrt(v[0][2] * v[0][2] + v[1][2] * v[1][2] + v[2][2] * v[2][2]);
  if (!(l > 0.0)) {
    n[0] = 0.0; n[1] = 0.0; n[2] = 1.0;
    return;
  }
  n[0] = v[0][2] / l; n[1] = v[1][2] / l; n[2] = v[2][2] / l;
}

F3R_HD inline void pc_cov_add(double cov[3][3], const double* p, const double* mean) {
  const double d[3] = {p[0] - mean[0], p[1] - mean[1], p[2] - mean[2]};
  for (int i = 0; i < 3; ++i)
    for (int j = i; j < 3; ++j) cov[i][j] += d[i] * d[j];
}

F3R_HD inline void pc_cov_finish(double cov[3][3], int k) {
  for (int i = 0; i < 3; ++i)
    for (int j = i; j < 3; ++j) {
      cov[i][j] /= k;
      cov[j][i] = cov[i][j];
    }
}

// Normal of the k points pt(0) .. pt(k-1) (each a const double[3]), Open3D's EstimateNormals: the eigenvector of the
// smallest eigenvalue of the fp64 covariance (two passes: mean, then centred outer products); fewer than 3 points or a
// degenerate solve give (0, 0, 1).
template <class Pt>
F3R_HD inline void pc_neighbourhood_normal(Pt pt, int k, double* n) {
  n[0] = 0.0; n[1] = 0.0; n[2] = 1.0;
  if (k < 3) return;
  double mean[3] = {0.0, 0.0, 0.0};
  for (int a = 0; a < k; ++a)
    for (int d = 0; d < 3; ++d) mean[d] += pt(a)[d];
  for (int d = 0; d < 3; ++d) mean[d] /= k;
  double cov[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
  for (int a = 0; a < k; ++a) pc_cov_add(cov, pt(a), mean);
  pc_cov_finish(cov, k);
  pc_normal_from_cov(cov, n);
}

// order-preserving unsigned image of a double (a < b <=> key(a) < key(b) for non-NaN values) and its inverse
F3R_HD inline uint64_t pc_dkey(double d) {
  union { double d; uint64_t u; } c;
  c.d = d;
  const uint64_t b = c.u;
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
F3R_HD inline double pc_dkey_inv(uint64_t u) {
  union { double d; uint64_t u; } c;
  c.u = (u & 0x8000000000000000ull) ? (u & 0x7fffffffffffffffull) : ~u;
  return c.d;
}

}  // namespace f3r
