// Host build of the per-point arithmetic of the reconstruction metrics (fast3r_b200/csrc/pointcloud_math.h), so the CPU
// suite checks that exact code against scipy and numpy.  Compiled by tests/test_recon_metric_cpu.py with g++
// -ffp-contract=off (the device code uses explicitly rounded operations).
#include <math.h>

#include "pointcloud_math.h"

// brute-force nearest neighbour with pc_dist2: dist = sqrt(min), idx = first index reaching it
extern "C" void f3r_test_nearest(const double* ref, int n, const double* query, int nq, double* dist, long long* idx) {
  for (int q = 0; q < nq; ++q) {
    double best = INFINITY;
    long long bi = n;
    for (int i = 0; i < n; ++i) {
      const double s = f3r::pc_dist2(query + 3 * q, ref + 3 * i);
      if (s < best) {
        best = s;
        bi = i;
      }
    }
    dist[q] = sqrt(best);
    idx[q] = bi;
  }
}

// normal of k points (fp64 [k][3]) as the kNN kernel computes it
extern "C" void f3r_test_normal(const double* pts, int k, double* n) {
  f3r::pc_neighbourhood_normal([&](int a) { return pts + 3 * a; }, k, n);
}

extern "C" void f3r_test_morton(const double* p, const double* origin, double inv_extent, unsigned long long* hi,
                                unsigned long long* lo) {
  uint64_t h, l;
  f3r::pc_morton(p, origin, inv_extent, &h, &l);
  *hi = h;
  *lo = l;
}

extern "C" unsigned long long f3r_test_dkey(double d) { return f3r::pc_dkey(d); }
extern "C" double f3r_test_dkey_inv(unsigned long long u) { return f3r::pc_dkey_inv(u); }
