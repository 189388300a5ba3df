// Ground-truth views (fast3r_b200/views.py): the depth half of the datasets' crop / rescale / crop, the unprojection to
// world points, the validity mask and the landscape transpose, one launch for every (view, item) of a call.
// (fast3r/dust3r/datasets/base/base_stereo_view_dataset.py:78-142, :165-221, :243-261; views_math.h has the per-pixel
// math.)  The image half runs through f3r_ingest_rgb8.
// One thread per output pixel, in output order, so the stores of a warp are contiguous; the depth reads are a gather
// through the nearest-neighbour map of the crop.  blockIdx.y is the (view, item); CTAs past its pixel count return.
#include <stdint.h>

#include "../../include/fast3r_b200.h"
#include "f3r_kernels.h"
#include "views_math.h"

namespace f3r {

namespace {

constexpr int VWT = 256;  // threads (output pixels) per CTA

__global__ void __launch_bounds__(VWT) view_geometry_kernel(const f3r_view_param* __restrict__ params,
                                                            float* __restrict__ out_pts,
                                                            uint8_t* __restrict__ out_valid,
                                                            float* __restrict__ out_depth) {
  const f3r_view_param& P = params[blockIdx.y];
  const int n = P.out_w * P.out_h;
  const int p = blockIdx.x * VWT + threadIdx.x;
  if (p >= n) return;
  // (u, v): column and row of the pixel in the crop before the transpose
  const int u = P.transpose ? p / P.out_h : p % P.out_w;
  const int v = P.transpose ? p % P.out_h : p / P.out_w;
  const int sx = P.crop_x + vw::nearest(u + P.box_x, P.crop_w, P.rs_w);
  const int sy = P.crop_y + vw::nearest(v + P.box_y, P.crop_h, P.rs_h);
  const float z = __ldg(P.depth + static_cast<long long>(sy) * P.src_w + sx);
  float k4[4], pose[12], w[3];
  for (int i = 0; i < 4; ++i) k4[i] = P.k[i];
  for (int i = 0; i < 12; ++i) pose[i] = P.pose[i];
  const bool ok = vw::point(u, v, z, k4, pose, w);
  const long long o = P.out_offset + p;
  out_pts[3 * o] = w[0];
  out_pts[3 * o + 1] = w[1];
  out_pts[3 * o + 2] = w[2];
  out_valid[o] = ok;
  out_depth[o] = z;
}

}  // namespace

cudaError_t launch_view_geometry(const f3r_view_param* params, int count, int max_pixels, float* out_pts,
                                 uint8_t* out_valid, float* out_depth, cudaStream_t st) {
  const dim3 grid(static_cast<unsigned>((max_pixels + VWT - 1) / VWT), static_cast<unsigned>(count));
  return launch(view_geometry_kernel, grid, VWT, 0, st, false, params, out_pts, out_valid, out_depth);
}

}  // namespace f3r
