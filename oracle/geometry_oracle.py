"""CPU restatement of the geometry tail that follows the forward in every caller (SURVEY.md §8 row f2, first slice).

TEST INFRASTRUCTURE ONLY - imported by tests/, tools/make_golden_geometry.py and bench.py's cpu leg, never by the
product (fast3r_b200/postprocess.py runs on the GPU through the C ABI and fails loudly without it).

What is restated, and from where:

* ``conf_quantile``      torch.quantile(conf.reshape(-1), q) as called at
                         fast3r/models/multiview_dust3r_module.py:477 and :1093 (linear interpolation between the two
                         neighbouring order statistics, rank = q*(n-1) evaluated in float32 like ATen does).
* ``umeyama``            roma.rigid_points_registration(x, y, compute_scaling=True) as called at
                         multiview_dust3r_module.py:515.  roma is a third-party dependency that is NOT vendored in
                         /root/reference and is unpinned there (requirements.txt:26 says just "roma"); what is restated
                         is its published algorithm (Umeyama 1991 / Kabsch with the det-sign correction):
                         M = sum (y-ym)(x-xm)^T = U S V^T, R = U diag(1,1,det(U V^T)) V^T,
                         s = (S1 + S2 + det(UV^T) S3) / sum |x-xm|^2, t = ym - s R xm.
                         PARITY UNPINNED against roma itself (the package is absent here); pinned instead on the
                         algorithm's defining properties (exact recovery of a known similarity, optimality against
                         perturbations) and on the reference's own call site run with this function standing in for roma.
* ``align_local_to_global``  MultiViewDUSt3RLitModule.align_local_pts3d_to_global, multiview_dust3r_module.py:427-549
                         (confidence-quantile mask & valid_mask, the two "fewer than 3 points" fallbacks, and the
                         similarity applied to ALL local points).
* ``focal_weiszfeld``    estimate_focal_knowing_depth_and_confidence_mask(..., focal_mode="weiszfeld")
                         fast3r/dust3r/post_process.py:82-142 (100 IRLS iterations, sums over the masked points) and
                         estimate_focal_knowing_depth(..., "weiszfeld") :19-79 (10 iterations, means over all points).
* ``estimate_focal``     multiview_dust3r_module.py:1081-1109 (10th-percentile confidence mask, pp = image centre).

The focal functions are pinned against the reference itself (pure torch, importable in the build container): see
tools/make_golden_geometry.py and tests/golden/geometry_tail.pt.
"""
import numpy as np


def conf_quantile(conf: np.ndarray, q: float) -> np.float32:
    """torch.quantile(conf_flat, q) for a float32 vector (ATen quantile_impl: ranks = q*(n-1) in the input dtype,
    below = floor, above = ceil, result = below.lerp(above, rank - below)).  ATen sends both ranks to the last sorted
    element, a NaN, when the vector holds a NaN of either sign, so the result is NaN."""
    v = np.sort(np.asarray(conf, np.float32).reshape(-1))
    if np.isnan(v).any():
        return np.float32(np.nan)
    n = v.size
    rank = np.float32(q) * np.float32(n - 1)
    lo = int(np.floor(rank))
    hi = int(np.ceil(rank))
    w = np.float32(rank - np.float32(lo))
    a, b = v[lo], v[hi]
    diff = np.float32(b - a)
    # ATen's lerp is a fused multiply-add (Lerp.h / cpu/LerpKernel.cpp lerp_vec: fmadd(coeff, end - start, base)); the
    # product of two float32 is exact in float64, so float64 arithmetic + one rounding reproduces it
    if abs(w) < 0.5:
        return np.float32(np.float64(w) * np.float64(diff) + np.float64(a))
    return np.float32(np.float64(np.float32(w - np.float32(1))) * np.float64(diff) + np.float64(b))


def umeyama(x: np.ndarray, y: np.ndarray):
    """Least-squares similarity (R, t, s) with y ~ s R x + t over rows of x, y (M,3).  float64 throughout."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    xm = x.mean(0)
    ym = y.mean(0)
    xh = x - xm
    yh = y - ym
    m = yh.T @ xh
    u, s, vt = np.linalg.svd(m)
    d = np.sign(np.linalg.det(u @ vt))
    if d == 0:
        d = 1.0
    dd = np.array([1.0, 1.0, d])
    r = (u * dd) @ vt
    scale = float((s * dd).sum() / (xh ** 2).sum())
    t = ym - scale * (r @ xm)
    return r, t, scale


def align_local_to_global(pts_local, conf_global, pts_global, valid=None, min_conf_thr_percentile=0.0):
    """One (view, batch) unit of align_local_pts3d_to_global.  pts (H,W,3), conf (H,W), valid (H,W) bool or None.
    Returns (aligned (H,W,3) float32, R, t, s)."""
    h, w, _ = pts_local.shape
    xl = np.asarray(pts_local, np.float32).reshape(-1, 3)
    yg = np.asarray(pts_global, np.float32).reshape(-1, 3)
    c = np.asarray(conf_global, np.float32).reshape(-1)
    vm = np.ones(c.shape, bool) if valid is None else np.asarray(valid, bool).reshape(-1)
    thr = conf_quantile(c, min_conf_thr_percentile / 100.0)
    mask = (c >= thr) & vm
    if mask.sum() < 3:
        mask = vm
    if mask.sum() < 3:
        r, t, s = np.eye(3), np.zeros(3), 1.0
    else:
        r, t, s = umeyama(xl[mask], yg[mask])
    out = s * (xl.astype(np.float64) @ r.T) + t
    return out.astype(np.float32).reshape(h, w, 3), r, t, s


def focal_weiszfeld(pts3d, pp, mask=None, iters=100):
    """Weiszfeld / IRLS focal: argmin_f sum | pixel - f (x,y)/z | over the selected points.  pts3d (H,W,3), pp (2,),
    mask (H,W) bool or None (all points).  Returns the focal clipped to [0, inf) as float (the reference's clip uses
    min_focal=0, max_focal=inf at both call sites).  With no selected point: max(H,W)/(2 tan 30deg) (post_process.py:108)."""
    h, w, _ = pts3d.shape
    p = np.asarray(pts3d, np.float32).reshape(-1, 3)
    uu, vv = np.meshgrid(np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32), indexing="xy")
    px = np.stack([uu.reshape(-1) - np.float32(pp[0]), vv.reshape(-1) - np.float32(pp[1])], -1).astype(np.float32)
    if mask is not None:
        sel = np.asarray(mask, bool).reshape(-1)
        p, px = p[sel], px[sel]
    if p.shape[0] == 0:
        return float(max(h, w) / (2 * np.tan(np.deg2rad(60) / 2)))
    with np.errstate(divide="ignore", invalid="ignore"):
        xyz = (p[:, :2] / p[:, 2:3]).astype(np.float32)
    xyz = np.nan_to_num(xyz, nan=0.0, posinf=0.0, neginf=0.0)
    dpx = (xyz * px).sum(-1).astype(np.float64)
    dxx = (xyz * xyz).sum(-1).astype(np.float64)
    xyz64, px64 = xyz.astype(np.float64), px.astype(np.float64)
    f = dpx.sum() / dxx.sum()
    for _ in range(iters):
        dis = np.sqrt(((px64 - f * xyz64) ** 2).sum(-1))
        wgt = 1.0 / np.maximum(dis, 1e-8)
        f = (wgt * dpx).sum() / (wgt * dxx).sum()
    return float(max(f, 0.0))


def estimate_focal(pts3d, conf, min_conf_thr_percentile=10.0, pp=None):
    """multiview_dust3r_module.py:1081-1109 for one (H,W,3)/(H,W) pair."""
    h, w, _ = pts3d.shape
    if pp is None:
        pp = (w / 2, h / 2)
    thr = conf_quantile(conf, min_conf_thr_percentile / 100.0)
    return focal_weiszfeld(pts3d, pp, np.asarray(conf, np.float32) >= thr, iters=100)
