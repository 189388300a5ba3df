"""CPU emulator of the camera-pose entry points of the C ABI (fast3r_b200.ops.pnp_gather / pnp_score / pnp_inliers),
TEST INFRASTRUCTURE ONLY: the same arguments and results as the ops, computed with numpy in OpenCV's arithmetic (the
rule of fast3r_b200/csrc/pose_math.h), so the host side of fast3r_b200.poses runs without a GPU and the GPU tests have
a host answer for every kernel."""
import numpy as np
import torch

from fast3r_b200 import lib as L


def project(hyp, pts):
    """projectPoints of fp32 pts (n, 3) under one PNP_HYP row: fp32 (n, 2), in pose_math.h's operation order."""
    r, t = hyp["r"], hyp["t"]
    X, Y, Z = (pts[:, i].astype(np.float64) for i in range(3))
    x = ((r[0] * X + r[1] * Y) + r[2] * Z) + t[0]
    y = ((r[3] * X + r[4] * Y) + r[5] * Z) + t[1]
    z = ((r[6] * X + r[7] * Y) + r[8] * Z) + t[2]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        w = np.where(z != 0, 1.0 / np.where(z != 0, z, 1.0), 1.0)
        x, y = x * w, y * w
        r2 = x * x + y * y
        bad = ~((r2 * r2) * r2 <= np.finfo(np.float64).max)
        x, y = np.where(bad, np.nan, x), np.where(bad, np.nan, y)
        return np.stack([(x * hyp["fx"] + hyp["cx"]).astype(np.float32), (y * hyp["fy"] + hyp["cy"]).astype(np.float32)], 1)


def error(pix, proj):
    """computeError's float32 (0 + dx^2) + dy^2."""
    with np.errstate(invalid="ignore", over="ignore"):
        d = pix.astype(np.float32) - proj
        return (np.float32(0) + d[:, 0] * d[:, 0]) + d[:, 1] * d[:, 1]


def inlier_mask(hyp, pts, pix, thr):
    with np.errstate(invalid="ignore"):
        return error(pix, project(hyp, pts)) <= np.float32(np.float64(np.float32(thr)) ** 2)


def pnp_gather(pts, conf=None, mask=None):
    views, h, w = pts.shape[0], pts.shape[1], pts.shape[2]
    sel = (conf > 1) if conf is not None else (mask != 0)
    grid = np.mgrid[:w, :h].T.astype(np.float32).reshape(-1, 2)  # pixel_grid(h, w)
    out_pts = torch.zeros(views, h * w, 3)
    out_pix = torch.zeros(views, h * w, 2)
    counts = torch.zeros(views, dtype=torch.int32)
    for v in range(views):
        m = sel[v].reshape(-1).numpy()
        c = int(m.sum())
        out_pts[v, :c] = pts[v].reshape(-1, 3)[torch.from_numpy(m)]
        out_pix[v, :c] = torch.from_numpy(grid[m])
        counts[v] = c
    return out_pts, out_pix, counts


def pnp_score(pts, pix, offsets, view_counts, hyps, thr):
    P, X = pts.numpy(), pix.numpy()
    hyps = np.asarray(hyps, L.PNP_HYP)
    out = np.zeros(len(hyps), np.int32)
    for i, h in enumerate(hyps):
        o, c = int(offsets[h["view"]]), int(view_counts[h["view"]])
        out[i] = int(inlier_mask(h, P[o:o + c], X[o:o + c], thr).sum())
    return torch.from_numpy(out)


def pnp_inliers(pts, pix, offsets, view_counts, hyps, thr):
    P, X = pts.numpy(), pix.numpy()
    hyps = np.asarray(hyps, L.PNP_HYP)
    m = int(sum(int(view_counts[h["view"]]) for h in hyps))
    out_pts, out_pix = np.zeros((m, 3), np.float32), np.zeros((m, 2), np.float32)
    counts, at = np.zeros(len(hyps), np.int32), 0
    for i, h in enumerate(hyps):
        o, c = int(offsets[h["view"]]), int(view_counts[h["view"]])
        sel = inlier_mask(h, P[o:o + c], X[o:o + c], thr)
        k = int(sel.sum())
        out_pts[at:at + k], out_pix[at:at + k] = P[o:o + c][sel], X[o:o + c][sel]
        counts[i] = k
        at += c
    return torch.from_numpy(out_pts), torch.from_numpy(out_pix), torch.from_numpy(counts)
