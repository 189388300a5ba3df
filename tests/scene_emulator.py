"""CPU emulator of the viewer-scene entry points of fast3r_b200.ops (sky_mask, scene_sort, scene_visible, ply_pack,
extent_percentiles): same arguments, the same results in numpy, on CPU tensors.  tests/test_scene_cpu.py runs
fast3r_b200.scene on it against the reference's goldens; tests/test_scene_gpu.py holds the kernels to it."""
import numpy as np
import torch

from tests import scene_oracle as O


def sky_mask(img, out=None):
    frames, _, h, w = img.shape
    masks = np.stack([O.detect_sky_mask(img[f].permute(1, 2, 0).cpu().numpy()).reshape(-1) for f in range(frames)])
    if out is None:
        out = torch.empty(frames, h * w, dtype=torch.int8)
    out.copy_(torch.from_numpy(masks))
    return out, torch.from_numpy(masks.astype(np.int64).sum(1).astype(np.int32))


def scene_sort(conf, pts, img, not_sky, offsets, out_pts, out_rgb, out_not_sky, max_conf):
    off = offsets.cpu().numpy()
    c, p, im, ns = conf.cpu().numpy(), pts.cpu().numpy().reshape(-1, 3), img.cpu().numpy(), not_sky.cpu().numpy()
    for f in range(len(off) - 1):
        a, b = int(off[f]), int(off[f + 1])
        o = O.order(c[a:b])
        rgb = O.to_u8(im[3 * a:3 * b].reshape(3, b - a).T)
        out_pts[a:b] = torch.from_numpy(p[a:b][o])
        out_rgb[a:b] = torch.from_numpy(rgb[o])
        out_not_sky[a:b] = torch.from_numpy(ns[a:b][o])
        max_conf[f] = float(c[a:b].max())


def scene_visible(segs, pts_g, pts_l, rgb_g, rgb_l, not_sky_g, not_sky_l, mask_sky):
    pts, cols = [], []
    for head, start, n, color in np.asarray(segs, np.int64).reshape(-1, 4):
        P, R, N = (pts_l, rgb_l, not_sky_l) if head else (pts_g, rgb_g, not_sky_g)
        sel = np.ones(n, bool) if not mask_sky else N[start:start + n].numpy() > 0
        pts.append(P[start:start + n].numpy()[sel])
        rgb = R[start:start + n].numpy()[sel]
        if color >= 0:
            rgb = np.tile(np.array([color >> 16, (color >> 8) & 255, color & 255], np.uint8), (len(rgb), 1))
        cols.append(rgb)
    if not pts:
        return torch.empty(0, 3), torch.empty(0, 3, dtype=torch.uint8)
    return torch.from_numpy(np.concatenate(pts)), torch.from_numpy(np.concatenate(cols))


def ply_pack(points, colors):
    rec = np.empty(len(points), dtype=[("xyz", "<f4", 3), ("rgb", "u1", 3)])
    rec["xyz"] = points.numpy()
    rec["rgb"] = colors.numpy()
    return torch.from_numpy(np.frombuffer(rec.tobytes(), np.uint8).copy())


def extent_percentiles(points, lo=20, hi=80):
    p = points.numpy()
    a, b = np.percentile(p, lo, axis=0), np.percentile(p, hi, axis=0)
    return torch.from_numpy(np.concatenate([a, b, [np.max(b - a)]]).astype(np.float32))
