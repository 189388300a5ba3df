"""A numpy / cv2 / scipy restatement of the reference viewer's scene (fast3r/viz/viser_visualizer.py), the oracle of
the fast3r_b200.scene tests: detect_sky_mask, the per-frame data of start_visualization, is_outdoor, max_extent, the
visible points of a state of the controls and the PLY bytes.  tests/test_scene_cpu.py pins it on the unmodified
reference.  The order is np.argsort(-conf, kind="stable"), the definition fast3r_b200.scene keeps."""
import colorsys

import cv2
import numpy as np
from scipy import ndimage

BOXES = (((105, 50, 140), (135, 255, 255)), ((95, 5, 150), (145, 100, 255)), ((0, 0, 235), (180, 10, 255)))


def to_u8(img):
    return ((img + 1) * 127.5).astype(np.uint8)


def sky_boxes(u8):
    """bool: the pixels of the three inRange boxes, and the HSV image."""
    hsv = cv2.cvtColor(np.ascontiguousarray(u8), cv2.COLOR_RGB2HSV)
    m = np.zeros(u8.shape[:2], bool)
    for lo, hi in BOXES:
        m |= cv2.inRange(hsv, np.array(lo), np.array(hi)) > 0
    return m, hsv


def detect_sky_mask(img, stats=None):
    """int8 not-sky mask of an (H, W, 3) image in [-1, 1]; `stats` (a dict) receives which selection case ran."""
    m, hsv = sky_boxes(to_u8(img))
    h, w = m.shape
    ut = int(h * 0.4)
    m[:ut] |= (hsv[:ut, :, 1] < 50) & (hsv[:ut, :, 2] > 150)
    k = np.ones((7, 7), np.uint8)
    m = cv2.dilate(m.astype(np.uint8), k)
    m = cv2.morphologyEx(m, cv2.MORPH_OPEN, k) > 0
    lab, num = ndimage.label(m)
    top = set(lab[0].tolist()) - {0}
    case = "empty" if num == 0 else ("no_top" if not top else "top")
    if top:
        cnt = np.bincount(lab.ravel(), minlength=num + 1)
        big = [l for l in top if cnt[l] > h * w * 0.01]
        case = "top_all_small" if not big else case
        m = np.isin(lab, big)
    if stats is not None:
        stats[case] = stats.get(case, 0) + 1
        lab8, _ = ndimage.label(lab > 0, structure=np.ones((3, 3)))
        if top and set(lab8[0].tolist()) - {0}:
            c8 = np.bincount(lab8.ravel())
            m8 = np.isin(lab8, [l for l in set(lab8[0].tolist()) - {0} if c8[l] > h * w * 0.01])
            if (m8 != m).any():  # 8-connectivity would select another sky: only 4-connectivity gives this mask
                stats["diagonal_4_vs_8"] = stats.get("diagonal_4_vs_8", 0) + 1
    return (~m).astype(np.int8)


def order(conf):
    return np.argsort(-conf, kind="stable")


def frame_data(pred, view, i, n, thr=1.5):
    """The frame arrays of frame i (batch size 1), with the u8 colours."""
    img = view["img"][0].permute(1, 2, 0).numpy()
    ns = detect_sky_mask(img).reshape(-1)
    rgb = to_u8(img.reshape(-1, 3))
    out = {}
    for head, pk, ck in (("global", "pts3d_in_other_view", "conf"), ("local", "pts3d_local_aligned_to_global", "conf_local")):
        conf = pred[ck][0].numpy().reshape(-1)
        o = order(conf)
        out[f"pts_{head}"] = pred[pk][0].numpy().reshape(-1, 3)[o]
        out[f"rgb_{head}"] = rgb[o]
        out[f"not_sky_{head}"] = ns[o]
    conf = pred["conf"][0].numpy().reshape(-1)
    out["max_conf_global"] = conf.max()
    out["is_high_confidence"] = bool(conf.max() >= thr)
    out["view_color"] = np.clip(np.array(colorsys.hsv_to_rgb(i / n, 1.0, 1.0)) * 255, 0, 255).astype(np.uint8)
    return out


def prepare_scene(output, thr=1.5):
    n = len(output["preds"])
    frames = [frame_data(p, v, i, n, thr) for i, (p, v) in enumerate(zip(output["preds"], output["views"]))]
    sig = sum(1 for fd in frames if 1.0 - np.mean(fd["not_sky_global"]) > 0.2)
    allp = np.concatenate([fd["pts_global"] for fd in frames])
    ext = np.max(np.percentile(allp, 80, axis=0) - np.percentile(allp, 20, axis=0))
    return dict(frames=frames, is_outdoor=sig >= n / 4, max_extent=ext)


def visible_points(scene, timestep=None, p=None, mask_sky=None, show_global=False, show_local=True, drop_low=False,
                   color="rgb"):
    frames = scene["frames"]
    last = len(frames) - 1 if timestep is None else timestep
    mask_sky = scene["is_outdoor"] if mask_sky is None else mask_sky
    pts, cols = [], []
    for i in range(last + 1):
        fd = frames[i]
        if drop_low and not fd["is_high_confidence"]:
            continue
        for head, shown in (("global", show_global), ("local", show_local)):
            if not shown:
                continue
            tot = len(fd[f"pts_{head}"])
            k = tot if p is None else max(1, int(tot * (100 - p) / 100))
            sel = np.ones(k, bool) if not mask_sky else fd[f"not_sky_{head}"][:k] > 0
            pts.append(fd[f"pts_{head}"][:k][sel])
            c = fd[f"rgb_{head}"][:k][sel] if color == "rgb" else np.tile(fd["view_color"], (int(sel.sum()), 1))
            cols.append(c)
    if not pts:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8)
    return np.concatenate(pts), np.concatenate(cols)


def ply_bytes(points, colors):
    header = "\n".join(["ply", "format binary_little_endian 1.0", f"element vertex {len(points)}", "property float x",
                        "property float y", "property float z", "property uchar red", "property uchar green",
                        "property uchar blue", "end_header"]).encode("ascii") + b"\n"
    rec = np.empty(len(points), dtype=[("xyz", "<f4", 3), ("rgb", "u1", 3)])
    rec["xyz"] = points
    rec["rgb"] = colors
    return header + rec.tobytes()
