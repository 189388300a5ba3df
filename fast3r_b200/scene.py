"""The viewer's scene on the GPU: the frame preparation of the reference's viewer and its point export, bit-identical to
the reference's numpy / cv2 / scipy code (fast3r/viz/viser_visualizer.py).

* ``detect_sky_mask(img_rgb)`` - viser_visualizer.py:24-72: the int8 not-sky mask of an (H, W, 3) image in [-1, 1].
* ``prepare_scene(output, global_conf_thr_value_to_drop_view=1.5)`` - the per-frame loop of ``start_visualization``
  (:343-427) and its scene tests (:74-81, :420-427): per frame the points of both heads, their u8 colours and not-sky
  values in descending confidence order, the frame's largest global confidence, whether it passes the threshold and
  its "Color by View" colour; ``is_outdoor`` and ``max_extent`` of the scene.
* ``Scene.visible_points(...)`` - the points the viewer shows for a state of its controls (:115-165, :487-533) and
  collects for "Download PLY" (:168-203); ``ply_bytes`` / ``save_ply`` - the file it sends (:228-254).

The one definition this module adds: frames are ordered by ``np.argsort(-conf, kind="stable")`` (ties by pixel index),
where the reference's default, unstable sort leaves the order of equal confidences to numpy's introsort.  The
viewer's server, its GIF rendering, camera frustums and the confidence (turbo) colouring are not here.

Inputs may live on the CPU or on a CUDA device; the results stay on the device.  There is no CPU path.
"""
from __future__ import annotations

import colorsys
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import ops

_GROUP = 64            # frames per sort launch: bounds the sort's keys and staging copies at N = 1000
_GROUP_ELEMS = 1 << 25  # ... and their pixels (a single larger frame still forms its own group)


def _device(t: torch.Tensor) -> torch.device:
    if t.is_cuda:
        return t.device
    if not torch.cuda.is_available():
        raise RuntimeError("fast3r_b200.scene needs a CUDA device (there is no CPU path)")
    return torch.device("cuda:0")


def _f32(t: torch.Tensor, dev: torch.device) -> torch.Tensor:
    return t.to(device=dev, dtype=torch.float32).contiguous()


def detect_sky_mask(img_rgb):
    """int8 (H, W) mask, 1 where the pixel is not sky, of an (H, W, 3) float32 RGB image in [-1, 1] (numpy in, numpy
    out; a tensor gives a tensor on the device)."""
    as_numpy = isinstance(img_rgb, np.ndarray)
    t = torch.from_numpy(np.ascontiguousarray(img_rgb)) if as_numpy else img_rgb
    if t.dtype != torch.float32:  # the u8 conversion rounds in the input's type: only float32 (load_images) is built
        raise TypeError(f"detect_sky_mask: expected a float32 image, got {t.dtype}")
    if t.dim() != 3 or t.shape[2] != 3:
        raise ValueError(f"detect_sky_mask: expected an (H, W, 3) image, got {tuple(t.shape)}")
    h, w = t.shape[0], t.shape[1]
    img = _f32(t, _device(t)).permute(2, 0, 1).contiguous().reshape(1, 3, h, w)
    not_sky, _ = ops.sky_mask(img)
    out = not_sky.reshape(h, w)
    return out.cpu().numpy() if as_numpy else out


@dataclass
class Scene:
    """The viewer's frame data, frames concatenated: frame i is rows offsets[i]:offsets[i + 1] of every frame array."""
    offsets: np.ndarray              # int64 [N + 1] (host)
    pts_global: torch.Tensor         # fp32 [T, 3]: pts3d_in_other_view, each frame in descending `conf` order
    pts_local: torch.Tensor          # fp32 [T, 3]: pts3d_local_aligned_to_global, descending `conf_local` order
    rgb_global: torch.Tensor         # uint8 [T, 3]: the pixels' colours in the global order
    rgb_local: torch.Tensor          # uint8 [T, 3]
    not_sky_global: torch.Tensor     # int8 [T]: detect_sky_mask in the global order
    not_sky_local: torch.Tensor      # int8 [T]
    max_conf_global: np.ndarray      # float32 [N]: conf.max() per frame
    is_high_confidence: np.ndarray   # bool [N]: max_conf_global >= the threshold (compared in float32, as numpy does)
    view_colors: np.ndarray          # uint8 [N, 3]: the frame's "Color by View" colour
    is_outdoor: bool
    max_extent: float                # max over axes of the 80th minus the 20th percentile of the global points (float32)

    @property
    def num_frames(self) -> int:
        return len(self.offsets) - 1

    def visible_points(self, timestep: Optional[int] = None, min_conf_thr_percentile: Optional[float] = None,
                       mask_sky: Optional[bool] = None, show_global: bool = False, show_local: bool = True,
                       drop_low_conf_views: bool = False, color: str = "rgb") -> Tuple[torch.Tensor, torch.Tensor]:
        """(points fp32 (M, 3), colours uint8 (M, 3)) on the device that the viewer shows, and exports, for a state of
        its controls.  Frames 0..timestep (default: the last) contribute in frame order, the global head before the
        local one, for each head shown; ``drop_low_conf_views`` hides frames that are not high-confidence.  Of each
        frame and head the first max(1, int(total * (100 - p) / 100)) points are kept when the percentile p is set,
        and of those only the not-sky points when ``mask_sky`` (default: ``is_outdoor``).  ``color`` is "rgb" (the
        pixels) or "view" (the frame's colour).  The defaults are the viewer's state at launch."""
        if color not in ("rgb", "view"):
            raise ValueError(f"color must be 'rgb' or 'view', got {color!r}")
        n = self.num_frames
        last = n - 1 if timestep is None else int(timestep)
        if not 0 <= last < n:
            raise ValueError(f"timestep {timestep} outside [0, {n})")
        mask_sky = self.is_outdoor if mask_sky is None else bool(mask_sky)
        segs = []
        for i in range(last + 1):
            if drop_low_conf_views and not self.is_high_confidence[i]:
                continue
            total = int(self.offsets[i + 1] - self.offsets[i])
            keep = total if min_conf_thr_percentile is None else max(1, int(total * (100 - min_conf_thr_percentile) / 100))
            c = self.view_colors[i]
            col = -1 if color == "rgb" else (int(c[0]) << 16) | (int(c[1]) << 8) | int(c[2])
            for head, shown in ((0, show_global), (1, show_local)):
                if shown:
                    segs.append((head, int(self.offsets[i]), keep, col))
        return ops.scene_visible(np.array(segs, dtype=np.int64).reshape(-1, 4), self.pts_global, self.pts_local,
                                 self.rgb_global, self.rgb_local, self.not_sky_global, self.not_sky_local, mask_sky)


def _view_color(i: int, n: int) -> np.ndarray:
    return np.clip(np.array(colorsys.hsv_to_rgb(i / n, 1.0, 1.0)) * 255, 0, 255).astype(np.uint8)


def _frame(pred: Dict, view: Dict, i: int):
    if view["img"].shape[0] != 1:
        raise ValueError(f"prepare_scene: view {i} has batch size {view['img'].shape[0]} (the viewer takes 1)")
    if view["img"].dtype != torch.float32:
        raise TypeError(f"prepare_scene: view {i} image is {view['img'].dtype}; the u8 conversion is built for float32")
    if "pts3d_local_aligned_to_global" not in pred:
        raise KeyError(f"pred {i} has no 'pts3d_local_aligned_to_global': run align_local_pts3d_to_global first")
    return tuple(view["img"].shape[2:])


def prepare_scene(output: Dict, global_conf_thr_value_to_drop_view: float = 1.5) -> Scene:
    """The viewer's frame data of ``output`` = {"views": [...], "preds": [...]} (batch size 1, any resolutions)."""
    views: List[Dict] = output["views"]
    preds: List[Dict] = output["preds"]
    n = len(preds)
    if n == 0 or len(views) != n:
        raise ValueError("prepare_scene: need one view per pred and at least one frame")
    shapes = [_frame(p, v, i) for i, (p, v) in enumerate(zip(preds, views))]
    dev = _device(preds[0]["conf"])
    hw = np.array([h * w for h, w in shapes], dtype=np.int64)
    offsets = np.concatenate([[0], np.cumsum(hw)]).astype(np.int64)
    total = int(offsets[-1])

    # sky masks, one call per run of consecutive frames of one shape (at most _GROUP frames)
    not_sky = torch.empty(total, dtype=torch.int8, device=dev)
    counts = []
    for i, j in _runs(n, lambda i, j: shapes[j] == shapes[i] and j - i < _GROUP):
        h, w = shapes[i]
        img = torch.cat([_f32(views[k]["img"], dev) for k in range(i, j)])
        counts.append(ops.sky_mask(img, out=not_sky[offsets[i]:offsets[j]].view(j - i, h * w))[1])
    counts = torch.cat(counts).cpu().numpy()

    # both heads in confidence order, in groups of consecutive frames of any shapes
    arrays = {}
    max_conf = torch.empty(n, dtype=torch.float32, device=dev)
    scratch = torch.empty(n, dtype=torch.float32, device=dev)
    for head, pts_key, conf_key in (("global", "pts3d_in_other_view", "conf"),
                                    ("local", "pts3d_local_aligned_to_global", "conf_local")):
        out_pts = torch.empty(total, 3, dtype=torch.float32, device=dev)
        out_rgb = torch.empty(total, 3, dtype=torch.uint8, device=dev)
        out_ns = torch.empty(total, dtype=torch.int8, device=dev)
        for i, j in _runs(n, lambda i, j: j - i < _GROUP and offsets[j + 1] - offsets[i] <= _GROUP_ELEMS):
            a, b = int(offsets[i]), int(offsets[j])
            conf = torch.cat([_f32(preds[k][conf_key], dev).reshape(-1) for k in range(i, j)])
            pts = torch.cat([_f32(preds[k][pts_key], dev).reshape(-1, 3) for k in range(i, j)])
            img = torch.cat([_f32(views[k]["img"], dev).reshape(-1) for k in range(i, j)])
            off = torch.from_numpy(offsets[i:j + 1] - a).to(dev)
            mc = max_conf if head == "global" else scratch
            ops.scene_sort(conf, pts, img, not_sky[a:b], off, out_pts[a:b], out_rgb[a:b], out_ns[a:b], mc[i:j])
        arrays[head] = (out_pts, out_rgb, out_ns)

    max_conf_np = max_conf.cpu().numpy()
    sky_ratios = 1.0 - counts.astype(np.float64) / hw  # 1 - np.mean(not_sky) of each frame, from exact counts
    is_outdoor = int((sky_ratios > 0.2).sum()) >= n / 4
    max_extent = float(ops.extent_percentiles(arrays["global"][0])[6].item())
    return Scene(offsets=offsets, pts_global=arrays["global"][0], pts_local=arrays["local"][0],
                 rgb_global=arrays["global"][1], rgb_local=arrays["local"][1], not_sky_global=arrays["global"][2],
                 not_sky_local=arrays["local"][2], max_conf_global=max_conf_np,
                 is_high_confidence=max_conf_np >= global_conf_thr_value_to_drop_view,
                 view_colors=np.stack([_view_color(i, n) for i in range(n)]), is_outdoor=bool(is_outdoor),
                 max_extent=max_extent)


def _runs(n: int, extend):
    """[i, j) runs of frames: a run grows by frame j while extend(i, j) holds."""
    i = 0
    while i < n:
        j = i + 1
        while j < n and extend(i, j):
            j += 1
        yield i, j
        i = j


_PLY_HEADER = ("ply\nformat binary_little_endian 1.0\nelement vertex {n}\nproperty float x\nproperty float y\n"
               "property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")


def ply_bytes(points: torch.Tensor, colors_u8: torch.Tensor) -> bytes:
    """The binary PLY file of the viewer's "Download PLY" for points fp32 (M, 3) and colours uint8 (M, 3): the records
    are packed on the device and copied to the host once."""
    if isinstance(points, np.ndarray):
        points = torch.from_numpy(points)
    if isinstance(colors_u8, np.ndarray):
        colors_u8 = torch.from_numpy(colors_u8)
    dev = _device(points)
    packed = ops.ply_pack(_f32(points, dev), colors_u8.to(device=dev, dtype=torch.uint8).contiguous())
    return _PLY_HEADER.format(n=points.shape[0]).encode("ascii") + packed.cpu().numpy().tobytes()


def save_ply(path, points: torch.Tensor, colors_u8: torch.Tensor) -> None:
    with open(path, "wb") as f:
        f.write(ply_bytes(points, colors_u8))
