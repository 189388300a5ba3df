"""Ground-truth views on the GPU: the per-view tail of the datasets' ``__getitem__``.

The reference makes every training, validation and evaluation view on the host, one at a time
(fast3r/dust3r/datasets/base/base_stereo_view_dataset.py): ``_crop_resize_if_necessary`` (:165-221) crops around the
principal point, picks the orientation, resizes with Pillow (LANCZOS / BICUBIC) and ``cv2.resize(INTER_NEAREST)`` and
crops again; ``__getitem__`` (:78-142) then applies ImgNorm, fills a missing pose with NaN, unprojects the depth map to
world points (fast3r/dust3r/utils/geometry.py:186-243), masks the invalid pixels and transposes portrait views to
landscape (:243-261).  The RE10K pose benchmark has an image-only variant (scripts/fast3r_re10k_pose_eval.py:84-134).

Here the geometry is planned on the host in numpy with the reference's dtypes and roundings (``plan_view``,
``plan_view_re10k``: cheap, and it consumes a loader's generator exactly as the reference does), and the pixel work runs
on the device: the image through ``f3r_ingest_rgb8`` (Pillow's 8-bit resampler, bit-exact), the depth map, points,
mask and transpose through one launch of ``f3r_view_geometry`` for every view of the call.  ``prepare_views`` returns
the views as ``default_collate`` gives them after ``__getitem__``, on the device, bit-identical to the reference.
File decoding, ColorJitter and the dataset classes stay with the loaders.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

from . import ingest, lib as L, ops

BICUBIC, LANCZOS = ingest.BICUBIC, ingest.LANCZOS
_KEYS = ("img", "depthmap", "camera_intrinsics", "camera_pose")


@dataclass(frozen=True)
class ViewPlan:
    """Geometry of one view: ``crop`` (left, top, right, bottom) around the principal point in the source image,
    ``size`` (width, height) the crop is resized to with ``filt`` (BICUBIC or LANCZOS), ``box`` (left, top, right,
    bottom) the final crop of the resized image, and ``intrinsics`` the float32 3x3 camera matrix of that final crop."""
    crop: Tuple[int, int, int, int]
    size: Tuple[int, int]
    filt: int
    box: Tuple[int, int, int, int]
    intrinsics: np.ndarray

    @property
    def shape(self):
        """(height, width) of the view before the landscape transpose: its ``true_shape``."""
        return self.box[3] - self.box[1], self.box[2] - self.box[0]


def _shift(K, left, top):
    """crop_image_depthmap's intrinsics (cropping.py): the principal point moves by the crop's corner; the float32
    entries are updated in place, through numpy's promotion of float32 with the corner's integer type."""
    K = K.copy()
    K[0, 2] -= left
    K[1, 2] -= top
    return K


def _crop_camera(K, in_size, out_size, scaling=1):
    """camera_matrix_of_crop (cropping.py) with offset_factor 0.5: scale the colmap-convention camera and move its
    principal point by half the margin; float32 entries rounded as numpy rounds them."""
    margins = np.asarray(in_size) * scaling - out_size
    assert np.all(margins >= 0.0)
    offset = 0.5 * margins
    C = K.copy()
    C[0, 2] += 0.5
    C[1, 2] += 0.5
    C[:2, :] *= scaling
    C[:2, 2] -= offset
    C = C.copy()
    C[0, 2] -= 0.5
    C[1, 2] -= 0.5
    return C


def _principal_crop(width, height, K):
    """The window of half-size (min margin x, min margin y) centred on the rounded principal point."""
    cx, cy = K[:2, 2].round().astype(int)
    mx, my = min(cx, width - cx), min(cy, height - cy)
    return (cx - mx, cy - my, cx + mx, cy + my), mx, my


def _finish(width, height, K, crop, resolution, target):
    """Rescale the principal-point crop so that it covers `target` (w, h), then crop `resolution` (w, h) around the
    principal point (rescale_image_depthmap, camera_matrix_of_crop, bbox_from_intrinsics_in_out of cropping.py)."""
    l, t, r, b = (int(v) for v in crop)
    if not (0 <= l < r <= width and 0 <= t < b <= height):
        raise ValueError(f"principal-point crop {crop} is empty or outside the {width}x{height} image")
    K = _shift(K, crop[0], crop[1])
    in_size = np.array((r - l, b - t))
    target = np.array(target)
    scale = max(target / (r - l, b - t)) + 1e-8
    size = np.floor(in_size * scale).astype(int)
    K = _crop_camera(K, in_size, size, scaling=scale)
    K2 = _crop_camera(K, (int(size[0]), int(size[1])), resolution)
    bl, bt = np.int32(np.round(K[:2, 2] - K2[:2, 2]))
    box = (int(bl), int(bt), int(bl) + resolution[0], int(bt) + resolution[1])
    if not (0 <= box[0] and box[2] <= size[0] and 0 <= box[1] and box[3] <= size[1]):
        raise ValueError(f"final crop {box} outside the resized {size[0]}x{size[1]} image")
    K = _shift(K, bl, bt)
    return ViewPlan((l, t, r, b), (int(size[0]), int(size[1])), LANCZOS if scale < 1 else BICUBIC, box, K)


def plan_view(width: int, height: int, intrinsics, resolution, rng: Optional[np.random.Generator] = None,
              aug_crop=False, info=None) -> ViewPlan:
    """The geometry of BaseStereoViewDataset._crop_resize_if_necessary for a width x height view with float32 camera
    matrix `intrinsics` at `resolution` (w, h) or a square size: the principal point must lie more than a fifth of the
    image from each edge (AssertionError otherwise, as in the reference); a crop more than 1.1 times taller than wide
    takes the portrait resolution, and a near-square one (0.9 < h / w < 1.1) at a non-square resolution draws
    ``rng.integers(2)``; ``aug_crop > 1`` draws ``rng.integers(0, aug_crop)`` once and adds it to both target
    dimensions.  Draws from `rng` in the reference's order."""
    K = np.array(intrinsics, dtype=np.float32)
    res = (resolution, resolution) if isinstance(resolution, int) else tuple(int(v) for v in resolution)
    crop, mx, my = _principal_crop(width, height, K)
    assert mx > width / 5, f"Bad principal point in view={info}"
    assert my > height / 5, f"Bad principal point in view={info}"
    W, H = crop[2] - crop[0], crop[3] - crop[1]
    assert res[0] >= res[1]
    portrait = H > 1.1 * W
    if not portrait and 0.9 < H / W < 1.1 and res[0] != res[1]:
        if rng is None:
            raise ValueError(f"a near-square view at a non-square resolution needs an rng (view={info})")
        portrait = bool(rng.integers(2))
    if portrait:
        res = res[::-1]
    target = np.array(res)
    if aug_crop > 1:
        if rng is None:
            raise ValueError(f"aug_crop needs an rng (view={info})")
        target += rng.integers(0, aug_crop)
    return _finish(width, height, K, crop, res, target)


def plan_view_re10k(width: int, height: int, intrinsics, target_resolution=(512, 288)) -> ViewPlan:
    """The geometry of the RE10K pose benchmark's crop_resize_if_necessary (scripts/fast3r_re10k_pose_eval.py:84-134):
    the principal-point crop without margin checks, the portrait target when the crop is taller than wide, no rng."""
    K = np.array(intrinsics, dtype=np.float32)
    crop, _, _ = _principal_crop(width, height, K)
    res = tuple(int(v) for v in target_resolution)
    if crop[3] - crop[1] > crop[2] - crop[0]:
        res = res[::-1]
    return _finish(width, height, K, crop, res, res)


def _need_cuda(device):
    ingest._need_cuda(device, "prepare_views makes CUDA views (there is no CPU path)")


def _upload(arr: np.ndarray, device) -> torch.Tensor:
    """Copies a host array to `device` through pinned staging (asynchronous on the current stream)."""
    return torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to(device, non_blocking=True)


_NP = {torch.uint8: np.uint8, torch.float32: np.float32}


def _on_device(x, dtype, device) -> torch.Tensor:
    """A raw view's array on `device`: CUDA tensors as they are (they must already be there), host arrays uploaded."""
    if torch.is_tensor(x):
        if x.device.type != "cpu":
            if x.device != device or x.dtype != dtype:
                raise ValueError(f"device input must be {dtype} on {device}, got {x.dtype} on {x.device}")
            return x.contiguous()
        x = x.numpy()
    return _upload(np.asarray(x, _NP[dtype]), device)


def _plan_sample(views, resolution, rng, aug_crop):
    plans = []
    for i, v in enumerate(views):
        h, w = v["img"].shape[:2]
        info = "/".join(str(v.get(k, "?")) for k in ("dataset", "label", "instance"))
        plans.append(plan_view(w, h, v["camera_intrinsics"], resolution, rng, aug_crop, info or i))
    return plans


def prepare_views(samples, resolution=None, plans=None, rngs=None, aug_crop=False, device="cuda"):
    """Views of a batch as ``default_collate`` gives them after ``BaseStereoViewDataset.__getitem__``, on `device`.

    samples: B lists of N raw views, each a dict with ``img`` (uint8 (H, W, 3) RGB), ``depthmap`` (float32 (H, W),
    metres, finite), ``camera_intrinsics`` (float32 3x3) and optionally ``camera_pose`` (float32 4x4 cam2world), as
    numpy arrays or CUDA tensors; other keys (``dataset``, ``label``, ``instance``, ...) pass through default_collate.
    plans: B lists of N ViewPlan (plan_view / plan_view_re10k), or None to plan each sample's views in order with
    ``plan_view(..., resolution, rngs[b], aug_crop)``.  rngs: one numpy Generator per sample, as the reference seeds one
    per item; after the views are planned, each sample draws ``rng.bytes(4)`` once per view, as ``__getitem__`` does,
    and the views get it as ``rng``.

    Returns N dicts with img (B, 3, H, W) float32 in [-1, 1], depthmap (B, H, W), pts3d (B, H, W, 3), valid_mask
    (B, H, W) bool, camera_intrinsics (B, 3, 3), camera_pose (B, 4, 4) (NaN when absent), true_shape (B, 2) int32
    (before the transpose), all on the device; portrait views are transposed to landscape.  No host synchronisation."""
    device = torch.device(device)
    _need_cuda(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    B = len(samples)
    if B == 0:
        raise ValueError("prepare_views needs at least one sample")
    N = len(samples[0])
    if N == 0 or any(len(s) != N for s in samples):
        raise ValueError("every sample must have the same number of views (at least one)")
    if rngs is not None and len(rngs) != B:
        raise ValueError(f"{len(rngs)} rngs for {B} samples")
    if plans is None:
        if resolution is None:
            raise ValueError("give a resolution or the plans")
        plans = [_plan_sample(s, resolution, None if rngs is None else rngs[b], aug_crop) for b, s in enumerate(samples)]
    if len(plans) != B or any(len(p) != N for p in plans):
        raise ValueError("plans must be B lists of N ViewPlan")
    tags = None if rngs is None else [[int.from_bytes(r.bytes(4), "big") for _ in range(N)] for r in rngs]

    # per-view output shapes (landscape) and offsets, laid out [view][item][pixel]
    shapes = []
    for n in range(N):
        hw = {p[n].shape for p in plans}
        land = {(min(h, w), max(h, w)) for h, w in hw}
        if len(land) != 1:
            raise ValueError(f"view {n}: the items' crops {sorted(hw)} do not collate to one landscape shape")
        shapes.append(land.pop())
    sizes = [h * w for h, w in shapes]
    total = B * sum(sizes)
    L.load()
    pts = torch.empty(total, 3, dtype=torch.float32, device=device)
    valid = torch.empty(total, dtype=torch.uint8, device=device)
    depth = torch.empty(total, dtype=torch.float32, device=device)
    imgs = [torch.empty(B, 3, h, w, dtype=torch.float32, device=device) for h, w in shapes]

    params = np.zeros(N * B, L.VIEW_PARAM)
    Ks = np.empty((N, B, 3, 3), np.float32)
    poses = np.empty((N, B, 4, 4), np.float32)
    true_shape = np.empty((N, B, 2), np.int32)
    keep = []  # the depth maps stay referenced until the launch that reads them is enqueued
    off = 0
    for n in range(N):
        for b in range(B):
            v, p = samples[b][n], plans[b][n]
            img = _on_device(v["img"], torch.uint8, device)
            dm = _on_device(v["depthmap"], torch.float32, device)
            sh, sw = img.shape[:2]
            if img.dim() != 3 or img.shape[2] != 3 or tuple(dm.shape) != (sh, sw):
                raise ValueError(f"view {n} of sample {b}: img must be (H, W, 3) and depthmap (H, W), got "
                                 f"{tuple(img.shape)} and {tuple(dm.shape)}")
            K = np.asarray(p.intrinsics, np.float32)
            if K[0, 1] != 0.0 or K[1, 0] != 0.0:
                raise AssertionError("camera intrinsics with skew")
            pose = v.get("camera_pose")
            pose = (np.full((4, 4), np.nan, np.float32) if pose is None else
                    np.asarray(pose.cpu().numpy() if torch.is_tensor(pose) else pose, np.float32))
            h, w = p.shape
            portrait = w < h
            l, t, r, bt = p.crop
            out = imgs[n][b]
            src = img[t:bt, l:r]
            if portrait:
                out.copy_(ingest.resize_crop_rgb8(src, p.size[0], p.size[1], p.filt, p.box).transpose(1, 2))
            else:
                ingest.resize_crop_rgb8(src, p.size[0], p.size[1], p.filt, p.box, out=out)
            rec = params[n * B + b]
            rec["depth"], rec["out_offset"], rec["src_w"], rec["src_h"] = dm.data_ptr(), off, sw, sh
            rec["crop_x"], rec["crop_y"], rec["crop_w"], rec["crop_h"] = l, t, r - l, bt - t
            rec["rs_w"], rec["rs_h"] = p.size
            rec["box_x"], rec["box_y"], rec["out_w"], rec["out_h"] = p.box[0], p.box[1], w, h
            rec["transpose"] = int(portrait)
            rec["k"] = (K[0, 0], K[1, 1], K[0, 2], K[1, 2])
            rec["pose"] = pose[:3, :4].reshape(-1)
            Ks[n, b] = K[[1, 0, 2]] if portrait else K
            poses[n, b] = pose
            true_shape[n, b] = (h, w)
            keep.append(dm)
            off += h * w
    ops.view_geometry(params, pts, valid, depth)
    small = _upload(np.concatenate([Ks.reshape(-1), poses.reshape(-1), true_shape.reshape(-1).view(np.float32)]),
                    device)
    nk, npo = Ks.size, poses.size
    Kd = small[:nk].view(N, B, 3, 3)
    Pd = small[nk:nk + npo].view(N, B, 4, 4)
    Td = small[nk + npo:].view(torch.int32).view(N, B, 2)
    tag_d = None if tags is None else _upload(np.array(tags, np.int64).T.copy(), device)

    res, start = [], 0
    for n, ((h, w), size) in enumerate(zip(shapes, sizes)):
        sl = slice(start, start + B * size)
        start += B * size
        view = dict(img=imgs[n], depthmap=depth[sl].view(B, h, w), camera_intrinsics=Kd[n], camera_pose=Pd[n],
                    pts3d=pts[sl].view(B, h, w, 3), valid_mask=valid[sl].view(torch.bool).view(B, h, w),
                    true_shape=Td[n])
        for k in samples[0][n]:
            if k not in _KEYS and k not in view:
                view[k] = torch.utils.data.default_collate([s[n][k] for s in samples])
        if tag_d is not None:
            view["rng"] = tag_d[n]
        res.append(view)
    return res
