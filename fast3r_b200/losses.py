"""The validation criterion of Fast3R on the GPU, forward only: ``ConfLossMultiviewV2(Regr3DMultiviewV4(L21Loss()))``
of fast3r/dust3r/losses.py, which every config uses for training and validation::

    _target_: fast3r_b200.losses.ConfLossMultiviewV2
    pixel_loss: {_target_: fast3r_b200.losses.Regr3DMultiviewV4, criterion: {_target_: fast3r_b200.losses.L21Loss},
                 norm_mode: avg_dis}
    alpha: 0.2

Same constructors, ``get_name()`` / ``repr`` and results as the reference: ``criterion(views, preds)`` returns
``(loss, details)``, the loss a 0-dim float32 tensor on the preds' device (a python float when no view has a valid
pixel), the details the reference's keys in its order - ``Regr3DMultiviewV3_pts3d_loss_{global,local}/{i:02d}`` (NaN for
a view without valid pixels), then ``ConfLossMultiviewV2_conf_loss_{global,local}/{i:02d}`` (the int 0 for such a view).

The pixel maps are stacked once per call (views of different heights at one width are padded with invalid pixels) and
run through three kernels (csrc/val_loss.cu); the host reads one small array of float64 sums back - the call's one
synchronisation - and forms the means, the loss and the details from it.  Inputs may be on the host or a CUDA device;
there is no CPU path and no backward: an input that requires grad raises.

Supported: norm_mode "avg_dis" and "avg_log1p", gt_scale, local_scale_consistent.  Other norm modes, ``dist_clip`` and
``*`` / ``+`` composition raise ``NotImplementedError``; ``Regr3DMultiviewV4`` runs only as the pixel_loss of
``ConfLossMultiviewV2`` (the reference's own standalone call fails in ``Sum`` for two views or more).
"""
from __future__ import annotations

from copy import copy, deepcopy

import torch
import torch.nn as nn

from . import ops

NORM_MODES = ("avg_dis", "avg_log1p")


def _device(t: torch.Tensor) -> torch.device:
    """The compute device: the tensor's own CUDA device, else cuda:0."""
    if t.is_cuda:
        return t.device
    if not torch.cuda.is_available():
        raise RuntimeError("fast3r_b200.losses needs a CUDA device (there is no CPU path)")
    return torch.device("cuda:0")


class L21Loss(nn.Module):
    """Euclidean distance between 3d points: the criterion of Regr3DMultiviewV4 (not callable on its own here)."""

    def __init__(self, reduction="mean"):
        super().__init__()
        self.reduction = reduction

    def forward(self, a, b):
        raise NotImplementedError("fast3r_b200.losses.L21Loss runs only as the criterion of Regr3DMultiviewV4")


class MultiLoss(nn.Module):
    """The reference's MultiLoss naming; ``*`` and ``+`` composition are not supported."""

    def __init__(self):
        super().__init__()
        self._alpha = 1
        self._loss2 = None

    def get_name(self):
        raise NotImplementedError()

    def __mul__(self, alpha):
        raise NotImplementedError(f"{type(self).__name__}: scaling a loss (`*`) is not supported")

    __rmul__ = __mul__

    def __add__(self, loss2):
        raise NotImplementedError(f"{type(self).__name__}: composing losses (`+`) is not supported")

    def __repr__(self):
        return self.get_name()


class Regr3DMultiviewV4(MultiLoss):
    """Regression of the global and the local pointmaps, normalised over all views of an item (global) and per view
    (local); see the module docstring."""

    def __init__(self, criterion, norm_mode="avg_dis", gt_scale=False, local_scale_consistent=False):
        super().__init__()
        if not isinstance(criterion, L21Loss):
            raise NotImplementedError(f"Regr3DMultiviewV4: criterion {criterion!r} is not supported (only L21Loss)")
        if norm_mode not in NORM_MODES:
            raise NotImplementedError(f"Regr3DMultiviewV4: norm_mode {norm_mode!r} is not supported (only {NORM_MODES})")
        self.criterion = copy(criterion)
        self.norm_mode = norm_mode
        self.gt_scale = gt_scale
        self.local_scale_consistent = local_scale_consistent

    def get_name(self):
        return f"{type(self).__name__}({self.criterion})"

    def with_reduction(self, mode):
        res = deepcopy(self)
        res.criterion.reduction = "none"
        return res

    def forward(self, gts, preds, **kw):
        raise NotImplementedError("Regr3DMultiviewV4 runs only as the pixel_loss of ConfLossMultiviewV2")


class ConfLossMultiviewV2(MultiLoss):
    """Confidence-weighted regression loss of all views, normalised by the number of global and local terms."""

    def __init__(self, pixel_loss, alpha=1):
        super().__init__()
        if not alpha > 0:
            raise ValueError(f"ConfLossMultiviewV2: alpha must be positive, got {alpha}")
        if not isinstance(pixel_loss, Regr3DMultiviewV4):
            raise NotImplementedError(f"ConfLossMultiviewV2: pixel_loss {pixel_loss!r} is not supported "
                                      "(only Regr3DMultiviewV4)")
        self.alpha = alpha
        self.pixel_loss = pixel_loss.with_reduction("none")

    def get_name(self):
        return f"ConfLossMultiviewV2({self.pixel_loss})"

    def forward(self, gts, preds, dist_clip=None):
        if dist_clip is not None:
            raise NotImplementedError(f"ConfLossMultiviewV2: dist_clip={dist_clip!r} is not supported")
        p = self.pixel_loss
        sums = view_sums(gts, preds, self.alpha, p.norm_mode == "avg_log1p", p.gt_scale, p.local_scale_consistent)
        return loss_and_details(sums, "pts3d_local" in preds[0], preds[0]["pts3d_in_other_view"].device)


def view_sums(gts, preds, alpha, log1p=False, gt_scale=False, local_scale_consistent=False) -> torch.Tensor:
    """float64 (views, ops.VL_SUMS) on the host: per view, over the valid pixels of all items, the sums of the global
    and the local term's d and d c - alpha log c, and the number of valid pixels.  One launch sequence, one sync."""
    maps = stack_maps(gts, preds, _device(preds[0]["pts3d_in_other_view"]))
    sums = ops.val_loss(**maps, alpha=float(alpha), log1p=log1p, gt_scale=gt_scale,
                        local_scale_consistent=local_scale_consistent)
    return sums.cpu().sum(1)


def stack_maps(gts, preds, dev) -> dict:
    """The arguments of ops.val_loss: every map stacked [views, items, n] in float32 (valid in uint8) on `dev`; views
    of different heights at one width are padded with invalid pixels to the largest."""
    nv = len(gts)
    if nv == 0 or len(preds) != nv:
        raise ValueError(f"val_loss: {nv} views and {len(preds)} preds")
    has_local = "pts3d_local" in preds[0]
    keys = ("pts3d_in_other_view", "conf") + (("pts3d_local", "conf_local") if has_local else ())
    for gt, pred in zip(gts, preds):
        for t in (gt["pts3d"], gt["camera_pose"]) + tuple(pred[k] for k in keys):
            if t.requires_grad:
                raise RuntimeError("fast3r_b200.losses computes the loss value only (no backward); an input "
                                   "requires grad")
    items, _, width = gts[0]["pts3d"].shape[:3]
    heights = [gt["pts3d"].shape[1] for gt in gts]
    for gt in gts:
        if gt["pts3d"].shape[0] != items or gt["pts3d"].shape[2] != width:
            raise ValueError("val_loss: every view needs the same batch size and width, got pts3d shapes "
                             f"{[tuple(g['pts3d'].shape) for g in gts]}")
    n = max(heights) * width
    srcs = [("gt", gts, "pts3d", (3,)), ("valid", gts, "valid_mask", ()), ("pr", preds, "pts3d_in_other_view", (3,)),
            ("conf", preds, "conf", ())]
    if has_local:
        srcs += [("pr_local", preds, "pts3d_local", (3,)), ("conf_local", preds, "conf_local", ())]
    dtype = lambda name: torch.uint8 if name == "valid" else torch.float32  # noqa: E731
    out = dict(poses=torch.stack([gt["camera_pose"] for gt in gts]).to(device=dev, dtype=torch.float32).contiguous())
    if len(set(heights)) == 1:
        for name, ds, k, tail in srcs:
            out[name] = torch.stack([d[k].reshape(items, n, *tail) for d in ds]).to(device=dev, dtype=dtype(name))
        return out
    for name, ds, k, tail in srcs:
        out[name] = (torch.zeros if name == "valid" else torch.empty)(nv, items, n, *tail, dtype=dtype(name), device=dev)
        for v, d in enumerate(ds):
            m = heights[v] * width
            out[name][v, :, :m].copy_(d[k].reshape(items, m, *tail), non_blocking=True)
    return out


def loss_and_details(sums: torch.Tensor, has_local: bool, device):
    """The reference's (loss, details) from view_sums: float32 means, the int 0 for a view without valid pixels, and
    the float32 sum of the conf terms over their number (a python float when every term is the int 0)."""
    nv = sums.shape[0]
    count = sums[:, 4]
    means = (sums[:, :4] / count[:, None]).float()  # 0 / 0: NaN, as the mean of an empty tensor
    terms = ("global", "local") if has_local else ("global",)
    details, conf_details = {}, {}
    total = 0
    for t, term in enumerate(terms):
        for i in range(nv):
            details[f"Regr3DMultiviewV3_pts3d_loss_{term}/{i:02d}"] = float(means[i, 2 * t])
    for t, term in enumerate(terms):
        for i in range(nv):
            conf_loss = means[i, 2 * t + 1] if count[i] > 0 else 0
            conf_details[f"ConfLossMultiviewV2_conf_loss_{term}/{i:02d}"] = float(conf_loss)
            total += conf_loss
    total /= nv * len(terms)
    details.update(conf_details)
    return (total.to(device) if torch.is_tensor(total) else total), details
