"""The camera-pose metric of Fast3R's pose evaluation on the GPU.  Same names, arguments and results as the reference,
down to the dtypes:

* ``camera_to_rel_deg(pred_cameras_c2w, gt_cameras_c2w, device, batch_size)`` - fast3r/eval/cam_pose_metric.py:17-38:
  the rotation and translation angles in degrees of every view pair (i < j, torch.combinations order) of the first
  ``batch_size`` views, as two (P,) tensors of the poses' dtype on the poses' device.
* ``calculate_auc(r_error, t_error, max_threshold=30)`` - cam_pose_metric.py:72-98: mAA, a 0-dim tensor of the errors'
  promoted dtype (float32 or float64); max_threshold from 1 to 63 (the reference takes any).

All pairs go through one kernel (csrc/pose_metric.cu) in the reference's CPU arithmetic (csrc/pose_metric_math.h):
every quantity before acos is bit-equal to what torch computes on the CPU, and acos is restated from basic IEEE
operations, within a few ulp of torch's.  The kernel reduces the angles to exact integer counts; the histogram's
normalisation, cumsum and mean run on the host as the reference's torch ops on those counts.  Inputs may be on the host
or a CUDA device; there is no CPU path.  ``evaluate_camera_poses`` (fast3r_b200.postprocess) is the caller that scores
a whole batch in one launch.
"""
from __future__ import annotations

import torch

from . import lib as L
from . import ops

RRA_THRESHOLDS = (5, 15, 30)
RTA_THRESHOLDS = (5, 15, 30)
TRACE_ERROR = "A matrix has trace outside valid range [-1-eps,3+eps]."


def _cuda(t: torch.Tensor, device=None) -> torch.device:
    if t.is_cuda:
        return t.device
    if device is not None and torch.device(device).type == "cuda":
        return torch.device(device)
    if not torch.cuda.is_available():
        raise RuntimeError("fast3r_b200.cam_pose_metric needs a CUDA device (there is no CPU path)")
    return torch.device("cuda:0")


def pose_counts(pred: torch.Tensor, gt: torch.Tensor, device=None, angles: bool = False):
    """pred, gt (items, views, 4, 4) of one dtype, views >= 2: (counts int64 (items, lib.PM_COUNTS) on the host, r, t)
    from one launch (r, t: (items, P) angles on the compute device with `angles`, else None).  Raises the reference's
    ValueError when a pair's trace is out of range."""
    if pred.dtype != gt.dtype:
        raise TypeError(f"pred and gt poses have different dtypes: {pred.dtype} and {gt.dtype}")
    dev = _cuda(pred, device)
    counts, r, t = ops.pose_metric(pred.to(dev).contiguous(), gt.to(dev).contiguous(), angles=angles)
    counts = counts.cpu()
    if bool((counts[:, 6] > 0).any()):
        raise ValueError(TRACE_ERROR)
    return counts, r, t


def below_ratio(count: int, pairs: int) -> float:
    """(x < tau).float().mean().item() for a (pairs,) tensor x with `count` elements below tau."""
    return float(torch.tensor(count, dtype=torch.float32) / pairs)


def auc_from_hist(hist: torch.Tensor, pairs: int) -> torch.Tensor:
    """calculate_auc's tail on the histogram counts (as a tensor of the errors' dtype): normalise, cumsum, mean."""
    return torch.cumsum(hist / float(pairs), dim=0).mean()


def camera_to_rel_deg(pred_cameras_c2w, gt_cameras_c2w, device, batch_size):
    n = int(batch_size)
    if n > pred_cameras_c2w.shape[0] or n > gt_cameras_c2w.shape[0]:
        raise IndexError(f"batch_size {n} exceeds the {min(pred_cameras_c2w.shape[0], gt_cameras_c2w.shape[0])} poses")
    src = pred_cameras_c2w.device
    if n < 2:  # no pair
        empty = torch.empty(0, dtype=pred_cameras_c2w.dtype, device=src)
        return empty, empty.clone()
    _, r, t = pose_counts(pred_cameras_c2w[None, :n], gt_cameras_c2w[None, :n], device, angles=True)
    return r[0].to(src), t[0].to(src)


def calculate_auc(r_error, t_error, max_threshold=30):
    dtype = torch.promote_types(r_error.dtype, t_error.dtype)  # as torch.stack((r_error, t_error)) promotes
    if dtype not in (torch.float32, torch.float64):
        raise TypeError(f"calculate_auc: errors must be float32 or float64, got {r_error.dtype} and {t_error.dtype}")
    if not 1 <= int(max_threshold) < L.PM_MAX_BINS:
        raise ValueError(f"max_threshold {max_threshold} not in [1, {L.PM_MAX_BINS})")
    dev = _cuda(r_error)
    r = r_error.to(device=dev, dtype=dtype).contiguous().reshape(-1)
    t = t_error.to(device=dev, dtype=dtype).contiguous().reshape(-1)
    counts = ops.pose_metric_counts(r, t, hist_max=int(max_threshold)).cpu()
    hist = counts[L.PM_HIST:L.PM_HIST + int(max_threshold) + 1].to(dtype)
    return auc_from_hist(hist, r_error.shape[0]).to(r_error.device)
