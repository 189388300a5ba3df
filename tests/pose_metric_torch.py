"""The reference's relative-pose metric (fast3r/eval/cam_pose_metric.py camera_to_rel_deg / calculate_auc with
fast3r/utils/so3_utils.py so3_relative_angle) restated in plain torch ops, TEST AND MEASUREMENT INFRASTRUCTURE ONLY.
It runs wherever its inputs live: on the CPU it is the arithmetic the kernels reproduce (the CPU tests hold
csrc/pose_metric_math.h to it bit for bit before acos), on cuda it is what the reference computes when its evaluation
runs on the device (cuBLAS bmm, CUDA acosf).  ``errors`` also returns the intermediates the tests compare."""
import math

import torch

BOUND = 1.0 - 1e-4


def _inverse(se3):
    """closed_form_inverse: [R^T | -R^T t] over [0 0 0 1]."""
    rt = se3[:, :3, :3].transpose(1, 2)
    out = torch.zeros_like(se3)
    out[:, :3, :3] = rt
    out[:, :3, 3] = -torch.bmm(rt, se3[:, :3, 3:4])[..., 0]
    out[:, 3, 3] = 1.0
    return out


def _extrapolated_acos(x):
    """acos inside (-BOUND, BOUND), first-order Taylor lines at +-BOUND outside."""
    slope = -1.0 / math.sqrt(1.0 - BOUND * BOUND)
    hi, lo = x >= BOUND, x <= -BOUND
    out = torch.empty_like(x)
    mid = ~(hi | lo)
    out[mid] = torch.acos(x[mid])
    out[hi] = (x[hi] - BOUND) * slope + math.acos(BOUND)
    out[lo] = (x[lo] - (-BOUND)) * slope + math.acos(-BOUND)
    return out


def errors(pred, gt):
    """pred, gt (n, 4, 4) cam-to-world: dict of per-pair (torch.combinations order) trace, r (degrees), u (1 - loss, whose
    sqrt's acos is the translation angle), t (degrees), and `bad` (trace outside [-1 - 1e-4, 3 + 1e-4])."""
    n = pred.shape[0]
    i, j = torch.combinations(torch.arange(n), 2).unbind(-1)
    rel_g = _inverse(gt[i]).bmm(gt[j])
    rel_p = _inverse(pred[i]).bmm(pred[j])
    r12 = torch.bmm(rel_g[:, :3, :3], rel_p[:, :3, :3].permute(0, 2, 1))
    trace = r12[:, 0, 0] + r12[:, 1, 1] + r12[:, 2, 2]
    bad = (trace < -1.0 - 1e-4) | (trace > 3.0 + 1e-4)
    r = _extrapolated_acos((trace - 1.0) * 0.5) * 180 / math.pi
    tp, tg = rel_p[:, :3, 3], rel_g[:, :3, 3]
    up = tp / (torch.norm(tp, dim=1, keepdim=True) + 1e-15)
    ug = tg / (torch.norm(tg, dim=1, keepdim=True) + 1e-15)
    loss = torch.clamp_min(1.0 - torch.sum(up * ug, dim=1) ** 2, 1e-15)
    u = 1 - loss
    a = torch.acos(torch.sqrt(u))
    a[~torch.isfinite(a)] = 1e6
    t = a * 180.0 / math.pi
    return dict(trace=trace, r=r, u=u, t=t, bad=bad)


def metrics(r, t):
    """evaluate_camera_poses' seven numbers from the pair errors of one item."""
    out = {f"RRA_at_{tau}": (r < tau).float().mean().item() for tau in (5, 15, 30)}
    out.update({f"RTA_at_{tau}": (t < tau).float().mean().item() for tau in (5, 15, 30)})
    worst = torch.stack((r, t), dim=1).max(dim=1).values
    hist = torch.histc(worst, bins=31, min=0, max=30)
    out["mAA_30"] = torch.cumsum(hist / float(worst.shape[0]), dim=0).mean().item()
    return out


def counts(r, t, bad=None):
    """The counts row of f3r_pose_metric (lib.PM_COUNTS int64) from the pair errors of one item, on the host."""
    from fast3r_b200 import lib as L
    r, t = r.cpu(), t.cpu()
    row = torch.zeros(L.PM_COUNTS, dtype=torch.int64)
    for k, tau in enumerate((5, 15, 30)):
        row[k] = int((r < tau).sum())
        row[3 + k] = int((t < tau).sum())
    row[6] = 0 if bad is None else int(bad.sum())
    row[7] = r.numel()
    worst = torch.stack((r, t), dim=1).max(dim=1).values
    row[L.PM_HIST:L.PM_HIST + 31] = torch.histc(worst, bins=31, min=0, max=30).to(torch.int64)
    return row
