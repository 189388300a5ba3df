"""Seeded inputs of the camera-pose metric tests (tests/test_pose_metric_cpu.py, tests/test_pose_metric_gpu.py) and of
tools/make_golden_pose_metrics.py, which stores the reference's outputs for them in tests/golden/pose_metrics.pt.

* ``pose_set(n, dtype, seed)``: (pred, gt) cam-to-world poses (n, 4, 4) with every quirk of the reference's metric: a
  prediction equal to the ground truth (0.4046 degrees, from the linear extrapolation of acos), two views at one place
  (a zero relative translation: 90 degrees), a NaN translation (1e6 before the conversion to degrees), a NaN rotation
  (fails every threshold, dropped by histc), and errors spread over [0, 60] degrees.
* ``eval_inputs(name)``: (views, preds) as a validation batch and inference() give them: ground-truth camera_pose and
  true_shape per view, pointmaps of tests/pose_plans.synth_view in view 0's camera frame; "b2_v4" has a portrait item.
"""
import torch

from tests import pose_plans as PP

POSE_SIZES = (2, 3, 10, 32, 320, 1000)
ANGLE_SIZES = (2, 3, 10, 32)  # the goldens keep the per-pair angles of these
# every focal mode; in the first-view modes the tests hand estimate_camera_poses the focal the reference solved with
# (stored in the goldens), as the GPU estimate_focal is within 1e-3 of the reference's, not bit-equal
MODES = ("individual", "first_view_from_global_head", "first_view_from_local_head")
EVAL_RUNS = {"b2_v4": [(m, n) for m in MODES for n in (10, 100)], "b1_v8": [(m, 10) for m in MODES]}


def _rotation(g, n, scale=None):
    """n rotations (float64): uniform, or of angle ~ scale * |N(0, 1)| radians about a random axis."""
    if scale is None:
        q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    else:
        axis = torch.randn(n, 3, generator=g, dtype=torch.float64)
        axis = axis / axis.norm(dim=1, keepdim=True)
        half = 0.5 * scale * torch.randn(n, generator=g, dtype=torch.float64).abs()
        q = torch.cat([torch.cos(half)[:, None], torch.sin(half)[:, None] * axis], 1)
    q = q / q.norm(dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                        2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                        2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).view(n, 3, 3)


def _se3(R, t):
    P = torch.eye(4, dtype=torch.float64).repeat(R.shape[0], 1, 1)
    P[:, :3, :3], P[:, :3, 3] = R, t
    return P


def pose_set(n, dtype=torch.float32, seed=0):
    g = torch.Generator().manual_seed(1000 * n + seed)
    gt = _se3(_rotation(g, n), 3 * torch.randn(n, 3, generator=g, dtype=torch.float64))
    dR = _rotation(g, n, scale=0.35)
    pred = _se3(dR @ gt[:, :3, :3], gt[:, :3, 3] + 0.4 * torch.randn(n, 3, generator=g, dtype=torch.float64))
    pred, gt = pred.to(dtype), gt.to(dtype)
    if n >= 3:
        pred[1] = gt[1]                   # equal rotations for the pairs of views 0 and 1 ... where view 0 is right too
        pred[0] = gt[0]
        gt[2, :3, 3] = gt[0, :3, 3]       # views 0 and 2 at one place: zero relative translation
    if n >= 10:
        pred[5, 1, 3] = float("nan")      # NaN translation
        pred[7, 0, 0] = float("nan")      # NaN rotation (and with it a NaN translation)
    return pred.contiguous(), gt.contiguous()


def eval_inputs(name):
    """(views, preds): ``b2_v4`` = 2 items x 4 views of 96x128, item 1 a portrait scene of 128x96 stored transposed to
    landscape as the data loader stores it (true_shape (128, 96)); ``b1_v8`` = 1 item x 8 views of 64x96.  Preds hold
    both heads (pts3d_in_other_view / conf and pts3d_local / conf_local, all in view 0's camera frame, the local head
    without outliers); camera_pose is float32 cam-to-world, view 0 of each item the world frame."""
    batch, nv, h, w = {"b2_v4": (2, 4, 96, 128), "b1_v8": (1, 8, 64, 96)}[name]
    portrait = [name == "b2_v4" and i == 1 for i in range(batch)]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    views, preds = [], []
    for k in range(nv):
        poses = [None if k == 0 else PP.random_pose(g) for _ in range(batch)]
        heads = []
        for outliers in ((0.0, 0.3)[k % 2], 0.0):
            pts, conf = [], []
            for i, p in enumerate(poses):
                hh, ww = (w, h) if portrait[i] else (h, w)      # the scene's true shape
                x, c = PP.synth_view(g, hh, ww, 0.9 * max(h, w), outliers, 1.0, pose=p)
                pts.append(x.transpose(0, 1) if portrait[i] else x)
                conf.append(c.transpose(0, 1) if portrait[i] else c)
            heads.append((torch.stack(pts).contiguous(), torch.stack(conf).contiguous()))
        c2w = torch.stack([torch.eye(4, dtype=torch.float64) if p is None else
                           torch.linalg.inv(_se3(p[0][None], p[1][None])[0]) for p in poses]).float()
        shape = torch.tensor([[w, h] if portrait[i] else [h, w] for i in range(batch)])
        views.append(dict(img=torch.zeros(batch, 3, h, w), true_shape=shape, camera_pose=c2w))
        preds.append(dict(pts3d_in_other_view=heads[0][0], conf=heads[0][1], pts3d_local=heads[1][0],
                          conf_local=heads[1][1]))
    return views, preds
