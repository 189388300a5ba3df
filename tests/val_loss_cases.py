"""Seeded inputs of the validation-criterion tests (tests/test_val_loss_*.py) and of tools/make_golden_val_loss.py, which
stores the reference's (loss, details) for them in tests/golden/val_loss.pt.

``inputs(name)`` gives (views, preds) as a validation batch and the forward give them: per view camera_pose (B, 4, 4),
pts3d (B, H, W, 3) in world coordinates and valid_mask (B, H, W); per pred pts3d_in_other_view near the ground truth in
view 0's frame, conf > 1, and with the local head pts3d_local near the ground truth in the view's own frame and
conf_local.  The predictions are the ground truth at another scale plus noise, so the losses are of the size a trained
model gives."""
import torch

# name: (B, N, H, W, local head, criterion keywords, specials); specials:
#   empty_view   view 1 has no valid pixel           empty_item   item 1 has no valid pixel in any view
#   all_invalid  no valid pixel at all (the reference returns a python float)
#   nan / inf    NaN and +-inf predictions at valid pixels
#   scaled       camera poses with a scale (not rigid)     heights      per-view heights at one width
CASES = {
    "b1_n1_64x96": (1, 1, 64, 96, True, {}, {}),
    "b2_n2_64x96": (2, 2, 64, 96, True, {}, {}),
    "b1_n8_64x96_global": (1, 8, 64, 96, False, {}, {}),
    "b2_n8_368x512": (2, 8, 368, 512, True, {}, {}),
    "b1_n2_368x512_global": (1, 2, 368, 512, False, {}, {}),
    "b2_n2_log1p": (2, 2, 64, 96, True, dict(norm_mode="avg_log1p"), {}),
    "b2_n2_gt_scale": (2, 2, 64, 96, True, dict(gt_scale=True), {}),
    "b2_n2_lsc": (2, 2, 64, 96, True, dict(local_scale_consistent=True), {}),
    "b2_n2_lsc_gt_scale_log1p": (2, 2, 64, 96, True, dict(local_scale_consistent=True, gt_scale=True,
                                                          norm_mode="avg_log1p"), {}),
    "b2_n3_empty_view": (2, 3, 64, 96, True, {}, dict(empty_view=True)),
    "b2_n2_empty_item": (2, 2, 64, 96, True, {}, dict(empty_item=True)),
    "b1_n2_all_invalid": (1, 2, 64, 96, True, {}, dict(all_invalid=True)),
    "b2_n2_all_invalid_global": (2, 2, 64, 96, False, {}, dict(all_invalid=True)),
    "b2_n3_nan": (2, 3, 64, 96, True, {}, dict(nan=True)),
    "b2_n2_inf": (2, 2, 64, 96, True, {}, dict(inf=True)),
    "b2_n3_scaled": (2, 3, 64, 96, True, {}, dict(scaled=True)),
    "b2_n3_heights": (2, 3, 64, 96, True, {}, dict(heights=(64, 48, 80))),
    "b1_n2_heights_global": (1, 2, 64, 96, False, {}, dict(heights=(32, 64))),
}
ALPHA = 0.2  # every config's alpha


def _rotation(g, n):
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    q = q / q.norm(dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                        2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                        2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).view(n, 3, 3)


def _apply(T, x):
    return torch.einsum("bij,bhwj->bhwi", T[:, :3, :3], x) + T[:, None, None, :3, 3]


def make(B, N, H, W, local=True, specials=None, seed=0):
    """(views, preds) of B items of N views; see the module docstring."""
    sp = specials or {}
    g = torch.Generator().manual_seed(seed)
    heights = sp.get("heights") or (H,) * N
    views, preds = [], []
    pose0 = None
    for i in range(N):
        h = heights[i]
        pose = torch.eye(4, dtype=torch.float64).repeat(B, 1, 1)
        pose[:, :3, :3] = _rotation(g, B)
        if sp.get("scaled"):
            pose[:, :3, :3] *= (0.5 + torch.rand(B, 1, 1, generator=g, dtype=torch.float64) * 2)
        pose[:, :3, 3] = torch.randn(B, 3, generator=g, dtype=torch.float64) * 3
        pose0 = pose if i == 0 else pose0
        cam = torch.randn(B, h, W, 3, generator=g, dtype=torch.float64) * 0.7
        cam[..., 2] = cam[..., 2].abs() + 2  # in front of the camera
        world = _apply(pose, cam)
        valid = torch.rand(B, h, W, generator=g) > 0.3
        in0 = _apply(torch.linalg.inv(pose0), world)
        noise = lambda: 0.05 * torch.randn(B, h, W, 3, generator=g, dtype=torch.float64)  # noqa: E731
        view = dict(camera_pose=pose.float(), pts3d=world.float(), valid_mask=valid)
        pred = dict(pts3d_in_other_view=(in0 * 0.3 + noise()).float(),
                    conf=(1 + torch.randn(B, h, W, generator=g).exp()))
        if local:
            pred["pts3d_local"] = (cam * 0.7 + noise()).float()
            pred["conf_local"] = 1 + torch.randn(B, h, W, generator=g).exp()
        views.append(view)
        preds.append(pred)
    if sp.get("empty_view"):
        views[1]["valid_mask"][:] = False
    if sp.get("empty_item"):
        for v in views:
            v["valid_mask"][1] = False
    if sp.get("all_invalid"):
        for v in views:
            v["valid_mask"][:] = False
    if sp.get("nan"):
        preds[1]["pts3d_in_other_view"][0, 3, 5, 1] = float("nan")  # skipped by item 0's factor, view 1 becomes NaN
        views[1]["valid_mask"][0, 3, 5] = True
        if "pts3d_local" in preds[2]:
            preds[2]["pts3d_local"][1, 7, 9] = float("nan")
            views[2]["valid_mask"][1, 7, 9] = True
    if sp.get("inf"):
        preds[0]["pts3d_in_other_view"][1, 2, 3, 0] = float("inf")  # item 1's factor becomes inf
        views[0]["valid_mask"][1, 2, 3] = True
        preds[1]["pts3d_local"][0, 4, 4, 2] = -float("inf")
        views[1]["valid_mask"][0, 4, 4] = True
    return views, preds


def inputs(name):
    B, N, H, W, local, _, sp = CASES[name]
    return make(B, N, H, W, local, sp, seed=sorted(CASES).index(name))


def criterion_kw(name):
    return CASES[name][5]
