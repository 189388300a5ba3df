"""Host restatement of the datasets' view pipeline with PIL, cv2 and numpy, TEST / MEASUREMENT INFRASTRUCTURE ONLY:
the checker of fast3r_b200.views.prepare_views on random inputs (tests/test_views_gpu.py) and the host arm of
tools/view_rates.py.  The geometry is fast3r_b200.views.plan_view (pinned bit for bit to the reference's goldens by
tests/test_views_cpu.py); every pixel is computed as the reference computes it: Pillow's crop and resize, ToTensor +
Normalize in float32, cv2.resize(INTER_NEAREST) of the depth map, the unprojection with numpy's float64 promotion and
np.einsum, the validity mask and the landscape transpose."""
import numpy as np
import PIL.Image
import torch


def host_view(raw, plan):
    """One view dict (numpy) from a raw view and its ViewPlan, as __getitem__ leaves it before collation."""
    import cv2
    l, t, r, b = plan.crop
    bl, bt, br, bb = plan.box
    im = PIL.Image.fromarray(np.asarray(raw["img"])).crop(plan.crop)
    im = im.resize(plan.size, PIL.Image.LANCZOS if plan.filt == 1 else PIL.Image.BICUBIC).crop(plan.box)
    img = ((np.asarray(im).astype(np.float32) / np.float32(255) - 0.5) / 0.5).transpose(2, 0, 1)
    depth = cv2.resize(np.ascontiguousarray(raw["depthmap"][t:b, l:r]), plan.size,
                       interpolation=cv2.INTER_NEAREST)[bt:bb, bl:br]
    K = plan.intrinsics
    pose = raw.get("camera_pose")
    pose = np.full((4, 4), np.nan, np.float32) if pose is None else np.asarray(pose, np.float32)
    H, W = depth.shape
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    with np.errstate(over="ignore", invalid="ignore"):
        cam = np.stack(((u - K[0, 2]) * depth / K[0, 0], (v - K[1, 2]) * depth / K[1, 1], depth), -1).astype(np.float32)
        pts = np.einsum("ik, vuk -> vui", pose[:3, :3], cam) + pose[:3, 3][None, None, :]
    valid = (depth > 0.0) & np.isfinite(pts).all(-1)
    view = dict(img=img, depthmap=depth, pts3d=pts, valid_mask=valid, camera_intrinsics=K, camera_pose=pose,
                true_shape=np.int32((H, W)))
    if W < H:
        view.update(img=img.swapaxes(1, 2), depthmap=depth.swapaxes(0, 1), pts3d=pts.swapaxes(0, 1),
                    valid_mask=valid.swapaxes(0, 1), camera_intrinsics=K[[1, 0, 2]])
    return view


def host_views(samples, plans, tags=None):
    """The collated views (CPU tensors) of B samples of N raw views with their plans; tags[b][n] become ``rng``."""
    items = []
    for b, (raw, ps) in enumerate(zip(samples, plans)):
        vs = []
        for n, (v, p) in enumerate(zip(raw, ps)):
            view = host_view(v, p)
            view.update({k: x for k, x in v.items() if k not in ("img", "depthmap", "camera_intrinsics", "camera_pose")})
            if tags is not None:
                view["rng"] = tags[b][n]
            vs.append(view)
        items.append(vs)
    return torch.utils.data.default_collate(items)
