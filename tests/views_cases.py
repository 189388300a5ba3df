"""Seeded raw views of the ground-truth view tests (tests/test_views_*.py) and of tools/make_golden_views.py, which runs
the reference's dataset pipeline on them and stores its outputs in tests/golden/views.pt.

A raw view is what a dataset loader hands to ``_crop_resize_if_necessary``: img uint8 (H, W, 3), depthmap float32
(H, W) in metres, camera_intrinsics float32 3x3, camera_pose float32 4x4 cam2world (absent when the case has no pose),
and dataset / label / instance strings."""
import numpy as np

# name: (kind, B, N, source (W, H), resolution, aug_crop, specials)
#   kind: "dataset" (BaseStereoViewDataset) or "re10k" (the RE10K benchmark's image-only crop, target (512, 288))
#   specials: pp = principal point (cx, cy) or None for the centre plus a little noise; no_pose; depth_specials (zeros,
#   negatives and a depth whose point overflows to inf); raises = the reference's AssertionError
CASES = {
    "sevenscenes_640x480": ("dataset", 1, 2, (640, 480), (512, 384), False, {}),
    "photo_1920x1440": ("dataset", 1, 1, (1920, 1440), (512, 384), False, {}),
    "photo_1600x1200": ("dataset", 1, 2, (1600, 1200), (512, 384), False, {}),
    "re10k_640x360": ("re10k", 1, 2, (640, 360), (512, 288), False, {}),
    "re10k_portrait_360x640": ("re10k", 1, 1, (360, 640), (512, 288), False, {}),
    "portrait_480x640": ("dataset", 1, 2, (480, 640), (512, 384), False, {}),
    "near_square_aug_crop": ("dataset", 2, 3, (500, 480), (512, 384), 16, {}),
    "near_square_square_res": ("dataset", 1, 2, (500, 480), (224, 224), False, {}),
    "upscale_320x240": ("dataset", 1, 2, (320, 240), (512, 384), False, {}),
    "margin_just_inside": ("dataset", 1, 1, (640, 480), (512, 384), False, dict(pp=(129, 240))),
    "margin_assert": ("dataset", 1, 1, (640, 480), (512, 384), False, dict(pp=(128, 240), raises=True)),
    "depth_specials": ("dataset", 1, 2, (640, 480), (512, 384), False, dict(depth_specials=True)),
    "missing_pose": ("dataset", 1, 2, (640, 480), (512, 384), False, dict(no_pose=True)),
    "batch2_mixed": ("dataset", 2, 2, (800, 600), (512, 384), False, {}),
    "exact_512x384": ("dataset", 1, 2, (512, 384), (512, 384), False, dict(pp=(256, 192))),
    "odd_resolution_500x375": ("dataset", 1, 1, (640, 480), (500, 375), False, {}),
}
OVERFLOW_DEPTH = np.float32(3e38)


def _rotation(rng):
    q = rng.standard_normal(4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def raw_view(rng, w, h, pp=None, pose=True, depth_specials=False):
    """One raw view of w x h: smooth colour gradients plus noise, a plane-and-bumps depth map, a pinhole camera with its
    principal point at `pp` (default: near the centre) and a random rigid pose."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([xx / w * 255, yy / h * 255, (xx + yy) / (w + h) * 255], -1)
    img = np.clip(base + rng.normal(0, 20, (h, w, 3)), 0, 255).astype(np.uint8)
    depth = (1.5 + 0.5 * np.sin(xx / 37.0) * np.cos(yy / 23.0) + rng.uniform(0, 0.05, (h, w))).astype(np.float32)
    if depth_specials:
        depth[: h // 8] = 0.0
        depth[h // 8: h // 4, : w // 3] = -1.0
        depth[h - 4:, :4] = OVERFLOW_DEPTH  # with the wide lens below, (u - cu) z / fu overflows to -inf here
        depth[h - 4:, w - 4:] = -OVERFLOW_DEPTH
    f = np.float32(max(w, h) * (0.3 if depth_specials else rng.uniform(0.8, 1.2)))
    cx, cy = pp if pp is not None else (w / 2 + rng.uniform(-3, 3), h / 2 + rng.uniform(-3, 3))
    K = np.array([[f, 0, cx], [0, f * np.float32(rng.uniform(0.98, 1.02)), cy], [0, 0, 1]], np.float32)
    v = dict(img=img, depthmap=depth, camera_intrinsics=K)
    if pose:
        T = np.eye(4)
        T[:3, :3] = _rotation(rng)
        T[:3, 3] = rng.normal(0, 2, 3)
        v["camera_pose"] = T.astype(np.float32)
    return v


def samples(name):
    """B lists of N raw views of case `name` (seeded by the name)."""
    kind, B, N, (w, h), res, aug, sp = CASES[name]
    rng = np.random.default_rng([ord(c) for c in name])
    out = []
    for b in range(B):
        views = []
        for n in range(N):
            v = raw_view(rng, w, h, sp.get("pp"), not sp.get("no_pose"), sp.get("depth_specials", False))
            v.update(dataset=name, label=f"scene{b}", instance=f"{n}")
            views.append(v)
        out.append(views)
    return out


def rng_seeds(name):
    """Seed of each sample's generator (the reference seeds one per item)."""
    return [1000 + 17 * b + len(name) for b in range(CASES[name][1])]
