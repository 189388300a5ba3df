"""Seeded inputs of the viewer-scene tests: procedural outdoor images (sky gradient, clouds, horizon, noisy ground),
images that reach each case of detect_sky_mask's selection rule, and preds shaped as the forward returns them after
align_local_pts3d_to_global."""
import numpy as np
import torch


def to_img(u8):
    """(H, W, 3) uint8 -> (H, W, 3) float32 in [-1, 1], as load_images normalises."""
    return ((u8.astype(np.float32) / 255.0 - 0.5) / 0.5).astype(np.float32)


def outdoor(rng, h, w, horizon=0.45, clouds=3):
    """Blue sky getting lighter towards a horizon, white clouds, green-brown ground with noise."""
    y = np.arange(h)[:, None] / max(h - 1, 1)
    x = np.arange(w)[None, :] / max(w - 1, 1)
    img = np.zeros((h, w, 3), np.float64)
    sky = y < horizon + 0.05 * np.sin(6 * x + rng.uniform(0, 6))
    t = np.clip(y / max(horizon, 1e-3), 0, 1)
    img[..., 0] = 60 + 120 * t
    img[..., 1] = 120 + 90 * t
    img[..., 2] = 235 - 10 * t
    for _ in range(clouds):
        cy, cx, r = rng.uniform(0, horizon), rng.uniform(0, 1), rng.uniform(0.03, 0.12)
        d = ((y - cy) / r) ** 2 + ((x - cx) / (1.6 * r)) ** 2
        img[d < 1] = 245
    ground = np.stack([90 + 40 * x + 0 * y, 110 - 30 * y + 0 * x, 50 + 0 * x * y], -1)
    img = np.where(sky[..., None], img, ground)
    img += rng.normal(0, 6, img.shape)
    return to_img(np.clip(img, 0, 255).astype(np.uint8))


def indoor(rng, h, w):
    """Warm, textured walls: no sky colour anywhere."""
    base = np.array([150, 110, 80], np.float64)
    img = base + rng.normal(0, 20, (h, w, 3))
    return to_img(np.clip(img, 0, 255).astype(np.uint8))


def flat(h, w, rgb):
    return to_img(np.broadcast_to(np.array(rgb, np.uint8), (h, w, 3)).copy())


SKY, WALL = (70, 130, 240), (150, 110, 80)


def quirk_images():
    """(name, image) reaching each case of the selection rule and the shape edge cases."""
    out = []
    im = flat(40, 40, WALL)
    im[20:30, 10:30] = to_img(np.array([[SKY]], np.uint8))
    out.append(("no_top", im))                                  # no component touches row 0: the whole mask is sky
    im = flat(60, 60, WALL)
    im[0:2, 0:2] = to_img(np.array([[SKY]], np.uint8))
    out.append(("top_small", im.copy()))                        # every row-0 component is small: nothing is sky
    diag = flat(40, 40, WALL)
    diag[3, 3] = diag[10, 10] = to_img(np.array([[SKY]], np.uint8))[0, 0]
    out.append(("diagonal", diag))  # two 7x7 squares meeting at one corner: 4-connectivity keeps the lower one apart
    out.append(("full_sky", flat(50, 70, SKY)))
    out.append(("empty", flat(30, 20, WALL)))
    rng = np.random.default_rng(7)
    for h, w in ((1, 5), (1, 1), (5, 3), (3, 9), (7, 9), (6, 6), (11, 13), (12, 5), (13, 40), (40, 33), (64, 96)):
        out.append((f"{h}x{w}", outdoor(rng, h, w)))
    return out


def all_triplets():
    """4096 x 4096 image holding every RGB triplet once (r, g, b) = (i >> 16, i >> 8, i) & 255 in raster order i."""
    i = np.arange(1 << 24, dtype=np.int64)
    u8 = np.stack([(i >> 16) & 255, (i >> 8) & 255, i & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    return to_img(u8)


def synth_output(seed, shapes, kinds=None):
    """{"views", "preds"} of len(shapes) frames (batch size 1), tie-free confidences 1 + exp(N(0, 1))."""
    rng = np.random.default_rng(seed)
    views, preds = [], []
    for i, (h, w) in enumerate(shapes):
        kind = (kinds or ["outdoor", "outdoor", "indoor"])[i % len(kinds or [0, 0, 0])]
        img = outdoor(rng, h, w) if kind == "outdoor" else indoor(rng, h, w)
        views.append({"img": torch.from_numpy(img).permute(2, 0, 1)[None].contiguous()})
        p = {}
        for pk, ck in (("pts3d_in_other_view", "conf"), ("pts3d_local_aligned_to_global", "conf_local")):
            p[pk] = torch.from_numpy(rng.normal(size=(1, h, w, 3)).astype(np.float32))
            p[ck] = torch.from_numpy((1 + np.exp(rng.normal(size=(1, h, w)))).astype(np.float32))
        p["pts3d_local"] = p["pts3d_local_aligned_to_global"]
        preds.append(p)
    return {"views": views, "preds": preds}


# viewer states: (timestep, p, mask_sky, show_global, show_local, drop_low, color); None = the launch default
def viewer_states(n):
    states = [(None, None, None, False, True, False, "rgb")]  # launch
    for t in (0, n // 2, n - 1):
        for p in (None, 0, 10, 65, 99.99, 100):
            states.append((t, p, True, False, True, False, "rgb"))
    for sky in (False, True):
        for g, l in ((True, False), (False, True), (True, True)):
            for drop in (False, True):
                for color in ("rgb", "view"):
                    states.append((n - 1, 10, sky, g, l, drop, color))
    return states
