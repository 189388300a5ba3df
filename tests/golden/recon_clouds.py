"""Seeded point clouds for the reconstruction-metric fixtures (tests/golden/recon_metric.json,
tools/make_golden_recon_metric.py): each case is a ground-truth and a reconstructed cloud, optionally with normals, of
the shapes these metrics see - uniform volumes, depth-map surfaces, tight clusters next to far outliers, exact
duplicates, collinear sets, single points."""
import numpy as np


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _surface(rng, views, h, w):
    """Depth-map-like cloud: `views` pinhole back-projections of a smooth wavy surface, fp32."""
    pts = []
    for _ in range(views):
        u, v = np.meshgrid(np.linspace(-1, 1, w), np.linspace(-0.75, 0.75, h))
        z = 2.0 + 0.2 * np.sin(3 * u + rng.uniform(0, 6)) * np.cos(2 * v) + 0.01 * rng.standard_normal(u.shape)
        p = np.stack([u * z, v * z, z], -1).reshape(-1, 3)
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)) * 0.1 + np.eye(3))
        pts.append(p @ q.T + rng.standard_normal(3) * 0.2)
    return np.concatenate(pts).astype(np.float32)


def make_case(kind: str, seed: int):
    """(gt, rec, gt_normals, rec_normals) of one fixture; normals are None unless the kind asks for them."""
    rng = np.random.default_rng(seed)
    gn = rn = None
    if kind == "uniform":
        gt = rng.random((20000, 3))
        rec = rng.random((15000, 3)).astype(np.float32)
    elif kind == "surface":
        gt = _surface(rng, 4, 48, 64)
        rec = (gt[rng.permutation(len(gt))[:9000]] + 0.003 * rng.standard_normal((9000, 3))).astype(np.float32)
    elif kind == "outliers":
        centres = rng.standard_normal((5, 3))
        gt = (centres[rng.integers(0, 5, 12000)] + 0.01 * rng.standard_normal((12000, 3)))
        gt[rng.permutation(12000)[:120]] = rng.choice([-1e6, 1e6], (120, 3)) + rng.standard_normal((120, 3))
        rec = (centres[rng.integers(0, 5, 8000)] + 0.012 * rng.standard_normal((8000, 3)))
        rec[:40] = rng.choice([-1e6, 1e6], (40, 3))
    elif kind == "duplicates":
        base = rng.random((300, 3)).astype(np.float32)
        gt = base[rng.integers(0, 300, 9000)]
        rec = np.concatenate([base[rng.integers(0, 300, 3000)], rng.random((3000, 3)).astype(np.float32)])
    elif kind == "collinear":
        d = np.array([1.0, 2.0, -0.5])
        gt = np.outer(rng.uniform(-3, 3, 10000), d) + np.array([0.5, -1.0, 2.0])
        rec = np.outer(rng.uniform(-3.5, 3.5, 7000), d) + np.array([0.5, -1.0, 2.0]) + 1e-3 * rng.standard_normal((7000, 3))
    elif kind == "one_gt":
        gt = rng.random((1, 3))
        rec = rng.random((500, 3))
    elif kind == "one_rec":
        gt = rng.random((700, 3)).astype(np.float32)
        rec = rng.random((1, 3)).astype(np.float32)
    elif kind == "normals":
        gt = _surface(rng, 2, 40, 50).astype(np.float64)
        rec = gt[rng.permutation(len(gt))[:3000]] + 0.002 * rng.standard_normal((3000, 3))
        gn = _unit(rng.standard_normal(gt.shape))
        rn = _unit(rng.standard_normal(rec.shape))
    else:
        raise ValueError(kind)
    return gt, rec, gn, rn


CASES = [("uniform", 11), ("surface", 12), ("outliers", 13), ("duplicates", 14), ("collinear", 15), ("one_gt", 16),
         ("one_rec", 17), ("normals", 18)]
