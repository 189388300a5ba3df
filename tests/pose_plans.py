"""Launch keys of the camera-pose kernels (fast3r_b200/csrc/pose.cu), the table of GPU cases that
tests/test_pose_gpu.py runs and tests/test_pose_plans_cpu.py checks the fast3r_b200.poses callers against, and the
seeded pointmaps of the pose tests.

A call is a plain dict ("descriptor") with its kernel and the arguments that decide the code path:
    gather   views, n, mask                 (mask: a mask is passed instead of conf)
    score    views, nh, chunks, counts      (counts: the per-view point counts)
    inliers  rows, counts                   (counts: the point counts of the rows' views)
The key restates the launchers' rules (each function cites the lines it restates)."""
import numpy as np
import torch

CB = 1024      # elements per compaction block: pose.cu:23
STILE = 1024   # points per scoring CTA: pose.cu:26
SHB = 32       # hypotheses per scoring chunk: pose.cu:27
MAX_CHUNKS = 65535  # chunks per scoring launch (grid.y): pose.cu, launch_pnp_score


def _flags(*pairs):
    return "".join(" " + f for f, on in pairs if on)


def gather_key(d):
    """pose.cu launch_pnp_gather: the mask or conf selection; a partial last block when n % 1024 != 0; one block per
    view when n <= 1024."""
    return "gather" + _flags(("mask", d["mask"]), ("tail", d["n"] % CB != 0), ("multiblock", d["n"] > CB))


def score_key(d):
    """pose.cu launch_pnp_score: more than one launch past 65535 chunks; a view with no points; views of different
    counts (CTAs past a view's tiles exit); a partial last tile."""
    counts = d["counts"]
    return "score" + _flags(("multilaunch", d["chunks"] > MAX_CHUNKS), ("empty", min(counts) == 0),
                            ("ragged", len(set(counts)) > 1), ("tail", any(c % STILE for c in counts)))


def inliers_key(d):
    """pose.cu launch_pnp_inliers: rows of different counts, a row of no points, partial last block."""
    counts = d["counts"]
    return "inliers" + _flags(("empty", min(counts) == 0), ("ragged", len(set(counts)) > 1),
                              ("tail", any(c % CB for c in counts)))


KEYS = dict(gather=gather_key, score=score_key, inliers=inliers_key)


def key(d):
    return KEYS[d["op"]](d)


def chunks_of(views_of_rows):
    """Chunks the launcher forms: runs of at most SHB consecutive rows of one view."""
    n, prev, run = 0, None, 0
    for v in views_of_rows:
        if v != prev or run == SHB:
            n, prev, run = n + 1, v, 0
        run += 1
    return n


# ------------------------------------------------------------------------------------------------------ the case table
LAND = (368, 512)
# gather: (name, views, H, W, mask, fraction selected (None: conf from a seeded lognormal))
GATHER = [
    ("g_land_v32_conf", 32, 368, 512, False, None),
    ("g_land_v2_mask", 2, 368, 512, True, 0.7),
    ("g_small_conf", 3, 17, 29, False, None),
    ("g_one_block_mask", 2, 16, 64, True, 0.5),
    ("g_1x1_mask", 2, 1, 1, True, 0.5),
    ("g_tail_conf_none", 3, 33, 33, False, 0.0),
]
# score / inliers: (name, view counts, hypotheses per view, interleave the views' rows)
SCORE = [
    ("s_land_v32_h10", [188416] * 32, 10, False),
    ("s_land_ragged_v32_h10", [169000 + 37 * k for k in range(32)], 10, False),
    ("s_ragged_empty", [0, 1, 1023, 1025, 5000], 40, False),
    ("s_one_view", [777], 3, False),
    ("s_interleaved_multilaunch", [7, 3], 32800, True),
]
INLIERS = [
    ("i_land_v32", [188416] * 32),
    ("i_land_ragged_v32", [169000 + 37 * k for k in range(32)]),
    ("i_one_tail", [777]),
    ("i_ragged_empty", [0, 1, 1023, 1025, 5000]),
    ("i_same", [4096, 4096]),
]


def gather_desc(c):
    return dict(op="gather", views=c[1], n=c[2] * c[3], mask=c[4])


def score_desc(c):
    views = len(c[1])
    rows = [v for _ in range(c[2]) for v in range(views)] if c[3] else [v for v in range(views) for _ in range(c[2])]
    return dict(op="score", views=views, nh=len(rows), chunks=chunks_of(rows), counts=list(c[1]))


def inliers_desc(c):
    return dict(op="inliers", rows=len(c[1]), counts=list(c[1]))


CASES = ([dict(name=c[0], key=gather_key(gather_desc(c)), **gather_desc(c)) for c in GATHER]
         + [dict(name=c[0], key=score_key(score_desc(c)), **score_desc(c)) for c in SCORE]
         + [dict(name=c[0], key=inliers_key(inliers_desc(c)), **inliers_desc(c)) for c in INLIERS])


# ------------------------------------------------------------------------------------------------ seeded pointmaps
def random_pose(g):
    """(R, t) float64: a uniformly random rotation and a N(0, 1) translation."""
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    if torch.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return q, torch.randn(3, generator=g, dtype=torch.float64)


def synth_view(g, h, w, focal, outliers, noise_px=0.0, planar=False, pose=None):
    """A pointmap of known pose: pixel (x, y) at depth z back-projected with `focal` about the image centre, in the
    camera's own frame (pose None) or moved into the frame in which the camera has pose = (R, t) (world-to-camera,
    cam = R world + t); a fraction `outliers` of the points is displaced; the confidence is 1 + exp(N(0, 1)) with a
    tenth of the pixels at or below 1 (masked out by conf > 1)."""
    v, u = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    z = torch.full((h, w), 2.0, dtype=torch.float64) if planar else 1.5 + 2.0 * torch.rand(h, w, generator=g, dtype=torch.float64)
    uu = u + noise_px * torch.randn(h, w, generator=g, dtype=torch.float64)
    vv = v + noise_px * torch.randn(h, w, generator=g, dtype=torch.float64)
    world = torch.stack([(uu - w / 2) * z / focal, (vv - h / 2) * z / focal, z], -1)
    if pose is not None:
        world = (world - pose[1]) @ pose[0]
    out = torch.rand(h, w, generator=g) < outliers
    world[out] += 2.0 * torch.randn(int(out.sum()), 3, generator=g, dtype=torch.float64)
    conf = 1 + torch.exp(torch.randn(h, w, generator=g))
    conf[torch.rand(h, w, generator=g) < 0.1] = 1.0
    return world.float(), conf


def synth_preds(seed, views, batch, h, w, outliers=(0.0, 0.3, 0.9), noise_px=1.0):
    """preds as inference() returns them: pts3d_in_other_view and pts3d_local_aligned_to_global in the frame of view 0's
    camera (so view 0's pointmaps are camera-frame pointmaps, as the forward's are, and the first-view focal modes find
    the focal), conf and conf_local.  Every other view has a random pose; its local pointmap has the same pose, its own
    noise and no outliers; the global pointmaps' outlier fractions cycle through `outliers`."""
    g = torch.Generator().manual_seed(seed)
    preds = []
    for k in range(views):
        poses = [None if k == 0 else random_pose(g) for _ in range(batch)]
        pv = [synth_view(g, h, w, 0.9 * max(h, w), outliers[k % len(outliers)], noise_px, pose=p) for p in poses]
        pl = [synth_view(g, h, w, 0.9 * max(h, w), 0.0, noise_px, pose=p) for p in poses]
        preds.append(dict(pts3d_in_other_view=torch.stack([p[0] for p in pv]), conf=torch.stack([p[1] for p in pv]),
                          pts3d_local_aligned_to_global=torch.stack([p[0] for p in pl]),
                          conf_local=torch.stack([p[1] for p in pl])))
    return preds


def threshold_view(seed, h, w, focal):
    """(points fp32 (h w, 3), pixels fp32 (h w, 2)) of a view whose errors pile up at the threshold: 40 % of the points
    are back-projected from their pixel moved by (3, 4) in one of four directions (error 25 = 5^2 under the true pose),
    20 % are displaced outliers, the rest exact.  Under a near-exact hypothesis the errors of the moved points spread
    over about 1e-4 around 25, so the rounding of the error decides some of them."""
    rs = np.random.default_rng(seed)
    pix = np.mgrid[:w, :h].T.reshape(-1, 2).astype(np.float64)
    z = rs.uniform(1.5, 3.5, len(pix))
    off = np.zeros_like(pix)
    ring = rs.random(len(pix)) < 0.4
    off[ring] = np.array([(3, 4), (-3, 4), (4, -3), (-4, -3)], float)[rs.choice(4, int(ring.sum()))]
    src = pix + off
    cam = np.stack([(src[:, 0] - w / 2) * z / focal, (src[:, 1] - h / 2) * z / focal, z], 1)
    q, _ = np.linalg.qr(rs.normal(size=(3, 3)))
    q *= np.sign(np.linalg.det(q))
    world = (cam - rs.normal(size=3)) @ q
    out = rs.random(len(pix)) < 0.2
    world[out] += 2 * rs.normal(size=(int(out.sum()), 3))
    return world.astype(np.float32), pix.astype(np.float32)
