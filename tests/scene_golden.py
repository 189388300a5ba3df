"""The reference viewer's goldens (tests/golden/scene.pt, made by tools/make_golden_scene.py) and the check of a
fast3r_b200.scene.Scene against them: frame arrays, sky masks, is_outdoor, max_extent, and the PLY bytes of the launch
state and of every replayed action."""
import hashlib
import os

import numpy as np
import torch

from tests import scene_reference as SR

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scene.pt")


def load():
    return torch.load(PATH, weights_only=False)


def output(g, device=None):
    views = [{"img": v if device is None else v.to(device)} for v in g["views"]]
    preds = [{k: (t if device is None else t.to(device)) for k, t in p.items()} for p in g["preds"]]
    return {"views": views, "preds": preds}


def ply_id(b):
    return None if b is None else (len(b), hashlib.sha256(b).hexdigest())


def check_scene(S, sc, g):
    """S: the fast3r_b200.scene module; sc: its Scene of the golden inputs."""
    assert sc.is_outdoor == g["is_outdoor"]
    assert np.float32(sc.max_extent) == np.float32(g["max_extent"])
    for i, fd in enumerate(g["frames"]):
        a, b = sc.offsets[i], sc.offsets[i + 1]
        for head in ("global", "local"):
            np.testing.assert_array_equal(getattr(sc, f"pts_{head}")[a:b].cpu().numpy(), fd[f"pts_{head}"].numpy())
            np.testing.assert_array_equal(getattr(sc, f"rgb_{head}")[a:b].cpu().numpy(), fd[f"rgb_{head}"].numpy())
        assert bool(sc.is_high_confidence[i]) == fd["is_high_confidence"]
        np.testing.assert_array_equal(sc.view_colors[i], fd["view_color"].numpy())
        img = g["views"][i][0].permute(1, 2, 0).contiguous().numpy()
        np.testing.assert_array_equal(S.detect_sky_mask(img), g["sky"][i].numpy())
    for k, (st, want) in enumerate(zip(SR.states(sc.num_frames, sc.is_outdoor), g["ply"])):
        pts, cols = sc.visible_points(**st)
        got = S.ply_bytes(pts, cols) if len(pts) else None  # the viewer sends nothing when no point is visible
        assert ply_id(got) == want, (k, st)
