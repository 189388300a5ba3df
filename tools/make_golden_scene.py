"""Writes tests/golden/scene.pt: the unmodified reference viewer (fast3r/viz/viser_visualizer.py) driven through
start_visualization with a fake server (tests/scene_reference.py) on two seeded scenes of procedural images, one
outdoor (sky masking on at launch, one low-confidence frame, one frame of another resolution) and one indoor.

Stored per scene: the inputs, the reference's sky mask of every frame (detect_sky_mask), the frame data the viewer
built (sorted points and u8 colours of both heads, is_high_confidence, rainbow colour), is_outdoor, max_extent, and the
length and SHA-256 of the PLY file "Download PLY" sends at launch and after each replayed action.

    python tools/make_golden_scene.py"""
import hashlib
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests import scene_cases as SC  # noqa: E402
from tests import scene_reference as SR  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "scene.pt")

SCENES = {
    "outdoor": dict(seed=21, shapes=[(24, 32)] * 4 + [(20, 28)] + [(24, 32)], kinds=["outdoor", "outdoor", "indoor"],
                    low_conf=[2]),
    "indoor": dict(seed=22, shapes=[(24, 32)] * 4, kinds=["indoor"], low_conf=[]),
}


def scene_inputs(seed, shapes, kinds, low_conf):
    out = SC.synth_output(seed, shapes, kinds)
    rng = np.random.default_rng(seed + 1000)
    for i, p in enumerate(out["preds"]):
        for k in ("conf", "conf_local"):
            # tie-free, so that numpy's default order is the stable one; max conf < 1.5 for the low-confidence frames
            # (hidden when low-confidence views are dropped)
            while True:
                shape = p[k].shape
                c = (1 + 0.4 * rng.random(shape) if (i in low_conf and k == "conf") else
                     1 + np.exp(rng.normal(size=shape))).astype(np.float32)
                if len(np.unique(c)) == c.size:
                    break
            p[k] = torch.from_numpy(c)
    return out


def record(ns, out):
    frames, is_outdoor, max_extent, plys = SR.run_viewer(ns, out)
    rec = dict(views=[v["img"] for v in out["views"]],
               preds=[{k: p[k] for k in ("pts3d_in_other_view", "conf", "pts3d_local_aligned_to_global", "conf_local")}
                      for p in out["preds"]],
               sky=[torch.from_numpy(ns["detect_sky_mask"](v["img"][0].permute(1, 2, 0).numpy())) for v in out["views"]],
               is_outdoor=is_outdoor, max_extent=float(max_extent), frames=[])
    for fd in frames:
        f = {}
        for head in ("global", "local"):
            c = np.asarray(fd[f"colors_{head}"])
            u8 = np.clip(c * 255, 0, 255).astype(np.uint8)  # what every export path makes of the stored floats
            assert np.array_equal(u8 / 255.0, c)
            f[f"pts_{head}"] = torch.from_numpy(np.asarray(fd[f"pts_{head}"]))
            f[f"rgb_{head}"] = torch.from_numpy(u8)
        f["is_high_confidence"] = fd["is_high_confidence"]
        f["view_color"] = torch.from_numpy(np.clip(fd["rainbow"] * 255, 0, 255).astype(np.uint8))
        rec["frames"].append(f)
    rec["ply"] = [None if b is None else (len(b), hashlib.sha256(b).hexdigest()) for b in plys]
    return rec


def main():
    ns = SR.import_reference_viewer()
    golden = {name: record(ns, scene_inputs(**cfg)) for name, cfg in SCENES.items()}
    torch.save(golden, OUT)
    for name, g in golden.items():
        print(name, "outdoor" if g["is_outdoor"] else "indoor", "max_extent", g["max_extent"],
              "ply", [p and p[0] for p in g["ply"]])


if __name__ == "__main__":
    main()
