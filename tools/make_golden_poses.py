"""Generates tests/golden/poses.pt by running the REFERENCE's unmodified
MultiViewDUSt3RLitModule.estimate_camera_poses (fast3r/models/multiview_dust3r_module.py:807-869, which calls
estimate_cam_pose_one_sample and fast_pnp -> cv2.solvePnPRansac) on seeded preds:

  * "geometry_tail": the preds of tests/golden/geometry_tail.pt (3 views, batch 2, 48x64), `individual` mode only:
    their view 0 is not in its own camera frame, so the first-view focal of these preds is 0;
  * "synth_small": tests/pose_plans.synth_preds(7, 4 views, batch 2, 96x128), known poses with 0 / 30 / 90 % outliers;
  * "synth_land32": tests/pose_plans.synth_preds(11, 32 views, batch 1, 368x512), the resolution of the benchmark.

Each entry holds the poses and focals of every (focal mode, niter_PnP) run and, in the first-view modes, the focal
estimate_focal gave each batch item; the file records the cv2 version that made them.  The inputs are regenerated from
the seeds by the tests, so only the outputs are stored.
Run: python tools/make_golden_poses.py   (about 8 minutes on 8 cores, most of it the 32-view `individual` runs)
"""
import os
import sys
import time

import cv2
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402
from tests import pose_plans as PP  # noqa: E402

MODES = ("individual", "first_view_from_global_head", "first_view_from_local_head")


def geometry_tail_preds():
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "geometry_tail.pt"), weights_only=False)
    return [dict(p) for p in gold["preds"]]


INPUTS = {
    "geometry_tail": (geometry_tail_preds, [("individual", 10), ("individual", 100)]),
    "synth_small": (lambda: PP.synth_preds(7, 4, 2, 96, 128), [(m, n) for m in MODES for n in (1, 10, 100)]),
    "synth_land32": (lambda: PP.synth_preds(11, 32, 1, 368, 512),
                     [("individual", 10), ("individual", 100), ("first_view_from_global_head", 100),
                      ("first_view_from_global_head", 10), ("first_view_from_local_head", 10),
                      ("first_view_from_local_head", 100)]),
}


def main():
    lit = ref_harness.import_reference_lit_module()
    out = {"cv2_version": cv2.__version__, "what": "reference outputs, see tools/make_golden_poses.py"}
    for name, (make, runs) in INPUTS.items():
        preds = make()
        out[name] = {}
        for mode, niter in runs:
            t0 = time.perf_counter()
            poses, focals = lit.MultiViewDUSt3RLitModule.estimate_camera_poses(
                [dict(p) for p in preds], niter_PnP=niter, focal_length_estimation_method=mode)
            # the focal each batch item's views were solved with (the reference's estimate_focal, :823-836)
            keys = {"first_view_from_global_head": ("pts3d_in_other_view", "conf"),
                    "first_view_from_local_head": ("pts3d_local_aligned_to_global", "conf_local")}.get(mode)
            given = [None if keys is None else
                     lit.estimate_focal(preds[0][keys[0]][i:i + 1], preds[0][keys[1]][i:i + 1], min_conf_thr_percentile=10)
                     for i in range(len(poses))]
            out[name][(mode, niter)] = {"poses": poses, "focals": focals, "estimated_focal": given}
            print(name, mode, niter, f"{time.perf_counter() - t0:.1f} s", flush=True)
    path = os.path.join(ROOT, "tests", "golden", "poses.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
