"""Generates tests/golden/pose_metrics.pt by running the REFERENCE's unmodified camera-pose metric:

  * "pose_sets": fast3r/eval/cam_pose_metric.py camera_to_rel_deg(pred, gt, "cpu", n) and calculate_auc on
    tests/pose_metric_cases.pose_set(n, dtype) for n in POSE_SIZES, float32 and float64: the angles (for n in
    ANGLE_SIZES only, to keep the file small), the seven metrics as evaluate_camera_poses forms them, and whether the
    call raised the trace ValueError;
  * "eval": MultiViewDUSt3RLitModule.evaluate_camera_poses (fast3r/models/multiview_dust3r_module.py:737-804) on
    tests/pose_metric_cases.eval_inputs(name) for each (focal mode, niter_PnP) of EVAL_RUNS: the per-item metrics and,
    in the first-view modes, the focal the reference's estimate_focal gave each item.  Its Lightning logging goes to
    no-op stand-ins; the third-party roma.rigid_points_registration its local-head alignment calls is supplied by
    oracle/geometry_oracle.umeyama (as in tools/make_golden_geometry.py).

Only outputs are stored; the tests regenerate the inputs from the seeds.
Run: python tools/make_golden_pose_metrics.py
"""
import os
import sys
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import geometry_oracle as go  # noqa: E402
from oracle import ref_harness  # noqa: E402
from tests import pose_metric_cases as PC  # noqa: E402


def metrics(cpm, r, t):
    out = {f"RRA_at_{tau}": (r < tau).float().mean().item() for tau in (5, 15, 30)}
    out.update({f"RTA_at_{tau}": (t < tau).float().mean().item() for tau in (5, 15, 30)})
    out["mAA_30"] = cpm.calculate_auc(r, t, max_threshold=30).item()
    return out


def roma_stub(x, y, compute_scaling=True):
    assert compute_scaling
    r, t, s = go.umeyama(x.double().numpy(), y.double().numpy())
    return torch.from_numpy(r).to(x.dtype), torch.from_numpy(t).to(x.dtype), torch.tensor(s, dtype=x.dtype)


def lit_self(M):
    """The attributes evaluate_camera_poses reads from the module, with its metric objects and self.log as no-ops."""
    noop = lambda *a, **k: None  # noqa: E731
    ns = types.SimpleNamespace(RRA_thresholds=[5, 15, 30], RTA_thresholds=[5, 15, 30], device=torch.device("cpu"),
                               correct_preds_orientation=M.correct_preds_orientation,
                               estimate_camera_poses=M.estimate_camera_poses, log=noop, val_mAA=noop)
    for tau in (5, 15, 30):
        setattr(ns, f"val_RRA_{tau}", noop)
        setattr(ns, f"val_RTA_{tau}", noop)
    ns.align_local_pts3d_to_global = types.MethodType(M.align_local_pts3d_to_global, ns)
    return ns


def main():
    lit = ref_harness.import_reference_lit_module(roma_registration=roma_stub)
    import fast3r.eval.cam_pose_metric as cpm
    out = {"what": "reference outputs, see tools/make_golden_pose_metrics.py", "pose_sets": {}, "eval": {}}
    for dtype in (torch.float32, torch.float64):
        for n in PC.POSE_SIZES:
            pred, gt = PC.pose_set(n, dtype)
            entry = {}
            try:
                r, t = cpm.camera_to_rel_deg(pred, gt, "cpu", n)
            except ValueError as e:
                entry["raised"] = str(e)
            else:
                entry["metrics"] = metrics(cpm, r, t)
                if n in PC.ANGLE_SIZES:
                    entry["r"], entry["t"] = r.clone(), t.clone()
            out["pose_sets"][(str(dtype).split(".")[-1], n)] = entry
    M = lit.MultiViewDUSt3RLitModule
    for name, runs in PC.EVAL_RUNS.items():
        for mode, niter in runs:
            t0 = time.perf_counter()
            views, preds = PC.eval_inputs(name)
            res = M.evaluate_camera_poses(lit_self(M), views, preds, niter_PnP=niter, focal_length_estimation_method=mode)
            # the focal each item was solved with: the reference's estimate_focal on view 0 of the item as
            # estimate_camera_poses hands it over (after the orientation fix and, for the local head, the alignment)
            keys = {"first_view_from_global_head": ("pts3d_in_other_view", "conf"),
                    "first_view_from_local_head": ("pts3d_local_aligned_to_global", "conf_local")}.get(mode)
            given = [None if keys is None else lit.estimate_focal(preds[0][keys[0]][i].unsqueeze(0),
                                                                   preds[0][keys[1]][i].unsqueeze(0),
                                                                   min_conf_thr_percentile=10)
                     for i in range(len(res))]
            out["eval"][(name, mode, niter)] = {"metrics": res, "estimated_focal": given}
            print(name, mode, niter, f"{time.perf_counter() - t0:.1f} s", flush=True)
    path = os.path.join(ROOT, "tests", "golden", "pose_metrics.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
