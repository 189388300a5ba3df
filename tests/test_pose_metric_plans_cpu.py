"""Every launch key of the camera-pose metric kernels that the callers reach (camera_to_rel_deg, calculate_auc and
evaluate_camera_poses at the reference's view counts: RE10K's 10 views, 32, 320 and 1000 views, 8 items of 32) has a
case in tests/pose_metric_plans.CASES, which tests/test_pose_metric_gpu.py runs; and each case reaches its key.  The
callers run on the CPU with the entry points replaced by recorders that answer through the host emulator."""
import pytest
import torch

from tests import pose_metric_cases as PC
from tests import pose_metric_emulator as E
from tests import pose_metric_plans as PM


def recorded_keys(monkeypatch):
    import fast3r_b200.cam_pose_metric as M
    import fast3r_b200.ops as O
    from fast3r_b200 import postprocess as P
    calls = []

    def pose_metric(pred, gt, hist_max=30, angles=False):
        calls.append(dict(op="pairs", dtype=str(pred.dtype).split(".")[-1], angles=angles, items=pred.shape[0],
                          pairs=PM.pairs_of(pred.shape[1])))
        return E.pose_metric(pred, gt, hist_max, angles)

    def pose_metric_counts(r, t, hist_max=30):
        calls.append(dict(op="counts", dtype=str(r.dtype).split(".")[-1], angles=False, items=1, pairs=r.numel()))
        return E.pose_metric_counts(r, t, hist_max)

    monkeypatch.setattr(M, "_cuda", lambda t, device=None: torch.device("cpu"))
    monkeypatch.setattr(O, "pose_metric", pose_metric)
    monkeypatch.setattr(O, "pose_metric_counts", pose_metric_counts)
    for dtype in (torch.float32, torch.float64):
        for n in (2, 3, 10, 32, 320, 1000):
            pred, gt = PC.pose_set(n, dtype)
            r, t = M.camera_to_rel_deg(pred, gt, "cpu", n)
            M.calculate_auc(r, t)
        for items, n in ((2, 4), (8, 10), (8, 32)):
            pred, gt = PC.pose_set(n, dtype)
            M.pose_counts(pred[None].repeat(items, 1, 1, 1), gt[None].repeat(items, 1, 1, 1))
    # evaluate_camera_poses reaches pose_counts with its batch; its poses step is covered by tests/test_pose_plans_cpu.py
    monkeypatch.setattr(P, "estimate_camera_poses", lambda preds, views, niter_PnP, focal_length_estimation_method: (
        [[v["camera_pose"][i].numpy() for v in views] for i in range(len(views[0]["camera_pose"]))], None))
    views, preds = PC.eval_inputs("b2_v4")
    P.evaluate_camera_poses(views, preds)
    return {PM.key(d) for d in calls}


def test_every_caller_key_has_a_gpu_case(monkeypatch):
    missing = recorded_keys(monkeypatch) - {c["key"] for c in PM.CASES}
    assert not missing, f"launch keys of the pose-metric callers without a case in tests/pose_metric_plans.CASES: {missing}"


def test_table_keys_are_what_the_cases_reach():
    names = [c["name"] for c in PM.CASES]
    assert len(names) == len(set(names))
    assert all(PM.key(c) == c["key"] for c in PM.CASES)


@pytest.mark.parametrize("flag", ["below-block", "one-block", "blocks ", "blocks-tail", "strided", "angles",
                                  "many-items", "float64"])
def test_table_reaches_every_flag(flag):
    assert any(flag in c["key"] + " " for c in PM.CASES)
