"""Every launch key of the camera-pose kernels that the fast3r_b200.poses callers reach is covered by a case of the GPU
table (tests/pose_plans.CASES, run by tests/test_pose_gpu.py), and each case reaches the key it declares.

The callers run on the CPU with poses._device_of pinned to the CPU and the three pose ops of fast3r_b200.ops replaced
by recorders: each records its descriptor; gather answers as the kernel does, score counts every point of a view as an
inlier and inliers returns all of them, so the callers go through sampling, bookkeeping and the refit at the callers'
shapes in seconds."""
from collections import Counter

import numpy as np
import pytest
import torch

pytest.importorskip("cv2")

from fast3r_b200 import lib as L  # noqa: E402
from tests import pose_emulator as E  # noqa: E402
from tests import pose_plans as PP  # noqa: E402


class Recorder:
    def __init__(self):
        self.calls = []
        self.where = ""

    def pnp_gather(self, pts, conf=None, mask=None):
        self.calls.append((dict(op="gather", views=pts.shape[0], n=pts.shape[1] * pts.shape[2], mask=mask is not None),
                           self.where))
        return E.pnp_gather(pts, conf, mask)

    def pnp_score(self, pts, pix, offsets, view_counts, hyps, thr):
        views = [int(v) for v in np.asarray(hyps, L.PNP_HYP)["view"]]
        self.calls.append((dict(op="score", views=len(offsets), nh=len(views), chunks=PP.chunks_of(views),
                                counts=[int(c) for c in view_counts]), self.where))
        return torch.tensor([int(view_counts[v]) for v in views], dtype=torch.int32)

    def pnp_inliers(self, pts, pix, offsets, view_counts, hyps, thr):
        views = [int(v) for v in np.asarray(hyps, L.PNP_HYP)["view"]]
        self.calls.append((dict(op="inliers", rows=len(views), counts=[int(view_counts[v]) for v in views]), self.where))
        sel = [torch.arange(int(offsets[v]), int(offsets[v]) + int(view_counts[v])) for v in views]
        idx = torch.cat(sel)
        return pts[idx], pix[idx], torch.tensor([len(s) for s in sel], dtype=torch.int32)


def all_pose_calls(monkeypatch):
    import fast3r_b200.ops as O
    import fast3r_b200.postprocess as P
    from fast3r_b200 import poses as PS
    rec = Recorder()
    monkeypatch.setattr(PS, "_device_of", lambda t, device=None: torch.device("cpu"))
    monkeypatch.setattr(P, "estimate_focal", lambda *a, **k: 400.0)
    for name in ("pnp_gather", "pnp_score", "pnp_inliers"):
        monkeypatch.setattr(O, name, getattr(rec, name))
    land = PP.synth_preds(3, 32, 1, *PP.LAND)
    for mode, niter in (("individual", 10), ("first_view_from_global_head", 100), ("first_view_from_local_head", 10)):
        rec.where = f"estimate_camera_poses 32 views {PP.LAND} {mode} niter {niter}"
        PS.estimate_camera_poses([dict(p) for p in land[:32]], niter_PnP=niter, focal_length_estimation_method=mode)
    p = land[0]
    rec.where = "fast_pnp one view"
    PS.fast_pnp(p["pts3d_in_other_view"][0], None, p["conf"][0] > 1, "cpu")
    rec.where = "estimate_cam_pose_one_sample"
    PS.estimate_cam_pose_one_sample([{k: v[0] for k, v in q.items()} for q in land[:4]])
    return rec.calls


@pytest.fixture(scope="module")
def recorded():
    mp = pytest.MonkeyPatch()
    try:
        yield all_pose_calls(mp)
    finally:
        mp.undo()


def test_recorder_sees_the_callers(recorded):
    """One gather, one score table and one refit round per call of the callers; `individual` scores 100 focals x 10
    hypotheses per view."""
    for where in {w for _, w in recorded}:
        assert Counter(d["op"] for d, w in recorded if w == where) == Counter(gather=1, score=1, inliers=1), where
    ind = [d for d, w in recorded if "individual" in w and d["op"] == "score"]
    assert ind[0]["nh"] == 32 * 100 * 10 and ind[0]["views"] == 32


def test_every_caller_key_has_a_gpu_case(recorded):
    table = {c["key"] for c in PP.CASES}
    missing = {}
    for d, where in recorded:
        k = PP.key(d)
        if k not in table:
            missing.setdefault(k, (where, {a: b for a, b in d.items() if a != "counts"}))
    assert not missing, "launch keys of the pose callers without a case in tests/pose_plans.CASES:\n" + \
        "\n".join(f"  {k}\n      from {where}: {d}" for k, (where, d) in sorted(missing.items()))


def test_table_keys_are_what_the_cases_reach():
    names = [c["name"] for c in PP.CASES]
    assert len(names) == len(set(names))
    wrong = [(c["name"], c["key"], PP.key(c)) for c in PP.CASES if PP.key(c) != c["key"]]
    assert not wrong, wrong


def test_table_reaches_every_flag():
    keys = {c["key"] for c in PP.CASES}
    for op, flags in (("gather", ("mask", "tail", "multiblock")), ("score", ("multilaunch", "empty", "ragged", "tail")),
                      ("inliers", ("empty", "ragged", "tail"))):
        ks = [k.split()[1:] for k in keys if k.split()[0] == op]
        for f in flags:
            assert any(f in k for k in ks) and any(f not in k for k in ks), (op, f)
