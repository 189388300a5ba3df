"""The camera-pose metric on the GPU.  Every case of tests/pose_metric_plans.CASES runs its kernel with canaries around
every output and equals the host build of the same math (tests/pose_metric_emulator.py) bit for bit: counts and, where
stored, the angles.  camera_to_rel_deg, calculate_auc and evaluate_camera_poses (all three focal modes, a portrait item)
equal the reference's goldens (tests/golden/pose_metrics.pt) from host and from device inputs, and the first-view modes
run end to end with the GPU focal."""
import pytest
import torch

from fast3r_b200 import lib as L
from fast3r_b200 import ops
from tests import canaries as CN
from tests import pose_metric_cases as PC
from tests import pose_metric_emulator as E
from tests import pose_metric_plans as PM
from tests.test_pose_metric_cpu import DTYPES, FOCAL_KEYS, THRESHOLDS, ULP_BOUND, golden, golden_focal, ulps

pytestmark = pytest.mark.gpu


def _bits(a, b):
    return bool(((a == b) | (a.isnan() & b.isnan())).all())


def _inputs(c):
    dtype = DTYPES[c["dtype"]]
    if c["op"] == "pairs":
        pred, gt = PC.pose_set(c["views"], dtype, seed=len(c["name"]))
        k = torch.arange(c["items"], dtype=dtype)[:, None, None, None]
        pred = (pred[None] + 0.01 * k * torch.eye(4, dtype=dtype)[None, None]).contiguous()  # items differ
        return pred, gt[None].repeat(c["items"], 1, 1, 1).contiguous()
    g = torch.Generator().manual_seed(c["views"])
    r = (torch.rand(c["views"], generator=g, dtype=torch.float64) * 40).to(dtype)
    t = (torch.rand(c["views"], generator=g, dtype=torch.float64) * 40).to(dtype)
    r[::97] = float("nan")
    return r, t


@pytest.mark.parametrize("case", PM.CASES, ids=[c["name"] for c in PM.CASES])
def test_plan_case_equals_emulator(case):
    a, b = _inputs(case)
    dtype = a.dtype
    ad, bd = a.cuda(), b.cuda()
    cb, cv = CN.buffer((case["items"], L.PM_COUNTS), torch.int64)
    before = cb.clone()
    if case["op"] == "pairs":
        want, wr, wt = E.pose_metric(a, b, 30, case["angles"])
        items, views = a.shape[0], a.shape[1]
        f64 = int(dtype == torch.float64)
        nbytes = L.load().f3r_pose_metric_workspace(f64, items, views)
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        rb = tb = rv = tv = None
        if case["angles"]:
            rb, rv = CN.buffer((items, case["pairs"]), dtype)
            tb, tv = CN.buffer((items, case["pairs"]), dtype)
            rbefore, tbefore = rb.clone(), tb.clone()
        ops._call("f3r_pose_metric", ad, f64, ad.data_ptr(), bd.data_ptr(), items, views, 30,
                  None if rv is None else rv.data_ptr(), None if tv is None else tv.data_ptr(), cv.data_ptr(),
                  ws.data_ptr(), nbytes)
        torch.cuda.synchronize()
        if case["angles"]:
            assert _bits(rv.cpu(), wr) and _bits(tv.cpu(), wt)
            n = items * case["pairs"]
            for name, buf, bef in (("r", rb, rbefore), ("t", tb, tbefore)):
                written = torch.zeros(buf.numel(), dtype=torch.bool, device="cuda")
                written[CN.PAD:CN.PAD + n] = True
                CN.untouched(name, buf, bef, written)
    else:
        want = E.pose_metric_counts(a, b)[None]
        ops._call("f3r_pose_metric_counts", ad, int(dtype == torch.float64), ad.data_ptr(), bd.data_ptr(), a.numel(), 30,
                  cv.data_ptr())
        torch.cuda.synchronize()
    assert torch.equal(cv.cpu(), want)
    written = torch.zeros(cb.numel(), dtype=torch.bool, device="cuda")
    written[CN.PAD:CN.PAD + cv.numel()] = True
    CN.untouched("counts", cb, before, written)


@pytest.mark.parametrize("on_device", [False, True])
@pytest.mark.parametrize("dname,n", [(d, n) for d in DTYPES for n in PC.POSE_SIZES])
def test_metric_equals_golden(dname, n, on_device):
    import fast3r_b200.cam_pose_metric as M
    want = golden()["pose_sets"][(dname, n)]
    pred, gt = PC.pose_set(n, DTYPES[dname])
    if on_device:
        pred, gt = pred.cuda(), gt.cuda()
    r, t = M.camera_to_rel_deg(pred, gt, pred.device, n)
    assert r.device == pred.device and r.dtype == DTYPES[dname]
    er, et = E.pose_metric(pred.cpu()[None], gt.cpu()[None], angles=True)[1:]
    assert _bits(r.cpu(), er[0]) and _bits(t.cpu(), et[0])
    if "r" in want:
        assert int(ulps(r.cpu(), want["r"]).max()) <= ULP_BOUND and int(ulps(t.cpu(), want["t"]).max()) <= ULP_BOUND
    got = {f"RRA_at_{int(k)}": M.below_ratio(int((r < k).sum()), len(r)) for k in THRESHOLDS}
    got.update({f"RTA_at_{int(k)}": M.below_ratio(int((t < k).sum()), len(t)) for k in THRESHOLDS})
    auc = M.calculate_auc(r, t)
    assert auc.device == r.device and auc.dtype == r.dtype
    got["mAA_30"] = auc.item()
    assert got == want["metrics"]


@pytest.mark.parametrize("on_device", [False, True])
@pytest.mark.parametrize("name,mode,niter", [(k, m, i) for k, runs in PC.EVAL_RUNS.items() for m, i in runs])
def test_evaluate_camera_poses_equals_golden(monkeypatch, name, mode, niter, on_device):
    """All three focal modes on a batch with a portrait item and both heads; the first-view modes are handed the
    reference's focal (and checked to receive view 0 of each item in its true orientation)."""
    from fast3r_b200 import postprocess as P
    want = golden()["eval"][(name, mode, niter)]
    views, preds = PC.eval_inputs(name)
    if on_device:
        views = [{k: v.cuda() for k, v in view.items()} for view in views]
        preds = [{k: v.cuda() for k, v in p.items()} for p in preds]
    if mode in FOCAL_KEYS:
        golden_focal(monkeypatch, views, preds, mode, want["estimated_focal"])
    got = P.evaluate_camera_poses(views, preds, niter_PnP=niter, focal_length_estimation_method=mode)
    assert got == want["metrics"]


@pytest.mark.parametrize("mode", list(FOCAL_KEYS))
def test_evaluate_camera_poses_with_the_gpu_focal(monkeypatch, mode):
    """The first-view modes end to end with the GPU estimate_focal (and, for the local head, the GPU alignment): its
    focal for each item, portrait included, is within 1e-3 of the reference's; where it equals the reference's the
    metrics equal the goldens."""
    from fast3r_b200 import postprocess as P
    want = golden()["eval"][("b2_v4", mode, 10)]
    views, preds = PC.eval_inputs("b2_v4")
    given = golden_focal(monkeypatch, views, preds, mode, want["estimated_focal"], real=P.estimate_focal)
    got = P.evaluate_camera_poses(views, preds, niter_PnP=10, focal_length_estimation_method=mode)
    print(mode, "GPU focal", given, "reference", want["estimated_focal"])
    assert len(got) == 2 and all(set(m) == set(want["metrics"][0]) for m in got)
    if given == want["estimated_focal"]:
        assert got == want["metrics"]
