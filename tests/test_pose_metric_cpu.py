"""The camera-pose metric without a GPU.  The kernels' math (csrc/pose_metric_math.h, built for the host by
tests/pose_metric_emulator.py) equals the reference's formula run by torch on the CPU (tests/pose_metric_torch.py): the
trace and 1 - loss_t bit for bit, the angles within ULP_BOUND, over 10^6 seeded pairs in float32 and float64; the
reference's quirks hold; and fast3r_b200.cam_pose_metric / postprocess.evaluate_camera_poses on a CPU emulator of the
entry points equal the reference's goldens (tests/golden/pose_metrics.pt, tools/make_golden_pose_metrics.py)."""
import math
import os

import numpy as np
import pytest
import torch

from fast3r_b200 import lib as L
from tests import pose_metric_cases as PC
from tests import pose_metric_emulator as E
from tests import pose_metric_torch as T
from tests.conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden", "pose_metrics.pt")
# the largest difference in ulp between the angles of the kernels' math and torch's (its CPU sqrt and acos are not
# correctly rounded), measured on the 10^6 pairs below in both precisions
ULP_BOUND = 3
THRESHOLDS = (5.0, 15.0, 30.0)
DTYPES = {"float32": torch.float32, "float64": torch.float64}


def golden():
    return torch.load(GOLDEN, weights_only=False)


def ulps(a, b):
    """|a - b| in units in the last place of the type (NaN == NaN counts as 0)."""
    it = torch.int32 if a.dtype == torch.float32 else torch.int64
    d = (a.view(it).long() - b.view(it).long()).abs()
    both_nan = a.isnan() & b.isnan()
    return torch.where(both_nan, torch.zeros_like(d), d)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_host_math_equals_torch_cpu(dtype):
    """10^6 pairs (1415 views): a third of the predictions uniform, the rest near the ground truth."""
    pred, gt = PC.pose_set(1415, dtype, seed=7)
    g = torch.Generator().manual_seed(3)
    pred[:470] = PC._se3(PC._rotation(g, 470), torch.randn(470, 3, generator=g, dtype=torch.float64)).to(dtype)
    ref = T.errors(pred, gt)
    counts, r, t, tr, u = E.run(pred[None], gt[None], intermediates=True)
    assert r.shape[1] >= 10 ** 6
    assert torch.equal(tr[0].view(-1), ref["trace"]) or bool(((tr[0] == ref["trace"]) | (tr[0].isnan() & ref["trace"].isnan())).all())
    same_u = (u[0] == ref["u"]) | (u[0].isnan() & ref["u"].isnan())
    assert bool(same_u.all()), int((~same_u).sum())
    assert int(ulps(r[0], ref["r"]).max()) <= ULP_BOUND
    assert int(ulps(t[0], ref["t"]).max()) <= ULP_BOUND
    assert torch.equal(counts[0], T.counts(ref["r"], ref["t"], ref["bad"]))


def test_scalars_are_the_references():
    """The constants of pose_metric_math.h, as the reference's Python forms them."""
    src = open(os.path.join(ROOT, "fast3r_b200", "csrc", "pose_metric_math.h")).read()
    const = {name: float.fromhex(src.split(f"constexpr double {name} = ")[1].split(";")[0])
             for name in ("TRACE_LO", "TRACE_HI", "BOUND", "SLOPE", "ACOS_HI", "ACOS_LO", "PI")}
    bound = 1.0 - 1e-4
    assert const["TRACE_LO"] == -1.0 - 1e-4 and const["TRACE_HI"] == 3.0 + 1e-4 and const["BOUND"] == bound
    assert const["SLOPE"] == (-1.0) / math.sqrt(1.0 - bound * bound) == (-1.0) / math.sqrt(1.0 - (-bound) * (-bound))
    assert const["ACOS_HI"] == math.acos(bound) and const["ACOS_LO"] == math.acos(-bound) and const["PI"] == np.pi


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_acos_is_close_to_correctly_rounded(dtype):
    x = torch.rand(10 ** 6, generator=torch.Generator().manual_seed(1), dtype=torch.float64).mul(2).sub(1).to(dtype)
    got = E.acos(x)
    exact = torch.from_numpy(np.arccos(x.double().numpy())).to(dtype)
    assert int(ulps(got, exact).max()) <= 1
    assert E.acos(torch.tensor([1.0, -1.0, 1.5, float("nan"), 0.0], dtype=dtype)).tolist()[:2] == [0.0, float(torch.tensor(math.pi, dtype=dtype))]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_quirks(dtype):
    pred, gt = PC.pose_set(10, dtype)
    _, r, t = E.pose_metric(pred[None], gt[None], angles=True)
    ref = T.errors(pred, gt)
    pair = {(int(i), int(j)): k for k, (i, j) in enumerate(torch.combinations(torch.arange(10), 2).tolist())}
    r, t = r[0], t[0]
    assert abs(float(r[pair[0, 1]]) - 0.4046) < 1e-3 and float(ref["r"][pair[0, 1]]) == float(r[pair[0, 1]])
    assert float(t[pair[0, 2]]) == pytest.approx(90.0, abs=1e-5)
    big = float(torch.tensor(1e6, dtype=dtype) * 180.0 / math.pi)
    assert float(t[pair[0, 5]]) == big and float(t[pair[5, 6]]) == big
    assert math.isnan(float(r[pair[0, 7]])) and math.isnan(float(r[pair[7, 9]]))
    counts = E.pose_metric(pred[None], gt[None])[0][0]
    assert int(counts[7]) == 45 and int(counts[6]) == 0
    assert int(counts[L.PM_HIST:L.PM_HIST + 31].sum()) < 45  # NaN and > 30 dropped, still in the denominator


def test_trace_out_of_range_raises(monkeypatch):
    import fast3r_b200.cam_pose_metric as M
    _emulate(monkeypatch)
    pred, gt = PC.pose_set(3)
    pred[1, :3, :3] *= 1.01
    with pytest.raises(ValueError, match=r"trace outside valid range \[-1-eps,3\+eps\]"):
        M.camera_to_rel_deg(pred, gt, "cpu", 3)
    pred[1, :3, :3] = float("nan")  # a NaN trace does not raise
    M.camera_to_rel_deg(pred, gt, "cpu", 3)


@pytest.mark.parametrize("pairs", [1, 3, 45, 496, 1953, 51040])
def test_below_ratio_is_the_float_mean(pairs):
    """below_ratio(count, P) == (x < tau).float().mean().item() for every count 0 .. P."""
    from fast3r_b200.cam_pose_metric import below_ratio
    x = torch.zeros(pairs)
    for c in range(pairs + 1):
        if c:
            x[c - 1] = 1.0
        assert below_ratio(c, pairs) == (x > 0.5).float().mean().item(), c


def _emulate(monkeypatch):
    import fast3r_b200.cam_pose_metric as M
    import fast3r_b200.ops as O
    import fast3r_b200.postprocess as P
    from fast3r_b200 import poses as PS
    from tests import abi_emulator as AE
    from tests import pose_emulator as PE
    monkeypatch.setattr(M, "_cuda", lambda t, device=None: torch.device("cpu"))
    monkeypatch.setattr(P, "_device_of", lambda t, device=None: torch.device("cpu"))
    for name in ("conf_quantile", "similarity_fit", "similarity_apply"):
        monkeypatch.setattr(O, name, getattr(AE, name))
    monkeypatch.setattr(PS, "_device_of", lambda t, device=None: torch.device("cpu"))
    monkeypatch.setattr(O, "pose_metric", E.pose_metric)
    monkeypatch.setattr(O, "pose_metric_counts", E.pose_metric_counts)
    for name in ("pnp_gather", "pnp_score", "pnp_inliers"):
        monkeypatch.setattr(O, name, getattr(PE, name))


def golden_pose_sets():
    return [(d, n) for d in DTYPES for n in PC.POSE_SIZES]


@pytest.mark.parametrize("dname,n", golden_pose_sets())
def test_emulated_metric_equals_golden(monkeypatch, dname, n):
    import fast3r_b200.cam_pose_metric as M
    _emulate(monkeypatch)
    want = golden()["pose_sets"][(dname, n)]
    pred, gt = PC.pose_set(n, DTYPES[dname])
    r, t = M.camera_to_rel_deg(pred, gt, "cpu", n)
    assert r.dtype == t.dtype == DTYPES[dname] and r.shape == (n * (n - 1) // 2,)
    if "r" in want:
        assert int(ulps(r, want["r"]).max()) <= ULP_BOUND and int(ulps(t, want["t"]).max()) <= ULP_BOUND
    got = {f"RRA_at_{int(k)}": M.below_ratio(int((r < k).sum()), len(r)) for k in THRESHOLDS}
    got.update({f"RTA_at_{int(k)}": M.below_ratio(int((t < k).sum()), len(t)) for k in THRESHOLDS})
    auc = M.calculate_auc(r, t)
    assert auc.dtype == DTYPES[dname] and auc.dim() == 0
    got["mAA_30"] = auc.item()
    assert got == want["metrics"]


def near_edge(x, edges, dtype):
    """Mask of the finite x within ULP_BOUND of their own ulps of any edge."""
    ulp = (torch.nextafter(x.abs(), torch.tensor(float("inf"), dtype=dtype)) - x.abs()).double()
    near = torch.zeros(x.shape, dtype=torch.bool)
    for e in edges:
        near |= torch.isfinite(x) & ((x.double() - float(torch.tensor(e, dtype=dtype))).abs() <= ULP_BOUND * ulp)
    return near


def decisions(r, t, hmax=30):
    """Per pair: the six threshold tests and the histc bin of max(r, t) (-1: dropped), as the counts see them."""
    worst = torch.stack((r, t), 1).max(1).values
    b = torch.where((worst >= 0) & (worst <= hmax), (worst * (hmax + 1) / hmax).long().clamp(max=hmax), -1)
    return torch.stack([r < 5, r < 15, r < 30, t < 5, t < 15, t < 30], 1), b


@pytest.mark.parametrize("dname,n", golden_pose_sets())
def test_golden_pairs_near_an_edge_fall_as_the_reference(dname, n):
    """A few ulp can only change a count at a pair within the ulp bound of a threshold or a histc edge.  The sets whose
    angles the goldens keep (n <= 32) have no such pair.  The larger sets have some (with 5 * 10^5 pairs a few land
    that close by chance); for each of them the kernels' math takes the same side of every edge as the reference's
    formula on the CPU, so the counts cannot differ there."""
    dtype = DTYPES[dname]
    edges = list(THRESHOLDS) + [30.0 * k / 31 for k in range(1, 32)]  # angles are >= 0: edge 0 cannot be crossed
    pred, gt = PC.pose_set(n, dtype)
    ref = T.errors(pred, gt)
    worst = torch.stack((ref["r"], ref["t"]), 1).max(1).values
    near = near_edge(ref["r"], edges, dtype) | near_edge(ref["t"], edges, dtype) | near_edge(worst, edges, dtype)
    if n in PC.ANGLE_SIZES:
        assert not bool(near.any())
    _, r, t = E.pose_metric(pred[None], gt[None], angles=True)
    (fk, bk), (fr, br) = decisions(r[0][near], t[0][near]), decisions(ref["r"][near], ref["t"][near])
    assert torch.equal(fk, fr) and torch.equal(bk, br)


FOCAL_KEYS = {"first_view_from_global_head": ("pts3d_in_other_view", "conf"),
              "first_view_from_local_head": ("pts3d_local_aligned_to_global", "conf_local")}


def golden_focal(monkeypatch, views, preds, mode, focals, real=None):
    """Replaces postprocess.estimate_focal (which estimate_camera_poses calls once per item, in item order) by one that
    checks it is handed view 0 of the item in its true orientation - the head's tensor after the orientation fix and,
    for the local head, the alignment - and returns the reference's focal for that item, or, with `real`, calls `real`
    and checks its focal is within 1e-3 of the reference's.  Returns the list of focals given."""
    from fast3r_b200 import postprocess as P
    items, given = iter(range(len(focals))), []

    def fake(pts3d_i, conf_i, min_conf_thr_percentile=10, **kw):
        i = next(items)
        kp, kc = FOCAL_KEYS[mode]
        h, w = views[0]["true_shape"][i].tolist()
        assert tuple(pts3d_i.shape) == (1, h, w, 3) and tuple(conf_i.shape) == (1, h, w)
        assert torch.equal(pts3d_i[0], preds[0][kp][i]) and torch.equal(conf_i[0], preds[0][kc][i])
        assert min_conf_thr_percentile == 10
        f = focals[i] if real is None else real(pts3d_i, conf_i, min_conf_thr_percentile=10, **kw)
        assert abs(f - focals[i]) <= 1e-3 * focals[i]
        given.append(f)
        return f

    monkeypatch.setattr(P, "estimate_focal", fake)
    return given


@pytest.mark.parametrize("name,mode,niter", [(k, m, i) for k, runs in PC.EVAL_RUNS.items() for m, i in runs])
def test_evaluate_camera_poses_emulated_equals_golden(monkeypatch, name, mode, niter):
    """All three focal modes on a batch with a portrait item; the first-view modes take the reference's focal."""
    pytest.importorskip("cv2")
    from fast3r_b200 import postprocess as P
    _emulate(monkeypatch)
    want = golden()["eval"][(name, mode, niter)]
    views, preds = PC.eval_inputs(name)
    given = golden_focal(monkeypatch, views, preds, mode, want["estimated_focal"]) if mode in FOCAL_KEYS else []
    got = P.evaluate_camera_poses(views, preds, niter_PnP=niter, focal_length_estimation_method=mode)
    assert got == want["metrics"]
    assert len(given) == (len(got) if mode in FOCAL_KEYS else 0)
    if name == "b2_v4":  # the portrait item's entries became lists holding it transposed back to its true shape
        keys = ["conf", "pts3d_in_other_view", "conf_local", "pts3d_local"]
        keys += ["pts3d_local_aligned_to_global"] if mode == "first_view_from_local_head" else []
        for k in keys:
            assert isinstance(preds[0][k], list) and preds[0][k][1].shape[:2] == (128, 96), k
            assert preds[0][k][0].shape[:2] == (96, 128), k


def test_evaluate_camera_poses_needs_two_views(monkeypatch):
    pytest.importorskip("cv2")
    from fast3r_b200 import postprocess as P
    _emulate(monkeypatch)
    views, preds = PC.eval_inputs("b1_v8")
    with pytest.raises(ValueError, match="Not enough camera poses"):
        P.evaluate_camera_poses(views[:1], preds[:1])


def test_cabi_rejects_bad_pose_metric_calls():
    lib = L.load()
    cnt = np.zeros(L.PM_COUNTS, np.int64)
    ws = np.zeros(64, np.uint8)
    p = ws.ctypes.data
    for args in ((0, p, p, 1, 1, 30, None, None, cnt.ctypes.data, p, 1 << 20, None),   # one view
                 (0, p, p, 0, 4, 30, None, None, cnt.ctypes.data, p, 1 << 20, None),   # no item
                 (0, p, p, 1, 4, 64, None, None, cnt.ctypes.data, p, 1 << 20, None),   # too many bins
                 (0, p, p, 1, 4, 30, p, None, cnt.ctypes.data, p, 1 << 20, None),      # r without t
                 (0, p, p, 1, 4, 30, None, None, cnt.ctypes.data, p, 16, None),        # workspace too small
                 (0, None, p, 1, 4, 30, None, None, cnt.ctypes.data, p, 1 << 20, None)):
        assert lib.f3r_pose_metric(*args) != 0
    assert lib.f3r_pose_metric_counts(0, p, p, 4, 0, cnt.ctypes.data, None) != 0
    assert lib.f3r_pose_metric_workspace(0, 1, 1) == 0
    assert lib.f3r_pose_metric_workspace(0, 32768, 65536) == 0  # items * views = 2^31
    assert lib.f3r_pose_metric(0, p, p, 32768, 65536, 30, None, None, cnt.ctypes.data, p, 1 << 62, None) != 0
    assert lib.f3r_pose_metric_workspace(1, 2, 10) == 8 * 24 * 2 * 10


def test_calculate_auc_promotes_mixed_dtypes(monkeypatch):
    """As torch.stack((r, t)) promotes: float32 and float64 errors give the float64 result."""
    import fast3r_b200.cam_pose_metric as M
    _emulate(monkeypatch)
    g = torch.Generator().manual_seed(5)
    r, t = torch.rand(500, generator=g, dtype=torch.float64) * 40, torch.rand(500, generator=g, dtype=torch.float64) * 40
    mixed = M.calculate_auc(r.float(), t)
    assert mixed.dtype == torch.float64 and mixed.item() == M.calculate_auc(r.float().double(), t).item()
    with pytest.raises(ValueError):
        M.calculate_auc(r, t, max_threshold=64)
