"""Camera poses on the GPU.  Every case of tests/pose_plans.CASES runs its kernel with canaries around every output and
equals the host answer (tests/pose_emulator.py, numpy in OpenCV's arithmetic) exactly: counts, compacted points and
pixels; on a view whose errors pile up at the threshold, the counts are the ones OpenCV's float error gives and not the
ones a double or fused sum gives.  fast_pnp and estimate_camera_poses on 32 views of 512x368 equal the reference's
goldens (tests/golden/poses.pt) and a live oracle - fast_pnp's loop around cv2.solvePnPRansac run here - with
np.array_equal, from host and device preds; `individual` mode with 10 and 100 iterations, the first-view modes with 10
and 100.  cv2 is imported unconditionally: without it these tests fail rather than skip."""
import cv2
import numpy as np
import pytest
import torch

from fast3r_b200 import lib as L  # noqa: E402
from fast3r_b200 import ops  # noqa: E402
from fast3r_b200 import poses as PS  # noqa: E402
from tests import canaries as CN  # noqa: E402
from tests import pose_emulator as E  # noqa: E402
from tests import pose_plans as PP  # noqa: E402
from tests.test_pose_cpu import _golden, _score, assert_matches_golden, golden_inputs, reference_fast_pnp  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def report_cv2():
    print(f"\ncomparing against OpenCV {cv2.__version__} (goldens: {_golden()['cv2_version']})")


def _ptr(t):
    return t.data_ptr()


def _call(name, anchor, *args):
    ops._call(name, anchor, *args)


def _canaried(shape, dtype):
    buf, view = CN.buffer(shape, dtype)
    return buf, view, buf.clone()


def _untouched(name, buf, before, n_written):
    written = torch.zeros(buf.numel(), dtype=torch.bool, device="cuda")
    written[CN.PAD:CN.PAD + n_written] = True
    CN.untouched(name, buf, before, written)


def _exact(name, got, want):
    assert torch.equal(got.cpu(), want.cpu()), name


# ------------------------------------------------------------------ the launch table
def _run_gather(c, g):
    views, n = c["views"], c["n"]
    spec = next(x for x in PP.GATHER if x[0] == c["name"])
    h, w, frac = spec[2], spec[3], spec[5]
    pts = torch.randn(views, h, w, 3, generator=g)
    conf = 1 + torch.exp(torch.randn(views, h, w, generator=g)) - 0.3
    if frac is not None:
        conf = torch.where(torch.rand(views, h, w, generator=g) < frac, 2.0, 0.5)
    mask = (conf > 1).to(torch.uint8) if c["mask"] else None
    want = E.pnp_gather(pts, conf=None if c["mask"] else conf, mask=mask)
    pb, po, pbefore = _canaried((views, n, 3), torch.float32)
    xb, xo, xbefore = _canaried((views, n, 2), torch.float32)
    cb, co, cbefore = _canaried((views,), torch.int32)
    pd = pts.cuda()
    cd = None if c["mask"] else conf.cuda()
    md = None if mask is None else mask.cuda()
    nbytes = L.load().f3r_pnp_gather_workspace(views, h, w)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    _call("f3r_pnp_gather", pd, _ptr(pd), None if cd is None else _ptr(cd), None if md is None else _ptr(md), views, h, w,
          _ptr(po), _ptr(xo), _ptr(co), _ptr(ws), nbytes)
    torch.cuda.synchronize()
    _exact("counts", co, want[2])
    for v in range(views):
        k = int(want[2][v])
        _exact(f"points of view {v}", po[v, :k], want[0][v, :k])
        _exact(f"pixels of view {v}", xo[v, :k], want[1][v, :k])
    _untouched("counts", cb, cbefore, views)
    # the slots past each view's count are not written: compare the whole buffer with the selected rows put in
    pexp, xexp = pbefore.clone(), xbefore.clone()
    for v in range(views):
        k = int(want[2][v])
        pexp[CN.PAD + v * n * 3:CN.PAD + (v * n + k) * 3] = want[0][v, :k].reshape(-1).cuda()
        xexp[CN.PAD + v * n * 2:CN.PAD + (v * n + k) * 2] = want[1][v, :k].reshape(-1).cuda()
    assert torch.equal(pb, pexp) and torch.equal(xb, xexp), "writes outside the selected rows"


def _points(g, counts, focal=300.0):
    """Points of views with `counts` points each, seen at pixels about a 512x368 grid by one camera, half of them
    displaced so that counts land anywhere between 0 and the view's count."""
    tot = sum(counts)
    pix = torch.stack([torch.randint(0, 512, (tot,), generator=g), torch.randint(0, 368, (tot,), generator=g)], 1).float()
    z = 1.5 + 2 * torch.rand(tot, generator=g, dtype=torch.float64)
    cam = torch.stack([(pix[:, 0] - 256) * z / focal, (pix[:, 1] - 184) * z / focal, z], 1)
    cam[torch.rand(tot, generator=g) < 0.5] += 0.05 * torch.randn(1, 3, generator=g, dtype=torch.float64)
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    return cam.float().contiguous(), pix.contiguous(), offsets


def _hyps(g, views_of_rows, focal=300.0):
    rows = np.zeros(len(views_of_rows), L.PNP_HYP)
    rv = (1e-3 * torch.randn(len(rows), 3, generator=g, dtype=torch.float64)).numpy()
    for i in range(len(rows)):
        rows["r"][i] = cv2.Rodrigues(rv[i].reshape(3, 1))[0].ravel()
    rows["t"] = (0.01 * torch.randn(len(rows), 3, generator=g, dtype=torch.float64)).numpy()
    rows["fx"], rows["fy"], rows["cx"], rows["cy"] = focal, focal * 1.001, 256.0, 184.0
    rows["view"] = views_of_rows
    return rows


def _run_score(c, g):
    counts = c["counts"]
    spec = next(x for x in PP.SCORE if x[0] == c["name"])
    views = len(counts)
    rows = ([v for _ in range(spec[2]) for v in range(views)] if spec[3] else
            [v for v in range(views) for _ in range(spec[2])])
    P, X, offs = _points(g, counts)
    hyps = _hyps(g, rows)
    want = E.pnp_score(P, X, offs, np.int32(counts), hyps, 5.0)
    assert int(want.max()) > 0
    cb, co, cbefore = _canaried((len(rows),), torch.int32)
    Pd, Xd = P.cuda(), X.cuda()
    nbytes = L.load().f3r_pnp_score_workspace(views, len(rows))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    cnt = np.int32(counts)
    _call("f3r_pnp_score", Pd, _ptr(Pd), _ptr(Xd), offs.ctypes.data, cnt.ctypes.data, views, hyps.ctypes.data, len(rows),
          5.0, _ptr(co), _ptr(ws), nbytes)
    torch.cuda.synchronize()
    _exact("counts", co, want)
    _untouched("counts", cb, cbefore, len(rows))


def _run_inliers(c, g):
    counts = c["counts"]
    P, X, offs = _points(g, counts)
    hyps = _hyps(g, list(range(len(counts))))
    want = E.pnp_inliers(P, X, offs, np.int32(counts), hyps, 5.0)
    m = sum(counts)
    pb, po, pbefore = _canaried((max(m, 1), 3), torch.float32)
    xb, xo, xbefore = _canaried((max(m, 1), 2), torch.float32)
    cb, co, cbefore = _canaried((len(counts),), torch.int32)
    Pd, Xd = P.cuda(), X.cuda()
    nbytes = L.load().f3r_pnp_inliers_workspace(len(counts), max(counts))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    cnt = np.int32(counts)
    _call("f3r_pnp_inliers", Pd, _ptr(Pd), _ptr(Xd), offs.ctypes.data, cnt.ctypes.data, len(counts), hyps.ctypes.data,
          len(counts), 5.0, _ptr(po), _ptr(xo), _ptr(co), _ptr(ws), nbytes)
    torch.cuda.synchronize()
    _exact("counts", co, want[2])
    _untouched("counts", cb, cbefore, len(counts))
    pexp, xexp = pbefore.clone(), xbefore.clone()
    for r in range(len(counts)):
        k, o = int(want[2][r]), int(offs[r])
        _exact(f"inliers of row {r}", po[o:o + k], want[0][o:o + k])
        _exact(f"inlier pixels of row {r}", xo[o:o + k], want[1][o:o + k])
        pexp[CN.PAD + 3 * o:CN.PAD + 3 * (o + k)] = want[0][o:o + k].reshape(-1).cuda()
        xexp[CN.PAD + 2 * o:CN.PAD + 2 * (o + k)] = want[1][o:o + k].reshape(-1).cuda()
    assert torch.equal(pb, pexp) and torch.equal(xb, xexp), "writes outside the inlier rows"


@pytest.mark.parametrize("case", PP.CASES, ids=[c["name"] for c in PP.CASES])
def test_pose_kernel_case(case):
    g = torch.Generator().manual_seed(sum(map(ord, case["name"])))
    {"gather": _run_gather, "score": _run_score, "inliers": _run_inliers}[case["op"]](case, g)


def test_score_decides_at_the_threshold_like_opencv():
    """The EPnP hypotheses of 100 RANSAC samples of tests/pose_plans.threshold_view, scored on the GPU: counts and the
    best hypothesis' inliers equal OpenCV's float error, and the table is one where the error summed in double or with
    the second square fused (a contracted FMA in pose_math.h's device branch) gives other counts."""
    P, X = PP.threshold_view(1, 92, 128, 115.0)
    K = PS.camera_matrix(115.0, (64, 46))
    S = PS.ransac_subsets(len(P), 100)
    ok, _, rv, tv = PS._epnp(P[S], X[S], K)
    table = PS._hyp_rows(rv[ok], tv[ok], K, 0)
    offs, cnt = np.zeros(1, np.int64), np.int32([len(P)])
    Pd, Xd = torch.from_numpy(P).cuda(), torch.from_numpy(X).cuda()
    got = ops.pnp_score(Pd, Xd, offs, cnt, table, 5.0).cpu().numpy()
    want = np.array([int(_score("cv")(h, P, X).sum()) for h in table])
    assert np.array_equal(got, want)
    for variant in ("double", "fma"):
        other = np.array([int(_score(variant)(h, P, X).sum()) for h in table])
        assert not np.array_equal(other, want), variant
    best = table[int(np.argmax(want))][None]
    ip, ix, ic = ops.pnp_inliers(Pd, Xd, offs, cnt, best, 5.0)
    sel = _score("cv")(best[0], P, X)
    k = int(ic[0])
    assert k == int(sel.sum())
    assert np.array_equal(ip[:k].cpu().numpy(), P[sel]) and np.array_equal(ix[:k].cpu().numpy(), X[sel])


# ------------------------------------------------------------------ the pose functions
@pytest.fixture(scope="module")
def land32():
    return golden_inputs("synth_land32")


INDIVIDUAL = [(10, False), (10, True), (100, False)]


@pytest.mark.parametrize("niter,on_device", INDIVIDUAL, ids=["it10_host_preds", "it10_device_preds", "it100_host_preds"])
def test_estimate_camera_poses_individual_equals_golden(land32, niter, on_device):
    """100 tentative focals per view (100 iterations: 320 000 EPnP hypotheses on the host, about a minute)."""
    preds = [{k: (v.cuda() if on_device else v) for k, v in p.items()} for p in land32]
    poses, focals = PS.estimate_camera_poses(preds, niter_PnP=niter, focal_length_estimation_method="individual")
    assert_matches_golden(poses, focals, _golden()["synth_land32"][("individual", niter)])


FIRST_VIEW = [(m, n) for m in ("first_view_from_global_head", "first_view_from_local_head") for n in (10, 100)]


@pytest.mark.parametrize("mode,niter", FIRST_VIEW)
@pytest.mark.parametrize("on_device", [False, True], ids=["host_preds", "device_preds"])
def test_estimate_camera_poses_first_view_equals_live_oracle(land32, mode, niter, on_device):
    """The focal comes from the GPU estimate_focal (within its tolerance of the reference's, tests/test_geometry_gpu.py);
    with it the poses equal fast_pnp's loop around cv2.solvePnPRansac, and they equal the goldens wherever the focal is
    the reference's to the bit."""
    from fast3r_b200.postprocess import estimate_focal
    preds = [{k: (v.cuda() if on_device else v) for k, v in p.items()} for p in land32]
    poses, focals = PS.estimate_camera_poses(preds, niter_PnP=niter, focal_length_estimation_method=mode)
    kp, kc = ("pts3d_in_other_view", "conf") if mode.endswith("global_head") else ("pts3d_local_aligned_to_global",
                                                                                   "conf_local")
    focal = estimate_focal(land32[0][kp][0:1], land32[0][kc][0:1], min_conf_thr_percentile=10)
    gold = _golden()["synth_land32"][(mode, niter)]
    assert abs(focal - gold["estimated_focal"][0]) <= 1e-3 * gold["estimated_focal"][0]
    assert focals[0][0] is not None  # view 0 is in its own camera frame: its pose is found
    for v, p in enumerate(land32):
        want = reference_fast_pnp(p["pts3d_in_other_view"][0].numpy(), focal, p["conf"][0].numpy() > 1.0, niter)
        if want[1] is None:
            assert focals[0][v] is None and poses[0][v].dtype == np.float64 and np.array_equal(poses[0][v], np.eye(4))
        else:
            assert focals[0][v] == want[0] and np.array_equal(poses[0][v], want[1].numpy()), v
    if gold["estimated_focal"][0] == focal:
        assert_matches_golden(poses, focals, gold)


@pytest.mark.parametrize("mode,niter", [("individual", 10)] + FIRST_VIEW)
def test_fast_pnp_equals_golden(land32, mode, niter):
    """fast_pnp itself, on device tensors, with the focal the reference solved with."""
    gold = _golden()["synth_land32"][(mode, niter)]
    for v in (0, 1, 2, 31):
        p = land32[v]
        got = PS.fast_pnp(p["pts3d_in_other_view"][0].cuda(), gold["estimated_focal"][0],
                          (p["conf"][0] > 1.0).cuda(), "cpu", niter_PnP=niter)
        if gold["focals"][0][v] is None:
            assert got == (None, None)
        else:
            assert got[0] == gold["focals"][0][v] and np.array_equal(got[1].numpy(), gold["poses"][0][v])
