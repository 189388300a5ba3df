"""Camera poses without a GPU: the host replay of cv2.solvePnPRansac (fast3r_b200.poses: OpenCV's samples, cv2's own
EPnP hypotheses, the RANSAC bookkeeping and the SQPnP refit around an exact inlier count) equals OpenCV bit for bit;
the scoring math of the kernel (csrc/pose_math.h) equals cv2.projectPoints; fast_pnp and estimate_camera_poses on a
CPU emulator of the three pose entry points (tests/pose_emulator.py) equal the reference's goldens; and the C ABI
rejects bad tables before any CUDA call."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from fast3r_b200 import lib as L  # noqa: E402
from fast3r_b200 import poses as PS  # noqa: E402
from tests import pose_emulator as E  # noqa: E402
from tests import pose_plans as PP  # noqa: E402
from tests.conftest import ROOT  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "fast3r_b200", "csrc")
GOLDEN = os.path.join(HERE, "golden", "poses.pt")


def fmaf(a, b, c):
    """Single-rounded float32 a * b + c, elementwise: a * b is exact in float64 (24 + 24 bits); TwoSum gives the exact
    sum as s + e; s rounds to float32 like the exact sum except when s is a float32 tie, where e breaks it."""
    p, c = a.astype(np.float64) * b.astype(np.float64), c.astype(np.float64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    f = s.astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        d = s - f.astype(np.float64)
        half = np.spacing(np.abs(f)).astype(np.float64) / 2
        tie = (np.abs(d) == half) & (e != 0)
        # at a tie s is the midpoint of f and its neighbour on d's side; when e points that way too, so does the sum
        away = tie & (np.sign(e) == np.sign(d))
        f = np.where(away, np.nextafter(f, np.float32(np.inf) * np.sign(d).astype(np.float32)), f)
    return f


def _score(variant):
    """Inlier rule: OpenCV's ("cv"), the error summed in double, or the second square fused into the float sum as a
    contracted build computes it, fmaf(dy, dy, 0 + dx^2)."""
    def rule(hyp, P, X):
        proj = E.project(hyp, P)
        if variant == "cv":
            return E.error(X, proj) <= np.float32(25)
        d = X - proj
        if variant == "double":
            return d[:, 0].astype(np.float64) ** 2 + d[:, 1].astype(np.float64) ** 2 <= 25.0
        with np.errstate(invalid="ignore", over="ignore"):
            return fmaf(d[:, 1], d[:, 1], np.float32(0) + d[:, 0] * d[:, 0]) <= np.float32(25)
    return rule


def replay(P, X, K, niter, rule=_score("cv")):
    """solvePnPRansac(P, X, K, None, iterationsCount=niter, reprojectionError=5, flags=SQPNP) from its parts; returns
    (success, rvec, tvec, inliers) or raises cv2.error like it."""
    n = len(P)
    S = PS.ransac_subsets(n, max(niter, 1))
    counts, ok, raised, masks = [], [], [], []
    for it in range(len(S)):
        try:
            good, rv, tv = cv2.solvePnP(P[S[it]], X[S[it]], K, None, flags=cv2.SOLVEPNP_EPNP)
        except cv2.error:
            good, rv, tv = False, None, None
            raised.append(True)
        else:
            raised.append(False)
        ok.append(bool(good))
        m = rule(PS._hyp_rows(rv.reshape(1, 3), tv.reshape(1, 3), K, 0)[0], P, X) if good else None
        masks.append(m)
        counts.append(0 if m is None else int(m.sum()))
    best = PS.ransac_replay(counts, ok, raised, n, niter)
    if best == "raised":
        raise cv2.error("EPnP raised")
    if best is None:
        return False, None, None, None
    inl = np.nonzero(masks[best])[0]
    good, rv, tv = cv2.solvePnP(P[inl].astype(np.float64), X[inl].astype(np.float64), K, None, flags=cv2.SOLVEPNP_SQPNP)
    return (True, rv, tv, inl.reshape(-1, 1).astype(np.int32)) if good else (False, None, None, None)


def _view(kind, n, outliers, seed):
    """(P fp32 (n, 3), X fp32 (n, 2), K): n pixels of a 368-wide grid seen by a camera of focal 400, exact or with
    displaced outliers; "planar" puts the points on one plane, "line" nearly on one line."""
    rs = np.random.default_rng(seed)
    X = np.stack([np.arange(n) % 368, np.arange(n) // 368], 1).astype(np.float64)
    f, c = 400.0, (184.0, 256.0)
    z = np.full(n, 2.0) if kind == "planar" else rs.uniform(1.5, 4.0, n)
    cam = np.stack([(X[:, 0] - c[0]) * z / f, (X[:, 1] - c[1]) * z / f, z], 1)
    if kind == "line":
        cam = np.outer(rs.uniform(1, 3, n), [0.3, 0.2, 1.0]) + 1e-4 * rs.normal(size=(n, 3))
    q, _ = np.linalg.qr(rs.normal(size=(3, 3)))
    q *= np.sign(np.linalg.det(q))
    world = (cam - rs.normal(size=3)) @ q
    out = rs.random(n) < outliers
    world[out] += 2 * rs.normal(size=(int(out.sum()), 3))
    return world.astype(np.float32), X.astype(np.float32), PS.camera_matrix(f * (1 + 0.1 * rs.normal()), c)


REPLAY_CASES = [(kind, n, niter, out) for n in (6, 100, 188416) for niter in (1, 10, 100) for out in (0.0, 0.3, 0.9)
                for kind in ("general",) if not (n == 188416 and niter == 100 and out == 0.9)]
REPLAY_CASES += [("planar", 100, 10, 0.0), ("planar", 5000, 100, 0.3), ("line", 100, 10, 0.0), ("line", 6, 100, 0.0),
                 ("line", 2000, 10, 0.3)]


def _same(a, b):
    if a[0] != b[0]:
        return False
    return not a[0] or all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:]))


@pytest.mark.parametrize("kind,n,niter,outliers", REPLAY_CASES, ids=[f"{k}_n{n}_it{i}_out{o}" for k, n, i, o in REPLAY_CASES])
def test_replay_equals_solvePnPRansac(kind, n, niter, outliers):
    """rvec, tvec and the inlier indices are bit-identical, including the "no model" result and the adaptive stop."""
    P, X, K = _view(kind, n, outliers, seed=n + niter + int(100 * outliers))
    try:
        want = cv2.solvePnPRansac(P, X, K, None, iterationsCount=niter, reprojectionError=5, flags=cv2.SOLVEPNP_SQPNP)
    except cv2.error:
        with pytest.raises(cv2.error):
            replay(P, X, K, niter)
        return
    got = replay(P, X, K, niter)
    assert _same(got, want), (kind, n, niter, outliers)


def test_replay_of_a_raising_solver():
    """All points equal: EPnP on the samples raises or fails and solvePnPRansac raises or reports no model; the
    replay does the same."""
    P = np.ones((50, 3), np.float32)
    X = np.tile(np.float32([[10, 20]]), (50, 1))
    K = PS.camera_matrix(300.0, (64, 48))
    try:
        want = cv2.solvePnPRansac(P, X, K, None, iterationsCount=10, reprojectionError=5, flags=cv2.SOLVEPNP_SQPNP)
    except cv2.error:
        with pytest.raises(cv2.error):
            replay(P, X, K, 10)
        return
    assert _same(replay(P, X, K, 10), want)


def test_replay_discriminates_the_error_arithmetic():
    """On a view with errors piled up at the threshold, OpenCV's float error reproduces solvePnPRansac while the error
    summed in double, or with the second square fused into the sum, changes the inlier set: a later edit to the
    scoring arithmetic cannot pass unnoticed."""
    P, X = PP.threshold_view(1, 92, 128, 115.0)
    K = PS.camera_matrix(115.0, (64, 46))
    want = cv2.solvePnPRansac(P, X, K, None, iterationsCount=10, reprojectionError=5, flags=cv2.SOLVEPNP_SQPNP)
    assert _same(replay(P, X, K, 10), want)
    for variant in ("double", "fma"):
        got = replay(P, X, K, 10, _score(variant))
        assert not np.array_equal(got[3], want[3]), variant


def test_update_num_iters():
    assert PS.update_num_iters(0.99, 0.0, 5, 100) == 0  # every point an inlier: stop
    assert PS.update_num_iters(0.99, 1.0, 5, 100) == 100
    assert PS.update_num_iters(0.99, 0.5, 5, 1000) == round(np.log(0.01) / np.log(1 - 0.5 ** 5)) == 145
    assert PS.update_num_iters(0.99, 0.3, 5, 3) == 3


# ------------------------------------------------------------------ the kernel's math against cv2.projectPoints
@pytest.fixture(scope="module")
def pose_math(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("pose_math") / "pose_math.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", CSRC,
                           os.path.join(HERE, "pose_math_host.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.f3r_test_pnp_project.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _host_project(lib, rv, tv, K, P, X):
    rt = np.ascontiguousarray(np.concatenate([cv2.Rodrigues(rv)[0].ravel(), tv.ravel()]), np.float64)
    k = np.float64([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    uv, err = np.empty((len(P), 2), np.float32), np.empty(len(P), np.float32)
    lib.f3r_test_pnp_project(rt.ctypes.data, k.ctypes.data, P.ctypes.data, X.ctypes.data, len(P), uv.ctypes.data,
                             err.ctypes.data)
    return uv, err


def _bits_equal(a, b):
    return bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


@pytest.mark.parametrize("trial", range(4))
def test_pose_math_equals_projectPoints(pose_math, trial):
    """1e6 seeded points at scales 1e-3 .. 1e3, with z = 0, z < 0, subnormal z (projections past the r^6 overflow give
    NaN as OpenCV's zero distortion does) and non-finite coordinates: the projection and the float error are cv2's bit
    for bit."""
    rs = np.random.default_rng(trial)
    n = 1_000_000 if trial == 0 else 250_000
    P = (rs.normal(size=(n, 3)) * rs.choice([1e-3, 1, 10, 1e3], size=(n, 1))).astype(np.float32)
    P[:1000, 2] = 0
    P[1000:2000, 2] *= -1
    P[2000:2100] = np.float32([1e10, 1, 1e-45])
    P[2100:2200] = np.float32([1e6, 1, 1e-45])
    P[2200:2210] = np.float32([np.inf, 1, 1])
    P[2210:2220] = np.float32([np.nan, 1, 1])
    X = rs.uniform(0, 512, size=(n, 2)).astype(np.float32)
    rv, tv = (np.zeros((3, 1)), np.zeros((3, 1))) if trial == 1 else (rs.normal(size=(3, 1)), rs.normal(size=(3, 1)))
    K = PS.camera_matrix(np.float32(rs.uniform(100, 900)), (256, 184))
    uv, err = _host_project(pose_math, rv, tv, K, P, X)
    want = cv2.projectPoints(P, rv, tv, K, None)[0].reshape(-1, 2)
    assert _bits_equal(uv, want)
    d = X - want
    with np.errstate(invalid="ignore", over="ignore"):
        assert _bits_equal(err, (np.float32(0) + d[:, 0] * d[:, 0]) + d[:, 1] * d[:, 1])
        assert _bits_equal(err, E.error(X, E.project(PS._hyp_rows(rv.reshape(1, 3), tv.reshape(1, 3), K, 0)[0], P)))


# ------------------------------------------------------------------ the pose functions on the emulator
@pytest.fixture
def emulated(monkeypatch):
    import fast3r_b200.ops as O
    monkeypatch.setattr(PS, "_device_of", lambda t, device=None: torch.device("cpu"))
    for name in ("pnp_gather", "pnp_score", "pnp_inliers"):
        monkeypatch.setattr(O, name, getattr(E, name))


def reference_fast_pnp(pts3d, focal, msk, niter_PnP=10, pp=None):
    """fast_pnp's loop (init_im_poses.py:300-350) restated around cv2.solvePnPRansac: (focal, pose) or (None, None)."""
    pts3d, msk = np.asarray(pts3d), np.asarray(msk)
    if msk.sum() < 4:
        return None, None
    H, W, _ = pts3d.shape
    pixels = np.mgrid[:W, :H].T.astype(np.float32)
    job = PS._Job(PS._tentative_focals(focal, H, W, 100), (W / 2, H / 2) if pp is None else pp, niter_PnP)
    return PS._reference_loop(pts3d[msk], pixels[msk], job, "cpu")


def _pose_equal(a, b):
    return (a[0] is None and b[0] is None and a[1] is None and b[1] is None) or (
        a[0] == b[0] and type(a[0]) is type(b[0]) and torch.equal(a[1], b[1]))


FAST_PNP_CASES = [(4, None, 10), (5, None, 10), (5, 150.0, 1), (6, None, 10), (3, None, 10), (100, 140.0, 100),
                  (900, None, 10), (2000, 300.0, 100)]


@pytest.mark.parametrize("count,focal,niter", FAST_PNP_CASES)
def test_fast_pnp_emulated_equals_reference(emulated, count, focal, niter):
    """Counts 3 (no pose), 4 (P3P), 5 (direct solve) and RANSAC sizes, with the 100 geometric focals or a given one."""
    g = torch.Generator().manual_seed(count)
    pts, conf = PP.synth_view(g, 40, 60, 60.0, 0.3, noise_px=1.0)
    msk = torch.zeros(40 * 60, dtype=torch.bool)
    msk[torch.randperm(40 * 60, generator=g)[:count]] = True
    msk = msk.reshape(40, 60)
    got = PS.fast_pnp(pts, focal, msk, "cpu", niter_PnP=niter)
    want = reference_fast_pnp(pts.numpy(), focal, msk.numpy(), niter)
    assert _pose_equal(got, want), (got, want)


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/poses.pt not generated")
    return torch.load(GOLDEN, weights_only=False)


def golden_inputs(name):
    if name == "geometry_tail":
        gold = torch.load(os.path.join(HERE, "golden", "geometry_tail.pt"), weights_only=False)
        return [dict(p) for p in gold["preds"]]
    if name == "synth_small":
        return PP.synth_preds(7, 4, 2, 96, 128)
    return PP.synth_preds(11, 32, 1, 368, 512)


def assert_matches_golden(poses, focals, want):
    assert len(poses) == len(want["poses"])
    for ps, fs, wp, wf in zip(poses, focals, want["poses"], want["focals"]):
        assert fs == wf and [type(f) for f in fs] == [type(f) for f in wf]
        for a, b in zip(ps, wp):
            assert a.dtype == b.dtype and np.array_equal(a, b)


def test_goldens_are_not_degenerate():
    """Every golden run solves real poses: the first-view modes have a positive focal and every view gets a pose."""
    gold = _golden()
    for name in ("geometry_tail", "synth_small", "synth_land32"):
        for (mode, niter), run in gold[name].items():
            if mode != "individual":
                assert all(f > 0 for f in run["estimated_focal"]), (name, mode, niter)
            for fs in run["focals"]:
                assert all(f is not None for f in fs), (name, mode, niter, fs)


@pytest.mark.parametrize("name", ["geometry_tail", "synth_small"])
def test_estimate_camera_poses_emulated_equals_golden(emulated, monkeypatch, name):
    """All three focal modes; the first-view modes take the golden focal of each batch item (the GPU estimate_focal is
    checked against the reference in tests/test_geometry_gpu.py)."""
    import fast3r_b200.postprocess as P
    gold = _golden()
    preds = golden_inputs(name)
    for (mode, niter), want in gold[name].items():
        it = iter(want["estimated_focal"])
        monkeypatch.setattr(P, "estimate_focal", lambda *a, **k: next(it))
        poses, focals = PS.estimate_camera_poses([dict(p) for p in preds], niter_PnP=niter,
                                                 focal_length_estimation_method=mode)
        assert_matches_golden(poses, focals, want)


def test_golden_records_its_opencv():
    print("goldens made with OpenCV", _golden()["cv2_version"], "- this host has", cv2.__version__)
    assert _golden()["cv2_version"]


# ------------------------------------------------------------------ argument checks before any CUDA call
def test_cabi_rejects_bad_pose_tables():
    from fast3r_b200.build import build
    build()
    lib = L.load()
    offs, cnts = np.zeros(2, np.int64), np.full(2, 10, np.int32)
    hyps = np.zeros(3, L.PNP_HYP)
    hyps["view"] = [0, 1, 2]
    f = C.c_float
    for name, args, what in (
            ("f3r_pnp_score", (8, 8, offs.ctypes.data, cnts.ctypes.data, 2, hyps.ctypes.data, 3, f(5), 8, 256, 1 << 20,
                               None), "names view 2 of 2"),
            ("f3r_pnp_score", (8, 8, offs.ctypes.data, cnts.ctypes.data, 3, hyps.ctypes.data, 3, f(float("nan")), 8, 256,
                               1 << 20, None), "not finite"),
            ("f3r_pnp_score", (8, 8, offs.ctypes.data, cnts.ctypes.data, 2, hyps.ctypes.data, 2, f(float("inf")), 8, 256,
                               1 << 20, None), "not finite"),
            ("f3r_pnp_score", (8, 8, None, cnts.ctypes.data, 2, hyps.ctypes.data, 2, f(5), 8, 256, 1 << 20, None),
             "null table"),
            ("f3r_pnp_score", (8, 8, offs.ctypes.data, np.int32([10, -1]).ctypes.data, 2, hyps.ctypes.data, 2, f(5), 8,
                               256, 1 << 20, None), "has offset"),
            ("f3r_pnp_score", (8, 8, offs.ctypes.data, cnts.ctypes.data, 2, hyps.ctypes.data, 2, f(5), 8, 256, 16, None),
             "workspace too small"),
            ("f3r_pnp_inliers", (8, 8, offs.ctypes.data, cnts.ctypes.data, 2, hyps.ctypes.data, 3, f(5), 8, 8, 8, 256,
                                 1 << 20, None), "names view 2 of 2"),
            ("f3r_pnp_inliers", (8, 8, offs.ctypes.data, cnts.ctypes.data, 2, hyps.ctypes.data, 0, f(5), 8, 8, 8, 256,
                                 1 << 20, None), "bad sizes"),
            ("f3r_pnp_gather", (8, 8, 8, 1, 4, 4, 8, 8, 8, 256, 1 << 20, None), "exactly one of conf and mask"),
            ("f3r_pnp_gather", (8, 8, None, 0, 4, 4, 8, 8, 8, 256, 1 << 20, None), "bad shape"),
            ("f3r_pnp_gather", (8, 8, None, 1, 4, 4, 8, 8, 8, 256, 0, None), "workspace too small")):
        assert getattr(lib, name)(*args) == 1, name
        assert what in lib.f3r_last_error().decode(), (name, lib.f3r_last_error().decode())
