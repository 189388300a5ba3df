"""Ground-truth views on the CPU: the host geometry of fast3r_b200.views against the reference's goldens
(tests/golden/views.pt, tools/make_golden_views.py) bit for bit; the host build of the kernel's math
(fast3r_b200/csrc/views_math.h) against cv2.resize and numpy; prepare_views on the CPU emulator of its device calls
(tests/views_emulator.py) against the goldens; and the refusals of f3r_view_geometry, which come before any CUDA call."""
import hashlib
import os

import numpy as np
import pytest
import torch

from tests import views_cases as VC
from tests import views_emulator as E

PIXEL_KEYS = ("img", "depthmap", "pts3d", "valid_mask")
SMALL_KEYS = ("camera_intrinsics", "camera_pose", "true_shape", "rng")
DATASET = [n for n, c in VC.CASES.items() if c[0] == "dataset"]
RE10K = [n for n, c in VC.CASES.items() if c[0] == "re10k"]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "views.pt"), weights_only=False)["cases"]


def digest(t):
    t = t.detach().cpu().contiguous()
    return f"{t.dtype}:{tuple(t.shape)}:" + hashlib.sha256(t.numpy().tobytes()).hexdigest()


def same_bits(a, b):
    a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
    return a.dtype == b.dtype and a.shape == b.shape and a.numpy().tobytes() == b.numpy().tobytes()


def check_plan(p, g):
    assert (p.crop, p.size, p.filt, p.box) == (g["crop"], g["size"], g["filt"], g["box"])
    assert p.intrinsics.dtype == np.float32 and p.intrinsics.tobytes() == g["intrinsics"].tobytes()


def run_case(name, device):
    """prepare_views on case `name` as a loader calls it; (views, rngs)."""
    from fast3r_b200 import views
    kind, B, N, _, res, aug, _ = VC.CASES[name]
    S = VC.samples(name)
    if kind == "re10k":
        plans = [[views.plan_view_re10k(v["img"].shape[1], v["img"].shape[0], v["camera_intrinsics"], res) for v in s]
                 for s in S]
        return views.prepare_views(S, plans=plans, device=device), None
    rngs = [np.random.default_rng(s) for s in VC.rng_seeds(name)]
    return views.prepare_views(S, res, rngs=rngs, aug_crop=aug, device=device), rngs


def check_golden(name, out, rngs, g):
    """The collated views of case `name` equal the reference's bit for bit."""
    if "images" in g:  # RE10K: the image and the intrinsics (the benchmark keeps the portrait orientation)
        for b, ims in enumerate(g["images"]):
            for n, im in enumerate(ims):
                img = out[n]["img"][b]
                K = out[n]["camera_intrinsics"][b]
                if im["intrinsics"][0, 0] != K[0, 0]:  # stored transposed
                    img, K = img.transpose(1, 2), K[[1, 0, 2]]
                assert digest(img) == im["img"], (b, n)
                assert same_bits(K, im["intrinsics"])
        return
    assert [r.bit_generator.state for r in rngs] == g["rng_states"]
    for n, gv in enumerate(g["views"]):
        for k in PIXEL_KEYS:
            assert digest(out[n][k]) == gv[k], (n, k)
        for k in SMALL_KEYS:
            assert same_bits(out[n][k], gv[k]), (n, k)


# ---------------------------------------------------------------- host geometry
@pytest.mark.parametrize("name", DATASET)
def test_plan_view_equals_golden(name, golden):
    from fast3r_b200 import views
    _, B, N, _, res, aug, sp = VC.CASES[name]
    g = golden[name]
    for b, (raw, seed) in enumerate(zip(VC.samples(name), VC.rng_seeds(name))):
        rng = np.random.default_rng(seed)
        if sp.get("raises"):
            assert g["raises"] == "AssertionError"
            with pytest.raises(AssertionError, match="Bad principal point"):
                views.plan_view(raw[0]["img"].shape[1], raw[0]["img"].shape[0], raw[0]["camera_intrinsics"], res, rng)
            return
        for n, v in enumerate(raw):
            h, w = v["img"].shape[:2]
            check_plan(views.plan_view(w, h, v["camera_intrinsics"], res, rng, aug), g["plans"][b][n])
        for _ in range(N):
            rng.bytes(4)
        assert rng.bit_generator.state == g["rng_states"][b]


@pytest.mark.parametrize("name", RE10K)
def test_plan_view_re10k_equals_golden(name, golden):
    from fast3r_b200 import views
    res = VC.CASES[name][4]
    for b, raw in enumerate(VC.samples(name)):
        for n, v in enumerate(raw):
            p = views.plan_view_re10k(v["img"].shape[1], v["img"].shape[0], v["camera_intrinsics"], res)
            check_plan(p, golden[name]["plans"][b][n])


def test_plan_view_needs_an_rng_where_the_reference_draws():
    from fast3r_b200 import views
    K = np.array([[500, 0, 250], [0, 500, 240], [0, 0, 1]], np.float32)
    with pytest.raises(ValueError, match="needs an rng"):
        views.plan_view(500, 480, K, (512, 384))
    with pytest.raises(ValueError, match="aug_crop needs an rng"):
        views.plan_view(640, 480, np.array([[500, 0, 320], [0, 500, 240], [0, 0, 1]], np.float32), (512, 384),
                        aug_crop=8)
    assert views.plan_view(500, 480, K, 224).shape == (224, 224)


# ---------------------------------------------------------------- math header
def test_nearest_rule_matches_cv2_resize():
    """The kernel's per-axis INTER_NEAREST rule gives cv2.resize's source index on 4000 random shape pairs; the naive
    floor(dst * ssize / dsize) does not."""
    import cv2
    rng = np.random.default_rng(0)
    naive_differs = 0
    for _ in range(4000):
        s, d = (int(x) for x in rng.integers(1, 2500, 2))
        ramp = np.arange(s, dtype=np.float32)[None, :]
        want = cv2.resize(ramp, (d, 1), interpolation=cv2.INTER_NEAREST)[0].astype(np.int32)
        assert np.array_equal(E.nearest(s, d), want), (s, d)
        naive_differs += not np.array_equal(np.minimum(np.arange(d) * s // d, s - 1), want)
    assert naive_differs > 100


def test_nearest_rule_2d_matches_cv2_resize():
    import cv2
    rng = np.random.default_rng(1)
    for _ in range(200):
        sw, sh, dw, dh = (int(x) for x in rng.integers(1, 300, 4))
        src = rng.standard_normal((sh, sw)).astype(np.float32)
        want = cv2.resize(src, (dw, dh), interpolation=cv2.INTER_NEAREST)
        assert np.array_equal(src[E.nearest(sh, dh)][:, E.nearest(sw, dw)], want)


def test_points_match_numpy():
    """Unprojection as depthmap_to_camera_coordinates' numpy promotes it (float64, cast to float32) and the world
    transform as np.einsum("ik, vuk -> vui") + t, bit for bit, on random data with zeros, negatives, overflows and NaN
    poses."""
    rng = np.random.default_rng(2)
    for trial in range(20):
        H, W = (int(x) for x in rng.integers(1, 90, 2))
        z = (rng.standard_normal((H, W)) * 10 ** rng.uniform(-3, 3)).astype(np.float32)
        z[rng.random((H, W)) < 0.1] = 0
        if trial % 5 == 4:
            z[0, 0] = np.float32(3e38)
        K = np.float32([[rng.uniform(0.1, 900), 0, rng.uniform(-50, 300)], [0, rng.uniform(0.1, 900),
                                                                          rng.uniform(-50, 300)], [0, 0, 1]])
        pose = np.eye(4, dtype=np.float32)
        pose[:3] = rng.standard_normal((3, 4)).astype(np.float32) * 3
        if trial == 7:
            pose[:] = np.nan
        u, v = np.meshgrid(np.arange(W), np.arange(H))
        fu, fv, cu, cv = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
        with np.errstate(over="ignore", invalid="ignore"):
            cam = np.stack(((u - cu) * z / fu, (v - cv) * z / fv, z), -1).astype(np.float32)
            world = np.einsum("ik, vuk -> vui", pose[:3, :3], cam) + pose[:3, 3][None, None, :]
        valid = (z > 0) & np.isfinite(world).all(-1)
        c, w, ok = E.points(u.ravel(), v.ravel(), z.ravel(), (fu, fv, cu, cv), pose[:3].ravel())
        assert c.tobytes() == cam.reshape(-1, 3).tobytes()
        assert w.tobytes() == world.reshape(-1, 3).tobytes()
        assert np.array_equal(ok, valid.ravel())


def test_view_param_layout_matches_header():
    from fast3r_b200 import lib as L
    lay = E.param_layout()
    assert lay[0] == L.VIEW_PARAM.itemsize
    assert list(lay[1:]) == [L.VIEW_PARAM.fields[f][1] for f in L.VIEW_PARAM.names]


# ---------------------------------------------------------------- prepare_views on the emulator
@pytest.mark.parametrize("name", [n for n in VC.CASES if not VC.CASES[n][6].get("raises")])
def test_prepare_views_emulator_equals_golden(name, golden, monkeypatch):
    E.patch(monkeypatch)
    out, rngs = run_case(name, "cpu")
    check_golden(name, out, rngs, golden[name])
    v = out[0]
    B, H, W = v["depthmap"].shape
    assert v["img"].shape == (B, 3, H, W) and v["pts3d"].shape == (B, H, W, 3) and v["valid_mask"].dtype == torch.bool
    assert v["dataset"] == [name] * B and v["instance"] == ["0"] * B


def test_prepare_views_refuses_a_host_device():
    from fast3r_b200 import views
    with pytest.raises(RuntimeError, match="no CPU path"):
        views.prepare_views(VC.samples("sevenscenes_640x480"), (512, 384), device="cpu")


def test_prepare_views_refuses_inconsistent_input(monkeypatch):
    from fast3r_b200 import views
    E.patch(monkeypatch)
    S = VC.samples("sevenscenes_640x480")
    with pytest.raises(ValueError, match="same number of views"):
        views.prepare_views([S[0], S[0][:1]], (512, 384), device="cpu")
    with pytest.raises(ValueError, match="resolution or the plans"):
        views.prepare_views(S, device="cpu")
    bad = [[dict(S[0][0], depthmap=S[0][0]["depthmap"][:-1])]]
    with pytest.raises(ValueError, match="depthmap"):
        views.prepare_views(bad, (512, 384), device="cpu")
    mixed = [S[0][:1], VC.samples("portrait_480x640")[0][:1]]
    assert len(views.prepare_views(mixed, (512, 384), device="cpu")) == 1  # both collate to 512x384 landscape
    with pytest.raises(ValueError, match="landscape shape"):
        views.prepare_views([S[0][:1], VC.samples("exact_512x384")[0][:1]], plans=[
            [views.plan_view(640, 480, S[0][0]["camera_intrinsics"], (512, 384))],
            [views.plan_view(640, 480, S[0][0]["camera_intrinsics"], (224, 224))]], device="cpu")


# ---------------------------------------------------------------- C ABI refusals
def _record(**kw):
    from fast3r_b200 import lib as L
    r = np.zeros(1, L.VIEW_PARAM)
    base = dict(depth=4096, out_offset=0, src_w=640, src_h=480, crop_x=0, crop_y=0, crop_w=640, crop_h=480, rs_w=512,
                rs_h=384, box_x=0, box_y=0, out_w=512, out_h=384, transpose=0)
    for k, v in {**base, **kw}.items():
        r[0][k] = v
    return r


@pytest.mark.parametrize("kw,count,pixels,msg", [
    (dict(), 0, 512 * 384, "views (1 to 65535)"),
    (dict(), 65536, 512 * 384, "views (1 to 65535)"),
    (dict(), 1, 1 << 31, "below 2^31"),
    (dict(depth=0), 1, 512 * 384, "null depth"),
    (dict(depth=4098), 1, 512 * 384, "not 4-byte aligned"),
    (dict(src_w=70000, src_h=70000), 1, 512 * 384, "bad source size"),
    (dict(crop_x=1), 1, 512 * 384, "crop outside the source"),
    (dict(crop_h=0), 1, 512 * 384, "crop outside the source"),
    (dict(box_y=1), 1, 512 * 384, "crop outside the resized image"),
    (dict(rs_w=0), 1, 512 * 384, "bad resized or output size"),
    (dict(transpose=2), 1, 512 * 384, "transpose must be 0 or 1"),
    (dict(out_offset=1), 1, 512 * 384, "outside the output buffers"),
    (dict(out_offset=-1), 1, 512 * 384, "outside the output buffers"),
])
def test_view_geometry_refuses_bad_arguments_before_any_cuda_call(kw, count, pixels, msg):
    from fast3r_b200 import lib as L
    lib = L.load()
    rec = _record(**kw)
    if count > 1:
        rec = np.repeat(rec, count)
    rc = lib.f3r_view_geometry(rec.ctypes.data, 8, count, 8, 8, 8, pixels, None)
    err = lib.f3r_last_error().decode()
    assert rc != 0 and err.startswith("f3r_view_geometry") and msg in err, err


def test_view_geometry_refuses_null_operands():
    from fast3r_b200 import lib as L
    lib = L.load()
    rec = _record()
    for args in ((None, 8, 8, 8, 8), (rec.ctypes.data, None, 8, 8, 8), (rec.ctypes.data, 8, None, 8, 8),
                 (rec.ctypes.data, 8, 8, None, 8), (rec.ctypes.data, 8, 8, 8, None)):
        p, d, a, b, c = args
        assert lib.f3r_view_geometry(p, d, 1, a, b, c, 512 * 384, None) != 0
        assert "null operand" in lib.f3r_last_error().decode()


def test_ops_view_geometry_checks_its_record_type():
    from fast3r_b200 import ops
    with pytest.raises(TypeError, match="VIEW_PARAM"):
        ops.view_geometry(np.zeros(3, np.int64), torch.empty(1, 3), torch.empty(1, dtype=torch.uint8), torch.empty(1))
