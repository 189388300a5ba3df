"""The viewer scene without a GPU: the oracle of the GPU tests (tests/scene_oracle.py) equals the unmodified
reference's functions, the per-pixel math of the kernels (csrc/scene_math.h, compiled for the host) equals numpy and
cv2 on every input it can meet, the stable order differs from numpy's default only inside runs of equal keys, and the
percentile plan of ops equals np.percentile."""
import colorsys
import ctypes as C
import os
import shutil
import subprocess
import types

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from fast3r_b200 import ops  # noqa: E402
from tests import scene_cases as SC  # noqa: E402
from tests import scene_oracle as O  # noqa: E402
from tests.conftest import ROOT  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "fast3r_b200", "csrc")


@pytest.fixture(scope="module")
def scene_math(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("scene_math") / "scene_math.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", CSRC,
                           os.path.join(HERE, "scene_math_host.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.f3r_test_scene_u8.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p]
    lib.f3r_test_scene_hsv.argtypes = [C.c_longlong, C.c_void_p, C.c_void_p]
    lib.f3r_test_scene_keys.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]
    return lib


def test_hsv_and_boxes_equal_cv2_on_every_triplet(scene_math):
    n = 1 << 24
    out = np.empty(n, np.uint8)
    hsv = np.empty((n, 3), np.uint8)
    scene_math.f3r_test_scene_hsv(n, out.ctypes.data, hsv.ctypes.data)
    i = np.arange(n, dtype=np.int64)
    rgb = np.stack([(i >> 16) & 255, (i >> 8) & 255, i & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    box, ref_hsv = O.sky_boxes(rgb)
    np.testing.assert_array_equal(hsv, ref_hsv.reshape(-1, 3))
    np.testing.assert_array_equal(out & 1, box.reshape(-1))
    upper = box.reshape(-1) | ((ref_hsv[..., 1] < 50) & (ref_hsv[..., 2] > 150)).reshape(-1)
    np.testing.assert_array_equal(out >> 1, upper)


def test_u8_conversion_equals_numpy(scene_math):
    loaded = ((np.arange(256, dtype=np.float32) / np.float32(255.0) - np.float32(0.5)) / np.float32(0.5)).astype(np.float32)
    x = np.concatenate([loaded, np.random.default_rng(0).uniform(-1, 1, 10 ** 7).astype(np.float32),
                        np.array([-1.0, 1.0, -0.0, 0.0], np.float32)])
    out = np.empty(len(x), np.uint8)
    scene_math.f3r_test_scene_u8(x.ctypes.data, len(x), out.ctypes.data)
    np.testing.assert_array_equal(out, O.to_u8(x))


def test_sort_key_orders_like_stable_argsort(scene_math):
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.normal(size=100000).astype(np.float32),
                        np.array([np.nan, -np.nan, 0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 3.4e38, -3.4e38], np.float32),
                        rng.integers(-5, 5, 10000).astype(np.float32)])
    rng.shuffle(x)
    key = np.empty(len(x), np.uint32)
    back = np.empty(len(x), np.float32)
    scene_math.f3r_test_scene_keys(x.ctypes.data, len(x), key.ctypes.data, back.ctypes.data)
    np.testing.assert_array_equal(np.argsort(key, kind="stable"), O.order(x))
    ok = ~np.isnan(x)
    np.testing.assert_array_equal(back[ok], np.where(x[ok] == 0, np.float32(0), x[ok]))
    assert np.isnan(back[~ok]).all()


def test_default_argsort_differs_only_inside_ties():
    """The reference's unstable np.argsort(-conf) and the stable order agree on every position's key: they can only
    permute elements of equal confidence."""
    rng = np.random.default_rng(2)
    conf = (1 + np.exp(rng.normal(size=188416))).astype(np.float32)
    conf[rng.integers(0, len(conf), 5000)] = conf[rng.integers(0, len(conf), 5000)]  # planted ties
    a, b = np.argsort(-conf), O.order(conf)
    np.testing.assert_array_equal(conf[a], conf[b])
    assert (a != b).any()  # the ties are really ordered differently


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 10, 1001, 188416 * 32, 188416 * 320 + 7, (1 << 24) + 3])
def test_percentile_plan_equals_numpy(n):
    rng = np.random.default_rng(n % 1000)
    x = np.sort(rng.normal(size=min(n, 3000)).astype(np.float32))
    for p in (20, 80):
        k, g = ops.percentile_plan(n, p)
        q = np.float32(n - 1) * np.true_divide(p, np.float32(100))
        assert k == min(int(np.floor(q)), n - 1)
        if n <= 3000:
            a, b = x[k], x[min(k + 1, n - 1)]
            d = np.float32(b - a)
            got = np.float32(b - d * (np.float32(1) - g)) if g >= 0.5 else np.float32(a + d * g)
            assert got == np.percentile(x, p)


# --------------------------------------------------------------------------------- the oracle against the reference
@pytest.fixture(scope="module")
def ref():
    from tests import scene_reference as SR
    if not os.path.exists(SR.reference_viewer_path()):
        pytest.skip("the reference viewer is not present")
    return SR.import_reference_viewer()


def test_oracle_sky_mask_equals_reference(ref):
    stats = {}
    rng = np.random.default_rng(4)
    images = SC.quirk_images() + [("outdoor", SC.outdoor(rng, 368, 512)), ("indoor", SC.indoor(rng, 368, 512)),
                                  ("small_outdoor", SC.outdoor(rng, 23, 31))]
    for h in range(1, 30):  # int(h * 0.4) rounds on several of these heights
        images.append((f"h{h}", SC.outdoor(rng, h, 17)))
    for name, img in images:
        np.testing.assert_array_equal(O.detect_sky_mask(img, stats), ref["detect_sky_mask"](img), err_msg=name)
    assert {"no_top", "top_all_small", "top", "empty", "diagonal_4_vs_8"} <= set(stats), stats


class _Node:
    def __init__(self, points, colors, visible):
        self.points, self.colors, self.visible = points, colors, visible


def test_oracle_frames_visible_points_and_ply_equal_reference(ref):
    """The oracle's frame arrays, is_outdoor, visible points and PLY bytes equal the reference's own is_outdoor_scene,
    update_points_filtering (through point nodes) and collect_visible_points + generate_ply_bytes."""
    out = SC.synth_output(5, [(37, 53)] * 5 + [(20, 30)], kinds=["outdoor", "indoor"])
    sc = O.prepare_scene(out)
    frames = sc["frames"]
    fdl = []
    for i, fd in enumerate(frames):
        rainbow = colorsys.hsv_to_rgb(i / len(frames), 1.0, 1.0)
        fdl.append({"sorted_pts3d_global": fd["pts_global"], "sorted_pts3d_local": fd["pts_local"],
                    "colors_rgb_global": fd["rgb_global"] / 255.0, "colors_rgb_local": fd["rgb_local"] / 255.0,
                    "colors_rainbow_global": np.tile(rainbow, (len(fd["pts_global"]), 1)),
                    "colors_rainbow_local": np.tile(rainbow, (len(fd["pts_local"]), 1)),
                    "sorted_not_sky_global": fd["not_sky_global"], "sorted_not_sky_local": fd["not_sky_local"]})
    assert ref["is_outdoor_scene"](fdl) == sc["is_outdoor"]

    class W:
        def __init__(self, v):
            self.value = v

    server = types.SimpleNamespace(flush=lambda: None)
    n = len(frames)
    for st in SC.viewer_states(n):
        t, p, sky, g, l, drop, color = st
        if p is None:
            continue  # the launch state: no percentile cut, which update_points_filtering does not express
        for fd in fdl:
            fd["point_node_global"], fd["point_node_local"] = _Node([], [], False), _Node([], [], False)
        sky_v = sc["is_outdoor"] if sky is None else sky
        ref["update_points_filtering"](server, fdl, W(t), W(p), W(sky_v), W(False), W(color == "view"))
        for i, fd in enumerate(fdl):
            shown = not drop or frames[i]["is_high_confidence"]
            fd["point_node_global"].visible = shown and g
            fd["point_node_local"].visible = shown and l
        rp, rc = ref["collect_visible_points"](fdl, t)
        op, oc = O.visible_points(sc, t, p, sky, g, l, drop, color)
        if rp is None:
            assert len(op) == 0
            continue
        np.testing.assert_array_equal(op, rp, err_msg=str(st))
        assert ref["generate_ply_bytes"](rp, rc) == O.ply_bytes(op, oc), st


# --------------------------------------------------------------------------------- the goldens of the reference viewer
from tests import scene_golden as G  # noqa: E402
from tests import scene_reference as SR  # noqa: E402


@pytest.mark.parametrize("name", ["outdoor", "indoor"])
def test_oracle_equals_reference_goldens(name):
    """The oracle's per-frame loop (order, gathers, u8 and view colours, is_high_confidence), is_outdoor, max_extent
    and PLY bytes equal what start_visualization built and sent."""
    g = G.load()[name]
    ref = O.prepare_scene(G.output(g))
    assert ref["is_outdoor"] == g["is_outdoor"] and ref["max_extent"] == np.float32(g["max_extent"])
    for fd, gd in zip(ref["frames"], g["frames"]):
        for head in ("global", "local"):
            np.testing.assert_array_equal(fd[f"pts_{head}"], gd[f"pts_{head}"].numpy())
            np.testing.assert_array_equal(fd[f"rgb_{head}"], gd[f"rgb_{head}"].numpy())
        assert fd["is_high_confidence"] == gd["is_high_confidence"]
        np.testing.assert_array_equal(fd["view_color"], gd["view_color"].numpy())
    assert not all(gd["is_high_confidence"] for gd in g["frames"]) or name == "indoor"
    for st, want in zip(SR.states(len(g["frames"]), ref["is_outdoor"]), g["ply"]):
        p, c = O.visible_points(ref, st["timestep"], st["min_conf_thr_percentile"], st["mask_sky"], st["show_global"],
                                st["show_local"], st["drop_low_conf_views"], st["color"])
        assert G.ply_id(O.ply_bytes(p, c) if len(p) else None) == want, st


@pytest.mark.parametrize("name", ["outdoor", "indoor"])
def test_emulated_scene_equals_reference_goldens(name, monkeypatch):
    """fast3r_b200.scene on the CPU emulator of its entry points (tests/scene_emulator.py) equals the goldens."""
    import fast3r_b200.ops as OPS
    from fast3r_b200 import scene as S
    from tests import scene_emulator as E
    monkeypatch.setattr(S, "_device", lambda t: torch.device("cpu"))
    for fn in ("sky_mask", "scene_sort", "scene_visible", "ply_pack", "extent_percentiles"):
        monkeypatch.setattr(OPS, fn, getattr(E, fn))
    g = G.load()[name]
    G.check_scene(S, S.prepare_scene(G.output(g)), g)


def test_goldens_reproduce_from_reference():
    """Driving the unmodified viewer again gives the stored goldens (skipped where the reference is not present)."""
    if not os.path.exists(SR.reference_viewer_path()):
        pytest.skip("the reference viewer is not present")
    ns = SR.import_reference_viewer()
    for name, g in G.load().items():
        frames, is_outdoor, max_extent, plys = SR.run_viewer(ns, G.output(g))
        assert is_outdoor == g["is_outdoor"] and float(max_extent) == g["max_extent"]
        assert [G.ply_id(b) for b in plys] == g["ply"], name
        for fd, gd in zip(frames, g["frames"]):
            np.testing.assert_array_equal(fd["pts_global"], gd["pts_global"].numpy())
            np.testing.assert_array_equal(fd["pts_local"], gd["pts_local"].numpy())
