"""Every launch key of the viewer-scene kernels that the fast3r_b200.scene callers reach is covered by a case of the GPU
table (tests/scene_plans.CASES, run by tests/test_scene_gpu.py).

The callers run on the CPU with scene._device pinned to the CPU and the scene ops of fast3r_b200.ops replaced by
recorders over the CPU emulator (tests/scene_emulator.py), at the callers' shapes: 32 views of 512x368, mixed
resolutions, more frames than one sort group holds, and every viewer state of the goldens."""
import numpy as np
import pytest
import torch

pytest.importorskip("cv2")

from tests import scene_cases as SC  # noqa: E402
from tests import scene_emulator as E  # noqa: E402
from tests import scene_plans as SP  # noqa: E402
from tests import scene_reference as SR  # noqa: E402


class Recorder:
    def __init__(self):
        self.calls = []

    def sky_mask(self, img, out=None):
        self.calls.append(dict(op="sky", frames=img.shape[0], h=img.shape[2], w=img.shape[3]))
        return E.sky_mask(img, out)

    def scene_sort(self, conf, pts, img, not_sky, offsets, *outs):
        off = offsets.numpy()
        self.calls.append(dict(op="sort", sizes=[int(b - a) for a, b in zip(off[:-1], off[1:])]))
        return E.scene_sort(conf, pts, img, not_sky, offsets, *outs)

    def scene_visible(self, segs, *args):
        segs = np.asarray(segs).reshape(-1, 4)
        if len(segs) and segs[:, 2].max() > 0:
            self.calls.append(dict(op="visible", lens=[int(x) for x in segs[:, 2]], mask_sky=bool(args[-1]),
                                   view=bool((segs[:, 3] >= 0).any())))
        return E.scene_visible(segs, *args)

    def ply_pack(self, points, colors):
        self.calls.append(dict(op="ply", n=points.shape[0]))
        return E.ply_pack(points, colors)

    def extent_percentiles(self, points, lo=20, hi=80):
        self.calls.append(dict(op="extent", n=points.shape[0]))
        return E.extent_percentiles(points, lo, hi)


def record_all(monkeypatch):
    import fast3r_b200.ops as O
    from fast3r_b200 import scene as S
    rec = Recorder()
    monkeypatch.setattr(S, "_device", lambda t: torch.device("cpu"))
    for name in ("sky_mask", "scene_sort", "scene_visible", "ply_pack", "extent_percentiles"):
        monkeypatch.setattr(O, name, getattr(rec, name))
    outs = [SC.synth_output(1, [SC_LAND] * 32), SC.synth_output(2, [SC_LAND, (64, 96), (1, 5), SC_LAND]),
            SC.synth_output(3, [(12, 16)] * 70), SC.synth_output(4, [(24, 32)] * 4, kinds=["indoor"])]
    for out in outs:
        sc = S.prepare_scene(out)
        for st in SR.states(sc.num_frames, sc.is_outdoor):
            S.ply_bytes(*sc.visible_points(**st))
    for _, img in SC.quirk_images():
        S.detect_sky_mask(img)
    return rec.calls


SC_LAND = (368, 512)


def test_every_reached_key_has_a_gpu_case(monkeypatch):
    calls = record_all(monkeypatch)
    table = {c["key"] for c in SP.CASES}
    reached = {SP.key(d) for d in calls}
    assert reached - table == set(), sorted(reached - table)
    assert any(d["op"] == "sort" and len(d["sizes"]) == 64 for d in calls)  # 70 frames: more than one sort group


def test_cases_declare_their_keys():
    for c in SP.CASES:
        assert SP.key(c) == c["key"], c["name"]
    assert len({c["name"] for c in SP.CASES}) == len(SP.CASES)
