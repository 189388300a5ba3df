"""Every launch key of the ground-truth view kernel that fast3r_b200.views reaches - on the golden cases and on 32 and
320 views from 1920x1440 and 640x480 photos to 512x384 - has a case in tests/views_plans.CASES, which
tests/test_views_gpu.py runs; and each case reaches exactly the keys the table gives it.  prepare_views runs on the CPU
with its device calls replaced by recorders (tests/views_record.py)."""
import numpy as np
import pytest

from tests import views_cases as VC
from tests import views_plans as VP
from tests.views_record import record


def _case_keys(monkeypatch, name):
    from fast3r_b200 import views
    kind, B, N, _, res, aug, _ = VC.CASES[name]
    S = VC.samples(name)
    if kind == "re10k":
        plans = [[views.plan_view_re10k(v["img"].shape[1], v["img"].shape[0], v["camera_intrinsics"], res) for v in s]
                 for s in S]
        fn = lambda: views.prepare_views(S, plans=plans, device="cpu")  # noqa: E731
    else:
        rngs = [np.random.default_rng(s) for s in VC.rng_seeds(name)]
        fn = lambda: views.prepare_views(S, res, rngs=rngs, aug_crop=aug, device="cpu")  # noqa: E731
    calls = record(monkeypatch, fn)
    assert len(calls) == 1
    return VP.call_keys(calls[0])


def _photos(n, w, h):
    rng = np.random.default_rng(5)
    v = VC.raw_view(rng, 8, 8)
    view = dict(img=np.broadcast_to(v["img"][:1, :1], (h, w, 3)), depthmap=np.broadcast_to(v["depthmap"][:1, :1], (h, w)),
                camera_intrinsics=np.array([[w, 0, w / 2], [0, w, h / 2], [0, 0, 1]], np.float32),
                camera_pose=v["camera_pose"])
    return [[view] * n]


@pytest.mark.parametrize("name", VP.CASES)
def test_case_reaches_its_keys(monkeypatch, name):
    assert _case_keys(monkeypatch, name) == VP.KEYS[name]


def test_every_caller_key_has_a_gpu_case(monkeypatch):
    from fast3r_b200 import views
    keys = set()
    for name in VP.CASES:
        keys |= _case_keys(monkeypatch, name)
    for n in (32, 320):
        for w, h in ((1920, 1440), (640, 480)):
            S = _photos(n, w, h)
            for c in record(monkeypatch, lambda: views.prepare_views(S, (512, 384), device="cpu")):
                keys |= VP.call_keys(c)
    covered = set().union(*VP.KEYS.values())
    assert keys <= covered, f"launch keys without a GPU case in tests/views_plans: {keys - covered}"
    assert len(keys) >= 7


def test_table_covers_every_case():
    assert set(VP.KEYS) == set(VP.CASES)
