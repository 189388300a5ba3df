"""Ground-truth views on the GPU.  prepare_views equals the reference's goldens (tests/golden/views.pt) bit for bit from
host and from device inputs; equals the PIL + cv2 + numpy restatement (tests/views_reference.py) on seeded random raw
views with the edge cases; every case of tests/views_plans runs f3r_view_geometry with canaries around its outputs and
equals the host build of the kernel's math (tests/views_emulator.py); two runs give the same bits; and views prepared
here give the same inference, validation loss and reconstruction metrics as the restatement's views."""
import numpy as np
import pytest
import torch

from fast3r_b200 import lib as L
from fast3r_b200 import ops
from tests import canaries as CN
from tests import views_cases as VC
from tests import views_emulator as E
from tests import views_plans as VP
from tests import views_reference as R
from tests.test_views_cpu import check_golden, golden, run_case, same_bits  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
KEYS = ("img", "depthmap", "pts3d", "valid_mask", "camera_intrinsics", "camera_pose", "true_shape")


def _cuda(samples):
    """The raw views with img and depthmap on the device, as a loader that decodes on the GPU gives them."""
    return [[{k: torch.from_numpy(np.array(x)).cuda() if k in ("img", "depthmap") else x for k, x in v.items()}
             for v in s] for s in samples]


@pytest.mark.parametrize("name", VP.CASES)
def test_golden_from_host_inputs(name, golden):
    out, rngs = run_case(name, "cuda")
    assert all(out[0][k].is_cuda for k in KEYS)
    check_golden(name, out, rngs, golden[name])


@pytest.mark.parametrize("name", ["sevenscenes_640x480", "portrait_480x640", "near_square_aug_crop", "depth_specials",
                                  "missing_pose", "re10k_640x360"])
def test_golden_from_device_inputs(name, golden, monkeypatch):
    from fast3r_b200 import views
    monkeypatch.setattr(VC, "samples", lambda n, f=VC.samples: _cuda(f(n)))
    upload = views._upload

    def small_only(arr, device):
        assert np.size(arr) < 4096, "a device input was uploaded again"
        return upload(arr, device)

    monkeypatch.setattr(views, "_upload", small_only)
    out, rngs = run_case(name, "cuda")
    check_golden(name, out, rngs, golden[name])


def _random_samples(seed):
    """Seeded random raw views: random sizes (landscape, portrait, near-square, tiny and large), principal points just
    inside the margin, depth zeros / negatives / overflows, missing poses."""
    rng = np.random.default_rng(seed)
    B, N = int(rng.integers(1, 4)), int(rng.integers(1, 4))
    w, h = int(rng.integers(200, 1300)), int(rng.integers(200, 1300))
    out = []
    for b in range(B):
        views = []
        for n in range(N):
            pp = None
            if rng.random() < 0.3:
                pp = (w // 5 + 1 + rng.uniform(0, 0.4), h / 2)
            v = VC.raw_view(rng, w, h, pp, pose=rng.random() > 0.2, depth_specials=rng.random() < 0.3)
            v.update(dataset="random", label=str(seed), instance=str(n))
            views.append(v)
        out.append(views)
    res = [(512, 384), (512, 288), (224, 224), (512, 336), (500, 375)][seed % 5]
    return out, res, int(rng.choice([0, 0, 16]))


@pytest.mark.parametrize("seed", range(12))
def test_equals_host_restatement_on_random_views(seed):
    from fast3r_b200 import views
    samples, res, aug = _random_samples(seed)
    seeds = [seed * 31 + b for b in range(len(samples))]
    try:
        want_plans = [views._plan_sample(s, res, np.random.default_rng(sd), aug) for s, sd in zip(samples, seeds)]
    except AssertionError:
        pytest.skip("principal point refused, as by the reference")
    tag_rngs = [np.random.default_rng(sd) for sd in seeds]
    for s, r in zip(samples, tag_rngs):
        views._plan_sample(s, res, r, aug)
    tags = [[int.from_bytes(r.bytes(4), "big") for _ in s] for s, r in zip(samples, tag_rngs)]
    want = R.host_views(samples, want_plans, tags)
    rngs = [np.random.default_rng(sd) for sd in seeds]
    got = views.prepare_views(samples, res, rngs=rngs, aug_crop=aug)
    for n, (g, w) in enumerate(zip(got, want)):
        for k in KEYS + ("rng",):
            assert same_bits(g[k], w[k]), (n, k)
        assert g["instance"] == w["instance"]


@pytest.mark.parametrize("name", VP.CASES)
def test_plan_case_equals_emulator_with_canaries(name, monkeypatch):
    """The records prepare_views builds for the case, run again through f3r_view_geometry into canary-guarded
    buffers, equal the host build of the kernel over the same records."""
    real, seen = ops.view_geometry, []

    def capture(params, out_pts, out_valid, out_depth):
        seen.append(params.copy())
        real(params, out_pts, out_valid, out_depth)

    monkeypatch.setattr(ops, "view_geometry", capture)
    S = _cuda(VC.samples(name))
    monkeypatch.setattr(VC, "samples", lambda n: S)
    run_case(name, "cuda")
    params = seen[0]
    total = int((params["out_w"].astype(np.int64) * params["out_h"]).sum())
    pb, pts = CN.buffer((total, 3), torch.float32)
    vb = torch.full((total + 2 * CN.PAD,), 0xA5, dtype=torch.uint8, device="cuda")  # uint8 canaries
    valid = vb[CN.PAD:CN.PAD + total]
    db, depth = CN.buffer((total,), torch.float32)
    before = [b.clone() for b in (pb, vb, db)]
    ops.view_geometry(params, pts, valid, depth)
    torch.cuda.synchronize()
    B = len(S)
    host = params.copy()
    hosts = []  # host copies of the depth maps, referenced by the records until the emulator has read them
    for i in range(len(host)):
        d = S[i % B][i // B]["depthmap"].cpu().contiguous()
        hosts.append(d)
        host[i]["depth"] = d.data_ptr()
    hp, hv, hd = torch.empty(total, 3), torch.empty(total, dtype=torch.uint8), torch.empty(total)
    E.view_geometry(host, hp, hv, hd)
    assert same_bits(pts, hp) and same_bits(valid, hv) and same_bits(depth, hd)
    for nm, buf, old, cnt in (("pts", pb, before[0], 3 * total), ("valid", vb, before[1], total),
                              ("depth", db, before[2], total)):
        written = torch.zeros(buf.numel(), dtype=torch.bool, device="cuda")
        written[CN.PAD:CN.PAD + cnt] = True
        CN.untouched(nm, buf, old, written)


def test_two_runs_give_the_same_bits():
    a, _ = run_case("near_square_aug_crop", "cuda")
    b, _ = run_case("near_square_aug_crop", "cuda")
    for va, vb in zip(a, b):
        for k in KEYS + ("rng",):
            assert same_bits(va[k], vb[k]), k


def test_launches_once_per_call():
    n0 = L.launch_count()
    out, _ = run_case("photo_1600x1200", "cuda")
    torch.cuda.synchronize()
    # one f3r_view_geometry launch, and the two resampling passes of f3r_ingest_rgb8 per view
    assert L.launch_count() - n0 == 1 + 2 * 2


def test_end_to_end_inference_loss_and_metrics():
    """Views from prepare_views and from the host restatement give the same preds, validation loss and reconstruction
    metrics (identical inputs, identical outputs)."""
    from fast3r_b200 import Fast3R, inference, tiny_args, views
    from fast3r_b200.losses import ConfLossMultiviewV2, L21Loss, Regr3DMultiviewV4
    from fast3r_b200.postprocess import evaluate_reconstruction
    from tests.golden.synth import synth_state_dict
    samples = [VC.samples("sevenscenes_640x480")[0] + VC.samples("photo_1600x1200")[0]]
    plans = [views._plan_sample(samples[0], (224, 224), None, False)]
    mine = views.prepare_views(samples, plans=plans)
    ref = R.host_views(samples, plans)
    enc, dec, head = tiny_args()
    model = Fast3R(enc, dec, head).eval()
    model.load_state_dict(synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=3))
    model = model.cuda()
    crit = ConfLossMultiviewV2(Regr3DMultiviewV4(L21Loss(), norm_mode="avg_dis"), alpha=0.2)
    results = []
    for vs in (mine, [{k: v.cuda() if torch.is_tensor(v) else v for k, v in view.items()} for view in ref]):
        torch.manual_seed(0)
        out = inference([dict(img=v["img"], true_shape=v["true_shape"], instance=v["instance"]) for v in vs], model,
                        "cuda", "fp32", verbose=False)
        preds = [{k: x.cuda() for k, x in p.items()} for p in out["preds"]]
        gts = [{k: v[k].cuda() for k in ("pts3d", "valid_mask", "camera_pose")} for v in vs]
        loss, details = crit(gts, preds)
        metrics = evaluate_reconstruction([dict(g, img=v["img"], label=["scene/0"]) for g, v in zip(gts, vs)], preds)
        results.append((out["preds"], loss, details, metrics))
    (p1, l1, d1, m1), (p2, l2, d2, m2) = results
    for a, b in zip(p1, p2):
        for k in a:
            assert same_bits(a[k], b[k]), k
    assert same_bits(l1, l2) and d1 == d2 and m1 == m2
    assert torch.isfinite(l1)
