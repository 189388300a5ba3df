"""End-to-end parity of the CUDA path against (a) the committed reference outputs (tests/golden, generated
by the UNMODIFIED reference) and (b) the CPU oracle on the same seeded inputs.  Needs an H100.

Tolerances (relative L2, stated per SURVEY.md §8(c) 'tolerance calibration'): the reference's OWN bf16-autocast
path differs from its fp32 path by the amount stored in the fixture (``ref_bf16_vs_fp32_relL2``: 1.2e-2 on
pts3d for this tiny model, 4.5e-3 on ViT-L).  The CUDA path (bf16 operands, fp32 accumulation/residual/statistics)
must be at least as close to the fp32 reference as that."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.conftest import rel_l2  # noqa: E402
from tests.golden.synth import synth_state_dict, synth_images  # noqa: E402


def _build(tag, golden_dir):
    from fast3r_b200 import Fast3R, tiny_args
    g = torch.load(os.path.join(golden_dir, f"{tag}.pt"))
    enc, dec, head = tiny_args()
    dec.update(g.get("dec_over", {}))
    head.update(g.get("head_over", {}))
    model = Fast3R(enc, dec, head).eval()
    model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
    model = model.cuda()
    if g.get("train_mode", False):
        model.train()  # forward semantics of training mode (attention scale 1/8); backward is not built
    imgs = synth_images(g["N"], g["B"], g["H"], g["W"])
    return g, model, imgs


@pytest.mark.parametrize("tag", ["tiny_b1_n3", "tiny_b2_n2", "tiny_noattnbias", "tiny_fixedidx", "tiny_nolocal_n2",
                                 "tiny_single_view", "tiny_trainmode"])
def test_tiny_vs_reference_golden(golden_dir, tag):
    g, model, imgs = _build(tag, golden_dir)
    views = [dict(img=im.cuda(), true_shape=torch.tensor([[g["H"], g["W"]]] * g["B"]), idx=i, instance=str(i))
             for i, im in enumerate(imgs)]
    model._taps = {}
    torch.manual_seed(g["rng_seed"])
    with torch.no_grad():
        preds = model(views)
    torch.cuda.synchronize()
    gap = g.get("ref_bf16_vs_fp32_relL2", {"pts3d_in_other_view": 1.2e-2, "pts3d_local": 1.3e-2, "conf": 2.7e-3,
                                           "conf_local": 3.8e-3})
    report = {}
    for k in g["preds"][0]:
        a = torch.cat([p[k].float().cpu().flatten() for p in preds])
        b = torch.cat([p[k].float().flatten() for p in g["preds"]])
        report[k] = rel_l2(a, b)
    for gk in ("patch_embed", "enc_block1", "dec_block0", "dec_block11", "layer_rn0", "layer_rn3"):
        if gk in g["taps"] and gk in model._taps:
            ref = g["taps"][gk]
            ours = model._taps[gk]
            if gk.startswith("layer_rn"):
                ours = ours.permute(0, 3, 1, 2)
            report["tap:" + gk] = rel_l2(ours.reshape(ref.shape), ref)
    print(tag, report)
    for k in g["preds"][0]:
        assert preds[0][k].shape == g["preds"][0][k].shape and preds[0][k].dtype == torch.float32
        # fast (bf16-operand) path: at least as close to fp32 as the reference's own bf16-autocast path on this fixture
        # (1.2e-2 / 1.3e-2 on pointmaps, stored in the fixture); measured 7e-3 .. 1.2e-2
        assert report[k] <= BF16_TOL, (k, report)
        assert report[k] <= 1.05 * gap[k] or report[k] <= 5e-3, (k, report, gap)


PARITY_TOL = 1e-3  # BASELINE.json north star: pointmaps within 1e-3 relative L2 of the reference PyTorch (fp32) path
BF16_TOL = 1.3e-2  # fast path; the reference's own bf16-autocast gap is 1.2e-2 .. 1.4e-2 on these fixtures


@pytest.mark.parametrize("tag", ["tiny_b1_n3", "tiny_b2_n2", "tiny_noattnbias", "tiny_fixedidx", "tiny_nolocal_n2",
                                 "tiny_single_view", "tiny_trainmode"])
def test_parity_path_tiny_vs_reference_golden(golden_dir, tag):
    """precision="fp32" (hi/lo-split bf16 tensor-core products, fp32 storage) against the reference's fp32 outputs."""
    g, model, imgs = _build(tag, golden_dir)
    model.set_precision("fp32")
    model._taps = {}
    torch.manual_seed(g["rng_seed"])
    with torch.no_grad():
        preds = model([dict(img=im.cuda()) for im in imgs])
    report = {}
    for k in g["preds"][0]:
        a = torch.cat([p[k].float().cpu().flatten() for p in preds])
        b = torch.cat([p[k].float().flatten() for p in g["preds"]])
        report[k] = rel_l2(a, b)
    for gk in ("patch_embed", "enc_block1", "dec_block0", "dec_block11", "layer_rn0", "layer_rn3"):
        if gk in g["taps"] and gk in model._taps:
            ref, ours = g["taps"][gk], model._taps[gk]
            if gk.startswith("layer_rn"):
                ours = ours.permute(0, 3, 1, 2)
            report["tap:" + gk] = rel_l2(ours.reshape(ref.shape), ref)
    print("parity", tag, report)
    assert all(v <= PARITY_TOL for v in report.values()), report


def test_parity_path_mixed_resolution(golden_dir):
    from fast3r_b200 import Fast3R, tiny_args
    g = torch.load(os.path.join(golden_dir, "tiny_mixed_res.pt"))
    model = Fast3R(*tiny_args()).eval().set_precision("fp32")
    model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
    model = model.cuda()
    imgs = [synth_images(1, g["B"], h, w, seed0=1234 + i)[0] for i, (h, w) in enumerate(g["sizes"])]
    torch.manual_seed(g["rng_seed"])
    preds = model([dict(img=im.cuda()) for im in imgs])
    rep = {k: rel_l2(torch.cat([p[k].float().cpu().flatten() for p in preds]),
                     torch.cat([p[k].float().flatten() for p in g["preds"]])) for k in g["preds"][0]}
    print("parity mixed", rep)
    assert all(v <= PARITY_TOL for v in rep.values()), rep


def test_vitl_n4_368x512_vs_reference_golden(golden_dir):
    """BASELINE.json configs[0] on the GPU: full ViT-L/512, N=4 views 512x368, through the reference-facing
    inference() API with dtype="32" (parity path, <= 1e-3) and dtype=torch.bfloat16 (fast path), against the outputs of
    the UNMODIFIED reference's inference(dtype="32") (tests/golden/make_golden.py run_vitl_n4; every 4th pixel)."""
    import numpy as np
    from fast3r_b200 import Fast3R, inference
    from tests.test_oracle_vs_golden import vitl_n4_model_inputs
    g = torch.load(os.path.join(golden_dir, "vitl_n4_368x512.pt"))
    cfg, sd, imgs = vitl_n4_model_inputs(g)
    model = Fast3R(*cfg).eval()
    model.load_state_dict(sd)
    model = model.cuda()
    st = g["stride"]
    rep = {}
    for dt in ("32", torch.bfloat16):
        views = [dict(img=im, true_shape=np.int32([[g["H"], g["W"]]]), idx=i, instance=str(i), dataset="synthetic",
                      label=f"v{i}") for i, im in enumerate(imgs)]
        torch.manual_seed(g["rng_seed"])
        res = inference(views, model, torch.device("cuda"), dtype=dt, verbose=False)
        rep[str(dt)] = {k: rel_l2(torch.cat([p[k][:, ::st, ::st].flatten() for p in res["preds"]]),
                                  torch.cat([q[k].flatten() for q in g["preds_sub"]])) for k in g["preds_sub"][0]}
        for i, p in enumerate(res["preds"]):
            for k, (mean, std, _amax) in g["moments"][i].items():
                assert abs(float(p[k].double().std()) - std) < (1e-3 if dt == "32" else 5e-2) * std, (dt, i, k)
    print("vitl_n4_368x512", rep, "reference's own bf16-vs-fp32 gap:", g["ref_bf16_vs_fp32_relL2"])
    assert all(v <= PARITY_TOL for v in rep["32"].values()), rep
    assert all(v <= BF16_TOL for v in rep[str(torch.bfloat16)].values()), rep


def test_vitl_n4_368x512_vs_oracle(golden_dir):
    """Same configuration against the CPU oracle run on this box (different seed for the weights / images / RNG than
    the committed fixture, so the check does not depend on the fixture's data)."""
    from fast3r_b200 import Fast3R, vit_large_args
    from oracle import fast3r_oracle as O
    enc, dec, head = vit_large_args()
    with torch.device("meta"):
        shapes = {k: tuple(v.shape) for k, v in Fast3R(enc, dec, head).state_dict().items()}
    sd = synth_state_dict(shapes, seed=11)
    imgs = synth_images(4, 1, 368, 512, seed0=4321)
    torch.manual_seed(13)
    ref = O.forward(sd, enc, dec, head, imgs)
    model = Fast3R(enc, dec, head).eval()
    model.load_state_dict(sd)
    model = model.cuda()
    rep = {}
    for prec in ("fp32", "bf16"):
        model.set_precision(prec)
        torch.manual_seed(13)
        preds = model([dict(img=im.cuda()) for im in imgs])
        rep[prec] = {k: rel_l2(torch.cat([p[k].cpu().flatten() for p in preds]), torch.cat([p[k].flatten() for p in ref]))
                     for k in ref[0]}
    print("vitl_n4 vs oracle", rep)
    assert all(v <= PARITY_TOL for v in rep["fp32"].values()), rep
    assert all(v <= BF16_TOL for v in rep["bf16"].values()), rep


def test_mixed_resolution_vs_reference_golden(golden_dir):
    """Views of different resolutions in one forward (reference per-view path) against reference outputs."""
    from fast3r_b200 import Fast3R, tiny_args
    g = torch.load(os.path.join(golden_dir, "tiny_mixed_res.pt"))
    model = Fast3R(*tiny_args()).eval()
    model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
    model = model.cuda()
    imgs = [synth_images(1, g["B"], h, w, seed0=1234 + i)[0] for i, (h, w) in enumerate(g["sizes"])]
    torch.manual_seed(g["rng_seed"])
    preds = model([dict(img=im.cuda()) for im in imgs])
    rep = {}
    for k in g["preds"][0]:
        a = torch.cat([p[k].float().cpu().flatten() for p in preds])
        b = torch.cat([p[k].float().flatten() for p in g["preds"]])
        rep[k] = rel_l2(a, b)
    print("mixed", rep)
    for i, q in enumerate(g["preds"]):
        for k in q:
            assert preds[i][k].shape == q[k].shape
    assert all(v <= BF16_TOL for v in rep.values()), rep


def test_inference_api_vs_golden(golden_dir):
    import numpy as np
    from fast3r_b200 import inference
    g, model, imgs = _build("tiny_b1_n3", golden_dir)
    views = [dict(img=im, true_shape=np.int32([[g["H"], g["W"]]]), idx=i, instance=str(i), dataset="synthetic",
                  label=f"v{i}") for i, im in enumerate(imgs)]
    torch.manual_seed(g["rng_seed"])
    res, prof = inference(views, model, torch.device("cuda"), dtype=torch.bfloat16, verbose=False, profiling=True)
    assert sorted(res.keys()) == g["inference_keys"]
    assert sorted(res["views"][0].keys()) == g["inference_view_keys"]
    assert set(prof) == {"encode_images_time", "pos_emb_time", "decoder_time", "head_prepare_input_time",
                         "head_forward_time", "total_time"}
    for p, q in zip(res["preds"], g["preds"]):
        assert sorted(p) == sorted(q)
        for k in q:
            assert p[k].device.type == "cpu" and p[k].shape == q[k].shape
            assert rel_l2(p[k], q[k]) <= BF16_TOL, k


def test_vitl_two_views_vs_oracle():
    """Full-width ViT-L (24+24 layers, D=1024) on 2 small views against the CPU fp32 oracle."""
    from fast3r_b200 import Fast3R, vit_large_args
    from oracle import fast3r_oracle as O
    enc, dec, head = vit_large_args()
    model = Fast3R(enc, dec, head).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    sd = synth_state_dict(shapes, seed=5)
    model.load_state_dict(sd)
    model = model.cuda()
    imgs = synth_images(2, 1, 96, 128)
    torch.manual_seed(7)
    ref = O.forward(sd, enc, dec, head, imgs)
    torch.manual_seed(7)
    preds = model([dict(img=im.cuda()) for im in imgs])
    rep = {k: rel_l2(torch.cat([p[k].cpu().flatten() for p in preds]), torch.cat([p[k].flatten() for p in ref]))
           for k in ref[0]}
    print("vitl", rep)
    for k, v in rep.items():
        assert v <= 1e-2, rep


@pytest.mark.parametrize("precision,tol", [("bf16", BF16_TOL), ("fp32", PARITY_TOL)])
def test_portrait_view_vs_reference_golden(golden_dir, precision, tol):
    """ManyAR_PatchEmbed + landscape_only heads, one portrait view stored transposed (fast3r/dust3r/patch_embed.py:59-105,
    fast3r/dust3r/utils/misc.py:74-104) against the reference's outputs."""
    from fast3r_b200 import Fast3R, tiny_args
    g = torch.load(os.path.join(golden_dir, "tiny_portrait.pt"))
    enc, dec, head = tiny_args()
    enc.update(g["enc_over"]); head.update(g["head_over"])
    model = Fast3R(enc, dec, head).eval().set_precision(precision)
    model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
    model = model.cuda()
    imgs = synth_images(g["N"], g["B"], g["H"], g["W"])
    views = [dict(img=im.cuda(), true_shape=torch.tensor([g["true_shapes"][i]] * g["B"], dtype=torch.int32))
             for i, im in enumerate(imgs)]
    torch.manual_seed(g["rng_seed"])
    preds = model(views)
    rep = {k: rel_l2(torch.cat([p[k].float().cpu().flatten() for p in preds]),
                     torch.cat([q[k].flatten() for q in g["preds"]])) for k in g["preds"][0]}
    print("portrait", precision, rep)
    for p, q in zip(preds, g["preds"]):
        for k in q:
            assert p[k].shape == q[k].shape
    assert all(v <= tol for v in rep.values()), rep


def test_full_size_n32_properties():
    """BASELINE configs[1] at full size (ViT-L/512, N=32 views 512x368 - too big for the CPU oracle inside a test): size-
    independent properties instead.  (1) the fast path stays within the bf16 tolerance of the parity path (itself pinned to
    the reference at N=4, 1.5e-4); (2) results do not depend on the head chunking; (3) same seed -> identical bits."""
    from fast3r_b200 import Fast3R, vit_large_args
    enc, dec, head = vit_large_args()
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = Fast3R(enc, dec, head).eval()
    views = [dict(img=im.cuda()) for im in synth_images(32, 1, 368, 512)]

    def run(precision, chunk=25):
        model.set_precision(precision)
        model.set_max_parallel_views_for_head(chunk)
        torch.manual_seed(7)
        out = model(views)
        return {k: torch.cat([p[k].flatten() for p in out]) for k in out[0]}

    fast = run("bf16")
    again = run("bf16")
    chunked = run("bf16", chunk=7)
    exact = run("fp32", chunk=8)
    for k in fast:
        assert torch.equal(fast[k], again[k]), k                      # deterministic
        assert torch.equal(fast[k], chunked[k]), k                    # head chunking is a pure batching choice
        assert torch.isfinite(fast[k]).all() and torch.isfinite(exact[k]).all()
    rep = {k: rel_l2(fast[k].cpu(), exact[k].cpu()) for k in fast}
    print("N=32 full size: fast vs parity path", rep)
    assert all(v <= BF16_TOL for v in rep.values()), rep
    assert float(fast["conf"].min()) >= 1.0 and float(exact["conf"].min()) >= 1.0   # conf = 1 + exp(.)
