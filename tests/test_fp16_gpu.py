"""precision="fp16" on the GPU: every GEMM and attention launch plan of the forward per element against float64 with fp16
operands, the fp16 forward against the reference goldens, and its launch count against the bf16 forward.  Needs an
H100.

The per-plan checks run the bf16 checks of tests/test_gemm_plans_gpu.py and tests/test_attention_plans_gpu.py with
fp16 in place of bf16 (their module's torch.bfloat16 reads as torch.float16; ops dispatches on the dtype).  The bounds
are those of the bf16 checks with the fp16 half-ulp 2^-11 in place of the bf16 one (2^-8) for every 16-bit rounding: the
stored outputs and, in attention, P.  fp16 has subnormals below 2^-14 where bf16 has none: a value under 2^-14 rounds to
within 2^-25 absolute, so every 16-bit output bound adds 2^-25 (SUB), and the attention bound 2^-25 per key of the slice
times max |v| for P.  The relative L2 tolerance of the 16-bit outputs is 1e-3 (the bf16 checks: 6e-3 / 6.2e-3; rounding
alone to fp16 gives ~3e-4)."""
import math
import os
import types

import numpy as np
import pytest
import torch

from tests import attention_plans as AP
from tests import gemm_plans as GP
from tests import test_attention_plans_gpu as APG
from tests import test_gemm_plans_gpu as GPG
from tests.conftest import rel_l2
from tests.packed_goldens import TAGS, scene, tiny_model

pytestmark = pytest.mark.gpu

F16 = torch.float16
FP16_TOL = 3e-3        # every pred key of the fp16 forward against the reference's fp32 result (relative L2)
U16, U8 = 2.0 ** -11, 2.0 ** -8
SUB = 2.0 ** -25       # half the spacing of fp16 subnormals
REL_L2_16 = 1e-3


class _Torch16(types.ModuleType):
    """torch, except that torch.bfloat16 is torch.float16."""

    def __init__(self):
        super().__init__("torch")
        self.bfloat16 = torch.float16

    def __getattr__(self, name):
        return getattr(torch, name)


@pytest.fixture
def fp16_checks(monkeypatch):
    """The per-plan check modules in fp16 (module docstring)."""
    from fast3r_b200 import ops
    t16 = _Torch16()
    monkeypatch.setattr(GPG, "torch", t16)
    monkeypatch.setattr(APG, "torch", t16)
    # the 16-bit outputs: half an fp16 ulp instead of half a bf16 ulp (bound = E + 2^-8 |ref| in the bf16 check)
    check = GPG._check

    def check16(name, out, ref, bound, kind):
        if kind == "bf16":
            bound = bound - (U8 - U16) * ref.abs() + SUB
        check(name, out, ref, bound, kind)

    monkeypatch.setattr(GPG, "_check", check16)
    monkeypatch.setitem(GPG.REL_L2, "bf16", REL_L2_16)
    for k in ("bf16", "f32"):
        monkeypatch.setitem(APG.REL_L2, k, REL_L2_16)

    def bounds16(R, nkv, sl2, x3, r):
        assert not x3
        r = U16 if r == U8 else r
        ew = APG._weight_err(R, nkv, sl2, False)
        c = ew + U16 + (129 * nkv + 4) * 2.0 ** -22 * (1 + U16)
        eL = ew + (33 * nkv + 4) * APG.U
        ref = R["ref"].abs()
        E = (c[:, None] * R["M"] + eL[:, None] * ref) / (1 - eL)[:, None] + 1.01 * 2.0 ** -23 * ref \
            + nkv * AP.KB * (2.0 ** -126 + 2.0 ** -25) * R["vmax"]
        E_lse = 1.01 * eL + 2.0 ** -21 * (R["lse"].abs() + APG.LN2 * R["T"] + 1)
        return E + r * (ref + E) + (SUB if r else 0.0), E_lse

    merge_bound = APG._merge_bound
    monkeypatch.setattr(APG, "_bounds", bounds16)
    monkeypatch.setattr(APG, "_merge_bound", lambda parts, ref, r: merge_bound(parts, ref, U16) + SUB)
    # the segments check calls the bf16 entry point by name
    call = ops._call
    monkeypatch.setattr(ops, "_call", lambda name, anchor, *a: call(
        name + "_f16" if name == "f3r_attention_segments" and anchor.dtype == F16 else name, anchor, *a))


# ------------------------------------------------------------------ every launch plan, per element
@pytest.mark.parametrize("case", GP.CASES, ids=[c["name"] for c in GP.CASES])
def test_gemm_case_fp16(case, fp16_checks):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if any(v.startswith("F3R_GEMM_") for v in os.environ) or sms != GP.H100_SMS:
        pytest.skip("the case table's plan keys are those of a 132-SM H100 SXM with the library's default plans")
    assert GP.plan_key(case, sms) == case["key"]
    GPG.run_case(case, seed=5000 + GP.CASES.index(case))


ATT16 = [c for c in AP.CASES if c["kind"] != "x3"]  # (attention_x3 is the parity path: no fp16 form)


@pytest.mark.parametrize("regime", ["flat", "grow"])
@pytest.mark.parametrize("case", ATT16, ids=[c["name"] for c in ATT16])
def test_attention_case_fp16(case, regime, fp16_checks):
    assert AP.case_keys(case) == case["keys"]
    APG.run_case(case, regime, seed=6000 + 2 * AP.CASES.index(case) + (regime == "grow"))


# ------------------------------------------------------------------ the 16-bit types are not mixed
# (the fp16 element-wise kernels are checked per element against float64 by tests/test_elementwise_plans_gpu.py)
def test_mixed_16bit_types_refused():
    from fast3r_b200 import ops
    a = torch.zeros(128, 64, dtype=F16, device="cuda")
    with pytest.raises(TypeError):
        ops.linear(a, torch.zeros(64, 64, dtype=torch.bfloat16, device="cuda"), out0=torch.empty(128, 64, dtype=F16,
                                                                                               device="cuda"))
    with pytest.raises(TypeError):
        ops.linear(a, torch.zeros(64, 64, dtype=F16, device="cuda"),
                   out0=torch.empty(128, 64, dtype=torch.bfloat16, device="cuda"))
    q, kv = torch.zeros(128, 64, dtype=F16, device="cuda"), torch.zeros(128, 128, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(TypeError):
        ops.attention(q, kv, torch.empty_like(q), batch=1, heads=1, sq=128, skv=128, scale=0.125)


# ------------------------------------------------------------------ the forward
def _build(tag, golden_dir):
    from fast3r_b200 import Fast3R, tiny_args
    from tests.golden.synth import synth_state_dict, synth_images
    g = torch.load(os.path.join(golden_dir, f"{tag}.pt"))
    enc, dec, head = tiny_args()
    dec.update(g.get("dec_over", {}))
    head.update(g.get("head_over", {}))
    model = Fast3R(enc, dec, head).eval()
    model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
    model = model.cuda().set_precision("fp16")
    if g.get("train_mode", False):
        model.train()
    return g, model, synth_images(g["N"], g["B"], g["H"], g["W"])


def _rel(preds, ref, k, sub=1):
    return rel_l2(torch.cat([p[k][:, ::sub, ::sub].float().cpu().flatten() for p in preds]),
                  torch.cat([q[k].float().flatten() for q in ref]))


@pytest.mark.parametrize("tag", ["tiny_b1_n3", "tiny_b2_n2", "tiny_noattnbias", "tiny_fixedidx", "tiny_nolocal_n2",
                                 "tiny_single_view", "tiny_trainmode"])
def test_tiny_fp16_vs_reference_golden(golden_dir, tag):
    g, model, imgs = _build(tag, golden_dir)
    views = [dict(img=im.cuda()) for im in imgs]
    torch.manual_seed(g["rng_seed"])
    with torch.no_grad():
        preds = model(views)
    rep = {k: _rel(preds, g["preds"], k) for k in g["preds"][0]}
    print(tag, "fp16", rep)
    for k in g["preds"][0]:
        assert preds[0][k].dtype == torch.float32 and preds[0][k].shape == g["preds"][0][k].shape
    assert all(v <= FP16_TOL for v in rep.values()), rep


@pytest.mark.parametrize("tag", ["tiny_mixed_res", "tiny_portrait"])
def test_tiny_fp16_mixed_and_portrait(golden_dir, tag):
    model = tiny_model(golden_dir).cuda().set_precision("fp16")
    views, ref, seed = scene(golden_dir, tag, "cuda")
    torch.manual_seed(seed)
    preds = model(views)
    rep = {k: _rel(preds, ref, k) for k in ref[0]}
    print(tag, "fp16", rep)
    assert all(v <= FP16_TOL for v in rep.values()), rep


def test_vitl_n4_fp16_vs_reference_golden(golden_dir):
    """ViT-L N=4 368x512 through inference() on an fp16 model: every key within FP16_TOL of the reference's fp32 result,
    and the pointmaps at most a quarter of the bf16 path's error on the same inputs."""
    from fast3r_b200 import Fast3R, inference
    from tests.test_oracle_vs_golden import vitl_n4_model_inputs
    g = torch.load(os.path.join(golden_dir, "vitl_n4_368x512.pt"))
    cfg, sd, imgs = vitl_n4_model_inputs(g)
    model = Fast3R(*cfg).eval()
    model.load_state_dict(sd)
    model = model.cuda()
    rep = {}
    for precision in ("bf16", "fp16"):
        model.set_precision(precision)
        views = [dict(img=im, true_shape=np.int32([[g["H"], g["W"]]]), idx=i, instance=str(i))
                 for i, im in enumerate(imgs)]
        torch.manual_seed(g["rng_seed"])
        res = inference(views, model, torch.device("cuda"), dtype=torch.bfloat16, verbose=False)
        assert model.precision == precision
        rep[precision] = {k: _rel(res["preds"], g["preds_sub"], k, g["stride"]) for k in g["preds_sub"][0]}
    print("vitl_n4_368x512", rep)
    assert all(v <= FP16_TOL for v in rep["fp16"].values()), rep
    for k in ("pts3d_in_other_view", "pts3d_local"):
        assert rep["fp16"][k] <= 0.25 * rep["bf16"][k], (k, rep)


def test_forward_many_fp16(golden_dir):
    """forward_many([scene]) is bit-identical to forward(scene) in fp16, and the tiny scenes packed into one call match
    their goldens within FP16_TOL."""
    from tests.packed_goldens import reseeded_ids
    model = tiny_model(golden_dir).cuda().set_precision("fp16")
    scenes = [scene(golden_dir, t, "cuda") for t in TAGS]
    for views, _, seed in scenes:
        torch.manual_seed(seed)
        ref = model(views)
        torch.manual_seed(seed)
        out, = model.forward_many([views])
        for p, q in zip(out, ref):
            for k in q:
                assert torch.equal(p[k], q[k]), k
    samples, refs, seeds = zip(*scenes)
    reseeded_ids(model, seeds)
    try:
        packed = model.forward_many(list(samples))
    finally:
        del model.decoder.draw_image_ids
    rep = {(t, k): _rel(p, r, k) for t, p, r in zip(TAGS, packed, refs) for k in r[0]}
    print("packed tiny fp16", rep)
    assert all(v <= FP16_TOL for v in rep.values()), rep


def test_fp16_forward_launch_count():
    """The fp16 forward makes exactly the launches of the bf16 forward (same plans, same kernels in another type)."""
    from fast3r_b200 import Fast3R, lib as L, vit_large_args
    from tests.golden.synth import synth_images
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = Fast3R(*vit_large_args()).eval()
    views = [dict(img=im.cuda()) for im in synth_images(4, 1, 368, 512)]
    counts = {}
    for precision in ("bf16", "fp16", "bf16"):
        model.set_precision(precision)
        model(views)  # packs the weights on the first call of each precision
        torch.cuda.synchronize()
        n0 = L.launch_count()
        model(views)
        torch.cuda.synchronize()
        counts.setdefault(precision, set()).add(L.launch_count() - n0)
    assert len(counts["bf16"]) == 1 and counts["fp16"] == counts["bf16"], counts
    assert math.prod(counts["fp16"]) > 0
