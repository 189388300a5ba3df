"""precision="fp16" without a GPU: the precision switch and inference()'s dtype rule, the refusal of a sharded fp16 model,
the launch plans of the fp16 forward (the same GEMM and attention plans as the bf16 forward, in the same order, with
every 16-bit operand fp16), and the tiny goldens through the ABI emulator (tests/abi_emulator.py) with fp16 storage."""
import os

import pytest
import torch

from tests import abi_emulator as E
from tests import attention_plans as AP
from tests import gemm_plans as GP
from tests import test_attention_plans_cpu as APC
from tests import test_gemm_plans_cpu as GPC
from tests.conftest import rel_l2
from tests.packed_goldens import TAGS, reseeded_ids, scene, tiny_model

F16, BF16 = torch.float16, torch.bfloat16
FP16_TOL = 3e-3  # tests/test_fp16_gpu.py


def _tiny():
    from fast3r_b200 import Fast3R, tiny_args
    return Fast3R(*tiny_args()).eval()


def test_set_precision_fp16():
    from fast3r_b200.model import PRECISIONS
    m = _tiny()
    assert "fp16" in PRECISIONS and m.precision == "bf16"
    assert m.set_precision("fp16") is m and m.precision == "fp16"
    for bad in ("float16", "f16", "half", "bf32", None):
        with pytest.raises(ValueError):
            m.set_precision(bad)
    assert m.precision == "fp16"


@pytest.mark.parametrize("model_precision,dtype,runs", [
    ("bf16", "32", "fp32"), ("bf16", torch.float32, "fp32"), ("bf16", torch.bfloat16, "bf16"), ("bf16", None, "bf16"),
    ("bf16", torch.float16, "bf16"),
    ("fp16", "32", "fp32"), ("fp16", torch.float32, "fp32"), ("fp16", torch.bfloat16, "fp16"), ("fp16", None, "fp16"),
    ("fp16", torch.float16, "fp16"),
])
def test_precision_scope(model_precision, dtype, runs):
    """inference()'s dtype picks the parity path or the fast path; the fast path of an fp16 model is fp16.  The model's
    own precision comes back afterwards."""
    from fast3r_b200.inference import _precision_scope, precision_of
    assert precision_of(torch.float16) == "bf16"  # unchanged: torch.float16 alone does not select fp16
    m = _tiny().set_precision(model_precision)
    with _precision_scope(m, dtype):
        assert m.precision == runs
    assert m.precision == model_precision


def test_sharded_fp16_model_refused():
    m = _tiny().set_precision("fp16")
    m.sp_group = object()  # any sequence-parallel group: refused before it is used
    views = [dict(img=torch.zeros(1, 3, 32, 48)) for _ in range(2)]
    with pytest.raises(NotImplementedError, match="fp16"):
        m(views)


# ------------------------------------------------------------------ launch plans
class _GemmRecorder(GPC.Recorder):
    """tests/test_gemm_plans_cpu.Recorder that also records the 16-bit type of each call and checks that one call does
    not mix bf16 and fp16."""

    def gemm(self, a, wt, **kw):
        types = {t.dtype for t in [a, wt] + [kw.get(k) for k in ("out0", "out0b", "out1", "res0", "res1")]
                 if t is not None and t.dtype != torch.float32}
        assert len(types) == 1, types
        super().gemm(a, wt, **kw)
        self.calls[-1] = self.calls[-1] + (types.pop(),)


class _AttnRecorder(APC.Recorder):
    """tests/test_attention_plans_cpu.Recorder that accepts the *_f16 entry points and records which form was called."""

    def _abi(self, name, anchor, *a):
        f16 = name.endswith("_f16")
        super()._abi(name[:-len("_f16")] if f16 else name, anchor, *a)
        self.calls[-1] = self.calls[-1] + (f16,)


def _gemm_calls(monkeypatch, precision, run):
    import fast3r_b200.model as M
    rec = _GemmRecorder()
    monkeypatch.setattr(M, "ops", rec)
    monkeypatch.setattr(M, "_require_cuda", lambda device: None)
    run(GPC._vitl(precision))
    return rec.calls


def _attn_calls(monkeypatch, precision, run):
    rec = _AttnRecorder(monkeypatch)
    APC._patch_model(monkeypatch, rec)
    run(APC._vitl(precision))
    return rec.calls


def _bench_forward(model):  # the benchmark forward: N = 32 views of 368x512
    torch.manual_seed(0)
    model([dict(img=torch.empty(1, 3, 368, 512, device="meta")) for _ in range(32)])


def _packed_forward(model):  # forward_many over the scenes of tests/test_attention_plans_cpu.py
    scenes = [[(368, 512)] * 4, [(384, 512)], [(512, 384)] * 2]
    model.forward_many([[dict(img=torch.empty(1, 3, h, w, device="meta")) for h, w in s] for s in scenes])


@pytest.mark.parametrize("run", [_bench_forward, _packed_forward], ids=["n32_368x512", "packed"])
def test_fp16_forward_has_the_plans_of_bf16(run):
    """The same GEMM plan keys (library rule, H100) and attention plan keys as bf16, call for call; every GEMM of the
    fp16 forward is fp16 throughout and every attention call goes to an *_f16 entry point."""
    mp = pytest.MonkeyPatch()
    try:
        g = {p: _gemm_calls(mp, p, run) for p in ("bf16", "fp16")}
        mp.undo()
        a = {p: _attn_calls(mp, p, run) for p in ("bf16", "fp16")}
    finally:
        mp.undo()
    assert len(g["fp16"]) == len(g["bf16"]) > 0
    assert [GP.plan_key(d) for d, _, _ in g["fp16"]] == [GP.plan_key(d) for d, _, _ in g["bf16"]]
    assert {t for _, _, t in g["fp16"]} == {F16} and {t for _, _, t in g["bf16"]} == {BF16}
    assert len(a["fp16"]) == len(a["bf16"]) > 0
    assert [AP.plan_keys(d) for d, _, _ in a["fp16"]] == [AP.plan_keys(d) for d, _, _ in a["bf16"]]
    assert all(f for _, _, f in a["fp16"]) and not any(f for _, _, f in a["bf16"])
    table = {k for c in AP.CASES if c["kind"] != "x3" for k in c["keys"]}
    # every one is a case that tests/test_fp16_gpu.py runs
    assert {k for d, _, _ in a["fp16"] for k in AP.plan_keys(d)} <= table


# ------------------------------------------------------------------ tiny goldens over the emulator
class _Emu16:
    """tests/abi_emulator with the fp16 cast of the hooks (a store into the fp16 tensor, like cast_bf16) and the
    block-diagonal attention as one emulated attention per segment."""

    def __getattr__(self, name):
        return getattr(E, name)

    cast_f16 = staticmethod(E.cast_bf16)

    @staticmethod
    def attention_segments(q, kv, out, seg_off, *, heads, scale, kv_split=None):
        off = seg_off.offsets
        for a, b in zip(off, off[1:]):
            if b > a:
                E.attention(q[a:b], kv[a:b], out[a:b], batch=1, heads=heads, sq=b - a, skv=b - a, scale=scale)


@pytest.fixture
def emulated(monkeypatch):
    import fast3r_b200.model as M
    monkeypatch.setattr(M, "ops", _Emu16())
    monkeypatch.setattr(M, "_require_cuda", lambda device: None)
    return M


def _err(preds, ref, k):
    return rel_l2(torch.cat([p[k].flatten() for p in preds]), torch.cat([q[k].float().flatten() for q in ref]))


@pytest.mark.parametrize("tag", ["tiny_b1_n3", "tiny_b2_n2", "tiny_nolocal_n2", "tiny_single_view"])
def test_tiny_golden_emulated_fp16(emulated, golden_dir, tag):
    """Every activation that feeds a GEMM or the attention is stored fp16 (the emulator rounds at each store); the
    predictions stay within FP16_TOL of the reference's fp32 result, and closer to it than with bf16 storage."""
    from fast3r_b200 import tiny_args
    from tests.golden.synth import synth_state_dict, synth_images
    g = torch.load(os.path.join(golden_dir, f"{tag}.pt"))
    enc, dec, head = tiny_args()
    dec.update(g.get("dec_over", {}))
    head.update(g.get("head_over", {}))
    model = emulated.Fast3R(enc, dec, head).eval()
    model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
    imgs = synth_images(g["N"], g["B"], g["H"], g["W"])
    rep = {}
    for precision in ("bf16", "fp16"):
        model.set_precision(precision)
        torch.manual_seed(g["rng_seed"])
        preds = model([dict(img=im) for im in imgs])
        rep[precision] = {k: _err(preds, g["preds"], k) for k in g["preds"][0]}
    print(tag, rep)
    assert all(v <= FP16_TOL for v in rep["fp16"].values()), rep
    for k in ("pts3d_in_other_view", "pts3d_local"):
        if k in rep["fp16"]:
            assert rep["fp16"][k] < rep["bf16"][k], (k, rep)


def test_packed_tiny_goldens_emulated_fp16(emulated, golden_dir):
    model = tiny_model(golden_dir, emulated).set_precision("fp16")
    samples, refs, seeds = zip(*[scene(golden_dir, t) for t in TAGS])
    reseeded_ids(model, seeds)
    packed = model.forward_many(list(samples))
    rep = {(t, k): _err(p, r, k) for t, p, r in zip(TAGS, packed, refs) for k in r[0]}
    assert all(v <= FP16_TOL for v in rep.values()), rep
