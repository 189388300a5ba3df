"""Host logic of Fast3R.forward_many / inference_many on the CPU: the kernels are replaced by tests/abi_emulator.py, with
f3r_attention_segments emulated by one emulated attention per segment (its contract: each segment exactly as a
single-segment attention over it alone).  Packing, image-id draws, regrouping by shape, splitting back per sample and
the refusals are the product code."""
import ctypes as C
import types

import pytest
import torch

from tests.conftest import rel_l2
from tests.packed_goldens import TAGS, reseeded_ids, scene, tiny_model

EMU_TOL = {"bf16": 2e-2, "fp32": 1e-3}  # emulator vs fixtures, as in tests/test_host_orchestration_cpu.py
MIXED_TOL = {"bf16": 3e-2, "fp32": 1e-3}


@pytest.fixture()
def emulated(monkeypatch):
    """fast3r_b200.model over the ABI emulator plus attention_segments; returns (module, list of segment calls)."""
    import fast3r_b200.model as M
    from fast3r_b200.ops import Segments
    from tests import abi_emulator as E
    calls = []

    def attention_segments(q, kv, out, seg_off, *, heads, scale, kv_split=None):
        offs = seg_off.offsets if isinstance(seg_off, Segments) else [int(v) for v in seg_off]
        calls.append(list(offs))
        for a, b in zip(offs, offs[1:]):
            E.attention(q[a:b], kv[a:b], out[a:b], batch=1, heads=heads, sq=b - a, skv=b - a, scale=scale)

    ops = types.SimpleNamespace(**{k: v for k, v in vars(E).items() if not k.startswith("__")})
    ops.attention_segments = attention_segments
    monkeypatch.setattr(M, "ops", ops)
    monkeypatch.setattr(M, "_require_cuda", lambda device: None)
    return M, calls


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_packed_goldens_match_fixtures(emulated, golden_dir, precision):
    M, calls = emulated
    model = tiny_model(golden_dir, M).set_precision(precision)
    scenes = [scene(golden_dir, t) for t in TAGS]
    reseeded_ids(model, [s[2] for s in scenes])
    preds = model.forward_many([s[0] for s in scenes])
    assert len(preds) == len(TAGS)
    for tag, (views, ref, _), out in zip(TAGS, scenes, preds):
        assert len(out) == len(views) == len(ref)
        tol = (MIXED_TOL if tag == "tiny_mixed_res" else EMU_TOL)[precision]
        for i, q in enumerate(ref):
            assert sorted(out[i]) == sorted(q), tag
            for k in q:
                assert out[i][k].shape == q[k].shape and out[i][k].dtype == torch.float32, (tag, i, k)
        for k in ref[0]:
            err = rel_l2(torch.cat([p[k].flatten() for p in out]), torch.cat([p[k].flatten() for p in ref]))
            assert err < tol, (tag, k, err)
    # bf16: one segmented attention per decoder layer, one segment per scene
    n_tok = [sum(v["img"].shape[-2] * v["img"].shape[-1] // 256 for v in s[0]) for s in scenes]
    expect = [0] + [sum(n_tok[:i + 1]) for i in range(len(n_tok))]
    assert calls == ([expect] * model.decoder.depth if precision == "bf16" else [])


def test_single_sample_equals_forward(emulated, golden_dir):
    M, _ = emulated
    model = tiny_model(golden_dir, M)
    for tag in TAGS:
        views, _, seed = scene(golden_dir, tag)
        torch.manual_seed(seed)
        ref = model(views)
        torch.manual_seed(seed)
        out, = model.forward_many([views])
        for p, q in zip(out, ref):
            assert sorted(p) == sorted(q)
            for k in q:
                assert torch.equal(p[k], q[k]), (tag, k)


@pytest.mark.parametrize("n_samples", [1, 2, 5])
def test_rng_and_one_segment_call_per_layer(emulated, golden_dir, n_samples):
    """Ids drawn and the RNG state left behind are those of forward on each sample in turn; the decoder makes one
    segmented attention call per layer whatever the number of samples."""
    M, calls = emulated
    model = tiny_model(golden_dir, M)
    samples = [scene(golden_dir, TAGS[k % len(TAGS)])[0] for k in range(n_samples)]
    drawn = []
    draw = model.decoder.draw_image_ids

    def recording(*a, **kw):
        drawn.append(draw(*a, **kw))
        return drawn[-1]

    model.decoder.draw_image_ids = recording
    torch.manual_seed(123)
    loop = [model(s) for s in samples]
    loop_ids, loop_state = list(drawn), torch.get_rng_state()
    drawn.clear()
    calls.clear()
    torch.manual_seed(123)
    packed = model.forward_many(samples)
    assert len(drawn) == n_samples
    assert all(torch.equal(a, b) for a, b in zip(drawn, loop_ids))
    assert torch.equal(torch.get_rng_state(), loop_state)
    assert len(calls) == model.decoder.depth and len(calls[0]) == n_samples + 1
    for a, b in zip(packed, loop):  # the emulator's matmuls round differently for other row counts (as in the
        # sequence-parallel test of tests/test_host_orchestration_cpu.py)
        for p, q in zip(a, b):
            for k in q:
                assert rel_l2(p[k], q[k]) < 1e-2, k


def test_profiling_info(emulated, golden_dir):
    M, _ = emulated
    model = tiny_model(golden_dir, M)
    samples = [scene(golden_dir, t)[0] for t in TAGS[:2]]
    preds, info = model.forward_many(samples, profiling=True)
    assert len(preds) == 2
    assert set(info) == {"encode_images_time", "pos_emb_time", "decoder_time", "head_prepare_input_time",
                         "head_forward_time", "total_time"}


def test_refusals(emulated, golden_dir):
    M, _ = emulated
    model = tiny_model(golden_dir, M)
    views = scene(golden_dir, "tiny_b1_n3")[0]
    with pytest.raises(ValueError, match="empty sample list"):
        model.forward_many([])
    with pytest.raises(ValueError, match="no views"):
        model.forward_many([views, []])
    b2 = [dict(img=torch.cat([v["img"], v["img"]])) for v in views]
    with pytest.raises(ValueError, match="batch size 1"):
        model.forward_many([views, b2])
    model.sp_group = object()
    with pytest.raises(NotImplementedError, match="sequence-parallel"):
        model.forward_many([views])


def test_inference_many_structure(emulated, golden_dir):
    """Element i of inference_many has the structure of inference(samples[i]) and its values up to the emulator's
    rounding for other row counts."""
    import numpy as np
    from fast3r_b200 import inference, inference_many
    M, _ = emulated
    model = tiny_model(golden_dir, M)

    def samples():
        out = []
        for t in TAGS:
            views = scene(golden_dir, t)[0]
            out.append([dict(v, idx=i, instance=str(i), true_shape=v.get("true_shape", np.int32([v["img"].shape[-2:]])))
                        for i, v in enumerate(views)])
        return out

    torch.manual_seed(5)
    loop = [inference(s, model, torch.device("cpu"), dtype=torch.bfloat16, verbose=False) for s in samples()]
    torch.manual_seed(5)
    packed = inference_many(samples(), model, torch.device("cpu"), dtype=torch.bfloat16, verbose=False)
    assert len(packed) == len(loop)
    for a, b in zip(packed, loop):
        assert sorted(a) == sorted(b) == ["loss", "preds", "views"] and a["loss"] is None
        assert [sorted(v) for v in a["views"]] == [sorted(v) for v in b["views"]]
        for p, q in zip(a["preds"], b["preds"]):
            assert sorted(p) == sorted(q)
            for k in q:
                assert p[k].device.type == "cpu" and p[k].shape == q[k].shape
                assert rel_l2(p[k], q[k]) < 1e-2, k


def test_segments_validation():
    from fast3r_b200.ops import Segments
    s = Segments([0, 5, 5, 12], "cpu")
    assert s.rows == 12 and s.lengths() == [5, 0, 7] and s.device_offsets.dtype == torch.int32
    for bad in ([0], [1, 4], [0, 5, 3]):
        with pytest.raises(ValueError):
            Segments(bad, "cpu")


def test_cabi_attention_segments_rejects_bad_arguments():
    """Argument checks of f3r_attention_segments run before any CUDA call (no GPU needed)."""
    from fast3r_b200 import lib as L
    lib = L.load()
    f = C.c_float(0.125)
    P = 256  # any 4-byte-aligned non-null pointer: the checks fail before it is dereferenced
    cases = [
        ((None, 128, P, 256, P, 128, P, 1, 100, 2, f, 1, None, None), "null operand"),
        ((P, 128, P, 256, P, 128, None, 1, 100, 2, f, 1, None, None), "null operand"),
        ((P, 128, P, 256, P, 128, P + 2, 1, 100, 2, f, 1, None, None), "not 4-byte aligned"),
        ((P, 128, P, 256, P, 128, P, 0, 100, 2, f, 1, None, None), "bad shape"),
        ((P, 120, P, 256, P, 128, P, 1, 100, 2, f, 1, None, None), "bad leading dimensions"),
        ((P, 128, P, 256, P, 128, P, 1, 100, 2, f, 2, None, None), "n_split=2 must be in"),
        ((P, 128, P, 256, P, 128, P, 1, 300, 2, f, 2, None, None), "part_o / part_lse needed"),
        ((P, 128, P, 256, P, 128, P, 1, 300, 2, f, 2, P, None), "given together"),
        ((P, 128, P, 256, None, 128, P, 1, 300, 2, f, 1, None, None), "null operand"),
    ]
    for args, msg in cases:
        assert lib.f3r_attention_segments(*args, None) != 0, msg
        err = lib.f3r_last_error().decode()
        assert err.startswith("f3r_attention_segments") and msg in err, (msg, err)
