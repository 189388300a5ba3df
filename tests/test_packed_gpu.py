"""Several scenes in one forward on the GPU: the segmented attention kernel (f3r_attention_segments) against single-
segment launches (bit for bit), an fp32 reference and poisoned neighbours; Fast3R.forward_many / inference_many against
forward and the reference fixtures.  Needs an H100."""
import math
import os
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.conftest import rel_l2  # noqa: E402
from tests.kernel_checks import attention_ref  # noqa: E402
from tests.packed_goldens import TAGS, reseeded_ids, scene, tiny_model  # noqa: E402

HEADS = 16
DEC_SCALE = 64 ** -0.5 * (math.log(137) / math.log(20)) ** 0.5
ENC_SCALE = 64 ** -0.5
LENGTHS = [1, 127, 128, 129, 191, 192, 193, 384, 736, 2944, 23552]
ATT_TOL = 8e-3        # tests/kernel_checks.check_attention
PARITY_TOL, BF16_TOL = 1e-3, 1.3e-2   # tests/test_model_gpu.py
PACK_VS_FORWARD = {"fp32": 1e-5, "bf16": 5e-3}


def _segment_lists():
    """Mixed orders of the lengths: all of them, shuffled; the short ones only (with repeats); and one long segment
    between short ones."""
    rnd = random.Random(17)
    every = list(LENGTHS)
    rnd.shuffle(every)
    short = [rnd.choice(LENGTHS[:9]) for _ in range(12)]
    return [every, short, [129, 23552, 1, 736]]


def _operands(rows, seed):
    g = torch.Generator().manual_seed(seed)
    D = HEADS * 64
    return (torch.randn(rows, D, generator=g).bfloat16().cuda(), torch.randn(rows, 2 * D, generator=g).bfloat16().cuda())


def _offsets(lens):
    off = [0]
    for n in lens:
        off.append(off[-1] + n)
    return off


def _ref(q, kv, scale):
    """fp32 attention of one segment, per head and in query chunks (the score matrix of 23552 rows does not fit)."""
    D = HEADS * 64
    out = torch.empty(q.shape[0], D, device="cuda")
    for h in range(HEADS):
        k, v = kv[:, h * 64:(h + 1) * 64], kv[:, D + h * 64:D + (h + 1) * 64]
        for a in range(0, q.shape[0], 4096):
            out[a:a + 4096, h * 64:(h + 1) * 64] = attention_ref(q[a:a + 4096, h * 64:(h + 1) * 64], k, v, scale)
    return out


@pytest.mark.parametrize("scale", [DEC_SCALE, ENC_SCALE], ids=["decoder", "encoder"])
@pytest.mark.parametrize("lens", _segment_lists(), ids=["all_lengths", "short", "long_between_short"])
def test_segments_bit_identical_to_single_segment_launches(lens, scale):
    from fast3r_b200 import ops
    off = _offsets(lens)
    rows = off[-1]
    q, kv = _operands(rows, seed=rows)
    seg = ops.Segments(off, q.device)
    worst = 0.0
    for ks in (1, 3):
        out = torch.full((rows, HEADS * 64), float("nan"), dtype=torch.bfloat16, device="cuda")
        ops.attention_segments(q, kv, out, seg, heads=HEADS, scale=scale, kv_split=ks)
        for a, b in zip(off, off[1:]):
            one = torch.empty(b - a, HEADS * 64, dtype=torch.bfloat16, device="cuda")
            ops.attention(q[a:b], kv[a:b], one, batch=1, heads=HEADS, sq=b - a, skv=b - a, scale=scale,
                          kv_split=min(ks, -(-(b - a) // 128)))
            assert torch.equal(out[a:b], one), (ks, a, b)
            if ks == 1:
                e = rel_l2(out[a:b].float(), _ref(q[a:b], kv[a:b], scale))
                worst = max(worst, e)
                assert e < ATT_TOL, (a, b, e)
    print("segments", lens, "worst rel-L2 vs fp32", worst)


def test_single_segment_picks_the_split_of_attention():
    """kv_split=None: one segment gets the key split ops.attention picks for it (what forward_many([s]) relies on)."""
    from fast3r_b200 import ops
    for n in (736, 2944, 23552):
        q, kv = _operands(n, seed=n + 1)
        a, b = (torch.empty(n, HEADS * 64, dtype=torch.bfloat16, device="cuda") for _ in range(2))
        ops.attention_segments(q, kv, a, [0, n], heads=HEADS, scale=DEC_SCALE)
        ops.attention(q, kv, b, batch=1, heads=HEADS, sq=n, skv=n, scale=DEC_SCALE)
        assert torch.equal(a, b), n


@pytest.mark.parametrize("ks", [1, 3])
def test_poisoned_neighbours_change_nothing(ks):
    """NaN and +-Inf in the q / k / v rows of the other segments leave a segment's output unchanged, bit for bit."""
    from fast3r_b200 import ops
    lens = _segment_lists()[0]
    off = _offsets(lens)
    rows = off[-1]
    q, kv = _operands(rows, seed=5)
    seg = ops.Segments(off, q.device)
    clean = torch.empty(rows, HEADS * 64, dtype=torch.bfloat16, device="cuda")
    ops.attention_segments(q, kv, clean, seg, heads=HEADS, scale=DEC_SCALE, kv_split=ks)
    poison = torch.tensor([float("nan"), float("inf"), -float("inf")], device="cuda").bfloat16()
    for parity in (0, 1):  # poison the odd segments, then the even ones
        qp, kvp = q.clone(), kv.clone()
        for s, (a, b) in enumerate(zip(off, off[1:])):
            if s % 2 != parity:
                qp[a:b] = poison[torch.arange(qp[a:b].numel(), device="cuda") % 3].view(b - a, -1)
                kvp[a:b] = poison[torch.arange(kvp[a:b].numel(), device="cuda") % 3].view(b - a, -1)
        out = torch.empty_like(clean)
        ops.attention_segments(qp, kvp, out, seg, heads=HEADS, scale=DEC_SCALE, kv_split=ks)
        for s, (a, b) in enumerate(zip(off, off[1:])):
            if s % 2 == parity:
                assert torch.equal(out[a:b], clean[a:b]), (parity, s, a, b)


_LAUNCH_COUNT = """
import json, sys
import torch
from fast3r_b200 import lib as L, ops
ks, path = int(sys.argv[1]), sys.argv[2]
off = [0, 736, 737, 3681]
g = torch.Generator().manual_seed(9)
q = torch.randn(off[-1], 1024, generator=g).bfloat16().cuda()
kv = torch.randn(off[-1], 2048, generator=g).bfloat16().cuda()
out = torch.empty(off[-1], 1024, dtype=torch.bfloat16, device="cuda")
seg = ops.Segments(off, q.device)
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    n0 = L.launch_count()
    ops.attention_segments(q, kv, out, seg, heads=16, scale=0.16, kv_split=ks)
    torch.cuda.synchronize()
    n = L.launch_count() - n0
prof.export_chrome_trace(path)
kernels = [e["name"] for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
print(json.dumps([n, kernels]))
"""


@pytest.mark.parametrize("ks", [1, 2])
def test_launch_count(ks, tmp_path):
    """lib.launch_count() against the CUDA trace (as tests/test_launch_count_gpu.py) for one call: one launch, plus the
    merge with key slices.  The trace is taken in a fresh process: after the long kernels of the tests above, the
    profiler of this process has been seen to record no kernel of a short traced window at all."""
    import json
    import subprocess
    import sys
    from tests.conftest import ROOT
    r = subprocess.run([sys.executable, "-c", _LAUNCH_COUNT, str(ks), str(tmp_path / "trace.json")], cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    n, kernels = json.loads(r.stdout.strip().splitlines()[-1])
    traced = [k for k in kernels if "f3r" in k]
    assert n == len(traced) == (1 if ks == 1 else 2), (n, kernels)


# ------------------------------------------------------------------ model
def _run(model, samples, seeds, packed):
    if packed:
        reseeded_ids(model, seeds)
        try:
            return model.forward_many(samples)
        finally:
            del model.decoder.draw_image_ids  # back to the class's method
    out = []
    for s, seed in zip(samples, seeds):
        torch.manual_seed(seed)
        out.append(model(s))
    return out


def _err(a, b, k):
    return rel_l2(torch.cat([p[k].float().cpu().flatten() for p in a]), torch.cat([p[k].float().cpu().flatten() for p in b]))


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_one_sample_bit_identical_to_forward(golden_dir, precision):
    from fast3r_b200 import Fast3R, tiny_args
    from tests.golden.synth import synth_state_dict
    model = tiny_model(golden_dir).cuda().set_precision(precision)
    for tag in TAGS:
        views, _, seed = scene(golden_dir, tag, "cuda")
        ref, = _run(model, [views], [seed], packed=False)
        out, = _run(model, [views], [seed], packed=True)
        for p, q in zip(out, ref):
            for k in q:
                assert torch.equal(p[k], q[k]), (tag, k)
    for tag in ("tiny_b1_n3", "tiny_noattnbias", "tiny_fixedidx", "tiny_nolocal_n2", "tiny_trainmode"):
        g = torch.load(os.path.join(golden_dir, f"{tag}.pt"))
        enc, dec, head = tiny_args()
        dec.update(g.get("dec_over", {}))
        head.update(g.get("head_over", {}))
        m = Fast3R(enc, dec, head).eval()
        m.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
        m = m.cuda().set_precision(precision)
        if g.get("train_mode", False):
            m.train()
        views = scene(golden_dir, tag, "cuda")[0]
        with torch.no_grad():
            ref, = _run(m, [views], [7], packed=False)
            torch.manual_seed(7)
            out, = m.forward_many([views])
        for p, q in zip(out, ref):
            for k in q:
                assert torch.equal(p[k], q[k]), (tag, k)


@pytest.mark.parametrize("precision,tol", [("bf16", BF16_TOL), ("fp32", PARITY_TOL)])
def test_packed_tiny_goldens(golden_dir, precision, tol):
    model = tiny_model(golden_dir).cuda().set_precision(precision)
    scenes = [scene(golden_dir, t, "cuda") for t in TAGS]
    samples, refs, seeds = zip(*scenes)
    packed = _run(model, samples, seeds, packed=True)
    loop = _run(model, samples, seeds, packed=False)
    rep = {}
    for tag, ref, a, b in zip(TAGS, refs, packed, loop):
        for k in ref[0]:
            rep[(tag, k)] = (_err(a, ref, k), _err(a, b, k))
    print("packed tiny", precision, {f"{t}:{k}": f"golden {e[0]:.2e} vs forward {e[1]:.2e}" for (t, k), e in rep.items()})
    for key, (golden, forward) in rep.items():
        assert golden <= tol, (key, golden)
        assert forward <= PACK_VS_FORWARD[precision], (key, forward)


def test_vitl_n4_packed_with_other_shapes(golden_dir):
    """The ViT-L N=4 368x512 fixture scene packed with a 1-view 384x512 and a 2-view 512x384 scene, through
    inference_many: the fixture scene stays within its golden tolerances; forward_many([scene]) is bit-identical to
    forward(scene)."""
    import numpy as np
    from fast3r_b200 import Fast3R, inference_many
    from tests.golden.synth import synth_images
    from tests.test_oracle_vs_golden import vitl_n4_model_inputs
    g = torch.load(os.path.join(golden_dir, "vitl_n4_368x512.pt"))
    cfg, sd, imgs = vitl_n4_model_inputs(g)
    model = Fast3R(*cfg).eval()
    model.load_state_dict(sd)
    model = model.cuda()
    st = g["stride"]
    for precision in ("fp32", "bf16"):
        model.set_precision(precision)
        views = [dict(img=im.cuda()) for im in imgs]
        torch.manual_seed(g["rng_seed"])
        ref = model(views)
        torch.manual_seed(g["rng_seed"])
        one, = model.forward_many([views])
        for p, q in zip(one, ref):
            for k in q:
                assert torch.equal(p[k], q[k]), (precision, k)
    rep = {}
    for dt, tol in (("32", PARITY_TOL), (torch.bfloat16, BF16_TOL)):
        def views_of(ims, h, w):
            return [dict(img=im, true_shape=np.int32([[h, w]]), idx=i, instance=str(i)) for i, im in enumerate(ims)]
        samples = [views_of(imgs, g["H"], g["W"]), views_of(synth_images(1, 1, 384, 512, seed0=77), 384, 512),
                   views_of(synth_images(2, 1, 512, 384, seed0=78), 512, 384)]
        torch.manual_seed(g["rng_seed"])  # the fixture scene draws first, from the fixture's seed
        res = inference_many(samples, model, torch.device("cuda"), dtype=dt, verbose=False)
        assert [len(r["preds"]) for r in res] == [4, 1, 2]
        assert res[1]["preds"][0]["pts3d_in_other_view"].shape == (1, 384, 512, 3)
        assert res[2]["preds"][1]["conf"].shape == (1, 512, 384)
        rep[str(dt)] = {k: rel_l2(torch.cat([p[k][:, ::st, ::st].flatten() for p in res[0]["preds"]]),
                                  torch.cat([q[k].flatten() for q in g["preds_sub"]])) for k in g["preds_sub"][0]}
        assert all(v <= tol for v in rep[str(dt)].values()), rep
    print("vitl_n4 packed with 1x384x512 + 2x512x384", rep)
