"""CPU side of the whole-forward checks of tests/test_forward_fp64_gpu.py.

* The slice checker (oracle/forward_slices.py) catches localized errors that the relative L2 over all views lets through.
* The float64 oracle agrees with the default float32 oracle, whose default call is unchanged.
* The host composition at large view counts (head chunks of 25 and 8, a chunk boundary inside a view, two encoder
  chunks, mixed shape groups, forward_many, the host sink of inference()) runs over the C-ABI emulator
  (tests/abi_emulator.py) and is checked slice by slice against the float64 oracle, in bf16 and on the parity path.
* Every host branch of that composition is reached by some GPU case of tests/forward_cases.py: each case runs here at
  small image sizes with its own view counts, batch size, shape groups, entry point and precisions, and the branches it
  takes are recorded from the calls the host code makes."""
import math
import types

import numpy as np
import pytest
import torch

from oracle import forward_slices as FS
from tests.conftest import rel_l2
from tests.forward_cases import BRANCHES, CASES, L368, L384, P512, scene_images, state_dict

# ------------------------------------------------------------------ checker sensitivity
NOISE = {"fp32": 1e-4, "bf16": 3e-3}  # relative noise of a healthy run, well inside T and spread evenly
CONCAT_TOL = {"fp32": 1e-3, "bf16": 1.3e-2}  # the suite's relative-L2 tolerance over all views concatenated
V, H, W = 32, 368, 512


def _field():
    """A smooth pointmap-like reference (V, H, W, 3) and conf (V, H, W) = 1 + exp(c): sums of a few sinusoids with
    wavelengths of 40 to 200 pixels, a different phase per view."""
    g = torch.Generator().manual_seed(0)
    y = torch.arange(H, dtype=torch.float64)[:, None]
    x = torch.arange(W, dtype=torch.float64)[None, :]
    pts = torch.empty(V, H, W, 3, dtype=torch.float64)
    c = torch.empty(V, H, W, dtype=torch.float64)
    for v in range(V):
        ph = torch.rand(8, generator=g, dtype=torch.float64) * 2 * math.pi
        pts[v, ..., 0] = torch.sin(2 * math.pi * x / 97 + ph[0]) + 0.5 * torch.cos(2 * math.pi * y / 41 + ph[1])
        pts[v, ..., 1] = torch.cos(2 * math.pi * y / 73 + ph[2]) + 0.5 * torch.sin(2 * math.pi * (x + y) / 53 + ph[3])
        pts[v, ..., 2] = 2 + torch.sin(2 * math.pi * x / 199 + ph[4]) * torch.cos(2 * math.pi * y / 151 + ph[5])
        c[v] = 0.5 * torch.sin(2 * math.pi * x / 61 + ph[6]) + 0.5 * torch.cos(2 * math.pi * y / 47 + ph[7]) - 1.0
    return pts, 1 + c.exp()


@pytest.fixture(scope="module")
def field():
    return _field()


def _noisy(ref, level, seed, conf=False):
    g = torch.Generator().manual_seed(seed)
    base = ref - 1 if conf else ref
    s = base.square().mean(dim=tuple(range(1, ref.dim())), keepdim=True).sqrt()
    return ref + NOISE[level] * s * torch.randn(ref.shape, generator=g, dtype=torch.float64)


def _shift_row(t, v=5, r=200):
    t = t.clone()
    t[v, r] = torch.roll(t[v, r], 1, dims=0)
    return t


def _swap_block(t, v=9, by=10, bx=14):
    t = t.clone()
    a = t[v, by * 16:(by + 1) * 16, bx * 16:(bx + 1) * 16].clone()
    t[v, by * 16:(by + 1) * 16, bx * 16:(bx + 1) * 16] = t[v, by * 16:(by + 1) * 16, (bx + 1) * 16:(bx + 2) * 16]
    t[v, by * 16:(by + 1) * 16, (bx + 1) * 16:(bx + 2) * 16] = a
    return t


def _scale_phase(t, eps):
    t = t.clone()
    t[:, :, 15::16] *= 1 + eps
    return t


def _scale_view(t, eps, v=17):
    t = t.clone()
    t[v] *= 1 + eps
    return t


# (name, level, output, perturbation of "ours"); each must fail check and pass the concatenated relative L2
PERTURB = [
    ("view_scaled_1e-3", "fp32", "pts3d", lambda t: _scale_view(t, 1e-3)),
    ("row_shifted_1px", "fp32", "pts3d", _shift_row),
    ("row_shifted_1px", "bf16", "pts3d", _shift_row),
    ("block_swapped", "bf16", "pts3d", _swap_block),
    ("phase_x15_scaled", "fp32", "pts3d", lambda t: _scale_phase(t, 2e-3)),
    ("phase_x15_scaled", "bf16", "pts3d", lambda t: _scale_phase(t, 4e-2)),
    ("conf_minus_1_view_scaled_1e-2", "fp32", "conf", lambda t: 1 + _scale_view(t - 1, 1e-2)),
]


@pytest.mark.parametrize("level", ["fp32", "bf16"])
def test_checker_passes_healthy_noise(field, level):
    pts, conf = field
    rep = FS.check_all({"pts3d": (_noisy(pts, level, 1), pts), "conf": (_noisy(conf, level, 2, conf=True), conf)},
                       level, "healthy")
    assert max(r["of_T"] for o in rep.values() for r in o.values()) < 0.5
    assert max(r["of_median"] for o in rep.values() for r in o.values()) < 1.5


@pytest.mark.parametrize("name,level,out,perturb", PERTURB, ids=[f"{p[0]}-{p[1]}" for p in PERTURB])
def test_checker_catches_what_concatenated_l2_misses(field, name, level, out, perturb):
    pts, conf = field
    ref = pts if out == "pts3d" else conf
    ours = perturb(_noisy(ref, level, 3, conf=out == "conf"))
    assert rel_l2(ours, ref) < CONCAT_TOL[level], (name, rel_l2(ours, ref))  # the gap: the old check passes
    with pytest.raises(AssertionError, match="out of bounds"):
        FS.check(ours, ref, level, out)


def test_checker_reports_worst_slice(field):
    pts, _ = field
    ours = _shift_row(_noisy(pts, "fp32", 4), v=3, r=77)
    with pytest.raises(AssertionError, match=r"view 3 row 77: .* > T"):
        FS.check(ours, pts, "fp32", "pts3d")


# ------------------------------------------------------------------ float64 oracle
def test_fp64_oracle_matches_fp32_oracle():
    from oracle import fast3r_oracle as O
    cfg, sd = state_dict("tiny", 1.0)
    imgs = scene_images([[(48, 64)] * 3], 2)[0]
    torch.manual_seed(5)
    a = O.forward(sd, *cfg, imgs)
    torch.manual_seed(5)
    b = O.forward(sd, *cfg, imgs, dtype=torch.float32, device="cpu")
    torch.manual_seed(5)
    c = O.forward(sd, *cfg, imgs, dtype=torch.float64, head_chunk=4)
    for p, q, r in zip(a, b, c):
        for k in p:
            assert p[k].dtype == torch.float32 and r[k].dtype == torch.float64
            assert torch.equal(p[k], q[k]), k  # the explicit defaults are the default call
            # fp32 against fp64: the float32 oracle's own rounding, ~1e-6 relative on this shape
            assert rel_l2(p[k], r[k]) < 2e-5, (k, rel_l2(p[k], r[k]))
    for k in a[0]:  # per slice: far inside the parity bound
        rep = FS.check(torch.cat([p[k] for p in a]), torch.cat([r[k] for r in c]), "fp32", k)
        assert max(v["of_T"] for v in rep.values()) < 0.05, (k, rep)


def test_oracle_head_chunks_are_per_image():
    from oracle import fast3r_oracle as O
    cfg, sd = state_dict("tiny", 1.0)
    imgs = scene_images([[(32, 48)] * 5], 1)[0]
    out = []
    for chunk in (None, 2):
        torch.manual_seed(5)
        out.append(O.forward(sd, *cfg, imgs, dtype=torch.float64, head_chunk=chunk))
    for p, q in zip(*out):
        for k in p:
            assert rel_l2(p[k], q[k]) < 1e-12, k


# ------------------------------------------------------------------ host composition over the emulator
class _SinkCheck:
    """Stands in for inference()'s host sink: at each chunk_done it snapshots the announced rows [start, start+count)
    of every buffer.  ``verify`` asserts that the chunks of each buffer tile it exactly once and that every row was
    final when announced (a chunk announced before its heads ran, or with a wrong start, fails)."""

    def __init__(self):
        self.snaps = {}

    def chunk_done(self, tensors, start, count):
        for t in tensors:
            key = (t.untyped_storage().data_ptr(), t.storage_offset())
            self.snaps.setdefault(key, (t, []))[1].append((start, count, t[start:start + count].clone()))

    def verify(self):
        for t, chunks in self.snaps.values():
            rows = sorted((s, c) for s, c, _ in chunks)
            ends = [0] + [s + c for s, c in rows]
            assert [s for s, _ in rows] == ends[:-1] and ends[-1] == t.shape[0], rows
            for s, c, snap in chunks:
                assert torch.equal(snap, t[s:s + c]), (s, c)
        return len(self.snaps)


class _Record:
    """Host branches taken, read off the calls the product code makes (ops namespace and Fast3R methods wrapped)."""

    def __init__(self, model, ops):
        self.seen = set()
        self._n_patch = 0
        self._enc_calls = 0
        self._B = 1
        im2col = ops.im2col_patch

        def im2col_patch(img, out):
            self._n_patch += 1
            return im2col(img, out)

        ops.im2col_patch = im2col_patch
        fwd, enc, dec, pack, dpt = model._forward, model._encode, model._decode, model._pack_tokens, model._dpt

        def _forward(samples, profiling=False, packed=False):
            self._enc_calls = 0
            r = fwd(samples, profiling, packed)
            if self._enc_calls > 1:
                self.seen.add("groups>1")
            return r

        def _encode(imgs, P_):
            n0 = self._n_patch
            self._enc_calls += 1
            r = enc(imgs, P_)
            if self._n_patch - n0 > 1:
                self.seen.add("encoder_chunks>1")
            return r

        def _decode(feats, ids, B, *a, **kw):
            self._B = B
            if B > 1:
                self.seen.add("batch>1")
            return dec(feats, ids, B, *a, **kw)

        def _pack_tokens(*a, **kw):
            self.seen.add("packed")
            return pack(*a, **kw)

        def _dpt(hooked, nv, gh, gw, H_, W_, hw, pts, conf):
            start = pts.storage_offset() // pts[0].numel()  # pts is rows [start, start+nv) of the group's buffer
            if start > 0:
                self.seen.add("head_chunks>1")
            if start % self._B:
                self.seen.add("head_chunk_splits_view")
            return dpt(hooked, nv, gh, gw, H_, W_, hw, pts, conf)

        model._forward, model._encode, model._decode = _forward, _encode, _decode
        model._pack_tokens, model._dpt = _pack_tokens, _dpt


@pytest.fixture()
def emulated(monkeypatch):
    """fast3r_b200.model over the ABI emulator, with attention_segments as one emulated attention per segment (its
    contract) and the fp16 hook cast as a store."""
    import fast3r_b200.model as M
    from fast3r_b200.ops import Segments
    from tests import abi_emulator as E

    def attention_segments(q, kv, out, seg_off, *, heads, scale, kv_split=None):
        offs = seg_off.offsets if isinstance(seg_off, Segments) else [int(v) for v in seg_off]
        for a, b in zip(offs, offs[1:]):
            E.attention(q[a:b], kv[a:b], out[a:b], batch=1, heads=heads, sq=b - a, skv=b - a, scale=scale)

    ops = types.SimpleNamespace(**{k: v for k, v in vars(E).items() if not k.startswith("__")})
    ops.attention_segments, ops.cast_f16 = attention_segments, E.cast_bf16
    monkeypatch.setattr(M, "ops", ops)
    monkeypatch.setattr(M, "_require_cuda", lambda device: None)
    return M, ops


def _run(M, ops, case, precision, imgs_per_scene, sink=None):
    """Runs a case's composition on the emulator; returns (per-view preds of all scenes, branches seen)."""
    from fast3r_b200 import inference, inference_many
    cfg, sd = state_dict(case["model_cpu"], case["gain"], M)
    model = M.Fast3R(*cfg).eval()
    model.load_state_dict(sd)
    model.set_precision(precision)
    rec = _Record(model, ops)
    dtype = "32" if precision == "fp32" else torch.bfloat16
    torch.manual_seed(7)
    entry = case["entry"]
    if entry in ("inference", "inference_many"):
        model._host_sink = sink if sink is not None else _SinkCheck()
        samples = [[dict(img=im, true_shape=np.int32([list(im.shape[-2:])] * im.shape[0]), idx=i, instance=str(i))
                    for i, im in enumerate(imgs)] for imgs in imgs_per_scene]
        if entry == "inference":
            preds = inference(samples[0], model, torch.device("cpu"), dtype=dtype, verbose=False)["preds"]
        else:
            preds = [p for r in inference_many(samples, model, torch.device("cpu"), dtype=dtype, verbose=False)
                     for p in r["preds"]]
        if sum(len(c) for _, c in model._host_sink.snaps.values()) > len(model._host_sink.snaps):
            rec.seen.add("sink_chunks>1")
        model._host_sink.verify()
    elif entry == "forward_many":
        preds = [p for s in model.forward_many([[dict(img=im) for im in imgs] for imgs in imgs_per_scene]) for p in s]
    else:
        preds, = [model([dict(img=im) for im in imgs]) for imgs in imgs_per_scene]
    return preds, rec.seen


# the same compositions as the GPU cases at small images (64x96 and friends), plus N=257 at 32x32 for two encoder chunks
SMALL = {L368: (64, 96), L384: (64, 128), P512: (96, 64)}
EMU_CASES = {
    "n32_inference": dict(scenes=[[(64, 96)] * 32], B=1, entry="inference"),
    "b2_n13": dict(scenes=[[(64, 96)] * 13], B=2, entry="forward"),
    "n257_32x32": dict(scenes=[[(32, 32)] * 257], B=1, entry="forward"),
    "mixed_n30": dict(scenes=[[(96, 64) if i % 7 == 2 else (64, 96) for i in range(30)]], B=1, entry="forward"),
    "many_3": dict(scenes=[[(64, 96)] * 20, [(64, 128)] * 7, [(96, 64)] * 5], B=1, entry="forward_many"),
}
EMU_BRANCHES = {  # what each composition must reach (bf16; the parity path's head chunks are 8)
    "n32_inference": {"head_chunks>1", "sink_chunks>1"},
    "b2_n13": {"batch>1", "head_chunks>1", "head_chunk_splits_view"},
    "n257_32x32": {"encoder_chunks>1", "head_chunks>1"},
    "mixed_n30": {"groups>1", "packed", "head_chunks>1"},
    "many_3": {"groups>1", "packed"},
}
_refs = {}


def _oracle(name):
    """float64 oracle of an emulated composition, one forward per scene in scene order (cached for both precisions)."""
    from oracle import fast3r_oracle as O
    if name not in _refs:
        c = EMU_CASES[name]
        cfg, sd = state_dict("tiny", 0.7)
        torch.manual_seed(7)
        _refs[name] = [p for imgs in scene_images(c["scenes"], c["B"])
                       for p in O.forward(sd, *cfg, imgs, dtype=torch.float64, head_chunk=16)]
    return _refs[name]


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("name", list(EMU_CASES))
def test_host_composition_vs_fp64_oracle(emulated, name, precision):
    M, ops = emulated
    c = EMU_CASES[name]
    case = dict(model_cpu="tiny", gain=0.7, entry=c["entry"])
    preds, seen = _run(M, ops, case, precision, scene_images(c["scenes"], c["B"]))
    want = set(EMU_BRANCHES[name])
    if precision == "fp32" and name == "b2_n13":
        want.discard("head_chunk_splits_view")  # 26 images in chunks of 8: every boundary falls between views
    assert want <= seen, (name, precision, want - seen)
    FS.check_all(FS.by_shape(preds, _oracle(name)), precision, f"emulated {name}")


def test_every_host_branch_has_a_gpu_case(emulated):
    """Each GPU case of tests/forward_cases.py at small images (its view counts, batch, shape groups, entry point and
    precisions kept): the union of the branches they reach must be every branch in BRANCHES."""
    M, ops = emulated
    reached = {}
    for name, c in CASES.items():
        imgs = scene_images(c["scenes"], c["B"], shape_map=SMALL if name != "tiny_n320" else {L368: (32, 32)})
        for precision in c["precisions"]:
            _, seen = _run(M, ops, dict(model_cpu="tiny", gain=c["gain"], entry=c["entry"]), precision, imgs)
            for b in seen:
                reached.setdefault(b, set()).add(f"{name}-{precision}")
    print({b: sorted(v) for b, v in reached.items()})
    missing = [b for b in BRANCHES if b not in reached]
    assert not missing, f"host branches without a GPU case: {missing}"
    assert set(reached) <= set(BRANCHES), set(reached) - set(BRANCHES)
