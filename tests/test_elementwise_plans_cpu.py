"""Every launch key of the element-wise kernels that the forward reaches is covered by a case of the GPU table
(tests/elementwise_plans.CASES, run by tests/test_elementwise_plans_gpu.py).  The forward runs on the meta device with
fast3r_b200.model.ops replaced by a recorder: the element-wise ops record their descriptor, every other op does
nothing."""
import pytest
import torch

from tests import elementwise_plans as EP

_DT = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: "f32"}


class Recorder:
    """Stand-in for fast3r_b200.ops: the element-wise ops append (descriptor, where) to `calls`.  ops.gemm_x3 splits its
    operand with split3 inside the library's host code, so it is recorded as that split3 call."""

    def __init__(self):
        self.calls = []
        self.where = ""

    def _rec(self, op, **d):
        self.calls.append((dict(op=op, **d), self.where))

    def layernorm(self, x, w, b, eps, out):
        dim = x.shape[-1]
        assert out.numel() == x.numel()
        self._rec("layernorm", rows=x.numel() // dim, dim=dim, out=_DT[out.dtype], eps=eps)

    def im2col_patch(self, img, out):
        n, _, H, W = img.shape
        self._rec("im2col_patch", n=n, H=H, W=W, out=_DT[out.dtype])

    def im2col3x3s2(self, x, out, n, h, w, c, ho, wo):
        assert x.numel() == n * h * w * c and out.numel() == n * ho * wo * 9 * c
        self._rec("im2col3x3s2", n=n, H=h, W=w, C=c, Ho=ho, Wo=wo)

    def upsample2x(self, x, out, n, h, w, c, ho, wo):
        assert x.dtype == out.dtype and out.numel() == n * ho * wo * c
        self._rec("upsample2x", n=n, H=h, W=w, C=c, Ho=ho, Wo=wo, dt=_DT[x.dtype])

    def cast_bf16(self, x, out):
        self._rec("cast", n=x.numel(), out="bf16")

    def cast_f16(self, x, out):
        self._rec("cast", n=x.numel(), out="f16")

    def split3(self, x, out, relu=False):
        k = x.shape[-1]
        self._rec("split3", rows=x.numel() // k, k=k, relu=bool(relu))

    def add_f32(self, dst, src):
        self._rec("add_f32", n=dst.numel())

    def gemm_x3(self, a, wt3, *, a_relu=False, **kw):
        self.split3(a, None, relu=a_relu)

    def __getattr__(self, name):
        return lambda *args, **kw: None


def _vitl(precision):
    from fast3r_b200 import Fast3R, vit_large_args
    enc, dec, head = vit_large_args()
    with torch.device("meta"):
        model = Fast3R(enc, dec, head).eval()
    return model.to("meta").set_precision(precision)


def _patch_model(monkeypatch, rec):
    import fast3r_b200.model as M
    monkeypatch.setattr(M, "ops", rec)
    monkeypatch.setattr(M, "_require_cuda", lambda device: None)


def forward_calls(monkeypatch, rec, precision, sizes):
    _patch_model(monkeypatch, rec)
    model = _vitl(precision)
    rec.where = f"forward {precision} {len(sizes)} views {sorted(set(sizes))}"
    model([dict(img=torch.empty(1, 3, h, w, device="meta")) for h, w in sizes])


def forward_many_calls(monkeypatch, rec, precision, scenes):
    _patch_model(monkeypatch, rec)
    model = _vitl(precision)
    rec.where = f"forward_many {precision} {scenes}"
    model.forward_many([[dict(img=torch.empty(1, 3, h, w, device="meta")) for h, w in s] for s in scenes])


def sharded_decoder_calls(monkeypatch, rec, precision, n_views, world, tok=736):
    """The fusion decoder of every rank when n_views views of `tok` tokens are sharded over `world` ranks (each rank runs
    the decoder's LayerNorms and hook casts on its own rows)."""
    from fast3r_b200.parallel import shard_views_weighted
    _patch_model(monkeypatch, rec)
    model = _vitl(precision)
    P_ = model._pack(torch.device("meta"))
    for rank, (lo, hi) in enumerate(shard_views_weighted([tok] * n_views, world)):
        rec.where = f"decoder {precision} N={n_views} rank {rank}/{world} ({hi - lo} views)"
        rows = (hi - lo) * tok
        feats = torch.empty(rows, model.encoder.embed_dim, dtype=P_.adt, device="meta")
        model._decode(feats, torch.zeros(1, hi - lo, dtype=torch.int32), 1, rows, tok, P_)


LAND, PORT = (368, 512), (512, 368)
BENCH = f"forward bf16 32 views {[LAND]}"


def all_forward_calls(monkeypatch):
    rec = Recorder()
    for precision in ("bf16", "fp16", "fp32"):
        forward_calls(monkeypatch, rec, precision, [LAND] * 32)        # the benchmark forward
        forward_calls(monkeypatch, rec, precision, [LAND] * 4)         # the golden configuration
        forward_calls(monkeypatch, rec, precision, [PORT])             # one portrait view
        forward_many_calls(monkeypatch, rec, precision, [[LAND] * 4, [(384, 512)], [(512, 384)] * 2])
    forward_calls(monkeypatch, rec, "bf16", [LAND] * 320)              # two encoder chunks (256 + 64 images)
    for precision in ("bf16", "fp32"):
        for world in (2, 4, 8):
            sharded_decoder_calls(monkeypatch, rec, precision, 32, world)
    return rec.calls


@pytest.fixture(scope="module")
def recorded():
    mp = pytest.MonkeyPatch()
    try:
        yield all_forward_calls(mp)
    finally:
        mp.undo()


def test_recorder_sees_the_forward(recorded):
    """Sanity of the recorder, from the model's structure: the benchmark forward makes 2 LayerNorms per block of the
    24 encoder and 24 decoder blocks, enc_norm and dec_norm; the 2 hook casts; and per head chunk (2 heads x 2 chunks
    of 25 + 7 views) 1 stride-2 im2col and 5 upsamples; plus 1 patch im2col."""
    from collections import Counter
    bench = Counter(d["op"] for d, where in recorded if where == BENCH)
    assert bench == Counter(layernorm=2 * 24 + 2 * 24 + 2, cast=2, im2col3x3s2=2 * 2, upsample2x=2 * 2 * 5,
                            im2col_patch=1), bench
    rows = {d["rows"] for d, where in recorded if where == BENCH and d["op"] == "layernorm"}
    assert rows == {32 * 736}, rows
    ops = {d["op"] for d, _ in recorded}
    assert ops == set(EP.KEYS), ops
    # the parity forward's splits: one per GEMM (ops.gemm_x3) and the explicit split of the stride-2 conv's operand
    x3 = [d for d, where in recorded if where == f"forward fp32 32 views {[LAND]}" and d["op"] == "split3"]
    assert any(d["relu"] for d in x3) and any(d["k"] == 768 and d["rows"] == 8 * 23 * 32 for d in x3)


def test_every_forward_key_has_a_gpu_case(recorded):
    table = {c["key"] for c in EP.CASES}
    missing = {}
    for d, where in recorded:
        k = EP.key(d)
        if k not in table:
            missing.setdefault(k, (d, where))
    assert not missing, "launch keys of the forward without a case in tests/elementwise_plans.CASES:\n" + "\n".join(
        f"  {k}\n      from {where}: {d}" for k, (d, where) in sorted(missing.items()))


def test_table_keys_are_what_the_cases_reach():
    """Each case of the GPU table reaches the key it declares, and no two cases share a name."""
    names = [c["name"] for c in EP.CASES]
    assert len(names) == len(set(names))
    wrong = [(c["name"], c["key"], EP.key(c)) for c in EP.CASES if EP.key(c) != c["key"]]
    assert not wrong, "\n".join(f"{n}: declares {k!r}, reaches {g!r}" for n, k, g in wrong)
