"""Every launch plan of f3r_gemm that the forward reaches is covered by a case of the GPU table
(tests/gemm_plans.CASES, run by tests/test_gemm_plans_gpu.py).  The forward runs on the meta device with
fast3r_b200.model.ops replaced by a recorder: each op is a no-op, gemm / gemm_x3 record their descriptor.  Each
descriptor is mapped to its plan key by the library's own rule (csrc/gemm_plan.h compiled for the host) for an H100
SXM (132 SMs)."""
import pytest
import torch

from tests import gemm_plans as GP

from fast3r_b200 import lib as L


class Recorder:
    """Stand-in for fast3r_b200.ops: gemm / gemm_x3 append (descriptor, where) to `calls`, everything else does
    nothing."""

    def __init__(self):
        self.calls = []
        self.where = ""

    def gemm(self, a, wt, *, w, h=1, nb=1, taps=1, bias=None, out0=None, out1=None, res0=None, res1=None,
             act=L.ACT_NONE, epi=L.EPI_STORE, split_col=0, ldo=None, ldo_b=0, tok_per_img=0, grid_w=0, rope_cols=0,
             ct_k=0, ct_cout=0, **_):
        dt = lambda t: None if t is None else ("f32" if t.dtype == torch.float32 else "bf16")  # noqa: E731
        r0 = dt(res0)
        if res0 is not None and res0 is out0:
            assert r0 == "f32"
            r0 = "f32_inplace"
        d = dict(n=wt.shape[0], k=wt.shape[-1], taps=taps, w=w, h=h, nb=nb, epi=epi, act=act, out0=dt(out0),
                 out1=out1 is not None, res0=r0, res1=res1 is not None, split_col=split_col, bias=bias is not None,
                 ldo=ldo, ldo_b=ldo_b, tok_per_img=tok_per_img, grid_w=grid_w, rope_cols=rope_cols, ct_k=ct_k,
                 ct_cout=ct_cout)
        assert a.numel() == nb * h * w * d["k"] and wt.numel() == d["n"] * taps * d["k"]
        self.calls.append((d, self.where))

    def gemm_x3(self, a, wt3, *, a_relu=False, **kw):  # the K = 3k GEMM over the [hi | lo | hi] split of a
        a3 = torch.empty(a.shape[:-1] + (3 * a.shape[-1],), dtype=torch.bfloat16, device=a.device)
        self.gemm(a3, wt3, **kw)
        self.calls[-1][0]["x3"] = True

    def linear(self, a, wt, bias=None, **kw):
        self.gemm(a, wt, w=a.numel() // a.shape[-1], bias=bias, **kw)

    def __getattr__(self, name):
        return lambda *args, **kw: None


def _vitl(precision):
    from fast3r_b200 import Fast3R, vit_large_args
    enc, dec, head = vit_large_args()
    with torch.device("meta"):
        model = Fast3R(enc, dec, head).eval()
    return model.to("meta").set_precision(precision)


def forward_calls(monkeypatch, precision, n_views, H, W):
    """Descriptors of every GEMM of one ViT-L forward over n_views views of H x W."""
    import fast3r_b200.model as M
    rec = Recorder()
    monkeypatch.setattr(M, "ops", rec)
    monkeypatch.setattr(M, "_require_cuda", lambda device: None)
    model = _vitl(precision)
    rec.where = f"forward {precision} N={n_views} {H}x{W}"
    views = [dict(img=torch.empty(1, 3, H, W, device="meta")) for _ in range(n_views)]
    torch.manual_seed(0)
    model(views)
    return rec.calls


def sharded_decoder_calls(monkeypatch, precision, n_views, world, tok=736):
    """Descriptors of the fusion-decoder GEMMs of every rank when n_views views of `tok` tokens are sharded over `world`
    ranks (sequence parallel: each rank runs the decoder's GEMMs on its own rows)."""
    import fast3r_b200.model as M
    from fast3r_b200.parallel import shard_views_weighted
    rec = Recorder()
    monkeypatch.setattr(M, "ops", rec)
    monkeypatch.setattr(M, "_require_cuda", lambda device: None)
    model = _vitl(precision)
    P_ = model._pack(torch.device("meta"))
    for rank, (lo, hi) in enumerate(shard_views_weighted([tok] * n_views, world)):
        rec.where = f"decoder {precision} N={n_views} rank {rank}/{world} ({hi - lo} views)"
        rows = (hi - lo) * tok
        feats = torch.empty(rows, model.encoder.embed_dim, dtype=P_.adt, device="meta")
        ids = torch.zeros(1, hi - lo, dtype=torch.int32)
        model._decode(feats, ids, 1, rows, tok, P_)
    return rec.calls


def all_forward_calls(monkeypatch):
    calls = []
    for precision in ("bf16", "fp32"):
        calls += forward_calls(monkeypatch, precision, 32, 368, 512)  # the benchmark forward
        for world in (2, 4, 8):
            calls += sharded_decoder_calls(monkeypatch, precision, 32, world)
    calls += forward_calls(monkeypatch, "bf16", 4, 368, 512)          # the golden configuration
    calls += forward_calls(monkeypatch, "bf16", 1, 512, 368)          # one portrait view
    return calls


@pytest.fixture(scope="module")
def recorded():
    mp = pytest.MonkeyPatch()
    try:
        yield all_forward_calls(mp)
    finally:
        mp.undo()


def test_recorder_sees_the_forward(recorded):
    """Sanity of the recorder: the benchmark forward makes the expected number of GEMMs (per block qkv, proj, fc1, fc2;
    patch embed; decoder embed; per DPT head 7 act_postprocess, 4 layer_rn, 4 out_conv, 7 residual units of 2 convs, 2
    head convs)."""
    bench = [d for d, where in recorded if where == "forward bf16 N=32 368x512"]
    per_head = 7 + 4 + 4 + 14 + 2
    assert len(bench) == 1 + 24 * 4 + 1 + 24 * 4 + 2 * 2 * per_head  # 2 heads (global, local) x 2 chunks (25 + 7)


def test_every_forward_plan_has_a_gpu_case(recorded):
    table = {c["key"] for c in GP.CASES}
    missing = {}
    for d, where in recorded:
        key = GP.plan_key(d)
        if key not in table:
            missing.setdefault(key, (d, where))
    assert not missing, "plan keys of the forward without a case in tests/gemm_plans.CASES:\n" + "\n".join(
        f"  {k}\n      from {where}: {d}" for k, (d, where) in sorted(missing.items()))


def test_every_parity_forward_plan_has_an_x3_case(recorded):
    """Every plan key of the fp32 (parity) forward has a case that runs it as the parity path computes it: fp32
    operands split into bf16 hi / lo parts, the weight packed [Whi | Whi | Wlo] by the model's own packing
    (tests/test_gemm_plans_gpu.run_case with x3=True).  The one GEMM of the parity forward that is not an ops.gemm_x3
    call, the stride-2 conv over its split3 + im2col3x3s2 columns, has the case x3="stride2"."""
    table = {c["key"] for c in GP.CASES if c["x3"]}
    missing = {}
    for d, where in recorded:
        if " fp32 " in where:
            key = GP.plan_key(d)
            if key not in table:
                missing.setdefault(key, (d, where))
    assert not missing, "plan keys of the parity forward without an x3 case in tests/gemm_plans.CASES:\n" + "\n".join(
        f"  {k}\n      from {where}: {d}" for k, (d, where) in sorted(missing.items()))
    assert all(c["k"] % 3 == 0 for c in GP.CASES if c["x3"])


def test_forward_never_needs_the_reduce_add_restriction(recorded):
    """The forward makes no call that the reduce-add epilogue refuses (an activation or the image-index embedding
    together with an in-place fp32 residual): those calls are planned as before, so the forward computes what it did
    before that restriction."""
    for d, where in recorded:
        if d["res0"] == "f32_inplace" and d["out0"] == "f32":
            assert d["act"] == L.ACT_NONE and d["epi"] != L.EPI_IDXEMB, (d, where)


def test_table_keys_are_what_the_cases_reach():
    """Each case of the GPU table reaches the plan key it declares (on an H100 SXM), and no two cases share a name."""
    names = [c["name"] for c in GP.CASES]
    assert len(names) == len(set(names))
    wrong = [(c["name"], c["key"], GP.plan_key(c)) for c in GP.CASES if GP.plan_key(c) != c["key"]]
    assert not wrong, "\n".join(f"{n}: declares {k!r}, reaches {g!r}" for n, k, g in wrong)


def test_reduce_add_plan_excludes_activation_and_embedding():
    """The in-place fp32 residual takes the TMA reduce-add only when out0 = res0 + (acc + bias [+ RoPE]): with an
    activation or the image-index embedding it takes the generic epilogue, without a K split."""
    base = dict(n=1024, k=4096, taps=1, w=300, h=1, nb=1, epi=L.EPI_STORE, act=L.ACT_NONE, out0="f32", out1=False,
                res0="f32_inplace", res1=False, split_col=0)
    p = GP.plan(base)
    assert p["tma_epi"] == 2 and p["k_split"] > 1
    for over in (dict(act=L.ACT_RELU), dict(act=L.ACT_GELU), dict(epi=L.EPI_IDXEMB)):
        p = GP.plan({**base, **over})
        assert (p["tma_epi"], p["k_split"]) == (0, 1), over
    assert GP.plan({**base, "epi": L.EPI_ROPE})["tma_epi"] == 2
    assert GP.plan(base, allow_k_split=False)["k_split"] == 1
    assert GP.plan(base, allow_tma_epi=False)["tma_epi"] == 0
