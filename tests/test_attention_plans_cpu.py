"""Every plan key of the attention kernels that the forward reaches is covered by a case of the GPU table
(tests/attention_plans.CASES, run by tests/test_attention_plans_gpu.py).  The forward runs on the meta device with
fast3r_b200.model.ops replaced by a recorder whose attention ops run the library's own host code (fast3r_b200.ops: the
key split, the partial buffers, the merge) down to the C-ABI call, which is recorded instead of made."""
import pytest
import torch

from tests import attention_plans as AP

from fast3r_b200 import ops


class Recorder:
    """Stand-in for fast3r_b200.ops (model and KVExchange): the attention ops run fast3r_b200.ops with its C-ABI call
    replaced by a recorder; every other op does nothing.  `calls`: (descriptor, where)."""

    def __init__(self, monkeypatch):
        self.calls = []
        self.where = ""
        self._offsets = None
        monkeypatch.setattr(ops, "_ptr", lambda t: None if t is None else 1)
        monkeypatch.setattr(ops, "_call", self._abi)

    def _abi(self, name, anchor, *a):
        if name == "f3r_attention":
            d = dict(entry="attention", ldo=a[5], lse=a[6] is not None, batch=a[7], heads=a[8], sq=a[9], skv=a[10])
        elif name == "f3r_attention_partial":
            d = dict(entry="partial", kv_rows_total=a[4], kv_row0=a[5], skv=a[6], n_split=a[7], part_base=a[10],
                     batch=a[11], heads=a[12], sq=a[13])
        elif name == "f3r_attention_segments":
            d = dict(entry="segments", ldo=a[5], offsets=list(self._offsets), heads=a[9], n_split=a[11],
                     part=a[12] is not None)
        elif name == "f3r_attention_merge":
            d = dict(entry="merge", n_parts=a[2], ldo=a[4], batch=a[5], heads=a[6], sq=a[7])
        else:
            raise AssertionError(f"unexpected library call {name}")
        self.calls.append((d, self.where))

    pick_kv_split = staticmethod(ops.pick_kv_split)
    Segments = ops.Segments

    def attention(self, *a, **kw):
        ops.attention(*a, **kw)

    def attention_partial(self, *a, **kw):
        ops.attention_partial(*a, **kw)

    def attention_merge(self, *a, **kw):
        ops.attention_merge(*a, **kw)

    def attention_segments(self, q, kv, out, seg_off, **kw):
        self._offsets = seg_off.offsets if isinstance(seg_off, ops.Segments) else [int(v) for v in seg_off]
        ops.attention_segments(q, kv, out, seg_off, **kw)

    def attention_x3(self, q, kv, out, *, batch, heads, sq, skv, scale, lse=None):
        assert q.dtype == kv.dtype == out.dtype == torch.float32
        assert q.numel() == batch * sq * q.shape[-1] and kv.numel() == batch * skv * kv.shape[-1]
        self.calls.append((dict(entry="x3", batch=batch, heads=heads, sq=sq, skv=skv, ldo=out.shape[-1],
                                lse=lse is not None), self.where))

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
    """One ViT-L forward over views of the given (H, W) sizes."""
    _patch_model(monkeypatch, rec)
    model = _vitl(precision)
    rec.where = f"forward {precision} {len(sizes)} views {sorted(set(sizes))}"
    model([dict(img=torch.empty(1, 3, h, w, device="meta")) for h, w in sizes])


def forward_many_calls(monkeypatch, rec, precision, scenes):
    """forward_many over scenes, each a list of (H, W) view sizes."""
    _patch_model(monkeypatch, rec)
    model = _vitl(precision)
    rec.where = f"forward_many {precision} {scenes}"
    model.forward_many([[dict(img=torch.empty(1, 3, h, w, device="meta")) for h, w in s] for s in scenes])


def exchange_calls(rec, rows, *, heads=16, use_local=False, x3=False):
    """The sequence-parallel attention of one decoder layer on every rank when the ranks hold `rows` tokens: the
    overlapped path (KVExchange.partials + the merge, as KVExchange.attend runs them) in bf16, or the parity path's
    all-gather call (one attention_x3 over all keys)."""
    from types import SimpleNamespace
    from fast3r_b200.parallel import KVExchange
    D = heads * 64
    for rank in range(len(rows)):
        sp = SimpleNamespace(rank=rank, world=len(rows))
        kvx = KVExchange(sp, 1, rows[rank], D, rows, mixed=len(set(rows)) > 1)
        sl = rows[rank]
        rec.where = (f"{'x3 all-gather' if x3 else 'KVExchange.partials'} rows {rows if len(rows) <= 8 else len(rows)}"
                     f" rank {rank}{' local' if use_local else ''}")
        if x3:
            f32 = dict(dtype=torch.float32, device="meta")
            rec.attention_x3(torch.empty(sl, D, **f32), torch.empty(sum(rows), 2 * D, **f32), torch.empty(sl, D, **f32),
                             batch=1, heads=heads, sq=sl, skv=sum(rows), scale=0.125)
            continue
        bf = dict(dtype=torch.bfloat16, device="meta")
        kvx.buf = torch.empty(len(rows), max(rows), 2 * D, **bf)
        local = torch.empty(sl, 2 * D, **bf) if use_local else None
        q = torch.empty(sl, D, **bf)
        n = kvx.partials(rec, q, local, heads=heads, scale=0.125, peers_landed=lambda: None)
        rec.attention_merge(kvx.parts[0], kvx.parts[1], n, torch.empty(sl, D, **bf), batch=1, heads=heads, sq=sl)


def _shard_rows(tokens, world):
    from fast3r_b200.parallel import shard_views_weighted
    return [sum(tokens[a:b]) for a, b in shard_views_weighted(tokens, world)]


LAND, PORT = (368, 512), (512, 368)


def all_forward_calls(monkeypatch):
    rec = Recorder(monkeypatch)
    for precision in ("bf16", "fp32"):
        forward_calls(monkeypatch, rec, precision, [LAND] * 32)        # the benchmark forward
        forward_calls(monkeypatch, rec, precision, [LAND] * 4)         # the golden configuration
        forward_calls(monkeypatch, rec, precision, [PORT])             # one portrait view
        forward_many_calls(monkeypatch, rec, precision, [[LAND] * 4, [(384, 512)], [(512, 384)] * 2])
    forward_calls(monkeypatch, rec, "bf16", [LAND] * 320)              # the benchmark's long-sequence configuration
    for world in (2, 4, 8):                                            # N=32 sharded, every rank
        for use_local in (False, True):
            exchange_calls(rec, _shard_rows([736] * 32, world), use_local=use_local)
        exchange_calls(rec, _shard_rows([736] * 32, world), x3=True)
    for n in (320, 1000):                                              # the benchmark's N=320 and N=1000 on 8 ranks
        exchange_calls(rec, _shard_rows([736] * n, 8))
        exchange_calls(rec, _shard_rows([736] * n, 8), use_local=True)
    mixed = _shard_rows([736, 736, 1024, 1024, 736, 736, 768, 1024], 3)  # views of mixed resolution over 3 ranks
    exchange_calls(rec, mixed)
    exchange_calls(rec, mixed, use_local=True)
    exchange_calls(rec, mixed, x3=True)
    return rec.calls


@pytest.fixture(scope="module")
def recorded():
    mp = pytest.MonkeyPatch()
    try:
        yield all_forward_calls(mp)
    finally:
        mp.undo()


def test_recorder_sees_the_forward(recorded):
    """Sanity of the recorder: the benchmark forward makes one attention per encoder block (24, batch = 32 views) and
    one per decoder block (24, one sequence of 23 552 tokens)."""
    bench = [d for d, where in recorded if where == f"forward bf16 32 views {[LAND]}"]
    assert len(bench) == 48
    assert sum(d["batch"] == 32 and d["sq"] == 736 for d in bench) == 24
    assert sum(d["batch"] == 1 and d["sq"] == d["skv"] == 23552 for d in bench) == 24
    entries = {d["entry"] for d, _ in recorded}
    assert entries == {"attention", "partial", "segments", "merge", "x3"}, entries
    assert any(d["entry"] == "partial" and d["kv_row0"] > 0 for d, _ in recorded)


def test_every_forward_plan_has_a_gpu_case(recorded):
    table = {k for c in AP.CASES for k in c["keys"]}
    missing = {}
    for d, where in recorded:
        for key in AP.plan_keys(d):
            if key not in table:
                missing.setdefault(key, (d, where))
    assert not missing, "plan keys of the forward without a case in tests/attention_plans.CASES:\n" + "\n".join(
        f"  {k}\n      from {where}: {d}" for k, (d, where) in sorted(missing.items()))


def test_table_keys_are_what_the_cases_reach():
    """Each case of the GPU table reaches the plan keys it declares, and no two cases share a name."""
    names = [c["name"] for c in AP.CASES]
    assert len(names) == len(set(names))
    wrong = [(c["name"], c["keys"], AP.case_keys(c)) for c in AP.CASES if AP.case_keys(c) != c["keys"]]
    assert not wrong, "\n".join(f"{n}: declares {k!r}, reaches {g!r}" for n, k, g in wrong)


def test_attention_refuses_lse_with_key_slices():
    """The key-slice path (attention_partial + attention_merge) has no log-sum-exp output: ops.attention refuses a call
    that asks for both before it touches a device."""
    q = torch.empty(300, 128, dtype=torch.bfloat16)
    kv = torch.empty(2000, 256, dtype=torch.bfloat16)
    out = torch.empty(300, 128, dtype=torch.bfloat16)
    lse = torch.empty(1, 2, 300, dtype=torch.float32)
    with pytest.raises(ValueError, match="lse"):
        ops.attention(q, kv, out, batch=1, heads=2, sq=300, skv=2000, scale=0.125, lse=lse, kv_split=2)


def test_plan_key_fields():
    """Hand-checked keys: tile rows per warpgroup, ring classes of uneven slices, the last key block and the flags."""
    d = dict(entry="partial", batch=1, heads=2, sq=193, skv=7 * 128 + 1, kv_rows_total=5000, kv_row0=128, n_split=3,
             part_base=1)
    assert AP.plan_keys(d) == ["partial tile1/3p kb:2..3 last:one split:uneven row0 tail"]
    d = dict(entry="attention", batch=2, heads=2, sq=384, skv=896, ldo=192, lse=True)
    assert AP.plan_keys(d) == ["attn+lse tile3/3 kb:7+ last:full split:1 batch ldo"]
    d = dict(entry="segments", offsets=[0, 100, 100, 900], heads=2, n_split=2, ldo=128, part=True)
    assert AP.plan_keys(d) == ["seg+part tile1/3p kb:3..4-6 last:part split:uneven unaligned",
                               "seg+part tile2/3p kb:1 last:part split:1 neutral short"]
    d = dict(entry="x3", batch=1, heads=2, sq=129, skv=5 * 128, ldo=128, lse=False)
    assert AP.plan_keys(d) == ["x3 tile1/2p kb:5+ last:full split:1"]
    assert AP.slices(7, 3) == [(0, 2), (2, 2), (4, 3)]
