"""Every launch key of the geometry tail that the postprocess entry points reach is covered by a case of the GPU table
(tests/geometry_plans.CASES, run by tests/test_geometry_plans_gpu.py), and the oracle's quantile is torch.quantile on
the inputs where the two could part: NaN, infinities, signed zeros and subnormals.

The entry points run on the CPU with postprocess._device_of pinned to the CPU and the four geometry ops of
fast3r_b200.ops replaced by recorders: each records its descriptor (alignment read off the tensors it is handed) and
answers with oracle/geometry_oracle, so the callers go on exactly as they would with the kernels."""
import numpy as np
import pytest
import torch

from oracle import geometry_oracle as go
from tests import geometry_plans as GP


def _al16(*ts):
    return all(t is None or t.data_ptr() % 16 == 0 for t in ts)


class Recorder:
    """Stand-in for the geometry ops of fast3r_b200.ops: appends (descriptor, where) to `calls`, returns the oracle's
    result."""

    def __init__(self):
        self.calls = []
        self.where = ""

    def _rec(self, op, **d):
        self.calls.append((dict(op=op, **d), self.where))

    def conf_quantile(self, conf, q):
        assert conf.dtype == torch.float32 and conf.is_contiguous() and conf.dim() == 2
        self._rec("quantile", views=conf.shape[0], n=conf.shape[1], q=float(q), aligned=_al16(conf))
        return torch.tensor([float(go.conf_quantile(c.numpy(), q)) for c in conf], dtype=torch.float32)

    def similarity_fit(self, x, y, conf=None, thr=None, valid=None):
        for t in (x, y, conf, valid):
            assert t is None or t.is_contiguous()
        views, n = x.shape[0], x.shape[1]
        self._rec("fit", views=views, n=n, conf=conf is not None and thr is not None, valid=valid is not None,
                  aligned=_al16(x, y, conf) and (valid is None or valid.data_ptr() % 4 == 0))
        rts = torch.zeros(views, 13, dtype=torch.float32)
        for v in range(views):
            vm = np.ones(n, bool) if valid is None else valid[v].numpy().astype(bool)
            sel = vm & (conf[v].numpy() >= thr[v].numpy()) if conf is not None else vm
            if sel.sum() < 3:
                sel = vm
            if sel.sum() < 3:
                r, t, s = np.eye(3), np.zeros(3), 1.0
            else:
                r, t, s = go.umeyama(x[v].numpy()[sel], y[v].numpy()[sel])
            rts[v] = torch.from_numpy(np.concatenate([r.reshape(-1), t, [s]]).astype(np.float32))
        return rts

    def similarity_apply(self, x, rts, out=None):
        assert x.is_contiguous()
        self._rec("apply", views=x.shape[0], n=x.shape[1], aligned=_al16(x, out),
                  alias=out is not None and out.data_ptr() == x.data_ptr())
        r = rts[:, :9].double().reshape(-1, 1, 3, 3)
        res = (rts[:, 12].double().reshape(-1, 1, 1) * (r @ x.double().unsqueeze(-1)).squeeze(-1)
               + rts[:, 9:12].double().reshape(-1, 1, 3)).float()
        if out is None:
            return res
        out.copy_(res)
        return out

    def focal_weiszfeld(self, pts, conf=None, thr=None, pp=None, iters=100):
        views, H, W = pts.shape[0], pts.shape[1], pts.shape[2]
        self._rec("focal", views=views, H=H, W=W, conf=conf is not None and thr is not None, pp=pp is not None,
                  iters=int(iters))
        out = []
        for v in range(views):
            c = (W / 2, H / 2) if pp is None else tuple(pp[v].tolist())
            mask = None if conf is None else (conf[v] >= thr[v]).numpy()
            out.append(go.focal_weiszfeld(pts[v].numpy(), c, mask, iters))
        return torch.tensor(out, dtype=torch.float32)


def _patch(monkeypatch, rec):
    import fast3r_b200.ops as O
    import fast3r_b200.postprocess as P
    import fast3r_b200.recon_metric as RM
    monkeypatch.setattr(P, "_device_of", lambda t, device: torch.device("cpu"))
    for name in ("conf_quantile", "similarity_fit", "similarity_apply", "focal_weiszfeld"):
        monkeypatch.setattr(O, name, getattr(rec, name))
    # the metric kernels (out of this table's scope) answer with placeholders
    monkeypatch.setattr(RM, "estimate_normals", lambda p: torch.zeros_like(p))
    monkeypatch.setattr(RM, "accuracy", lambda *a: (0.0, 0.0, 0.0, 0.0))
    monkeypatch.setattr(RM, "completion", lambda *a: (0.0, 0.0, 0.0, 0.0))


def _pred(g, b, h, w):
    x = torch.randn(b, h, w, 3, generator=g)
    return dict(pts3d_local=x, pts3d_in_other_view=1.5 * x + 0.3 + 0.01 * torch.randn(b, h, w, 3, generator=g),
                conf=1 + torch.rand(b, h, w, generator=g), conf_local=1 + torch.rand(b, h, w, generator=g))


def _view(g, pred, valid):
    b, h, w, _ = pred["pts3d_local"].shape
    v = dict(img=torch.empty(b, 3, h, w), pts3d=pred["pts3d_in_other_view"].clone())
    if valid:
        v["valid_mask"] = torch.rand(b, h, w, generator=g) > 0.1
    return v


LAND, PORT, FOUR3, CROP = (368, 512), (512, 368), (384, 512), (224, 224)


def all_postprocess_calls(monkeypatch):
    from fast3r_b200 import postprocess as P
    rec = Recorder()
    _patch(monkeypatch, rec)
    g = torch.Generator().manual_seed(0)
    # align_local_pts3d_to_global: the same pred object repeated keeps the inputs small; torch.cat copies them anyway
    for nviews, hw, valid, pct in ((1, LAND, False, 0), (2, PORT, True, 0), (32, LAND, True, 0), (64, CROP, False, 0),
                                   (65, FOUR3, True, 0), (1, FOUR3, False, 30)):
        p = _pred(g, 1, *hw)
        vw = _view(g, p, valid)
        rec.where = f"align {nviews} views {hw} valid={valid} p{pct}"
        P.align_local_pts3d_to_global([dict(p) for _ in range(nviews)], [vw] * nviews, min_conf_thr_percentile=pct)
    preds = [_pred(g, 1, *hw) for hw in (LAND, PORT, FOUR3, CROP)]
    rec.where = "align mixed resolutions"
    P.align_local_pts3d_to_global(preds, [_view(g, p, True) for p in preds])
    for hw in (LAND, PORT, CROP):
        p = _pred(g, 1, *hw)
        rec.where = f"estimate_focal {hw}"
        P.estimate_focal(p["pts3d_local"], p["conf_local"])
        rec.where = f"estimate_focal {hw} pp"
        P.estimate_focal(p["pts3d_local"], p["conf_local"], pp=torch.tensor([hw[1] / 2 + 1.5, hw[0] / 2 - 2.0]))
        rec.where = f"estimate_focal_knowing_depth {hw}"
        P.estimate_focal_knowing_depth(torch.cat([p["pts3d_local"]] * 2), torch.tensor([hw[1] / 2, hw[0] / 2]))
    for nviews, local in ((4, True), (4, False), (32, True)):
        p = _pred(g, 1, *LAND)
        rec.where = f"evaluate_reconstruction {nviews} views local={local}"
        P.evaluate_reconstruction([_view(g, p, True) for _ in range(nviews)], [dict(p) for _ in range(nviews)],
                                  use_pts3d_from_local_head=local)
    return rec.calls


@pytest.fixture(scope="module")
def recorded():
    mp = pytest.MonkeyPatch()
    try:
        yield all_postprocess_calls(mp)
    finally:
        mp.undo()


def test_recorder_sees_the_callers(recorded):
    """Sanity of the recorder, from postprocess.py: 65 views stack as 64 + 1 (_GROUP); mixed resolutions run one call
    per pred; evaluate_reconstruction fits and applies one "view" of V H W points after two quantiles of its V views (and, from the local head, the alignment's)."""
    from collections import Counter
    by = lambda where: [d for d, w in recorded if w == where]  # noqa: E731
    assert [d["views"] for d in by(f"align 65 views {FOUR3} valid=True p0") if d["op"] == "fit"] == [64, 1]
    mixed = by("align mixed resolutions")
    assert Counter(d["op"] for d in mixed) == Counter(quantile=4, fit=4, apply=4)
    assert {d["n"] for d in mixed} == {368 * 512, 384 * 512, 224 * 224}
    ev = by("evaluate_reconstruction 32 views local=True")
    assert [(d["op"], d["views"]) for d in ev if d["n"] == 32 * 368 * 512] == [("fit", 1), ("apply", 1)]
    assert sum(d["op"] == "quantile" and d["views"] == 32 for d in ev) == 3  # the local alignment's and two masks
    assert {d["op"] for d, _ in recorded} == set(GP.KEYS)


def test_every_caller_key_has_a_gpu_case(recorded):
    table = {c["key"] for c in GP.CASES}
    missing = {}
    for d, where in recorded:
        k = GP.key(d)
        if k not in table:
            missing.setdefault(k, (d, where))
    assert not missing, "launch keys of the postprocess callers without a case in tests/geometry_plans.CASES:\n" + \
        "\n".join(f"  {k}\n      from {where}: {d}" for k, (d, where) in sorted(missing.items()))


def test_table_keys_are_what_the_cases_reach():
    """Each case of the GPU table reaches the key it declares, and no two cases share a name."""
    names = [c["name"] for c in GP.CASES]
    assert len(names) == len(set(names))
    wrong = [(c["name"], c["key"], GP.key(c)) for c in GP.CASES if GP.key(c) != c["key"]]
    assert not wrong, "\n".join(f"{n}: declares {k!r}, reaches {g!r}" for n, k, g in wrong)


def test_table_reaches_the_contract_flags():
    """The contract part of the table reaches every flag of every kernel, on and off."""
    keys = {c["key"] for c in GP.CASES}
    for op, flags in (("quantile", ("vec", "interp", "empty")), ("fit", ("vec", "conf", "valid", "empty")),
                      ("apply", ("vec", "alias")), ("focal", ("conf", "pp", "iters0", "empty"))):
        ks = [k.split()[1:] for k in keys if k.split()[0] == op]
        for f in flags:
            assert any(f in k for k in ks) and any(f not in k for k in ks), (op, f)


# ------------------------------------------------------------------ the oracle's quantile is torch.quantile
NEG_NAN = np.array([0xFFC00000], np.uint32).view(np.float32)[0]
POS_NAN = np.array([0x7FC00001], np.uint32).view(np.float32)[0]


def _same(a, b):
    a, b = float(a), float(b)
    return a == b or (np.isnan(a) and np.isnan(b))


def _pin(v, tag):
    t = torch.from_numpy(np.asarray(v, np.float32).copy())
    with np.errstate(invalid="ignore"):
        for q in GP.QS:
            want = float(torch.quantile(t, q))
            got = go.conf_quantile(v, q)
            assert _same(got, want), (tag, q, v.tolist(), float(got), want)


@pytest.mark.parametrize("nan", [POS_NAN, NEG_NAN], ids=["pos_nan", "neg_nan"])
def test_oracle_quantile_nan_is_torch(nan):
    """One NaN of either sign at every position of small vectors (with ties and infinities around it) gives NaN."""
    assert np.isnan(nan)
    rng = np.random.default_rng(1)
    for n in (1, 2, 3, 5, 8):
        base = rng.standard_normal(n).astype(np.float32)
        for pos in range(n):
            for extra in (None, np.inf, -np.inf):
                v = base.copy()
                if extra is not None and n > 1:
                    v[(pos + 1) % n] = extra
                v[pos] = nan
                _pin(v, (n, pos, extra))


def test_oracle_quantile_edges_are_torch():
    """Infinities at and next to the order statistics, signed zeros, subnormals, constants."""
    rng = np.random.default_rng(2)
    f = np.float32
    cases = [
        np.array([np.inf, 1, 2], f), np.array([-np.inf, 1, 2], f), np.array([np.inf, np.inf, -np.inf, 0], f),
        np.array([-np.inf] * 3 + [1.0], f), np.array([1.0, np.inf, np.inf, np.inf], f),
        np.array([-0.0, 0.0, -0.0, 0.0, 1.0], f), np.array([0.0, -0.0], f), np.array([-0.0] * 5, f),
        np.array([1e-45, -1e-45, 3e-39, -3e-39, 0.0], f), np.array([1e-40, 2e-40, 1.2e-38, 1e-38], f),
        np.full(7, 3.25, f), np.full(4, np.inf, f), np.full(3, -np.inf, f),
    ]
    for n in (5, 17, 100):
        v = rng.standard_normal(n).astype(f)
        for lo in range(n):
            w = np.sort(v)
            w[lo:] = np.inf
            cases.append(rng.permutation(w))
            w = np.sort(v)
            w[:lo + 1] = -np.inf
            cases.append(rng.permutation(w))
        cases.append((rng.standard_normal(n) * 1e-40).astype(f))
        cases.append(np.where(rng.random(n) < 0.5, f(-0.0), f(0.0)).astype(f))
    for i, v in enumerate(cases):
        _pin(v, i)
