"""Every launch key of the reconstruction metrics that the recon_metric entry points and evaluate_reconstruction reach is
covered by a case of the GPU table (tests/pointcloud_plans, run by tests/test_pointcloud_plans_gpu.py), every contract
flag is reached on and off, and every case reaches the flags it is built for.

The callers run on the CPU with recon_metric._device and postprocess._device_of pinned to the CPU.  The point-cloud ops
of fast3r_b200.ops are replaced by recorders that record each call's descriptor (read off the operands it is handed) and
answer with scipy's cKDTree and numpy; the geometry ops answer through the recorder of tests/test_geometry_plans_cpu.
So the callers go on exactly as they would with the kernels."""
import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from tests import pointcloud_plans as PP
from tests.test_geometry_plans_cpu import Recorder as GeometryRecorder

EXACT_NORMALS_MAX = 1 << 17  # larger clouds get (0, 0, 1) normals: no key depends on their values


class _Index:
    def __init__(self, pts):
        self.pts, self.n = pts, len(pts)


class Recorder:
    """Stand-in for the point-cloud ops of fast3r_b200.ops: appends (descriptor, where) to `calls`."""

    def __init__(self):
        self.calls = []
        self.where = ""

    def _rec(self, d):
        self.calls.append((d, self.where))

    def pc_index(self, pts):
        assert pts.dtype in (torch.float32, torch.float64) and pts.is_contiguous() and pts.shape[1] == 3
        a = pts.numpy()
        if len(a):
            self._rec(PP.index_desc(a))
        return _Index(a)

    def pc_nearest(self, index, query):
        q = query.numpy()
        self._rec(PP.nearest_desc(index.pts, q))
        if index.n == 0:
            return torch.full((len(q),), np.inf, dtype=torch.float64), torch.zeros(len(q), dtype=torch.int64)
        d, i = cKDTree(index.pts.astype(np.float64)).query(q.astype(np.float64), workers=-1)
        return torch.from_numpy(np.asarray(d, np.float64)), torch.from_numpy(np.asarray(i, np.int64))

    def pc_knn_normals(self, index, k=30):
        if index.n:
            self._rec(PP.knn_desc(index.n, int(k)))
        out = np.tile([0.0, 0.0, 1.0], (index.n, 1))
        if 3 <= index.n <= EXACT_NORMALS_MAX:
            p = index.pts.astype(np.float64)
            _, nb = cKDTree(p).query(p, k=min(k, index.n), workers=-1)
            if nb.ndim == 1:
                nb = nb[:, None]
            if nb.shape[1] >= 3:
                x = p[nb]
                x = x - x.mean(1, keepdims=True)
                out = np.linalg.eigh(np.einsum("nki,nkj->nij", x, x) / x.shape[1])[1][:, :, 0]
        return torch.from_numpy(np.ascontiguousarray(out))

    def pc_count_nonfinite(self, pts):
        self._rec(PP.nonfinite_desc(pts.numpy()))
        return torch.tensor([int((~np.isfinite(pts.numpy())).sum())], dtype=torch.int32)

    def pc_abs_dot(self, a, b, a_idx=None, b_idx=None):
        assert a.dtype == b.dtype == torch.float64
        n = (a_idx if a_idx is not None else b_idx if b_idx is not None else a).shape[0]
        self._rec(PP.abs_dot_desc(n, a_idx is not None, b_idx is not None))
        an, bn = a.numpy(), b.numpy()
        an = an[a_idx.numpy()] if a_idx is not None else an
        bn = bn[b_idx.numpy()] if b_idx is not None else bn
        return torch.from_numpy(np.abs(np.sum(an * bn, -1)))

    def f64_mean(self, x):
        self._rec(PP.mean_desc(x.numel()))
        return torch.tensor(np.mean(x.numpy()), dtype=torch.float64)

    def f64_median(self, x):
        self._rec(PP.median_desc(x.numpy()))
        return torch.tensor(np.median(x.numpy()), dtype=torch.float64)

    def f64_count_below(self, x, th):
        self._rec(PP.count_below_desc(x.numel()))
        return torch.tensor([int((x.numpy() < th).sum())], dtype=torch.int64)


POINT_OPS = ("pc_index", "pc_nearest", "pc_knn_normals", "pc_count_nonfinite", "pc_abs_dot", "f64_mean", "f64_median",
             "f64_count_below")
LAND = (368, 512)


def _scene(g, v, b, h, w):
    """views / preds of evaluate_reconstruction: a wavy surface per view, the prediction a similarity of it plus noise."""
    yy, xx = torch.meshgrid(torch.linspace(-0.75, 0.75, h), torch.linspace(-1, 1, w), indexing="ij")
    views, preds = [], []
    for j in range(v):
        z = 2 + 0.2 * torch.sin(3 * xx + j) * torch.cos(2 * yy) + 0.01 * torch.randn(b, h, w, generator=g)
        gt = torch.stack([xx * z + 0.3 * j, yy * z, z], -1)
        pr = 0.8 * gt + 0.1 + 0.001 * torch.randn(b, h, w, 3, generator=g)
        views.append(dict(img=torch.empty(b, 3, h, w), pts3d=gt, valid_mask=torch.rand(b, h, w, generator=g) > 0.1,
                          label=[f"scene{j}/frame{k}" for k in range(b)]))
        conf = 1 + torch.rand(b, h, w, generator=g)
        preds.append(dict(pts3d_in_other_view=pr, conf=conf, pts3d_local=pr.clone(), conf_local=conf.clone()))
    return views, preds


def all_metric_calls(monkeypatch):
    import fast3r_b200.ops as O
    import fast3r_b200.postprocess as P
    import fast3r_b200.recon_metric as RM
    rec, geo = Recorder(), GeometryRecorder()
    monkeypatch.setattr(RM, "_device", lambda xs, device: torch.device("cpu"))
    monkeypatch.setattr(P, "_device_of", lambda t, device: torch.device("cpu"))
    for name in POINT_OPS:
        monkeypatch.setattr(O, name, getattr(rec, name))
    for name in ("conf_quantile", "similarity_fit", "similarity_apply", "focal_weiszfeld"):
        monkeypatch.setattr(O, name, getattr(geo, name))
    rng = np.random.default_rng(0)
    for n_gt, n_rec in ((1, 1), (2, 3), (33, 4097), (4097, 2049), (262145, 100), (0, 5), (5, 0), (0, 0)):
        gt, rc = rng.standard_normal((n_gt, 3)), rng.standard_normal((n_rec, 3))
        gn, rn = rng.standard_normal((n_gt, 3)), rng.standard_normal((n_rec, 3))
        for kind, conv in (("numpy f64", lambda a: a), ("numpy f32", lambda a: a.astype(np.float32)),
                           ("torch f32", lambda a: torch.from_numpy(a.astype(np.float32))),
                           ("torch f64", torch.from_numpy), ("int", lambda a: (a * 10).astype(np.int64))):
            rec.where = f"{kind} gt {n_gt} rec {n_rec}"
            g_, r_ = conv(gt), conv(rc)
            RM.accuracy(g_, r_)
            RM.completion(g_, r_)
            if n_gt and n_rec:
                RM.accuracy(g_, r_, gn, rn)
                RM.completion(g_, r_, gn, rn)
            RM.completion_ratio(g_, r_)
            RM.nearest_neighbors(g_, r_)
            for k in (1, 3, 30, 32):
                RM.estimate_normals(g_, knn=k)
    g = torch.Generator().manual_seed(1)
    for v, b in ((32, 1), (4, 2)):
        views, preds = _scene(g, v, b, *LAND)
        for local in (True, False):
            rec.where = f"evaluate_reconstruction {v} views B={b} local={local}"
            P.evaluate_reconstruction(views, [dict(p) for p in preds], use_pts3d_from_local_head=local)
    return rec.calls


@pytest.fixture(scope="module")
def recorded():
    mp = pytest.MonkeyPatch()
    try:
        yield all_metric_calls(mp)
    finally:
        mp.undo()


@pytest.fixture(scope="module")
def table_keys():
    """key -> names of the cases that reach it, from the cases' own data."""
    out = {}
    for c in PP.CASES:
        for d in PP.case_descs(c):
            out.setdefault(PP.key(d), []).append(c["name"])
    return out


def test_recorder_sees_the_callers(recorded):
    """Sanity of the recorder: evaluate_reconstruction at 32 views indexes both 6 029 312-point clouds (less the masked
    pixels), and every op was recorded."""
    ev = [d for d, w in recorded if w.startswith("evaluate_reconstruction 32")]
    assert {d["op"] for d in ev} >= {"index", "nearest", "knn", "mean", "median", "abs_dot", "nonfinite"}
    assert max(d["n"] for d in ev if d["op"] == "index") > 5_000_000
    assert {d["op"] for d, _ in recorded} == set(PP.KEYS)
    assert any(d["op"] == "nearest" and d["n_ref"] == 0 for d, _ in recorded)


def test_every_caller_key_has_a_gpu_case(recorded, table_keys):
    missing = {}
    for d, where in recorded:
        k = PP.key(d)
        if k not in table_keys:
            missing.setdefault(k, (d, where))
    assert not missing, "launch keys of the recon_metric callers without a case in tests/pointcloud_plans.CASES:\n" + \
        "\n".join(f"  {k}\n      from {where}: {d}" for k, (d, where) in sorted(missing.items()))


def test_cases_reach_what_they_are_built_for():
    """Case names are unique; each nearest case's data reaches the flags it is built for (pointcloud_plans.
    expected_flags), and each knn case its (n, k) key."""
    names = [c["name"] for c in PP.CASES]
    assert len(names) == len(set(names))
    wrong = []
    for c in PP.NEAREST:
        descs = PP.case_descs(c)
        ix = PP.key(descs[0]).split() if c["n"] else []
        got = set(ix[3:]) & {"flat", "flataxis"} | set(PP.key(descs[-1]).split()[2:])
        checked = {"flat", "flataxis", "outside", "tiles"} | ({"past"} if c["qmode"] == "far" else set())
        if got & checked != set(c["expect"]):
            wrong.append((c["name"], c["expect"], sorted(got)))
    assert not wrong, "\n".join(f"{n}: built for {e}, reaches {g}" for n, e, g in wrong)


def test_table_reaches_the_contract(table_keys):
    """The table reaches every flag of every op, on and off; every size, geometry, k and dtype pair of the contract
    matrix has a case, and the callers' shapes have theirs."""
    keys = set(table_keys)
    for op, flags in (("index", ("small", "partial", "ppart", "tiles", "scanloop", "bboxcap", "flat", "flataxis")),
                      ("nearest", ("tiles", "outside", "past")),
                      ("knn", ("k<3", "k32", "k>n", "k=n", "spill")), ("mean", ("one", "stride")),
                      ("median", ("odd", "even", "tie", "cap", "nan")), ("count_below", ("cap",)),
                      ("nonfinite", ("cap",)), ("abs_dot", ("aidx", "bidx", "partial"))):
        ks = [k.split()[1:] for k in keys if k.split()[0] == op]
        for f in flags:
            assert any(f in k for k in ks) and any(f not in k for k in ks), (op, f)
    for a in ("f32", "f64"):
        assert any(k.startswith(f"index {a}") for k in keys)
        for b in ("f32", "f64"):
            assert any(k.startswith(f"nearest {a}x{b}") for k in keys), (a, b)
    assert {len(PP.tree_counts(n)) for n in PP.SIZES + PP.CALLER_N} <= {int(k.split()[2][1:]) for k in keys
                                                                     if k.startswith("index")}
    nn = PP.NEAREST
    assert set(PP.SIZES) <= {c["n"] for c in nn if c["geometry"] == "gauss"}
    assert set(PP.CALLER_N) <= {c["n"] for c in nn} and set(PP.CALLER_N) <= {c["n"] for c in PP.KNN}
    for g in PP.GEOMETRIES:
        assert {"near", "far"} <= {c["qmode"] for c in nn if c["geometry"] == g}, g
    assert any(c["geometry"] == "cluster" and c["n"] >= 1 << 20 for c in nn)
    for k in PP.KS:
        ks = {c["geometry"] for c in PP.KNN if c["k"] == k}
        assert {"surface", "dup", "lattice", "plane", "line", "same"} <= ks, k
        assert {c["n"] for c in PP.KNN if c["k"] == k and c["geometry"] == "surface"} >= {1, 2, 3, 4, 31, 33, 4097}
    assert set(PP.CALLER_N) <= {c["n"] for c in PP.REDUCTIONS}
