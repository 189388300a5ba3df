"""Reconstruction metrics on the GPU (csrc/pointcloud.cu through fast3r_b200.recon_metric) against the reference-generated
golden values, scipy's cKDTree run here, and numpy restatements.

Exact: distances (bit-equal to cKDTree), indices wherever the nearest point is unique, medians, completion_ratio.
Means are fixed-order fp64 sums, within 1e-12 relative of numpy's pairwise sums."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from tests.golden.recon_clouds import CASES, make_case

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "recon_metric.json")


def dig(a):
    return hashlib.sha256(np.ascontiguousarray(a, "<f8").tobytes()).hexdigest()


def close(a, b, rel=1e-12):
    return abs(float(a) - float(b)) <= rel * abs(float(b)) or float(a) == float(b)


@pytest.fixture(scope="module")
def rm():
    from fast3r_b200 import recon_metric
    return recon_metric


def test_golden_cases(rm):
    with open(GOLDEN) as f:
        gold = json.load(f)
    for c in gold["cases"]:
        gt, rec, gn, rn = make_case(c["kind"], c["seed"])
        d_acc, _ = rm.nearest_neighbors(gt, rec)
        d_comp, _ = rm.nearest_neighbors(rec, gt)
        assert isinstance(d_acc, np.ndarray) and d_acc.dtype == np.float64
        assert dig(d_acc) == c["dist_accuracy_sha256"] and dig(d_comp) == c["dist_completion_sha256"], c["kind"]
        acc, comp = rm.accuracy(gt, rec, gn, rn), rm.completion(gt, rec, gn, rn)
        assert all(isinstance(v, np.float64) for v in acc + comp)
        for got, want in ((acc, c["accuracy"]), (comp, c["completion"])):
            assert len(got) == len(want)
            assert got[1] == want[1] and close(got[0], want[0]), (c["kind"], got, want)
            if len(got) == 4:
                assert got[3] == want[3] and close(got[2], want[2]), (c["kind"], got, want)
        ratio = rm.completion_ratio(gt, rec)
        assert isinstance(ratio, np.float32) and float(ratio) == c["completion_ratio"], c["kind"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_nearest_matches_ckdtree(rm, dtype):
    g = torch.Generator().manual_seed(3)
    for n, nq in ((1, 50), (7, 1000), (40000, 30000), (100000, 5)):
        ref = torch.randn(n, 3, generator=g, dtype=torch.float64).to(dtype)
        ref[: n // 10] = ref[0]  # exact duplicates
        query = (torch.randn(nq, 3, generator=g, dtype=torch.float64) * 1.3).to(dtype)
        d, i = rm.nearest_neighbors(ref.cuda(), query.cuda())
        assert d.is_cuda and d.dtype == torch.float64 and i.dtype == torch.int64
        k = 2 if n > 1 else 1  # the second distance tells whether the nearest point is unique
        d_ref, i_ref = cKDTree(ref.numpy()).query(query.numpy(), k=k)
        first_d = d_ref if k == 1 else d_ref[:, 0]
        first_i = i_ref if k == 1 else i_ref[:, 0]
        assert np.array_equal(d.cpu().numpy(), first_d), (n, nq)
        unique = np.ones(nq, bool) if k == 1 else d_ref[:, 0] < d_ref[:, 1]
        assert np.array_equal(i.cpu().numpy()[unique], first_i[unique]), (n, nq)
        # a tie returns one of the equidistant points
        r = ref.double().numpy()[i.cpu().numpy()]
        q = query.double().numpy()
        dx, dy, dz = (q - r).T
        assert np.array_equal(np.sqrt((dx * dx + dy * dy) + dz * dz), first_d)


def test_full_size_device_clouds(rm):
    """32 depth-map views of 512x368 each side (6.03 M points), as device tensors."""
    g = torch.Generator().manual_seed(4)
    views, h, w = 32, 368, 512
    v, u = torch.meshgrid(torch.linspace(-0.75, 0.75, h), torch.linspace(-1, 1, w), indexing="ij")
    clouds = []
    for side in range(2):
        pts = []
        for k in range(views):
            z = 2 + 0.3 * torch.sin(3 * u + k + side * 0.01) * torch.cos(2 * v) + 0.01 * torch.randn(h, w, generator=g)
            p = torch.stack([u * z + 0.05 * k, v * z, z], -1).reshape(-1, 3)
            pts.append(p)
        clouds.append(torch.cat(pts).cuda())
    gt, rec = clouds
    assert gt.shape[0] == 6_029_312
    d, i = rm.nearest_neighbors(gt, rec)
    d_ref, i_ref = cKDTree(gt.cpu().numpy()).query(rec.cpu().numpy(), workers=-1)
    assert np.array_equal(d.cpu().numpy(), d_ref)
    acc = rm.accuracy(gt, rec)
    assert acc[1] == np.median(d_ref) and close(acc[0], np.mean(d_ref))
    ratio = rm.completion_ratio(rec, gt, dist_th=0.01)
    assert ratio == np.mean((d_ref < 0.01).astype(np.float32))


def test_reductions_match_numpy():
    from fast3r_b200 import ops
    rng = np.random.default_rng(8)
    for n in (1, 2, 3, 10, 1001, 65536, 1_000_003):
        x = np.abs(rng.standard_normal(n)) * 10 ** rng.uniform(-3, 3)
        if n > 10:
            x[: n // 4] = x[0]  # ties
            x[5] = np.inf
        t = torch.from_numpy(x).cuda()
        assert float(ops.f64_median(t)) == np.median(x), n
        if np.isfinite(x).all():
            assert close(float(ops.f64_mean(t)), np.mean(x)), n
        th = float(np.median(x))
        assert int(ops.f64_count_below(t, th)) == int((x < th).sum())


def test_normals_match_knn_eigh_restatement(rm):
    """estimate_normals: the smallest-eigenvalue eigenvector of the 30-NN covariance (scipy kNN + numpy eigh), away from
    near-degenerate neighbourhoods; (0, 0, 1) below 3 points."""
    rng = np.random.default_rng(9)
    u, v = rng.uniform(-1, 1, (2, 20000))
    pts = np.stack([u, v, 0.3 * np.sin(2 * u) * np.cos(3 * v)], -1) + 0.002 * rng.standard_normal((20000, 3))
    n = rm.estimate_normals(pts)
    assert n.shape == pts.shape and n.dtype == np.float64
    _, nb = cKDTree(pts).query(pts, k=30)
    checked = 0
    for i in range(0, len(pts), 7):
        c = np.cov(pts[nb[i]].T, bias=True)
        lam, vec = np.linalg.eigh(c)
        if lam[1] - lam[0] > 1e-2 * lam[1]:
            assert abs(n[i] @ vec[:, 0]) >= 1 - 1e-6, i
            checked += 1
    assert checked > 2000
    assert np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-12)
    two = rm.estimate_normals(np.array([[0.0, 0, 0], [1.0, 1, 1]]))
    assert np.array_equal(two, [[0, 0, 1], [0, 0, 1]])
    with pytest.raises(ValueError):
        rm.estimate_normals(pts, knn=33)


def test_nonfinite_input_raises_and_empty_reference(rm):
    pts = np.random.default_rng(10).random((1000, 3))
    for bad in (np.nan, np.inf, -np.inf):
        p = pts.copy()
        p[17, 1] = bad
        for fn in (lambda: rm.accuracy(p, pts), lambda: rm.accuracy(pts, p), lambda: rm.completion(p, pts),
                   lambda: rm.completion_ratio(pts, p), lambda: rm.nearest_neighbors(p, pts), lambda: rm.estimate_normals(p)):
            with pytest.raises(ValueError, match="finite"):
                fn()
    torch.cuda.synchronize()
    d, i = rm.nearest_neighbors(np.zeros((0, 3)), pts)
    assert np.isinf(d).all() and (i == 0).all()
    acc = rm.accuracy(np.zeros((0, 3)), pts)
    assert np.isinf(acc[0]) and np.isinf(acc[1])


def _rot(rng):
    q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    return q if np.linalg.det(q) > 0 else -q


@pytest.mark.parametrize("use_local", [False, True])
def test_evaluate_reconstruction_recovers_similarity(rm, use_local):
    from fast3r_b200 import postprocess as pp
    rng = np.random.default_rng(11)
    V, B, H, W = 3, 2, 48, 64
    truths = [(_rot(rng), rng.uniform(0.5, 2.0), rng.standard_normal(3)) for _ in range(B)]
    views, preds = [], []
    for j in range(V):
        gt = np.empty((B, H, W, 3), np.float32)
        pr = np.empty_like(gt)
        for b, (r, s, t) in enumerate(truths):
            uu, vv = np.meshgrid(np.linspace(-1, 1, W), np.linspace(-0.75, 0.75, H))
            z = 2 + 0.2 * np.sin(3 * uu + j + b) * np.cos(2 * vv)
            g = np.stack([uu * z + 0.3 * j, vv * z, z], -1)
            gt[b] = g
            pr[b] = ((g - t) @ r) / s  # gt = s R pr + t
        valid = torch.from_numpy(rng.random((B, H, W)) > 0.1)
        views.append({"img": torch.zeros(B, 3, H, W), "pts3d": torch.from_numpy(gt), "valid_mask": valid,
                      "label": [f"scene{j}/frame{k}" for k in range(B)]})
        conf = torch.from_numpy(1 + rng.random((B, H, W)).astype(np.float32))
        p = {"pts3d_in_other_view": torch.from_numpy(pr), "conf": conf}
        if use_local:
            p.update(pts3d_local=torch.from_numpy(pr), conf_local=conf)
        preds.append(p)
    res = pp.evaluate_reconstruction(views, preds, 30, 10, use_pts3d_from_local_head=use_local)
    assert len(res) == B and list(res[0]) == ["scene0"] and list(res[1]) == ["scene1"]
    dev = torch.device("cuda:0")
    for b, (r, s, t) in enumerate(truths):
        aligned, gt_pts, rts = pp._registered_clouds(views, preds, b, 30, 10, use_local, dev)
        rts = rts.cpu().double().numpy()
        assert np.allclose(rts[:9].reshape(3, 3), r, atol=1e-6) and abs(rts[12] - s) < 1e-6 * s
        assert np.allclose(rts[9:12], t, atol=1e-5)
        m = res[b][f"scene{b}"]
        a_np, g_np = aligned.cpu().numpy().astype(np.float64), gt_pts.cpu().numpy().astype(np.float64)
        d_acc, i_acc = cKDTree(g_np).query(a_np)
        d_comp, i_comp = cKDTree(a_np).query(g_np)
        assert m["accuracy_median"] == np.median(d_acc) and close(m["accuracy"], np.mean(d_acc))
        assert m["completion_median"] == np.median(d_comp) and close(m["completion"], np.mean(d_comp))
        # NC on the same normals, as numpy computes it
        gn, an = rm.estimate_normals(g_np), rm.estimate_normals(a_np)
        nc1 = np.abs(np.sum(gn[i_acc] * an, axis=-1))
        nc2 = np.abs(np.sum(gn * an[i_comp], axis=-1))
        assert m["nc1_median"] == np.median(nc1) and close(m["nc1"], np.mean(nc1))
        assert m["nc2_median"] == np.median(nc2) and close(m["nc2"], np.mean(nc2))
        assert all(isinstance(v, np.float64) for v in m.values())
