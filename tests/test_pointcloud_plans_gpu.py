"""The reconstruction metrics (csrc/pointcloud.cu) per element against scipy, numpy and long-double references, one case
per launch key of tests/pointcloud_plans.CASES.  Needs an H100.

Every output, the index block and the query workspace sit between canaries that must keep their bytes.  u = 2^-53 is
the fp64 unit roundoff, gamma_k = k u / (1 - k u).

Nearest.  Distances bit-equal to cKDTree.query; indices equal wherever the second-nearest distance is larger; at a tie,
the distance recomputed to the returned point with scipy's rounding, sqrt((dx dx + dy dy) + dz dz), is bit-equal too.
Where every squared distance overflows (coordinates near 1e160) scipy returns inf and index n, and so must the kernel.

Normals.  For each checked point the reference takes the fp64 neighbour set of cKDTree(k) (the point included) and
forms the covariance in long double, two-pass: C = sum (p - m)(p - m)^T / k', k' = min(k, n).  The kernel's fp64
covariance differs from C in two ways.  Its mean m^ = fl(sum p / k') is off by at most delta = gamma_k' sum|p| / k' per
axis, which adds exactly delta delta^T to the centred sum (sum (p - m) = 0).  Its differences, products, k'-term sum
and division round each entry by at most gamma_{k'+4} D_ij, D_ij = sum (|d_i| + delta_i)(|d_j| + delta_j) / k'.  So
    ||C^ - C||_F <= ||delta||^2 + gamma_{k'+4} ||D||_F =: e_C.
The Jacobi solve (geometry_math.h:18-62) stops when off^2 <= 1e-34 diag^2, i.e. off <= 1e-17 ||C^||_F < u ||C^||_F, and
runs at most 32 sweeps of 3 rotations, each an orthogonal transform up to a few u; its eigenvector v of the smallest
eigenvalue is therefore the exact one of a matrix within e_J = 96 * 8 u ||C^||_F of C^ (plus u for the stopping rule),
and normalising costs 4 u ||C^||.  The Rayleigh residual of the returned unit normal n against the reference,
    r = n^T C n - lambda_min(C) <= 2 e_C + 2 e_J + 4 u ||C||_F + 8 u ||C||_F =: eps,
where the last term covers eigh's lambda_min and the rounding of C to fp64.  The residual holds in degenerate
eigenspaces (a plane's normal is unique, a line's is any vector orthogonal to it, identical points allow any unit
vector) and gives the angle wherever there is a gap: sin^2(theta) <= eps / (lambda_2 - lambda_1).  ||n|| = 1 within 8 u.
Fewer than 3 neighbours give (0, 0, 1) exactly.  When distances tie at the k-th neighbour, the admissible sets are the
strictly nearer points plus any choice from the tied group: if the tied points coincide, every choice is the same
cloud; else up to 20 choices are enumerated and one must pass; lattices and planes are built so that every admissible
set is planar with normal +-z, and any one set is checked.  At 6 M points a strided sample is checked.

Reductions.  Median bit-equal to np.median (NaN of either sign anywhere gives NaN; the sign of a zero median is free,
numpy's partition leaves it unspecified).  count_below and count_nonfinite exact.  abs_dot bit-equal to
np.abs(np.sum(a[ia] * b[ib], -1)).  The mean (f64_sum_kernel and f64_mean_final_kernel, pointcloud.cu:563-584): each of 65 536 threads adds its
ceil(n / 65 536) strided elements in order from 0, then 5 shuffle levels, 8 warp partials in order and 256 block
partials in order, then one division; so every term passes through K = ceil(n / 65 536) + 5 + 8 + 256 roundings and
    |mean - fsum(x) / n| <= gamma_K sum|x| / n + 2 u |mean_ref|
(the reference is math.fsum rounded once, then divided once).

completion_ratio at n in {2^24 - 1, 2^24 + 3, 20 000 001} ground-truth points equals numpy's own expression
np.mean((d < th).astype(np.float32)) on the distances of nearest_neighbors (pinned bit-equal above)."""
import itertools
import math

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from tests import pointcloud_plans as PP
from tests.canaries import PAD, buffer, untouched

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
BYTE_PAD = 256
CANARY_BYTE = 0xA5


def gamma(k):
    return k * U / (1 - k * U)


def _ops():
    from fast3r_b200 import ops
    return ops


def _call(name, anchor, *args):
    ops = _ops()
    ops._call(name, anchor, *[ops._ptr(a) if isinstance(a, torch.Tensor) or a is None else a for a in args])


def _block(nbytes):
    """(full uint8 buffer, 256-byte-aligned view of nbytes in its middle); the canary bytes hold CANARY_BYTE."""
    buf = torch.full((nbytes + 2 * BYTE_PAD,), CANARY_BYTE, dtype=torch.uint8, device="cuda")
    assert buf.data_ptr() % 256 == 0
    return buf, buf[BYTE_PAD:BYTE_PAD + nbytes]


def _block_canaries(name, buf):
    c = torch.cat([buf[:BYTE_PAD], buf[-BYTE_PAD:]])
    assert bool((c == CANARY_BYTE).all()), f"{name}: a canary byte around the block changed"


def _out(n, dtype):
    fill = -7 if dtype == torch.int64 else None
    if fill is None:
        return buffer((n,), dtype)
    buf = torch.full((n + 2 * PAD,), fill, dtype=dtype, device="cuda")
    return buf, buf[PAD:PAD + n]


def _sent(buf):
    return torch.full_like(buf, -7 if buf.dtype == torch.int64 else -1234.5)


def _check_out(name, buf):
    written = torch.zeros_like(buf, dtype=torch.bool)
    written[PAD:buf.numel() - PAD] = True
    untouched(name, buf, _sent(buf), written)


def _report(kind, name, ratio):
    print(f"\nERROR/BOUND {kind} {name}: {ratio:.3g}")


def build_index(name, pts):
    """pts: CUDA (n, 3) float32 / float64 -> (full block buffer, block view), canaries checked."""
    lib = _ops().L.load()
    n = pts.shape[0]
    nbytes = lib.f3r_pc_index_workspace(n)
    buf, blk = _block(nbytes)
    _call("f3r_pc_index_build", pts, pts, int(pts.dtype == torch.float64), n, blk, nbytes)
    torch.cuda.synchronize()
    _block_canaries(f"{name} index", buf)
    return buf, blk


# ------------------------------------------------------------------ nearest
def run_nearest(name, ref, query):
    """Kernel (dist, idx) of every query as numpy, with canaries around the index, workspace and outputs."""
    lib = _ops().L.load()
    r = torch.from_numpy(ref).cuda()
    q = torch.from_numpy(query).cuda()
    n, nq = len(ref), len(query)
    dbuf, dist = _out(nq, torch.float64)
    ibuf, idx = _out(nq, torch.int64)
    if n:
        ib, blk = build_index(name, r)
        ws_bytes = lib.f3r_pc_query_workspace(nq)
        wbuf, ws = _block(ws_bytes)
        _call("f3r_pc_nearest", q, blk, blk.numel(), n, q, int(q.dtype == torch.float64), nq, dist, idx, ws, ws_bytes)
    else:
        _call("f3r_pc_nearest", q, None, 0, 0, q, int(q.dtype == torch.float64), nq, dist, idx, None, 0)
    torch.cuda.synchronize()
    if n:
        _block_canaries(f"{name} index", ib)
        _block_canaries(f"{name} workspace", wbuf)
    _check_out(f"{name} dist", dbuf)
    _check_out(f"{name} idx", ibuf)
    return dist.cpu().numpy(), idx.cpu().numpy()


def check_nearest(name, ref, query, d, i):
    n = len(ref)
    if n == 0:
        assert np.isinf(d).all() and (i == 0).all(), name
        return
    r64, q64 = ref.astype(np.float64), query.astype(np.float64)
    k = 2 if n > 1 else 1
    dr, ir = cKDTree(r64).query(q64, k=k, workers=-1)
    d1, i1 = (dr, ir) if k == 1 else (dr[:, 0], ir[:, 0])
    bad = np.flatnonzero(d.view(np.uint64) != d1.view(np.uint64))
    assert not len(bad), f"{name}: {len(bad)} of {len(d)} distances differ from cKDTree; first {bad[:5].tolist()}: " \
                         f"got {d[bad[:5]].tolist()} want {d1[bad[:5]].tolist()}"
    unique = np.ones(len(d), bool) if k == 1 else d1 < dr[:, 1]
    wrong = np.flatnonzero(unique & (i != i1))
    assert not len(wrong), f"{name}: {len(wrong)} unique nearest indices differ; first {wrong[:5].tolist()}"
    none = i == n  # every squared distance overflowed: scipy's inf and n
    assert np.array_equal(none, i1 == n) and np.isinf(d[none]).all(), name
    p = r64[i[~none]]
    dx, dy, dz = (q64[~none] - p).T
    with np.errstate(over="ignore"):
        again = np.sqrt((dx * dx + dy * dy) + dz * dz)
    assert np.array_equal(again.view(np.uint64), d[~none].view(np.uint64)), f"{name}: a tie returned a farther point"


@pytest.mark.parametrize("case", PP.NEAREST, ids=[c["name"] for c in PP.NEAREST])
def test_nearest(case):
    ref, q = PP.nearest_inputs(case)
    d, i = run_nearest(case["name"], ref, q)
    check_nearest(case["name"], ref, q, d, i)


# ------------------------------------------------------------------ normals
def run_normals(name, pts, k):
    t = torch.from_numpy(pts).cuda()
    ib, blk = build_index(name, t)
    obuf, out = buffer((len(pts) * 3,), torch.float64)
    _call("f3r_pc_knn_normals", t, blk, blk.numel(), len(pts), k, out)
    torch.cuda.synchronize()
    _block_canaries(f"{name} index", ib)
    _check_out(f"{name} normals", obuf)
    return out.view(-1, 3).cpu().numpy()


def _residual(p, nrm):
    """(r, eps) of one neighbour set p (k', 3) float64 and the kernel's normal."""
    L = np.longdouble
    kk = len(p)
    pl = p.astype(L)
    m = pl.sum(0) / kk
    d = pl - m
    C = (d[:, :, None] * d[:, None, :]).sum(0) / kk
    delta = gamma(kk) * np.abs(p).sum(0) / kk
    ad = np.abs(d).astype(np.float64) + delta
    D = (ad[:, :, None] * ad[:, None, :]).sum(0) / kk
    cf = float(np.sqrt((C.astype(np.float64) ** 2).sum()))
    e_c = float(delta @ delta) + gamma(kk + 4) * float(np.sqrt((D ** 2).sum()))
    c_hat = cf + e_c
    eps = 2 * e_c + 2 * (96 * 8 * U + U) * c_hat + 12 * U * cf
    nl = nrm.astype(L)
    nl = nl / np.sqrt((nl * nl).sum())
    lam = float(np.linalg.eigvalsh(C.astype(np.float64))[0])
    r = float(nl @ C @ nl) - lam
    return r, max(eps, 1e-300)


def check_normals(case, pts, nrm):
    name, k, n = case["name"], case["k"], len(pts)
    assert np.isfinite(nrm).all(), name
    kk = min(k, n)
    if kk < 3:
        assert np.array_equal(nrm, np.tile([0.0, 0.0, 1.0], (n, 1))), name
        return 0.0
    assert np.abs(np.sqrt((nrm ** 2).sum(1)) - 1).max() <= 8 * U, name
    p64 = pts.astype(np.float64)
    tree = cKDTree(p64)
    rows = np.arange(0, n, max(1, n // case.get("sample", 1024)))
    kq = min(n, kk + 40)
    dd, nb = tree.query(p64[rows], k=kq, workers=-1)
    dd, nb = dd.reshape(len(rows), -1), nb.reshape(len(rows), -1)
    shared = case["geometry"] in ("lattice", "plane", "same", "dup")
    worst, skipped = 0.0, 0
    for j, row in enumerate(rows):
        dk = dd[j, kk - 1]
        strict = nb[j, dd[j] < dk]
        group = nb[j, dd[j] == dk]
        need = kk - len(strict)
        sets = [np.concatenate([strict, group[:need]])]
        if len(group) > need:
            open_ended = kq < n and dd[j, -1] == dk
            same = (p64[group] == p64[group[0]]).all()
            if not same and not shared:
                if open_ended or math.comb(len(group), need) > 20:
                    skipped += 1
                    continue
                sets = [np.concatenate([strict, list(c)]) for c in itertools.combinations(group, need)]
        best = min((r / e for r, e in (_residual(p64[s], nrm[row]) for s in sets)))
        assert best <= 1.0, f"{name}: point {row}: Rayleigh residual {best:.3g}x its bound"
        worst = max(worst, best)
    assert skipped <= len(rows) // 10, f"{name}: {skipped} of {len(rows)} points tied beyond enumeration"
    return worst


@pytest.mark.parametrize("case", PP.KNN, ids=[c["name"] for c in PP.KNN])
def test_normals(case):
    pts = PP.knn_cloud(case)
    nrm = run_normals(case["name"], pts, case["k"])
    _report("normals", case["name"], check_normals(case, pts, nrm))


# ------------------------------------------------------------------ reductions
def _reduce(name, x):
    lib = _ops().L.load()
    t = torch.from_numpy(x).cuda()
    nbytes = lib.f3r_f64_reduce_workspace()
    wbuf, ws = _block(nbytes)
    obuf, out = buffer((1,), torch.float64)
    _call(name, t, t, t.numel(), out, ws, nbytes)
    torch.cuda.synchronize()
    _block_canaries(name, wbuf)
    _check_out(name, obuf)
    return float(out.cpu()[0])


def _same_median(got, want):
    return (np.isnan(got) and np.isnan(want)) or got == want


def _count_below(x, th):
    t = torch.from_numpy(x).cuda()
    thr = torch.tensor([th], dtype=torch.float64, device="cuda")
    buf = torch.full((2 * PAD + 1,), -7, dtype=torch.int64, device="cuda")
    _call("f3r_f64_count_below", t, t, t.numel(), thr, buf[PAD:PAD + 1])
    torch.cuda.synchronize()
    _check_out("count_below", buf)
    return int(buf[PAD].cpu())


def _nonfinite(pts):
    t = torch.from_numpy(pts).cuda()
    buf = torch.full((2 * PAD + 1,), -7, dtype=torch.int32, device="cuda")
    _call("f3r_pc_count_nonfinite", t, t, int(t.dtype == torch.float64), len(pts), buf[PAD:PAD + 1])
    torch.cuda.synchronize()
    assert bool((buf[:PAD] == -7).all() and (buf[PAD + 1:] == -7).all()), "count_nonfinite canaries"
    return int(buf[PAD].cpu())


@pytest.mark.parametrize("case", PP.REDUCTIONS, ids=[c["name"] for c in PP.REDUCTIONS])
def test_reductions(case):
    n = case["n"]
    worst = 0.0
    with np.errstate(invalid="ignore"):
        for regime, x in PP.reduction_inputs(n, n).items():
            got, want = _reduce("f3r_f64_median", x), float(np.median(x))
            assert _same_median(got, want), (case["name"], regime, got, want)
            if np.isfinite(x).all():
                mean = _reduce("f3r_f64_mean", x)
                ref = math.fsum(x.tolist()) / n
                K = -(-n // PP.RED) + 5 + 8 + 256
                bound = gamma(K) * float(np.abs(x).sum()) / n + 2 * U * abs(ref)
                assert abs(mean - ref) <= bound, (case["name"], regime, mean, ref, bound)
                worst = max(worst, abs(mean - ref) / max(bound, 1e-300))
            fin = x[np.isfinite(x)]
            for th in (x[0], x[n - 1], x[n // 2], np.inf, -np.inf, np.nan, 0.0, float(np.median(fin)) if len(fin) else 0.0):
                assert _count_below(x, float(th)) == int((x < th).sum()), (case["name"], regime, th)
    _report("mean", case["name"], worst)
    rng = np.random.default_rng(n)
    for dt in (np.float32, np.float64):
        p = rng.standard_normal((n, 3)).astype(dt)
        assert _nonfinite(p) == 0
        for v in (np.nan, np.inf, -np.inf):
            q = p.copy()
            q[0, 0] = v
            q[n - 1, 2] = v
            q[n // 2, 1] = -np.inf
            assert _nonfinite(q) == int((~np.isfinite(q)).sum()), (case["name"], dt, v)
    a, b = rng.standard_normal((n, 3)), rng.standard_normal((n, 3))
    ia = rng.integers(0, n, n)
    ib = rng.integers(0, n, n)
    for use_a, use_b in ((False, False), (True, False), (False, True), (True, True)):
        ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        xa = torch.from_numpy(ia).cuda() if use_a else None
        xb = torch.from_numpy(ib).cuda() if use_b else None
        obuf, out = buffer((n,), torch.float64)
        _call("f3r_pc_abs_dot", ta, ta, xa, tb, xb, n, out)
        torch.cuda.synchronize()
        _check_out("abs_dot", obuf)
        want = np.abs(np.sum((a[ia] if use_a else a) * (b[ib] if use_b else b), -1))
        assert np.array_equal(out.cpu().numpy().view(np.uint64), want.view(np.uint64)), (case["name"], use_a, use_b)


# ------------------------------------------------------------------ completion_ratio past 2^24 points
@pytest.mark.parametrize("n", PP.COMPLETION_RATIO_N)
def test_completion_ratio_matches_numpy(n):
    from fast3r_b200 import recon_metric as rm
    rng = np.random.default_rng(n)
    gt = torch.from_numpy(rng.random((n, 3), dtype=np.float32)).cuda()
    rec = torch.from_numpy(rng.random((4096, 3), dtype=np.float32)).cuda()
    d, _ = rm.nearest_neighbors(rec, gt)
    d = d.cpu().numpy()
    for th in (0.02, 0.05, float(np.median(d))):
        got = rm.completion_ratio(gt, rec, dist_th=th)
        want = np.mean((d < th).astype(np.float32))
        assert isinstance(got, np.float32) and got == want, (n, th, float(got), float(want))


# ------------------------------------------------------------------ evaluate_reconstruction at 32 views x 368 x 512
def test_evaluate_reconstruction_32_views():
    from fast3r_b200 import postprocess as pp
    from fast3r_b200 import recon_metric as rm
    from tests.test_pointcloud_plans_cpu import _scene
    g = torch.Generator().manual_seed(3)
    views, preds = _scene(g, 32, 1, 368, 512)
    res = pp.evaluate_reconstruction(views, preds, use_pts3d_from_local_head=False)
    m = res[0]["scene0"]
    aligned, gt_pts, _ = pp._registered_clouds(views, preds, 0, 0, 0, False, torch.device("cuda:0"))
    a, gp = aligned.cpu().numpy().astype(np.float64), gt_pts.cpu().numpy().astype(np.float64)
    assert len(gp) > 5_000_000
    d_acc, i_acc = cKDTree(gp).query(a, workers=-1)
    d_comp, i_comp = cKDTree(a).query(gp, workers=-1)
    gn, an = rm.estimate_normals(gt_pts).cpu().numpy(), rm.estimate_normals(aligned).cpu().numpy()
    for pts, nrm, tag in ((gp, gn, "gt"), (a, an, "pred")):
        _report("normals", f"evaluate_32_views {tag}",
                check_normals(dict(name=f"evaluate {tag}", k=30, geometry="surface", sample=4000), pts, nrm))
    nc1 = np.abs(np.sum(gn[i_acc] * an, -1))
    nc2 = np.abs(np.sum(gn * an[i_comp], -1))
    for key, x in (("accuracy", d_acc), ("completion", d_comp), ("nc1", nc1), ("nc2", nc2)):
        assert m[f"{key}_median"] == np.median(x), key
        K = -(-len(x) // PP.RED) + 5 + 8 + 256
        ref = math.fsum(x.tolist()) / len(x)
        assert abs(m[key] - ref) <= gamma(K) * float(np.abs(x).sum()) / len(x) + 2 * U * abs(ref), key
