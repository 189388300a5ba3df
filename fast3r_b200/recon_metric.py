"""Reconstruction metrics on the GPU: drop-ins for ``fast3r.eval.recon_metric`` (fast3r/eval/recon_metric.py:14-49).

* ``accuracy(gt_points, rec_points, gt_normals=None, rec_normals=None, device=None)`` - distance of every reconstructed
  point to its nearest ground-truth point: (mean, median), plus (mean, median) of the normal consistency |n_gt . n_rec|
  over those pairs when both normal arrays are given.
* ``completion(...)`` - the same from every ground-truth point to the reconstruction.
* ``completion_ratio(gt_points, rec_points, dist_th=0.05)`` - share of ground-truth points nearer than ``dist_th``.

Same arguments and result types as the reference (numpy float64 scalars, ``completion_ratio`` a numpy float32).  The
nearest neighbours are exact: every distance is bit-equal to scipy's ``cKDTree.query`` (fp64, the same rounding), the
medians are exact and the means are fixed-order fp64 sums (equal to numpy's pairwise sums to a few ulp).  Inputs may be
numpy arrays or torch tensors on the host or on a CUDA device; host inputs are uploaded to ``device`` (default cuda:0).
Points with a non-finite coordinate raise ``ValueError`` as in scipy; an empty reference cloud gives infinite distances.
There is no CPU path: without CUDA this raises.

Building blocks: ``nearest_neighbors(ref, query) -> (dist, idx)`` and ``estimate_normals(points, knn=30)`` (Open3D's
``estimate_normals`` with a k-nearest neighbourhood, as ``evaluate_reconstruction`` uses it).  They return numpy arrays
for numpy input and tensors on the input's device otherwise.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops


def _device(xs, device) -> torch.device:
    for x in xs:
        if isinstance(x, torch.Tensor) and x.is_cuda:
            return x.device
    if not torch.cuda.is_available():
        raise RuntimeError("fast3r_b200.recon_metric needs a CUDA device (there is no CPU path)")
    return torch.device(device if device is not None else "cuda:0")


def _upload(x, dev: torch.device, what: str) -> torch.Tensor:
    """(n, 3) float32 / float64 contiguous tensor on dev; other dtypes are converted to float64, as scipy does."""
    t = torch.as_tensor(np.asarray(x) if not isinstance(x, torch.Tensor) else x)
    if t.dtype not in (torch.float32, torch.float64):
        t = t.to(torch.float64)
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{what}: expected an (n, 3) point array, got shape {tuple(t.shape)}")
    return t.to(dev, non_blocking=True).contiguous()


def _check_finite(*named) -> None:
    counts = [ops.pc_count_nonfinite(t) for _, t in named]
    for (what, _), c in zip(named, counts):
        if int(c.item()) != 0:
            raise ValueError(f"{what} must be finite")


def _normals(x, dev: torch.device) -> torch.Tensor:
    t = torch.as_tensor(np.asarray(x) if not isinstance(x, torch.Tensor) else x)
    return t.to(device=dev, dtype=torch.float64).contiguous()


def _host(x, like):
    """Result tensor back in the caller's world: numpy for numpy input, a tensor on the input's device otherwise."""
    if isinstance(like, torch.Tensor):
        return x.to(like.device)
    return x.cpu().numpy()


def _nn(ref: torch.Tensor, query: torch.Tensor):
    return ops.pc_nearest(ops.pc_index(ref), query)


def _mean_median(x: torch.Tensor):
    if x.numel() == 0:
        return np.float64(np.nan), np.float64(np.nan)
    return np.float64(ops.f64_mean(x).item()), np.float64(ops.f64_median(x).item())


def _metric(ref, query, ref_normals, query_normals, device, gather_ref: bool):
    """Distances from every query point to the reference cloud: (mean, median), and with normals (mean, median) of
    |dot| of the pairs, the gathered reference normal first (accuracy) or second (completion) as numpy multiplies them."""
    dev = _device((ref, query, ref_normals, query_normals), device)
    r, q = _upload(ref, dev, "reference points"), _upload(query, dev, "query points")
    _check_finite(("reference points", r), ("query points", q))
    dist, idx = _nn(r, q)
    out = _mean_median(dist)
    if ref_normals is None or query_normals is None:
        return out
    rn, qn = _normals(ref_normals, dev), _normals(query_normals, dev)
    if r.shape[0] == 0 and q.shape[0] > 0:
        raise IndexError("normal consistency against an empty cloud: no nearest point to take a normal from")
    if rn.shape != r.shape or qn.shape != q.shape:
        raise ValueError("normals must have the shape of their points")
    dots = ops.pc_abs_dot(rn, qn, a_idx=idx) if gather_ref else ops.pc_abs_dot(qn, rn, b_idx=idx)
    return out + _mean_median(dots)


def accuracy(gt_points, rec_points, gt_normals=None, rec_normals=None, device=None):
    """Every reconstructed point against its nearest ground-truth point (recon_metric.py:21-35)."""
    return _metric(gt_points, rec_points, gt_normals, rec_normals, device, gather_ref=True)


def completion(gt_points, rec_points, gt_normals=None, rec_normals=None, device=None):
    """Every ground-truth point against its nearest reconstructed point (recon_metric.py:38-49)."""
    return _metric(rec_points, gt_points, rec_normals, gt_normals, device, gather_ref=False)


EXACT_F32_SUM = 1 << 24  # numpy's float32 sum of n ones and zeros is exact (every partial sum an integer <= 2^24)


def completion_ratio(gt_points, rec_points, dist_th=0.05):
    """np.mean((dist < dist_th).astype(np.float32)) over the ground-truth points (recon_metric.py:14-18).  Up to 2^24
    points numpy's float32 sum is the exact count, so this is float32(count) / float32(n) from a device count.  Past
    that, numpy's pairwise float32 partial sums round and its result depends on where the ones lie; the distances are
    copied to the host and the reference's own expression is evaluated on them."""
    dev = _device((gt_points, rec_points), None)
    r, q = _upload(rec_points, dev, "reconstructed points"), _upload(gt_points, dev, "ground-truth points")
    _check_finite(("reconstructed points", r), ("ground-truth points", q))
    n = q.shape[0]
    if n == 0:
        return np.float32(np.nan)
    dist, _ = _nn(r, q)
    if n > EXACT_F32_SUM:
        return np.mean((dist.cpu().numpy() < dist_th).astype(np.float32))
    count = int(ops.f64_count_below(dist, float(dist_th)).item())
    return np.float32(count) / np.float32(n)


def nearest_neighbors(ref, query, device=None):
    """(dist float64 (nq,), idx int64 (nq,)) of cKDTree(ref).query(query): exact, idx = len(ref) for an empty ref."""
    dev = _device((ref, query), device)
    r, q = _upload(ref, dev, "ref"), _upload(query, dev, "query")
    _check_finite(("ref", r), ("query", q))
    dist, idx = _nn(r, q)
    return _host(dist, query), _host(idx, query)


def estimate_normals(points, knn: int = 30, device=None):
    """float64 (n, 3) unit normals: per point the smallest-eigenvalue eigenvector of the covariance of its knn nearest
    points, itself included (fewer than 3 points: (0, 0, 1)); the sign is unspecified."""
    if not 1 <= int(knn) <= 32:
        raise ValueError(f"knn={knn} must be in [1, 32]")
    dev = _device((points,), device)
    p = _upload(points, dev, "points")
    _check_finite(("points", p))
    return _host(ops.pc_knn_normals(ops.pc_index(p), int(knn)), points)
