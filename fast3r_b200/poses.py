"""Camera poses from the forward's pointmaps, with the RANSAC scoring on the GPU.  Same names, arguments and results as
the reference, down to the dtypes:

* ``fast_pnp(pts3d, focal, msk, device, pp=None, niter_PnP=10, num_guessed_focals=100)`` -
  fast3r/dust3r/cloud_opt/init_im_poses.py:300-350: ``(focal, cam-to-world float32 (4, 4) tensor)`` or ``(None, None)``.
* ``estimate_cam_pose_one_sample(sample_preds, device='cpu', niter_PnP=10, min_conf_thr_percentile=0)`` -
  fast3r/models/multiview_dust3r_module.py:1038-1078: per view a float32 (4, 4) numpy pose and its focal, or the
  float64 identity and None where no pose is found.
* ``estimate_camera_poses(preds, views=None, niter_PnP=10, focal_length_estimation_method='individual')`` -
  MultiViewDUSt3RLitModule.estimate_camera_poses (multiview_dust3r_module.py:807-869).

The reference calls ``cv2.solvePnPRansac(pts, pixels, K, None, iterationsCount=niter_PnP, reprojectionError=5,
flags=SOLVEPNP_SQPNP)`` once per tentative focal and keeps the focal of the most inliers.  With a non-USAC flag OpenCV
runs its classic RANSACPointSetRegistrator, whose parts separate:

1. samples: every call seeds a fresh cv::RNG((uint64)-1), so the 5-point subsets depend only on the point count
   (``ransac_subsets`` replays the generator);
2. hypotheses: ``solvePnP(subset, SOLVEPNP_EPNP)`` on the fp32 subset - called here on the host, through cv2 itself;
3. scoring: the inlier count of every hypothesis over every point - the GPU (``ops.pnp_score``, csrc/pose.cu), all
   hypotheses of all focals of all views in one table;
4. bookkeeping: keep the first hypothesis whose count beats max(best, 4), shrink the iteration count by
   RANSACUpdateNumIters(0.99, ...) and stop where OpenCV stops - replayed on the host from the counts;
5. refit: ``solvePnP(inliers as float64, SOLVEPNP_SQPNP)`` on the inliers of the best hypothesis (``ops.pnp_inliers``
   compacts them in index order).  fast_pnp scores a focal by its RANSAC inlier count, so only the focal it would keep
   is refit; if that refit fails or raises, the next focal in the same order is.

So the results equal the reference's bit for bit.  4 and 5 points take OpenCV's special paths (P3P, a direct solve):
those views call cv2.solvePnPRansac itself.  Like the reference, these functions need cv2 (imported on first use).
"""
from __future__ import annotations

import functools
import logging
import math
import os
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, List

import numpy as np
import torch

from . import lib as L
from . import ops

log = logging.getLogger(__name__)

MODEL_POINTS = 5       # OpenCV's sample size with the EPnP kernel
CONFIDENCE = 0.99      # cv2.solvePnPRansac's default
REPROJ_ERROR = 5.0     # fast_pnp's reprojectionError
_DBL_MIN = 2.2250738585072014e-308


def _cv2():
    import cv2
    return cv2


@functools.lru_cache(maxsize=64)
def ransac_subsets(count: int, iters: int) -> np.ndarray:
    """(iters, 5) int64: the point subsets RANSACPointSetRegistrator::run draws for `count` points.  cv::RNG is a
    multiply-with-carry generator, state = (uint32)state * 4164903690 + (state >> 32), seeded with (uint64)-1 on every
    call; getSubset takes rng.uniform(0, count) = next() % count and redraws an index already in the subset."""
    state = 0xFFFFFFFFFFFFFFFF
    out = np.empty((iters, MODEL_POINTS), np.int64)
    for it in range(iters):
        for i in range(MODEL_POINTS):
            while True:
                state = (state & 0xFFFFFFFF) * 4164903690 + (state >> 32)
                j = (state & 0xFFFFFFFF) % count
                if j not in out[it, :i]:
                    break
            out[it, i] = j
    out.setflags(write=False)
    return out


def update_num_iters(p: float, ep: float, model_points: int, max_iters: int) -> int:
    """cv::RANSACUpdateNumIters."""
    p = min(max(p, 0.0), 1.0)
    ep = min(max(ep, 0.0), 1.0)
    num = max(1.0 - p, _DBL_MIN)
    denom = 1.0 - math.pow(1.0 - ep, model_points)
    if denom < _DBL_MIN:
        return 0
    num, denom = math.log(num), math.log(denom)
    return max_iters if (denom >= 0 or -num >= max_iters * (-denom)) else int(round(num / denom))


def ransac_replay(counts, ok, raised, count: int, niter: int):
    """The loop of RANSACPointSetRegistrator::run over precomputed hypotheses: counts[i] inliers of hypothesis i, ok[i]
    its EPnP solve succeeded, raised[i] it threw (which ends solvePnPRansac with the exception).  Returns the index of
    the kept hypothesis, None when none beats 4 inliers ("no model"), or "raised"."""
    niters, best, best_i, it = max(niter, 1), 0, None, 0
    while it < niters:
        if raised[it]:
            return "raised"
        if ok[it]:
            g = int(counts[it])
            if g > max(best, MODEL_POINTS - 1):
                best, best_i = g, it
                niters = update_num_iters(CONFIDENCE, (count - g) / count, MODEL_POINTS, niters)
        it += 1
    return best_i


def camera_matrix(focal, pp) -> np.ndarray:
    """K exactly as fast_pnp builds it (init_im_poses.py:325)."""
    return np.float32([(focal, 0, pp[0]), (0, focal, pp[1]), (0, 0, 1)])


def _epnp(pts: np.ndarray, pix: np.ndarray, K: np.ndarray):
    """EPnP hypotheses of one focal: pts (iters, 5, 3), pix (iters, 5, 2) fp32.  Returns (ok, raised, rvec, tvec)."""
    cv2 = _cv2()
    n = len(pts)
    ok, raised = np.zeros(n, bool), np.zeros(n, bool)
    rv, tv = np.zeros((n, 3)), np.zeros((n, 3))
    for i in range(n):
        try:
            ok[i], r, t = cv2.solvePnP(pts[i], pix[i], K, None, flags=cv2.SOLVEPNP_EPNP)
        except cv2.error:
            raised[i] = True
            continue
        if ok[i]:
            rv[i], tv[i] = r.ravel(), t.ravel()
    return ok, raised, rv, tv


def _hyp_rows(rv: np.ndarray, tv: np.ndarray, K: np.ndarray, view: int) -> np.ndarray:
    cv2 = _cv2()
    rows = np.zeros(len(rv), L.PNP_HYP)
    for i in range(len(rv)):
        rows["r"][i] = cv2.Rodrigues(rv[i].reshape(3, 1))[0].ravel()
    rows["t"] = tv
    kd = K.astype(np.float64)
    rows["fx"], rows["fy"], rows["cx"], rows["cy"] = kd[0, 0], kd[1, 1], kd[0, 2], kd[1, 2]
    rows["view"] = view
    return rows


def _pose_c2w(rvec, tvec, device):
    """init_im_poses.py:346-350 and sRT_to_4x4 (:277-281): the inverse of the float32 world-to-camera matrix."""
    R = torch.from_numpy(_cv2().Rodrigues(rvec)[0])
    T = torch.from_numpy(tvec)
    trf = torch.eye(4, device=device)
    trf[:3, :3] = R * 1
    trf[:3, 3] = T.ravel()
    return torch.linalg.inv(trf)


class _Job:
    """One fast_pnp call: a view of the gathered points with its tentative focals."""

    def __init__(self, focals, pp, niter):
        self.focals, self.pp, self.niter = focals, pp, niter
        self.result = (None, None)


def _solve(jobs: List[_Job], pts: torch.Tensor, pix: torch.Tensor, counts: np.ndarray, device, pool) -> None:
    """fast_pnp for every job; job j's masked points are pts/pix[j], the first counts[j] of them."""
    cv2 = _cv2()
    nj, slot = pts.shape[0], pts.shape[1]
    flat_pts, flat_pix = pts.reshape(-1, 3), pix.reshape(-1, 2)
    offsets = np.arange(nj, dtype=np.int64) * slot
    ransac = [j for j in range(nj) if counts[j] > MODEL_POINTS]
    for j in range(nj):
        if 4 <= counts[j] <= MODEL_POINTS:  # OpenCV's P3P / direct paths: the reference's own loop
            jobs[j].result = _reference_loop(pts[j, :counts[j]].cpu().numpy(), pix[j, :counts[j]].cpu().numpy(),
                                             jobs[j], device)
    if not ransac:
        return
    # 1. samples, gathered on the device and copied back
    subsets = {j: ransac_subsets(int(counts[j]), max(jobs[j].niter, 1)) for j in ransac}
    idx = torch.from_numpy(np.concatenate([subsets[j].ravel() + offsets[j] for j in ransac])).to(pts.device)
    sub_pts = flat_pts.index_select(0, idx).cpu().numpy()
    sub_pix = flat_pix.index_select(0, idx).cpu().numpy()
    # 2. EPnP hypotheses per (job, focal) on the thread pool
    tasks, at = [], 0
    for j in ransac:
        m = subsets[j].size
        jp, jx = sub_pts[at:at + m].reshape(-1, MODEL_POINTS, 3), sub_pix[at:at + m].reshape(-1, MODEL_POINTS, 2)
        at += m
        for fi, f in enumerate(jobs[j].focals):
            tasks.append((j, fi, jp, jx, camera_matrix(f, jobs[j].pp)))
    def solve_focal(task):
        j, _, jp, jx, K = task
        ok, raised, rv, tv = _epnp(jp, jx, K)
        return (ok, raised), _hyp_rows(rv[ok], tv[ok], K, j)

    solved = list(pool.map(solve_focal, tasks))
    hyps, rows = [s[0] for s in solved], [s[1] for s in solved]
    # 3. one table, scored on the GPU
    table = np.concatenate(rows)
    scores = np.zeros(0, np.int32)
    if len(table):
        scores = ops.pnp_score(flat_pts, flat_pix, offsets, counts, table, REPROJ_ERROR).cpu().numpy()
    # 4. the RANSAC loop of every (job, focal); candidates ordered as fast_pnp's "score > best" keeps them
    cands = {j: [] for j in ransac}
    at = 0
    for (j, fi, _, _, K), (ok, raised), r in zip(tasks, hyps, rows):
        full = np.zeros(len(ok), np.int64)
        full[ok] = scores[at:at + len(r)]
        at += len(r)
        best = ransac_replay(full, ok, raised, int(counts[j]), jobs[j].niter)
        if best is not None and best != "raised":
            cands[j].append((-int(full[best]), fi, r[int(np.count_nonzero(ok[:best]))], K))
    for j in ransac:
        cands[j].sort(key=lambda c: (c[0], c[1]))
    # 5. refit the best candidate of every job; a failed refit moves that job on to its next candidate
    pending = [j for j in ransac if cands[j]]
    while pending:
        heads = [cands[j].pop(0) for j in pending]
        table = np.array([h[2] for h in heads], L.PNP_HYP)
        ip, ix, ic = ops.pnp_inliers(flat_pts, flat_pix, offsets, counts, table, REPROJ_ERROR)
        ip, ix, ic = ip.cpu().numpy(), ix.cpu().numpy(), ic.cpu().numpy()
        starts = np.concatenate([[0], np.cumsum(counts[table["view"]].astype(np.int64))])

        def refit(k):
            n = int(ic[k])
            P, X = ip[starts[k]:starts[k] + n].astype(np.float64), ix[starts[k]:starts[k] + n].astype(np.float64)
            try:
                ok, r, t = cv2.solvePnP(P, X, heads[k][3], None, flags=cv2.SOLVEPNP_SQPNP)
            except cv2.error:
                return None
            return (r, t) if ok else None

        nxt = []
        for k, (j, res) in enumerate(zip(pending, pool.map(refit, range(len(pending))))):
            if res is None:
                if cands[j]:
                    nxt.append(j)
                continue
            jobs[j].result = (jobs[j].focals[heads[k][1]], _pose_c2w(res[0], res[1], device))
        pending = nxt


def _reference_loop(P: np.ndarray, X: np.ndarray, job: _Job, device):
    """fast_pnp's loop around cv2.solvePnPRansac (init_im_poses.py:323-350), for the point counts where OpenCV does not
    run RANSAC."""
    cv2 = _cv2()
    best = (0,)
    for focal in job.focals:
        K = camera_matrix(focal, job.pp)
        try:
            success, R, T, inliers = cv2.solvePnPRansac(P, X, K, None, iterationsCount=job.niter,
                                                        reprojectionError=REPROJ_ERROR, flags=cv2.SOLVEPNP_SQPNP)
            if not success:
                continue
        except cv2.error:
            continue
        if len(inliers) > best[0]:
            best = len(inliers), R, T, focal
    if not best[0]:
        return None, None
    _, R, T, focal = best
    return focal, _pose_c2w(R, T, device)


def _tentative_focals(focal, H, W, num_guessed_focals):
    if focal is None:
        S = max(W, H)
        return np.geomspace(S / 2, S * 3, num=num_guessed_focals)
    return [focal]


def _device_of(t, device=None) -> torch.device:
    if isinstance(t, torch.Tensor) and t.is_cuda:
        return t.device
    if not torch.cuda.is_available():
        raise RuntimeError("fast3r_b200.poses needs a CUDA device (there is no CPU path for the scoring)")
    return torch.device(device if device is not None else "cuda:0")


def _pool():
    return ThreadPoolExecutor(max_workers=os.cpu_count() or 1)


def _to_tensor(x) -> torch.Tensor:
    return x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x))


def fast_pnp(pts3d, focal, msk, device, pp=None, niter_PnP=10, num_guessed_focals=100):
    """init_im_poses.py:300-350, with the RANSAC scoring on pts3d's GPU (cuda:0 for host tensors and arrays)."""
    pts3d, msk = _to_tensor(pts3d), _to_tensor(msk)
    if msk.sum() < 4:
        return None, None
    H, W, THREE = pts3d.shape
    assert THREE == 3
    dev = _device_of(pts3d)
    pp = (W / 2, H / 2) if pp is None else _to_tensor(pp).cpu().numpy()
    job = _Job(_tentative_focals(focal, H, W, num_guessed_focals), pp, niter_PnP)
    p = pts3d.to(dev).to(torch.float32).reshape(1, H, W, 3).contiguous()
    m = msk.to(dev).to(torch.uint8).reshape(1, H, W).contiguous()
    g_pts, g_pix, cnt = ops.pnp_gather(p, mask=m)
    with _pool() as pool:
        _solve([job], g_pts, g_pix, cnt.cpu().numpy(), device, pool)
    return job.result


def _run_views(items, niter_PnP, pool):
    """items: (pts3d (H, W, 3), conf (H, W), focal or None) per view, any device.  Returns [(pose, focal)] as
    estimate_cam_pose_one_sample's process_view does (multiview_dust3r_module.py:1044-1066).  Views of one resolution
    share one gather."""
    out = [None] * len(items)
    groups: Dict[tuple, List[int]] = {}
    for k, (p, _, _) in enumerate(items):
        groups.setdefault(tuple(p.shape), []).append(k)
    for (H, W, _), ks in groups.items():
        dev = _device_of(items[ks[0]][0])
        pts = torch.stack([items[k][0].to(dev) for k in ks]).to(torch.float32).contiguous()
        conf = torch.stack([items[k][1].to(dev) for k in ks])
        if conf.dtype == torch.float32:
            g_pts, g_pix, cnt = ops.pnp_gather(pts, conf=conf.contiguous())
        else:  # the comparison in the confidences' own precision
            g_pts, g_pix, cnt = ops.pnp_gather(pts, mask=(conf > 1.0).to(torch.uint8).contiguous())
        cnt = cnt.cpu().numpy()
        jobs = [_Job(_tentative_focals(items[k][2], H, W, 100), (W / 2, H / 2), niter_PnP) for k in ks]
        _solve(jobs, g_pts, g_pix, cnt, "cpu", pool)
        for k, job in zip(ks, jobs):
            focal, pose = job.result
            if pose is None or focal is None:
                log.warning(f"Failed to estimate pose for view {k}")
                out[k] = (np.eye(4), focal)
            else:
                out[k] = (pose.cpu().numpy(), focal)
    return out


def estimate_cam_pose_one_sample(sample_preds, device="cpu", niter_PnP=10, min_conf_thr_percentile=0):
    """multiview_dust3r_module.py:1038-1078: (poses_c2w, focals) of one batch item's views."""
    items = [(p["pts3d_in_other_view"].squeeze(), p["conf"].squeeze(),
              float(p["focal_length"]) if "focal_length" in p else None) for p in sample_preds]
    with _pool() as pool:
        res = _run_views(items, niter_PnP, pool)
    return [r[0] for r in res], [r[1] for r in res]


def estimate_camera_poses(preds, views=None, niter_PnP=10, focal_length_estimation_method="individual"):
    """MultiViewDUSt3RLitModule.estimate_camera_poses (multiview_dust3r_module.py:807-869): ([poses_c2w per item],
    [focals per item]); all views of all batch items are solved together."""
    from .postprocess import estimate_focal
    batch_size = len(preds[0]["pts3d_in_other_view"])
    keys = {"first_view_from_global_head": ("pts3d_in_other_view", "conf"),
            "first_view_from_local_head": ("pts3d_local_aligned_to_global", "conf_local")}
    if focal_length_estimation_method not in keys and focal_length_estimation_method != "individual":
        raise ValueError(f"Unknown focal_length_estimation_method: {focal_length_estimation_method}")
    items = []
    for i in range(batch_size):
        focal = None
        if focal_length_estimation_method in keys:
            kp, kc = keys[focal_length_estimation_method]
            # [i][None], not [i:i + 1]: correct_preds_orientation leaves lists of per-item tensors
            focal = estimate_focal(preds[0][kp][i][None], preds[0][kc][i][None], min_conf_thr_percentile=10)
        items += [(p["pts3d_in_other_view"][i], p["conf"][i], focal) for p in preds]
    with _pool() as pool:
        res = _run_views(items, niter_PnP, pool)
    nv = len(preds)
    return ([[r[0] for r in res[i * nv:(i + 1) * nv]] for i in range(batch_size)],
            [[r[1] for r in res[i * nv:(i + 1) * nv]] for i in range(batch_size)])
