"""The geometry tail every caller runs on the forward's outputs (SURVEY.md §8 row f2, first slice), on the GPU.

Same names, arguments and results as the reference:

* ``align_local_pts3d_to_global(preds, views, min_conf_thr_percentile=0)`` -
  MultiViewDUSt3RLitModule.align_local_pts3d_to_global (fast3r/models/multiview_dust3r_module.py:427-549): adds
  ``pts3d_local_aligned_to_global`` (B, H, W, 3) to every pred.  The reference loops over (view, batch item) pairs in a
  CPU thread pool (torch.quantile + boolean gathers + roma SVD per pair); here all pairs go through three kernels
  (exact radix-select quantile, masked moments + Umeyama solve, streaming apply).
* ``estimate_focal(pts3d_i, conf_i, pp=None, min_conf_thr_percentile=10)`` - multiview_dust3r_module.py:1081-1109
  (returns a python float), and ``estimate_focal_knowing_depth(pts3d, pp, focal_mode="weiszfeld")`` -
  fast3r/dust3r/post_process.py:19-79 (returns a (B,) tensor).
* ``evaluate_reconstruction(views, preds, ...)`` - MultiViewDUSt3RLitModule.evaluate_reconstruction
  (multiview_dust3r_module.py:551-735): registration, normals and the metrics of fast3r_b200.recon_metric per batch item.

* ``fast_pnp``, ``estimate_cam_pose_one_sample`` and ``estimate_camera_poses`` - the camera poses, re-exported from
  fast3r_b200.poses (RANSAC scoring on the GPU, bit-identical to cv2.solvePnPRansac).
* ``correct_preds_orientation(preds, views)`` and ``evaluate_camera_poses(views, preds, niter_PnP=10,
  focal_length_estimation_method='individual')`` - multiview_dust3r_module.py:871-937 and :737-804: RRA / RTA / mAA
  per batch item, all pairs of all items in one launch (fast3r_b200.cam_pose_metric).

NOT here (documented in DESIGN.md §1): the "median" focal mode.  Tensors may live on the CPU (what ``inference()`` returns) or on a CUDA device; CPU inputs are
copied to ``device`` (default cuda:0) and the results copied back, so the function is a drop-in either way.  There is
no CPU implementation: without the CUDA library this raises.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from . import ops

_GROUP = 64  # (view, batch) pairs stacked per kernel call: bounds the staging copy to ~64 x 5.3 MB at 512x368


def _device_of(t: torch.Tensor, device) -> torch.device:
    if t.is_cuda:
        return t.device
    if not torch.cuda.is_available():
        raise RuntimeError("fast3r_b200.postprocess needs a CUDA device (there is no CPU path)")
    return torch.device(device if device is not None else "cuda:0")


def _f32(t: torch.Tensor, dev: torch.device) -> torch.Tensor:
    return t.to(device=dev, dtype=torch.float32, non_blocking=True).contiguous()


def align_local_pts3d_to_global(preds: List[Dict], views: List[Dict], min_conf_thr_percentile: float = 0, device=None) -> None:
    for pred in preds:
        for key, what in (("pts3d_local", "Key 'pts3d_local' not found in preds."),
                          ("conf_local", "Key 'conf_local' not found in preds."),
                          ("pts3d_in_other_view", "Key 'pts3d_in_other_view' not found in preds."),
                          ("conf", "Key 'conf' (global head confidence) not found in preds.")):
            if key not in pred:
                raise ValueError(what)
    if not preds:
        return
    dev = _device_of(preds[0]["pts3d_local"], device)
    q = float(min_conf_thr_percentile) / 100.0
    for g0 in range(0, len(preds), _GROUP):
        group = preds[g0:g0 + _GROUP]
        gviews = views[g0:g0 + _GROUP] if views is not None else [{}] * len(group)
        shapes = {tuple(p["pts3d_local"].shape) for p in group}
        if len(shapes) != 1:  # mixed resolutions: one call per pred
            for p, v in zip(group, gviews):
                _align_group([p], [v], q, dev)
        else:
            _align_group(group, gviews, q, dev)


def _align_group(group: List[Dict], gviews: List[Dict], q: float, dev: torch.device) -> None:
    b, h, w, _ = group[0]["pts3d_local"].shape
    n = h * w
    x = torch.cat([_f32(p["pts3d_local"], dev).reshape(b, n, 3) for p in group])
    y = torch.cat([_f32(p["pts3d_in_other_view"], dev).reshape(b, n, 3) for p in group])
    conf = torch.cat([_f32(p["conf"], dev).reshape(b, n) for p in group])
    valid = None
    if any("valid_mask" in v for v in gviews):
        valid = torch.cat([
            (v["valid_mask"].to(dev).reshape(b, n) if "valid_mask" in v else torch.ones(b, n, dtype=torch.bool, device=dev))
            .to(torch.uint8) for v in gviews]).contiguous()
    thr = ops.conf_quantile(conf, q)
    rts = ops.similarity_fit(x, y, conf, thr, valid)
    out = ops.similarity_apply(x, rts)
    for i, p in enumerate(group):
        src = p["pts3d_local"]
        aligned = out[i * b:(i + 1) * b].reshape(b, h, w, 3)
        p["pts3d_local_aligned_to_global"] = aligned.to(device=src.device, dtype=src.dtype)  # no copy if already there


def estimate_focal(pts3d_i: torch.Tensor, conf_i: torch.Tensor, pp: Optional[torch.Tensor] = None,
                   min_conf_thr_percentile: float = 10, device=None) -> float:
    b, h, w, three = pts3d_i.shape
    assert three == 3
    assert b == 1  # the reference processes one sample at a time
    dev = _device_of(pts3d_i, device)
    pts = _f32(pts3d_i, dev)
    conf = _f32(conf_i, dev).reshape(b, h, w)
    thr = ops.conf_quantile(conf.reshape(b, h * w), float(min_conf_thr_percentile) / 100.0)
    ppt = None if pp is None else _f32(torch.as_tensor(pp), dev).reshape(b, 2)
    return float(ops.focal_weiszfeld(pts, conf, thr, ppt, iters=100)[0])


from .poses import estimate_cam_pose_one_sample, estimate_camera_poses, fast_pnp  # noqa: E402,F401


def estimate_focal_knowing_depth(pts3d: torch.Tensor, pp: torch.Tensor, focal_mode: str = "weiszfeld", device=None) -> torch.Tensor:
    if focal_mode != "weiszfeld":
        raise ValueError(f"bad {focal_mode=} (only 'weiszfeld' is implemented on the GPU)")
    b, h, w, three = pts3d.shape
    assert three == 3
    dev = _device_of(pts3d, device)
    ppt = _f32(torch.as_tensor(pp), dev).reshape(-1, 2).expand(b, 2).contiguous()
    return ops.focal_weiszfeld(_f32(pts3d, dev), None, None, ppt, iters=10).to(pts3d.device)


def evaluate_reconstruction(views: List[Dict], preds: List[Dict], min_conf_thr_percentile_for_local_alignment_and_icp=0,
                            min_conf_thr_percentile_for_metric_cacluation=0, use_pts3d_from_local_head=True,
                            device=None) -> List[Dict]:
    """MultiViewDUSt3RLitModule.evaluate_reconstruction (multiview_dust3r_module.py:551-735) on the GPU, without the
    Lightning side: returns one ``{scene_name: {accuracy, accuracy_median, completion, completion_median, nc1,
    nc1_median, nc2, nc2_median}}`` per batch item instead of accumulating them in the module.

    Per item: per-view quantile masks, the similarity of the masked predicted points onto the ground truth over all views
    at once (the boolean-weighted roma.rigid_points_registration is Umeyama over the points of weight 1), Open3D-style
    k=30 normals of both clouds, then accuracy / completion / normal consistency (fast3r_b200.recon_metric).  One
    difference: with fewer than 3 registration points the fit returns the identity (the fallback of similarity_fit);
    roma has no such fallback."""
    from . import recon_metric as rm
    if use_pts3d_from_local_head:
        align_local_pts3d_to_global(preds, views, min_conf_thr_percentile=min_conf_thr_percentile_for_local_alignment_and_icp,
                                    device=device)
    assert min_conf_thr_percentile_for_local_alignment_and_icp >= min_conf_thr_percentile_for_metric_cacluation
    if not views:
        return []
    dev = _device_of(preds[0]["pts3d_in_other_view"], device)
    results = []
    for i in range(len(views[0]["img"])):
        # the reference names the scene after views[i] (the view with the item's index), kept as is
        scene_name = "/".join(views[i]["label"][0].split("/")[:-1]) if "label" in views[i] else "unknown"
        pred_aligned, gt_pts, _ = _registered_clouds(views, preds, i, min_conf_thr_percentile_for_local_alignment_and_icp,
                                                      min_conf_thr_percentile_for_metric_cacluation,
                                                      use_pts3d_from_local_head, dev)
        pred_normals = rm.estimate_normals(pred_aligned)
        gt_normals = rm.estimate_normals(gt_pts)
        acc, acc_med, nc1, nc1_med = rm.accuracy(gt_pts, pred_aligned, gt_normals, pred_normals)
        comp, comp_med, nc2, nc2_med = rm.completion(gt_pts, pred_aligned, gt_normals, pred_normals)
        results.append({scene_name: {
            "accuracy": acc, "accuracy_median": acc_med, "completion": comp, "completion_median": comp_med,
            "nc1": nc1, "nc1_median": nc1_med, "nc2": nc2, "nc2_median": nc2_med,
        }})
    return results


def _registered_clouds(views, preds, i: int, pct_icp: float, pct_metric: float, use_local: bool, dev: torch.device):
    """Batch item i of evaluate_reconstruction up to the metrics (multiview_dust3r_module.py:565-660): the predicted
    points with valid & conf >= quantile(pct_metric) of their view, registered onto the ground truth by the similarity
    fitted over those of them that also pass quantile(pct_icp); and all valid ground-truth points.  Returns
    (pred_aligned fp32 (m, 3), gt fp32 (g, 3), rts fp32 (13,)), points view-major in raster order as the reference
    concatenates them."""
    key_pts, key_conf = ("pts3d_local_aligned_to_global", "conf_local") if use_local else ("pts3d_in_other_view", "conf")
    x = torch.stack([_f32(p[key_pts][i], dev) for p in preds])              # (V, H, W, 3)
    conf = torch.stack([_f32(p[key_conf][i], dev) for p in preds])          # (V, H, W)
    y = torch.stack([_f32(v["pts3d"][i], dev) for v in views])
    valid = torch.stack([v["valid_mask"][i].to(dev, torch.bool) for v in views])
    nv = x.shape[0]
    n = x[0, ..., 0].numel()
    conf_v = conf.reshape(nv, n).contiguous()
    thr_metric = ops.conf_quantile(conf_v, float(pct_metric) / 100.0)
    thr_icp = ops.conf_quantile(conf_v, float(pct_icp) / 100.0)
    mask_pred = valid.reshape(nv, n) & (conf_v >= thr_metric[:, None])
    weights = mask_pred & (conf_v >= thr_icp[:, None])
    xs, ys = x.reshape(1, nv * n, 3).contiguous(), y.reshape(1, nv * n, 3).contiguous()
    rts = ops.similarity_fit(xs, ys, None, None, weights.reshape(1, nv * n).to(torch.uint8).contiguous())
    aligned = ops.similarity_apply(xs, rts)[0]
    return aligned[mask_pred.reshape(-1)].contiguous(), y[valid].contiguous(), rts[0]


def correct_preds_orientation(preds: List[Dict], views: List[Dict]) -> None:
    """MultiViewDUSt3RLitModule.correct_preds_orientation (multiview_dust3r_module.py:871-937), in place: the items whose
    true_shape (H, W) is portrait get their pointmaps and confidences transposed back (the data loader transposed
    them to landscape), and those entries become lists of per-item tensors."""
    if views is None:
        return
    for pred, view in zip(preds, views):
        portrait = [bool(h > w) for h, w in view["true_shape"].tolist()]
        keys = ["conf", "pts3d_in_other_view"]
        if "pts3d_local" in pred:
            keys += ["conf_local", "pts3d_local"] + (["pts3d_local_aligned_to_global"]
                                                     if "pts3d_local_aligned_to_global" in pred else [])
        for key in keys:
            pred[key] = [x.transpose(0, 1) if p else x for x, p in zip(pred[key], portrait)]


def evaluate_camera_poses(views: List[Dict], preds: List[Dict], niter_PnP: int = 10,
                          focal_length_estimation_method: str = "individual", device=None) -> List[Dict]:
    """MultiViewDUSt3RLitModule.evaluate_camera_poses (multiview_dust3r_module.py:737-804) without the Lightning side:
    returns one dict of RRA_at_{5,15,30}, RTA_at_{5,15,30} and mAA_30 (python floats) per batch item instead of
    logging them.

    The first-view-from-local-head alignment, the in-place portrait correction and estimate_camera_poses run as in the
    reference; the estimated poses are cast to the dtype of the ground-truth camera_pose and every pair of every item
    is scored in one launch (fast3r_b200.cam_pose_metric).  Two differences: with fewer than 2 views this raises
    ValueError (the reference logs a warning and then fails on an unbound name), and nothing is printed per item."""
    import numpy as np

    from . import cam_pose_metric as cpm
    from . import lib as L
    if focal_length_estimation_method == "first_view_from_local_head":
        align_local_pts3d_to_global(preds, views, device=device)
    correct_preds_orientation(preds, views)
    poses_c2w, _ = estimate_camera_poses(preds=preds, views=views, niter_PnP=niter_PnP,
                                         focal_length_estimation_method=focal_length_estimation_method)
    gt_list = [view["camera_pose"] for view in views]
    pred_cameras = torch.tensor(np.stack(poses_c2w), dtype=gt_list[0].dtype)   # (B, N, 4, 4)
    gt_cameras = torch.stack(gt_list).transpose(0, 1)                           # (B, N, 4, 4)
    nv = pred_cameras.shape[1]
    if nv < 2:
        raise ValueError("Not enough camera poses to compute relative errors.")
    counts, _, _ = cpm.pose_counts(pred_cameras, gt_cameras, device)
    pairs = nv * (nv - 1) // 2
    results = []
    for row in counts.tolist():
        res = {f"RRA_at_{tau}": cpm.below_ratio(row[k], pairs) for k, tau in enumerate(cpm.RRA_THRESHOLDS)}
        res.update({f"RTA_at_{tau}": cpm.below_ratio(row[3 + k], pairs) for k, tau in enumerate(cpm.RTA_THRESHOLDS)})
        hist = torch.tensor(row[L.PM_HIST:L.PM_HIST + 31], dtype=gt_cameras.dtype)
        res["mAA_30"] = cpm.auc_from_hist(hist, pairs).item()
        results.append(res)
    return results
