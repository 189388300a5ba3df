"""The reference's validation criterion (fast3r/dust3r/losses.py:570-848, ConfLossMultiviewV2 over Regr3DMultiviewV4
with L21Loss) restated in torch at a chosen precision, TEST INFRASTRUCTURE ONLY: per view, over the valid pixels of all
items, the sums f3r_val_loss forms (sum d and sum d c - alpha log c of the global and the local term, the count) and the
sums of their absolute values, which scale the tests' bounds."""
import torch


def _apply(T, x):
    return torch.einsum("bij,bhwj->bhwi", T[:, :3, :3], x) + T[:, None, None, :3, 3]


def view_sums(views, preds, alpha, norm_mode="avg_dis", gt_scale=False, local_scale_consistent=False,
              dtype=torch.float64):
    """(sums [views, 5], absolute sums [views, 4]) in `dtype`."""
    log1p = norm_mode == "avg_log1p"
    B = views[0]["pts3d"].shape[0]
    has_local = "pts3d_local" in preds[0]
    valid = [v["valid_mask"].bool() for v in views]

    def dis(p, m):
        d = p.norm(dim=-1)
        d = torch.log1p(d) if log1p else d
        return d.masked_fill(~m, float("nan")).reshape(B, -1)

    def factor(pts, masks):  # nanmean over the given maps of each item, clip(min=1e-8); NaN stays
        d = torch.cat([dis(p, m) for p, m in zip(pts, masks)], 1)
        return d.nanmean(1).clamp(min=1e-8)[:, None, None, None]

    poses = [v["camera_pose"].to(dtype) for v in views]
    gts = [v["pts3d"].to(dtype) for v in views]
    inv0 = torch.linalg.inv(poses[0])
    terms = [([_apply(inv0, g) for g in gts], [p["pts3d_in_other_view"].to(dtype) for p in preds],
              [p["conf"].to(dtype) for p in preds])]
    fg = [factor(terms[0][1], valid)] * len(views)
    ft = [torch.ones_like(fg[0]) if gt_scale else factor(terms[0][0], valid)] * len(views)
    scales = [(fg, ft)]
    if has_local:
        gl = [_apply(torch.linalg.inv(P), g) for P, g in zip(poses, gts)]
        pl = [p["pts3d_local"].to(dtype) for p in preds]
        terms.append((gl, pl, [p["conf_local"].to(dtype) for p in preds]))
        if local_scale_consistent:
            scales.append((fg, ft))
        else:
            scales.append(([factor([p], [m]) for p, m in zip(pl, valid)],
                           [torch.ones_like(fg[0]) if gt_scale else factor([g], [m]) for g, m in zip(gl, valid)]))
    sums = torch.zeros(len(views), 5, dtype=dtype)
    mags = torch.zeros(len(views), 4, dtype=dtype)
    for t, ((g, p, c), (fp, fgt)) in enumerate(zip(terms, scales)):
        for i, m in enumerate(valid):
            d = (p[i] / fp[i] - g[i] / fgt[i]).norm(dim=-1)[m]
            ci = c[i][m]
            cl = d * ci - alpha * torch.log(ci)
            sums[i, 2 * t], sums[i, 2 * t + 1] = d.sum(), cl.sum()
            mags[i, 2 * t], mags[i, 2 * t + 1] = d.abs().sum(), cl.abs().sum()
            sums[i, 4] = m.sum()
    return sums, mags
