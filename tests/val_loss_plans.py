"""Launch keys of the validation-criterion kernels (fast3r_b200/csrc/val_loss.cu) and the table of GPU cases that
tests/test_val_loss_gpu.py runs and tests/test_val_loss_plans_cpu.py checks the callers against.

A call is a dict with the arguments that decide the code path: the local term, the criterion's flags (log1p,
gt_scale, local_scale_consistent), items, views and the pixels n per (view, item).  The pixel kernels run VPX = 4096
pixels per CTA (val_loss.cu:21); one item or one view skips no code but changes which CTA sums a group last."""
VPX = 4096


def _chunks(n):
    if n < VPX:
        return "below-chunk"
    if n == VPX:
        return "one-chunk"
    return "chunks" if n % VPX == 0 else "chunks-tail"


def key(d):
    k = f"{'local' if d['local'] else 'global'} {_chunks(d['n'])}"
    for flag in ("log1p", "gt_scale", "local_scale_consistent"):
        k += f" {flag}" if d[flag] else ""
    return k + (" many-items" if d["items"] > 1 else "") + (" many-views" if d["views"] > 1 else "")


# (name, items, views, H, W, local head, criterion keywords)
CASES_SPEC = [
    ("l_b1_v1_32x64", 1, 1, 32, 64, True, {}),
    ("l_b2_v3_64x64", 2, 3, 64, 64, True, {}),
    ("g_b1_v2_64x96", 1, 2, 64, 96, False, {}),
    ("l_b1_v32_368x512", 1, 32, 368, 512, True, {}),
    ("g_b1_v32_64x128", 1, 32, 64, 128, False, {}),
    ("l_b8_v20_64x128", 8, 20, 64, 128, True, {}),
    ("g_b8_v20_96x128", 8, 20, 96, 128, False, {}),
    ("l_b2_v2_log1p", 2, 2, 64, 96, True, dict(norm_mode="avg_log1p")),
    ("l_b2_v2_gt_scale", 2, 2, 64, 96, True, dict(gt_scale=True)),
    ("l_b2_v2_lsc", 2, 2, 64, 96, True, dict(local_scale_consistent=True)),
    ("g_b3_v5_17x31", 3, 5, 17, 31, False, dict(norm_mode="avg_log1p", gt_scale=True)),
]


def desc(c):
    name, items, views, h, w, local, kw = c
    return dict(name=name, items=items, views=views, H=h, W=w, local=local, kw=kw, n=h * w,
                log1p=kw.get("norm_mode") == "avg_log1p", gt_scale=kw.get("gt_scale", False),
                local_scale_consistent=kw.get("local_scale_consistent", False))


CASES = [dict(key=key(desc(c)), **desc(c)) for c in CASES_SPEC]
