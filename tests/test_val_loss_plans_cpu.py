"""Every launch key of the validation-criterion kernels that fast3r_b200.losses reaches at the reference's sizes
(32 and 320 views of 368x512, and 8 items of 20 views of 384x512, with and without the local head) has a case in
tests/val_loss_plans.CASES, which tests/test_val_loss_gpu.py runs; and each case reaches its key.  The criterion runs on
the CPU with its maps stacked on the meta device (no memory) and the entry point replaced by a recorder."""
import pytest
import torch

from tests import val_loss_plans as VP


def _inputs(items, views, h, w, local):
    z3 = torch.zeros(1, 1, 1, 3).expand(items, h, w, 3)
    z1 = torch.ones(1, 1, 1).expand(items, h, w)
    gts = [dict(pts3d=z3, valid_mask=z1.bool(), camera_pose=torch.eye(4).expand(items, 4, 4)) for _ in range(views)]
    preds = [dict(pts3d_in_other_view=z3, conf=z1, **(dict(pts3d_local=z3, conf_local=z1) if local else {}))
             for _ in range(views)]
    return gts, preds


def recorded_keys(monkeypatch):
    import fast3r_b200.losses as LS
    import fast3r_b200.ops as O
    calls = []

    def val_loss(gt, valid, pr, conf, poses, pr_local=None, conf_local=None, alpha=1.0, log1p=False, gt_scale=False,
                 local_scale_consistent=False):
        views, items, n = valid.shape
        calls.append(dict(local=pr_local is not None, log1p=log1p, gt_scale=gt_scale,
                          local_scale_consistent=local_scale_consistent, items=items, views=views, n=n))
        return torch.zeros(views, items, O.VL_SUMS, dtype=torch.float64)

    monkeypatch.setattr(LS, "_device", lambda t: torch.device("meta"))
    monkeypatch.setattr(O, "val_loss", val_loss)
    crit = LS.ConfLossMultiviewV2(LS.Regr3DMultiviewV4(LS.L21Loss(), norm_mode="avg_dis"), alpha=0.2)
    for items, views, h, w in ((1, 32, 368, 512), (1, 320, 368, 512), (8, 20, 384, 512)):
        for local in (True, False):
            crit(*_inputs(items, views, h, w, local))
    return {VP.key(d) for d in calls}


def test_every_caller_key_has_a_gpu_case(monkeypatch):
    keys = recorded_keys(monkeypatch)
    assert len(keys) == 4
    missing = keys - {c["key"] for c in VP.CASES}
    assert not missing, f"launch keys of the criterion without a case in tests/val_loss_plans.CASES: {missing}"


def test_table_keys_are_what_the_cases_reach():
    names = [c["name"] for c in VP.CASES]
    assert len(names) == len(set(names))
    assert all(VP.key(c) == c["key"] for c in VP.CASES)


@pytest.mark.parametrize("flag", ["local", "global", "below-chunk", "one-chunk", "chunks ", "chunks-tail", "log1p",
                                  "gt_scale", "local_scale_consistent", "many-items", "many-views"])
def test_table_reaches_every_flag(flag):
    assert any(flag in c["key"] + " " for c in VP.CASES)
