"""The validation criterion on the GPU.  Every case of tests/val_loss_plans.CASES runs f3r_val_loss with canaries around
its output and its workspace and equals the host build of the same math (tests/val_loss_emulator.py): counts exactly,
sums within 1e-6 of the sum of their terms' magnitudes (the float64 sums run in another order and logf / log1pf come
from another library).  fast3r_b200.losses equals the reference's goldens (tests/golden/val_loss.pt) from host and device
inputs, gives the same bits on a second run, and works as the criterion of loss_of_one_batch with the real model."""
import os

import pytest
import torch

from fast3r_b200 import lib as L
from fast3r_b200 import ops
from tests import canaries as CN
from tests import val_loss_cases as VC
from tests import val_loss_emulator as E
from tests import val_loss_plans as VP
from tests.test_val_loss_cpu import check_golden, criterion

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", VP.CASES, ids=[c["name"] for c in VP.CASES])
def test_plan_case_equals_emulator(case):
    from fast3r_b200 import losses as LS
    views, preds = VC.make(case["items"], case["views"], case["H"], case["W"], case["local"],
                           seed=len(case["name"]))
    m = LS.stack_maps(views, preds, torch.device("cuda"))
    flags = dict(alpha=VC.ALPHA, log1p=case["log1p"], gt_scale=case["gt_scale"],
                 local_scale_consistent=case["local_scale_consistent"])
    want, mags = E.run(**m, **flags)
    nv, items, n = m["valid"].shape
    nbytes = L.load().f3r_val_loss_workspace(nv, items, n)
    wb, ws = CN.buffer(((nbytes + 7) // 8,), torch.float64)
    ob, out = CN.buffer((nv, items, ops.VL_SUMS), torch.float64)
    obefore, wbefore = ob.clone(), wb.clone()
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    ops._call("f3r_val_loss", out, ptr(m["gt"]), ptr(m["valid"]), ptr(m["pr"]), ptr(m.get("pr_local")),
              ptr(m["conf"]), ptr(m.get("conf_local")), ptr(m["poses"]), nv, items, n, VC.ALPHA, int(case["log1p"]),
              int(case["gt_scale"]), int(case["local_scale_consistent"]), int(case["local"]), out.data_ptr(),
              ws.data_ptr(), nbytes)
    torch.cuda.synchronize()
    got = out.cpu()
    assert torch.equal(got[..., 4], want[..., 4])
    assert torch.equal(got.isnan(), want.isnan())
    err = (got[..., :4] - want[..., :4]).abs()
    assert bool((want[..., :4].isnan() | (err <= 1e-6 * mags)).all()), float((err / mags).nan_to_num(0).max())
    for name, buf, before, cnt in (("out", ob, obefore, out.numel()), ("workspace", wb, wbefore, ws.numel())):
        written = torch.zeros(buf.numel(), dtype=torch.bool, device="cuda")
        written[CN.PAD:CN.PAD + cnt] = True
        CN.untouched(name, buf, before, written)


@pytest.mark.parametrize("on_device", [False, True])
@pytest.mark.parametrize("name", list(VC.CASES))
def test_losses_equal_golden(name, on_device):
    views, preds = VC.inputs(name)
    if on_device:
        views = [{k: v.cuda() for k, v in view.items()} for view in views]
        preds = [{k: v.cuda() for k, v in p.items()} for p in preds]
    loss, details = criterion(name)(views, preds)
    check_golden(name, loss, details, device="cuda" if on_device else "cpu")


@pytest.mark.parametrize("name", ["b2_n8_368x512", "b2_n3_heights", "b2_n3_nan"])
def test_two_runs_give_the_same_bits(name):
    from fast3r_b200 import losses as LS
    views, preds = VC.inputs(name)
    preds = [{k: v.cuda() for k, v in p.items()} for p in preds]
    kw = VC.criterion_kw(name)
    args = (views, preds, VC.ALPHA, kw.get("norm_mode") == "avg_log1p", kw.get("gt_scale", False),
            kw.get("local_scale_consistent", False))
    a, b = LS.view_sums(*args), LS.view_sums(*args)
    assert torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())


def test_criterion_of_loss_of_one_batch(golden_dir):
    """loss_of_one_batch(batch, model, criterion) with the tiny model: the loss and details equal the criterion applied
    to the preds it returns."""
    from fast3r_b200 import Fast3R, loss_of_one_batch, tiny_args
    from tests.golden.synth import synth_images, synth_state_dict
    g = torch.load(os.path.join(golden_dir, "tiny_b1_n3.pt"))
    enc, dec, head = tiny_args()
    dec.update(g.get("dec_over", {}))
    head.update(g.get("head_over", {}))
    model = Fast3R(enc, dec, head).eval()
    model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
    model = model.cuda()
    imgs = synth_images(g["N"], g["B"], g["H"], g["W"])
    gts, _ = VC.make(g["B"], g["N"], g["H"], g["W"], local=False, seed=11)
    batch = [dict(img=im, true_shape=torch.tensor([[g["H"], g["W"]]] * g["B"]), idx=i, instance=str(i), **gt)
             for i, (im, gt) in enumerate(zip(imgs, gts))]
    crit = criterion("b2_n2_64x96")
    with torch.no_grad():
        res = loss_of_one_batch(batch, model, crit, "cuda", "32")
    loss, details = res["loss"]
    assert loss.is_cuda and loss.dtype == torch.float32 and torch.isfinite(loss)
    assert len(details) == (4 if "pts3d_local" in res["preds"][0] else 2) * g["N"]
    again, details2 = crit(res["views"], res["preds"])
    assert torch.equal(loss, again) and details2 == details
