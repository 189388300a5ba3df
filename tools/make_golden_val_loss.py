"""Generates tests/golden/val_loss.pt by running the REFERENCE's unmodified validation criterion,
ConfLossMultiviewV2(Regr3DMultiviewV4(L21Loss(), norm_mode, gt_scale, local_scale_consistent), alpha=0.2) of
fast3r/dust3r/losses.py, on tests/val_loss_cases.inputs(name) for every case of tests/val_loss_cases.CASES, on the CPU.

Stored per case: the loss (a float) and its type ("tensor" for the 0-dim float32 tensor, "float" for the python float
the reference returns when every conf term is the int 0), and the details dict as returned (key order and value types
kept).  Only outputs are stored; the tests regenerate the inputs from the seeds.
Run: python tools/make_golden_val_loss.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402
from tests import val_loss_cases as VC  # noqa: E402


def reference_losses():
    # fast3r/dust3r/losses.py imports `dust3r.*`, which resolves inside the reference's fast3r directory
    for p in (ref_harness.REFERENCE_ROOT, os.path.join(ref_harness.REFERENCE_ROOT, "fast3r")):
        if p not in sys.path:
            sys.path.insert(0, p)
    from fast3r.dust3r import losses
    return losses


def main():
    R = reference_losses()
    out = {"what": "reference outputs, see tools/make_golden_val_loss.py", "alpha": VC.ALPHA, "cases": {}}
    for name in VC.CASES:
        views, preds = VC.inputs(name)
        crit = R.ConfLossMultiviewV2(R.Regr3DMultiviewV4(R.L21Loss(), **{"norm_mode": "avg_dis",
                                                                          **VC.criterion_kw(name)}), alpha=VC.ALPHA)
        loss, details = crit(views, preds)
        out["cases"][name] = dict(loss=float(loss), loss_type="tensor" if torch.is_tensor(loss) else type(loss).__name__,
                                  details=details, name=repr(crit))
        print(name, out["cases"][name]["loss_type"], float(loss))
    path = os.path.join(ROOT, "tests", "golden", "val_loss.pt")
    torch.save(out, path)
    print("wrote", path)


if __name__ == "__main__":
    main()
