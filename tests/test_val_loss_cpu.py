"""The validation criterion without a GPU: the host build of csrc/val_loss_math.h against an fp64 torch restatement of
the reference's formula, fast3r_b200.losses on the CPU emulator of its entry point (tests/val_loss_emulator.py) against
the reference's goldens (tests/golden/val_loss.pt: keys, key order, value types and values), and the module's
constructors, names and refusals."""
import math
import os

import pytest
import torch

from tests import val_loss_cases as VC
from tests import val_loss_emulator as E
from tests import val_loss_torch as VT
from tests.conftest import ROOT

BOUND = 1e-6  # of the mean magnitude of a value's per-pixel terms (about 10x the reference's own float32 error)


def golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "val_loss.pt"))


def criterion(name):
    from fast3r_b200 import losses as LS
    kw = {"norm_mode": "avg_dis", **VC.criterion_kw(name)}
    return LS.ConfLossMultiviewV2(LS.Regr3DMultiviewV4(LS.L21Loss(), **kw), alpha=VC.ALPHA)


def _close(got, want, scale):
    if math.isnan(want):
        return math.isnan(got)
    return got == want or abs(got - want) <= BOUND * scale


def check_golden(name, loss, details, device="cpu"):
    """(loss, details) of fast3r_b200.losses equal the reference's for golden case `name`: the same keys in the same
    order, the int 0 where the reference has it, NaN where it has NaN, values within BOUND of the mean magnitude of
    their per-pixel terms (from the fp64 restatement)."""
    want = golden()["cases"][name]
    assert list(details) == list(want["details"])
    views, preds = VC.inputs(name)
    _, mags = VT.view_sums(views, preds, VC.ALPHA, **VC.criterion_kw(name))
    counts = torch.stack([v["valid_mask"].sum() for v in views]).double()
    mean_mag = mags / counts[:, None]  # NaN for a view without valid pixels
    nv = len(views)
    terms = ["global", "local"] if "pts3d_local" in preds[0] else ["global"]
    conf_scale = 0.0
    for k, w in want["details"].items():
        g = details[k]
        assert type(g) is type(w), (k, g, w)
        t = terms.index("local" if "_local/" in k else "global")
        i = int(k[-2:])
        j = 2 * t + (1 if k.startswith("ConfLoss") else 0)
        if k.startswith("ConfLoss") and w != 0:
            conf_scale += float(mean_mag[i, j])
        assert _close(g, w, float(mean_mag[i, j])), (k, g, w, float(mean_mag[i, j]))
    if want["loss_type"] == "float":
        assert type(loss) is float and loss == want["loss"]
    else:
        assert torch.is_tensor(loss) and loss.dim() == 0 and loss.dtype == torch.float32
        assert loss.device.type == torch.device(device).type
        assert _close(float(loss), want["loss"], conf_scale / (nv * len(terms))), (float(loss), want["loss"])


@pytest.fixture
def emulated(monkeypatch):
    import fast3r_b200.losses as LS
    import fast3r_b200.ops as O
    monkeypatch.setattr(LS, "_device", lambda t: torch.device("cpu"))
    monkeypatch.setattr(O, "val_loss", E.val_loss)


def test_inverse_is_fp64_rounded():
    g = torch.Generator().manual_seed(3)
    m = torch.randn(500, 4, 4, generator=g, dtype=torch.float64).float()
    m[:, 3] = torch.tensor([0.0, 0.0, 0.0, 1.0])
    m[:250, 3, :3] = torch.randn(250, 3, generator=g).float()  # general (projective) matrices too
    want = torch.linalg.inv(m.double())
    got = E.inverse(m).double()
    ulp = want.float().abs().double() * 2.0 ** -23
    assert bool(((got - want).abs() <= 0.5 * ulp + 1e-30).all())


@pytest.mark.parametrize("name", [n for n in VC.CASES if "368x512" not in n])
def test_host_math_equals_fp64_restatement(emulated, name):
    """Per view: the host build's sums equal the fp64 restatement's within BOUND of their absolute sums, the counts
    exactly, NaN where it has NaN."""
    from fast3r_b200 import losses as LS
    views, preds = VC.inputs(name)
    kw = VC.criterion_kw(name)
    got = LS.view_sums(views, preds, VC.ALPHA, kw.get("norm_mode") == "avg_log1p", kw.get("gt_scale", False),
                       kw.get("local_scale_consistent", False))
    want, mags = VT.view_sums(views, preds, VC.ALPHA, **kw)
    assert torch.equal(got[:, 4], want[:, 4])
    w = want[:, :4] if "pts3d_local" in preds[0] else want[:, :2]
    g = got[:, :w.shape[1]]
    assert torch.equal(g.isnan(), w.isnan())
    ok = g.isnan() | ((g - w).abs() <= BOUND * mags[:, :w.shape[1]])
    assert bool(ok.all()), (g, w)
    if "pts3d_local" not in preds[0]:
        assert bool((got[:, 2:4] == 0).all())


@pytest.mark.parametrize("name", list(VC.CASES))
def test_losses_equal_golden_on_the_emulator(emulated, name):
    views, preds = VC.inputs(name)
    crit = criterion(name)
    assert repr(crit) == golden()["cases"][name]["name"]
    loss, details = crit(views, preds)
    check_golden(name, loss, details)


def test_names_and_repr():
    from fast3r_b200 import losses as LS
    crit = LS.ConfLossMultiviewV2(LS.Regr3DMultiviewV4(LS.L21Loss(), norm_mode="avg_dis"), alpha=0.2)
    assert repr(crit) == crit.get_name() == "ConfLossMultiviewV2(Regr3DMultiviewV4(L21Loss()))"
    assert crit.alpha == 0.2 and crit.pixel_loss.criterion.reduction == "none"
    assert crit.pixel_loss.get_name() == "Regr3DMultiviewV4(L21Loss())"


@pytest.mark.parametrize("mode", ["median_dis", "avg_warp-log1p", "median_log1p", None, ""])
def test_unsupported_norm_modes_raise(mode):
    from fast3r_b200 import losses as LS
    with pytest.raises(NotImplementedError, match=repr(mode)):
        LS.Regr3DMultiviewV4(LS.L21Loss(), norm_mode=mode)


def test_refusals(emulated):
    from fast3r_b200 import losses as LS
    crit = criterion("b2_n2_64x96")
    views, preds = VC.inputs("b2_n2_64x96")
    with pytest.raises(NotImplementedError, match="dist_clip"):
        crit(views, preds, dist_clip=10.0)
    with pytest.raises(NotImplementedError):
        crit * 2
    with pytest.raises(NotImplementedError):
        crit + crit
    with pytest.raises(NotImplementedError, match="pixel_loss"):
        LS.Regr3DMultiviewV4(LS.L21Loss())(views, preds)
    with pytest.raises(ValueError):
        LS.ConfLossMultiviewV2(LS.Regr3DMultiviewV4(LS.L21Loss()), alpha=0)
    preds[1]["conf"].requires_grad_(True)
    with pytest.raises(RuntimeError, match="grad"):
        crit(views, preds)


def test_widths_must_match(emulated):
    views, preds = VC.inputs("b2_n2_64x96")
    views[1]["pts3d"] = views[1]["pts3d"][:, :, :90]
    with pytest.raises(ValueError, match="width"):
        criterion("b2_n2_64x96")(views, preds)
