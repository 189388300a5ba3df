"""Making the reference code base use this model unchanged.

`MultiViewDUSt3RLitModule.forward(views)` is literally ``self.net(views)`` and `load_for_inference(net)` only stores
`net` (fast3r/models/multiview_dust3r_module.py:119-126), so an instance of ``fast3r_b200.Fast3R`` can be handed to it
directly.  The one place that looks at the class is ``isinstance(self.net, Fast3R)`` when pretrained weights are loaded
(multiview_dust3r_module.py:1005): `install()` rebinds the name ``fast3r.models.fast3r.Fast3R`` (and the copy already
imported into the Lightning module, if any) to this package's class, so that check - and Hydra configs whose ``_target_`` is
``fast3r.models.fast3r.Fast3R`` - resolve to this implementation.  Call it once, before building the Lightning module."""
import importlib
import sys


def install() -> type:
    from .model import Fast3R
    ref = importlib.import_module("fast3r.models.fast3r")  # the reference package must be importable
    if getattr(ref.Fast3R, "__module__", "") != Fast3R.__module__:
        ref.ReferenceFast3R = ref.Fast3R  # keep the original reachable
        ref.Fast3R = Fast3R
    lit = sys.modules.get("fast3r.models.multiview_dust3r_module")
    if lit is not None:
        lit.Fast3R = Fast3R
    return Fast3R


def uninstall() -> None:
    ref = sys.modules.get("fast3r.models.fast3r")
    if ref is not None and hasattr(ref, "ReferenceFast3R"):
        ref.Fast3R = ref.ReferenceFast3R
        del ref.ReferenceFast3R
        lit = sys.modules.get("fast3r.models.multiview_dust3r_module")
        if lit is not None:
            lit.Fast3R = ref.Fast3R
