"""Per-slice comparison of one forward output against its float64 reference (TEST INFRASTRUCTURE ONLY: used by
tests/ and tools/sp_check.py, never by the product).

A relative L2 over all views concatenated averages a localized error away: at N=32 and 368x512, one view 7 % off or one
pixel row entirely wrong still passes the bf16 tolerance 1.3e-2, and one view 0.5 % off passes the parity tolerance 1e-3.
Wrong chunk offsets, a wrong view <-> image-id pairing, a race in a chunk's copy or an off-by-one at a group boundary
produce exactly such errors.  ``check`` therefore measures the error of many small slices of each view separately.

Error measure.  ``d = ours - ref``.  For a slice S of view v:

    e(S) = RMS(d over S) / s_v,   s_v = RMS(ref over all of view v)       (pts3d*)
                                  s_v = RMS(ref - 1 over all of view v)   (conf*)

The normaliser is the whole view's, not the slice's: a slice where the field happens to be small is not judged more
strictly than the view as a whole, and one where it is large not more loosely.  ``conf = 1 + exp(c)``: against
``ref - 1`` the constant 1 no longer dilutes the error of the exp term.  e(view v) is the per-view relative L2, and the
relative L2 over all views concatenated is the s_v-weighted RMS of those.  A slice spanning all views (a phase class, a
channel) is measured on ``d / s_v`` of each view.

Slice kinds (H and W are multiples of the 16-pixel patch):
  * ``view``   each view;
  * ``row``    each pixel row of each view, ``col`` each pixel column of each view;
  * ``patch``  each 16x16 block of each view, one token's footprint (a wrong token, a wrong block of a GEMM tile);
  * ``phase``  each pixel phase class (y mod 16, x mod 16) over all views (tile and upsample-phase faults: the heads
    upsample by 4, 2, 2, 2, 2 from the patch grid, so a phase fault repeats every 16 pixels);
  * ``channel`` each output channel over all views (x, y, z of a pointmap; conf has one).

Rules:
  (1) Absolute bound: e(S) <= T for every slice.  T is the tolerance the suite already applies to the concatenated
      relative L2 of the same precision: 1e-3 for the parity path ("fp32", the north-star tolerance), 3e-3 for
      "fp16" (the fp16 golden tolerance), 1.3e-2 for "bf16".  The concatenated figure is an s_v-weighted RMS of the
      per-view e(view), so a run whose error is spread evenly over its slices has e(S) close to that figure
      everywhere, and the rule costs a healthy run only the spread of e(S) around it, which rule (2) bounds.
  (2) No outliers: e(S) <= R * median(e over all slices of the same kind of the same output), R = 4.  A healthy
      run's error is rounding noise spread over the whole forward; every slice of one kind holds the same number of
      elements, drawn from the same process, so their e(S) scatter only by the sampling noise of an RMS over n
      elements (relative spread ~ 1/sqrt(2n); n >= 256 for every kind at the sizes tested, so a few per cent) and by
      how unevenly the field's sensitivity is spread over the image.  A fault confined to one slice (a view, a row, a
      token, a phase) raises that slice alone, by a factor that does not shrink with the number of slices.  R = 4
      leaves room for smooth variation of the sensitivity across an image while any slice several times worse than
      its peers fails.
      Border group.  Rows and columns within one patch (16 pixels) of the image edge, and the patches of the outer
      ring, form a group of their own with its own median.  Their error is systematically larger: the 3x3
      convolutions of the heads see zero padding there and the align_corners upsamples pin their edge samples, so
      the field and its rounding error differ in kind from the interior.  Measured on an H100 against the float64
      oracle: in every tiny-model case of the parity path the worst conf row was row 1, and in ViT-L at N=32 the
      parity path's conf_local columns 6 to 10 were 4.2-4.4x the median of all columns, across many views.  Mixed
      with the interior they raise R*median's bar for nobody and fail only by being border slices; in their own group
      they are held to R like every other slice.

On failure the worst slices are listed with kind, view, index, value and the bound they broke.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch

PATCH = 16
T = {"fp32": 1e-3, "fp16": 3e-3, "bf16": 1.3e-2}
R = 4.0
KINDS = ("view", "row", "col", "patch", "phase", "channel")


def _as_vhwc(t: torch.Tensor) -> torch.Tensor:
    t = t.detach().to(device="cpu", dtype=torch.float64)
    return t[..., None] if t.dim() == 3 else t


def slice_errors(ours: torch.Tensor, ref: torch.Tensor, name: str) -> Dict[str, torch.Tensor]:
    """e(S) of every slice, per kind: view (V,), row (V, H), col (V, W), patch (V, H/16, W/16), phase (16, 16),
    channel (C,).  ``ours`` / ``ref``: (V, H, W, 3) pointmaps or (V, H, W) confidences; ``name`` starting with "conf"
    selects the conf normaliser."""
    a, b = _as_vhwc(ours), _as_vhwc(ref)
    if a.shape != b.shape:
        raise ValueError(f"{name}: shape {tuple(a.shape)} != reference {tuple(b.shape)}")
    V, H, W, C = b.shape
    if H % PATCH or W % PATCH:
        raise ValueError(f"{name}: {H}x{W} is not a multiple of the {PATCH}-pixel patch")
    base = b - 1.0 if name.startswith("conf") else b
    s = base.square().mean(dim=(1, 2, 3)).sqrt()  # (V,)
    if not bool((s > 0).all()):
        raise ValueError(f"{name}: a reference view is identically zero")
    e2 = ((a - b) / s[:, None, None, None]).square()  # normalised squared error, (V, H, W, C)
    blocks = e2.reshape(V, H // PATCH, PATCH, W // PATCH, PATCH, C)
    return dict(
        view=e2.mean(dim=(1, 2, 3)).sqrt(),
        row=e2.mean(dim=(2, 3)).sqrt(),
        col=e2.mean(dim=(1, 3)).sqrt(),
        patch=blocks.mean(dim=(2, 4, 5)).sqrt(),
        phase=blocks.mean(dim=(0, 1, 3, 5)).sqrt(),
        channel=e2.mean(dim=(0, 1, 2)).sqrt(),
    )


def _label(kind: str, idx: Tuple[int, ...]) -> str:
    if kind in ("view", "channel"):
        return f"{kind} {idx[0]}"
    if kind == "phase":
        return f"phase (y%16={idx[0]}, x%16={idx[1]})"
    if kind == "patch":
        return f"view {idx[0]} patch ({idx[1]}, {idx[2]})"
    return f"view {idx[0]} {kind} {idx[1]}"


def summary(errs: Dict[str, torch.Tensor], precision: str) -> Dict[str, dict]:
    """Per kind: the worst slice, its value as a fraction of T (rule 1) and the worst ratio to the median (rule 2)."""
    out = {}
    for kind, e in errs.items():
        flat = e.flatten()
        k = int(flat.argmax())
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(k), e.shape))
        ratio = (e / medians(kind, e)).flatten()
        j = int(ratio.argmax())
        jdx = tuple(int(i) for i in torch.unravel_index(torch.tensor(j), e.shape))
        out[kind] = dict(worst=_label(kind, idx), value=float(flat[k]), of_T=float(flat[k]) / T[precision],
                         of_median=float(ratio[j]), worst_ratio=_label(kind, jdx))
    return out


def border(kind: str, e: torch.Tensor) -> torch.Tensor:
    """Mask of the slices of the border group: rows / columns within one patch of the edge, patches of the outer ring
    (no slice of the other kinds)."""
    m = torch.zeros(e.shape, dtype=torch.bool)
    if kind in ("row", "col"):
        m[:, :PATCH] = m[:, -PATCH:] = True
    elif kind == "patch":
        m[:, 0] = m[:, -1] = m[:, :, 0] = m[:, :, -1] = True
    return m


def medians(kind: str, e: torch.Tensor) -> torch.Tensor:
    """Per slice, the median of its group (border or interior) for rule 2."""
    m = border(kind, e)
    med = torch.full(e.shape, float(e[~m].median()), dtype=e.dtype)
    if bool(m.any()):
        med[m] = float(e[m].median())
    return med


def violations(errs: Dict[str, torch.Tensor], precision: str) -> List[Tuple[float, str]]:
    """(excess over the bound, description) of every slice that breaks rule 1 or rule 2."""
    bad = []
    for kind, e in errs.items():
        med = medians(kind, e)
        for idx in (e > T[precision]).nonzero().tolist():
            v = float(e[tuple(idx)])
            bad.append((v / T[precision], f"{_label(kind, tuple(idx))}: {v:.3e} > T = {T[precision]:.3e}"))
        for idx in (e > R * med).nonzero().tolist():
            v, m = float(e[tuple(idx)]), float(med[tuple(idx)])
            bad.append((v / (R * m) if m > 0 else float("inf"),
                        f"{_label(kind, tuple(idx))}: {v:.3e} > R*median ({R:g} x {m:.3g}) = {R * m:.3e}"))
    return sorted(bad, reverse=True)


def check(ours: torch.Tensor, ref: torch.Tensor, precision: str, name: str, show: int = 12) -> Dict[str, dict]:
    """Asserts rules (1) and (2) for one output; returns its ``summary``.  ``precision``: "bf16", "fp16" or "fp32"."""
    errs = slice_errors(ours, ref, name)
    if not all(bool(torch.isfinite(e).all()) for e in errs.values()):
        raise AssertionError(f"{name} [{precision}]: non-finite error (NaN or inf in the output)")
    bad = violations(errs, precision)
    if bad:
        lines = "\n  ".join(d for _, d in bad[:show])
        raise AssertionError(f"{name} [{precision}]: {len(bad)} slice(s) out of bounds; worst first:\n  {lines}")
    return summary(errs, precision)


def check_all(pairs: Dict[str, Tuple[torch.Tensor, torch.Tensor]], precision: str, tag: str) -> Dict[str, dict]:
    """``check`` of every output in ``pairs`` (name -> (ours, ref)); every output is checked before the first failure is
    raised, and the summary of each is printed."""
    report, failures = {}, []
    for name, (ours, ref) in pairs.items():
        errs = slice_errors(ours, ref, name)
        report[name] = summary(errs, precision)
        worst = max(report[name].values(), key=lambda r: r["of_T"])
        ratio = max(report[name].values(), key=lambda r: r["of_median"])
        print(f"{tag} [{precision}] {name}: worst {worst['worst']} = {worst['of_T']:.3f} T; "
              f"worst ratio to its group's median {ratio['of_median']:.2f} ({ratio['worst_ratio']})")
        try:
            check(ours, ref, precision, name)
        except AssertionError as exc:
            failures.append(f"{tag}: {exc}")
    if failures:
        raise AssertionError("\n".join(failures))
    return report


def by_shape(preds_flat, refs_flat):
    """{(H, W): (ours, ref)} per output key and shape: the views of each shape stacked to (V*B, H, W[, 3]) in view order.
    ``preds_flat`` / ``refs_flat``: per-view prediction dicts of the whole case (scenes concatenated)."""
    out = {}
    for k in refs_flat[0]:
        groups = {}
        for p, q in zip(preds_flat, refs_flat):
            groups.setdefault(tuple(q[k].shape[1:3]), []).append((p[k], q[k]))
        for hw, pairs in groups.items():
            name = k if len(groups) == 1 else f"{k}@{hw[0]}x{hw[1]}"
            out[name] = (torch.cat([a.detach().cpu() for a, _ in pairs]), torch.cat([b.detach().cpu() for _, b in pairs]))
    return out
