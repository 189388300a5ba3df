"""Output buffers with canaries and the per-element bound check, shared by the per-element kernel tests
(tests/test_gemm_plans_gpu.py, tests/test_attention_plans_gpu.py)."""
import math

import torch

PAD = 64  # canary elements before and after every output (keeps 16-byte alignment)
SENTINEL = -1234.5


def buffer(shape, dtype, fill=None):
    """(full flat buffer, contiguous view of `shape` in its middle); the canaries hold SENTINEL."""
    n = math.prod(shape)
    buf = torch.full((n + 2 * PAD,), SENTINEL, dtype=dtype, device="cuda")
    view = buf[PAD:PAD + n].view(shape)
    if fill is not None:
        view.copy_(fill)
    return buf, view


def check_elements(name, out, ref, bound):
    """|out - ref| <= bound element by element (NaN counts as outside)."""
    out = out.double()
    err = (out - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        idx = bad.nonzero()[:5].tolist()
        worst = float((err / bound.clamp_min(1e-300)).nan_to_num(float("inf")).max())
        raise AssertionError(f"{name}: {int(bad.sum())} of {out.numel()} elements outside the bound (worst {worst:.3g}x "
                             f"the bound); first at {idx}: out {[float(out[tuple(i)]) for i in idx]} "
                             f"ref {[float(ref[tuple(i)]) for i in idx]}")


def untouched(name, buf, before, written):
    """Elements of buf outside `written` (a bool mask of buf's shape) still hold their old bits."""
    keep = ~written
    a, b = buf[keep], before[keep]
    same = (a == b) | (a.isnan() & b.isnan())
    assert bool(same.all()), f"{name}: {int((~same).sum())} elements outside the written region changed"


def region(buf_len, rows, ld, cols, offset=PAD):
    """Mask of a buffer from `buffer`: the first `cols` columns of `rows` rows of stride `ld` after the leading canary."""
    m = torch.zeros(buf_len, dtype=torch.bool, device="cuda")
    m[offset:offset + rows * ld].view(rows, ld)[:, :cols] = True
    return m
