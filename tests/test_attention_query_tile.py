"""Query tiles of the bf16 attention kernel (192 rows = three consumer warpgroups of 64 rows): the host's unit count
agrees with the kernel's tile height, and on the GPU the partial-tile layouts that no other case reaches are exact."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_attention_units_match_kernel_tile():
    """ops.ATT_Q_TILE (used to count work units for the key-slice choice) is the kernel's ATT_Q_TILE."""
    from fast3r_b200 import ops
    with open(os.path.join(ROOT, "fast3r_b200", "csrc", "f3r_kernels.h")) as f:
        m = re.search(r"constexpr int ATT_Q_TILE = (\d+);", f.read())
    assert m is not None and int(m.group(1)) == ops.ATT_Q_TILE
    assert ops.attention_units(1, 16, 736 * 32) == 16 * 123   # N=32 fusion decoder: 23 552 tokens
    assert ops.attention_units(2, 3, 192) == 6
    assert ops.attention_units(2, 3, 193) == 12


def _gpu_cases():
    from tests import kernel_checks as KC
    cases = [
        # the last tile holds one row, in its first warpgroup; the other two run the key loop with no rows to store
        ("attn_sq193_ranges", KC.check_attention_ranges, dict(heads=2, sq=193, chunk=200, world=2, rank=1)),
        # the last tile holds one row, in its third warpgroup (rows 320 = 192 + 128)
        ("attn_sq321", KC.check_attention, dict(batch=2, heads=2, sq=321, skv=300, scale=0.16019)),
        # whole tiles only
        ("attn_sq384", KC.check_attention, dict(batch=1, heads=2, sq=384, skv=384)),
    ]
    return [pytest.param(fn, kw, id=name) for name, fn, kw in cases]


@pytest.mark.gpu
@pytest.mark.parametrize("fn,kw", _gpu_cases())
def test_attention_partial_query_tiles(fn, kw):
    import torch
    assert torch.cuda.is_available()
    err, tol, info = fn(**kw)
    torch.cuda.synchronize()
    assert err <= tol, (err, tol, info)
