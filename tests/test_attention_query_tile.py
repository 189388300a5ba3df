"""Query tiles of the bf16 attention kernel (192 rows = three consumer warpgroups of 64 rows): the host's unit count
agrees with the kernel's tile height (the partial-tile layouts run on the GPU in tests/test_attention_plans_gpu.py)."""
import os
import re

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

