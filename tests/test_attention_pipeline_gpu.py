"""Pipeline edges of the bf16 attention kernel: short key ranges where the prologue (block 0), the steady-state trip and
the last block (PV only) meet, with and without a partial last key block, in full and key-slice mode.  Needs an H100."""
import pytest

pytestmark = pytest.mark.gpu


def _cases():
    from tests import kernel_checks as KC
    cases = [
        # full mode: 2 key blocks with a partial last block (72 / 1 keys), 2 full blocks, 4 blocks with 1 key in the last
        ("attn_skv200", KC.check_attention, dict(batch=1, heads=2, sq=300, skv=200, scale=0.16019)),
        ("attn_skv129", KC.check_attention, dict(batch=2, heads=1, sq=130, skv=129, scale=0.16019)),
        ("attn_skv256", KC.check_attention, dict(batch=1, heads=2, sq=256, skv=256)),
        ("attn_skv385_peaky", KC.check_attention, dict(batch=1, heads=2, sq=200, skv=385, scale=0.5, qscale=3.0)),
        # key-slice mode: slices of 1 and 2 key blocks (full and partial) merged by their log-sum-exp
        ("attn_ranges_skv200", KC.check_attention_ranges, dict(heads=2, sq=300, chunk=200, world=2, rank=0)),
        ("attn_ranges_skv330", KC.check_attention_ranges, dict(heads=2, sq=300, chunk=330, world=3, rank=1)),
    ]
    return [pytest.param(fn, kw, id=name) for name, fn, kw in cases]


@pytest.mark.parametrize("fn,kw", _cases())
def test_attention_pipeline_edges(fn, kw):
    import torch
    assert torch.cuda.is_available()
    err, tol, info = fn(**kw)
    torch.cuda.synchronize()
    assert err <= tol, (err, tol, info)
