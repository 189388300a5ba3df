"""Each CUDA kernel (through the C ABI) vs a plain PyTorch fp32 reference of the same op.  Needs an H100."""
import pytest

pytestmark = pytest.mark.gpu


def _cases():
    from tests import kernel_checks as KC
    return [pytest.param(fn, kw, id=name) for name, fn, kw in KC.ALL]


@pytest.mark.parametrize("fn,kw", _cases())
def test_kernel(fn, kw):
    import torch
    assert torch.cuda.is_available()
    err, tol, info = fn(**kw)
    torch.cuda.synchronize()
    assert err <= tol, (err, tol, info)
