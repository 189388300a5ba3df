"""Sequence-parallel forward over views of mixed resolution == single-GPU forward (tools/sp_mixed_check.py): two ranks
sharing one GPU over gloo, and one GPU per rank over NCCL when two or more GPUs are present."""
import os
import socket
import subprocess
import sys

import pytest

from tests.conftest import ROOT

pytestmark = pytest.mark.gpu


def _run(nproc, env):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "sp_mixed_check.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, **env))
    assert "SP_MIXED_OK" in p.stdout, (p.stdout[-3000:], p.stderr[-3000:])
    return p.stdout


def test_mixed_resolution_two_ranks_on_one_gpu():
    import torch
    assert torch.cuda.device_count() >= 1
    out = _run(2, dict(SP_ONE_GPU="1"))
    assert "bit-identical" in out and "overlapped partials" in out


def test_mixed_resolution_over_nccl():
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    out = _run(2, dict(SP_ONE_GPU="0"))
    assert "overlapped partials" in out


def _rand(shape, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * 0.5).bfloat16().cuda()


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


@pytest.mark.parametrize("rows", [[736, 1024, 576], [2496, 1760], [1472, 1024]])
@pytest.mark.parametrize("use_local", [False, True])
def test_overlapped_partials_ignore_nan_padding(rows, use_local):
    """The overlapped path over a gather buffer whose padding rows hold NaN (as reused device memory may): every key
    range ends inside a 128-row block, and the rows past it must not reach the PV product.  Equal to one attention over the
    assembled real keys, for every rank."""
    import torch
    from types import SimpleNamespace
    from fast3r_b200 import ops
    from fast3r_b200.parallel import KVExchange, assemble_kv
    heads, mx = 2, max(rows)
    D = heads * 64
    for rank in range(len(rows)):
        kvx = KVExchange(SimpleNamespace(rank=rank, world=len(rows), overlap=True), 1, rows[rank], D, rows, mixed=True)
        kvx.buf = torch.full((len(rows), mx, 2 * D), float("nan"), dtype=torch.bfloat16, device="cuda")
        for p, n in enumerate(rows):
            kvx.buf[p, :n] = _rand((n, 2 * D), 10 + p)
        q = _rand((rows[rank], D), 20 + rank)
        local = kvx.buf[rank, :rows[rank]].clone() if use_local else None
        n_parts = kvx.partials(ops, q, local, heads=heads, scale=0.16, peers_landed=lambda: None)
        out = torch.empty(rows[rank], D, dtype=torch.bfloat16, device="cuda")
        ops.attention_merge(kvx.parts[0], kvx.parts[1], n_parts, out, batch=1, heads=heads, sq=rows[rank])
        ref = torch.empty_like(out)
        ops.attention(q, assemble_kv(kvx.buf, 1, rows), ref, batch=1, heads=heads, sq=rows[rank], skv=sum(rows), scale=0.16)
        torch.cuda.synchronize()
        assert not torch.isnan(out.float()).any(), (rows, rank)
        assert _rel(out, ref) < 8e-3, (rows, rank, _rel(out, ref))


def test_partial_key_range_ignores_rows_past_it_batch2():
    """f3r_attention_partial with batch 2 on a buffer of kv_rows_total rows per sample: the rows after the range (NaN here)
    are not read; equal to f3r_attention on the range alone."""
    import torch
    from fast3r_b200 import ops
    heads, sq, total, row0, skv = 2, 300, 1200, 200, 700
    D = heads * 64
    kv = torch.full((2, total, 2 * D), float("nan"), dtype=torch.bfloat16, device="cuda")
    kv[:, row0:row0 + skv] = _rand((2, skv, 2 * D), 3)
    q = _rand((2 * sq, D), 4)
    part_o = torch.empty(1, 2 * sq, D, dtype=torch.float32, device="cuda")
    part_lse = torch.empty(1, 2, heads, sq, dtype=torch.float32, device="cuda")
    ops.attention_partial(q, kv.view(-1, 2 * D), part_o, part_lse, part_base=0, n_split=1, batch=2, heads=heads, sq=sq,
                          kv_rows_total=total, kv_row0=row0, skv=skv, scale=0.16)
    out = torch.empty(2 * sq, D, dtype=torch.bfloat16, device="cuda")
    ops.attention_merge(part_o, part_lse, 1, out, batch=2, heads=heads, sq=sq)
    ref = torch.empty_like(out)
    ops.attention(q, kv[:, row0:row0 + skv].contiguous().view(-1, 2 * D), ref, batch=2, heads=heads, sq=sq, skv=skv,
                  scale=0.16, kv_split=1)
    torch.cuda.synchronize()
    assert not torch.isnan(out.float()).any()
    assert _rel(out, ref) < 8e-3
