"""The C-ABI emulator used by the CPU host-orchestration tests (tests/abi_emulator.py) must describe the real
kernels: same call, same inputs, outputs compared (bf16 rounding tolerance).  Needs an H100."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _both(fn_name, make_args):
    """Runs ops.<fn> on CUDA copies and abi_emulator.<fn> on CPU copies of the same arguments; returns the pairs of
    output tensors (those whose key starts with 'out', or 'pts'/'conf'/'lse')."""
    from fast3r_b200 import ops
    from tests import abi_emulator as E
    args_cpu, kw_cpu = make_args()
    to_gpu = lambda t: t.cuda() if torch.is_tensor(t) else t  # noqa: E731
    args_gpu = [to_gpu(a) for a in args_cpu]
    kw_gpu = {k: to_gpu(v) for k, v in kw_cpu.items()}
    getattr(ops, fn_name)(*args_gpu, **kw_gpu)
    torch.cuda.synchronize()
    getattr(E, fn_name)(*args_cpu, **kw_cpu)
    outs = []
    for k in kw_cpu:
        if torch.is_tensor(kw_cpu[k]) and (k.startswith("out") or k in ("pts", "conf", "lse")):
            outs.append((k, kw_gpu[k], kw_cpu[k]))
    return outs


def _r(shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype)


CASES = {}


def case(f):
    CASES[f.__name__] = f
    return f


@case
def gemm_rope_split():
    from fast3r_b200 import lib as L
    n_img, gh, gw, D = 2, 3, 4, 128
    P = gh * gw
    M = n_img * P
    j = torch.arange(16, dtype=torch.float32)
    ang = torch.arange(8, dtype=torch.float32)[:, None] * (1.0 / (100.0 ** (j / 16.0)))[None]
    return "gemm", lambda: ([_r((M, D), 1), _r((3 * D, 1, D), 2, D ** -0.5)],
                            dict(w=M, bias=_r((3 * D,), 3, 1.0, torch.float32),
                                 out0=torch.zeros(M, D, dtype=torch.bfloat16), ldo=D, split_col=D,
                                 out0b=torch.zeros(M, 2 * D, dtype=torch.bfloat16), ldo_b=2 * D, epi=L.EPI_ROPE,
                                 tok_per_img=P, grid_w=gw, rope_cols=2 * D, rope_cos=ang.cos().contiguous(),
                                 rope_sin=ang.sin().contiguous()))


@case
def gemm_idxemb_per_row():
    from fast3r_b200 import lib as L
    M, D = 50, 128
    return "gemm", lambda: ([_r((M, D), 4), _r((D, 1, D), 5, D ** -0.5)],
                            dict(w=M, bias=_r((D,), 6, 1.0, torch.float32), out0=torch.zeros(M, D), epi=L.EPI_IDXEMB,
                                 tok_per_img=0, emb_table=_r((1000, D), 7, 1.0, torch.float32),
                                 emb_ids=torch.randint(0, 1000, (M,), generator=torch.Generator().manual_seed(8),
                                                       dtype=torch.int32)))


@case
def gemm_conv3x3_res_out1():
    nb, H, W, C, N = 2, 5, 6, 96, 256
    return "gemm", lambda: ([_r((nb, H, W, C), 9), _r((N, 9, C), 10, (9 * C) ** -0.5)],
                            dict(w=W, h=H, nb=nb, taps=9, bias=_r((N,), 11, 1.0, torch.float32),
                                 out0=torch.zeros(nb, H, W, N, dtype=torch.bfloat16),
                                 out1=torch.zeros(nb, H, W, N, dtype=torch.bfloat16),
                                 res0=_r((nb, H, W, N), 12), res1=_r((nb, H, W, N), 13)))


@case
def gemm_convt():
    from fast3r_b200 import lib as L
    nb, H, W, C, k = 2, 3, 4, 96, 4
    return "gemm", lambda: ([_r((nb, H, W, C), 14), _r((k * k * C, 1, C), 15, C ** -0.5)],
                            dict(w=W, h=H, nb=nb, bias=_r((C,), 16, 1.0, torch.float32),
                                 out0=torch.zeros(nb, H * k, W * k, C, dtype=torch.bfloat16), epi=L.EPI_CONVT,
                                 ct_k=k, ct_cout=C))


@case
def gemm_final():
    from fast3r_b200 import lib as L
    nb, H, W, C = 1, 8, 48, 128
    return "gemm", lambda: ([_r((nb, H, W, C), 17), _r((128, 9, C), 18, (9 * C) ** -0.5)],
                            dict(w=W, h=H, nb=nb, taps=9, bias=_r((128,), 19, 0.5, torch.float32), epi=L.EPI_FINAL,
                                 w4=_r((4, 128), 20, 128 ** -0.5, torch.float32), b4=_r((4,), 21, 0.5, torch.float32),
                                 pts=torch.zeros(nb, H, W, 3), conf=torch.zeros(nb, H, W)))


@case
def gemm_resid_f32_gelu():
    from fast3r_b200 import lib as L
    M, K, N = 300, 256, 512
    return "gemm", lambda: ([_r((M, K), 22), _r((N, 1, K), 23, K ** -0.5)],
                            dict(w=M, bias=_r((N,), 24, 1.0, torch.float32),
                                 out0=torch.zeros(M, N, dtype=torch.bfloat16), act=L.ACT_GELU))


@case
def attention_tails():
    batch, heads, sq, skv = 2, 2, 200, 333
    D = heads * 64
    return "attention", lambda: ([_r((batch * sq, D), 25), _r((batch * skv, 2 * D), 26),
                                  ], dict(out=torch.zeros(batch * sq, D, dtype=torch.bfloat16), batch=batch,
                                          heads=heads, sq=sq, skv=skv, scale=0.16019,
                                          lse=torch.zeros(batch, heads, sq)))


@pytest.mark.parametrize("name", sorted(CASES))
def test_kernel_matches_emulator(name):
    fn_name, make = CASES[name]()
    if fn_name == "attention":  # ops.attention takes `out` positionally
        orig = make

        def make():
            a, kw = orig()
            return a + [kw.pop("out")], kw
        from fast3r_b200 import ops
        from tests import abi_emulator as E
        a_cpu, kw_cpu = make()
        a_gpu = [t.cuda() for t in a_cpu]
        kw_gpu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in kw_cpu.items()}
        ops.attention(*a_gpu, **kw_gpu)
        torch.cuda.synchronize()
        E.attention(*a_cpu, **kw_cpu)
        assert _rel(a_gpu[2], a_cpu[2]) < 8e-3
        assert _rel(kw_gpu["lse"], kw_cpu["lse"]) < 1e-5
        return
    for key, got, want in _both(fn_name, make):
        tol = 2e-5 if got.dtype == torch.float32 and key not in ("pts", "conf") else 6e-3
        if key in ("pts", "conf"):
            tol = 2e-3
        assert _rel(got, want) < tol, (name, key, _rel(got, want))
