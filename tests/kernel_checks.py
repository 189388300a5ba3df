"""Per-kernel numerics checks: each CUDA op (through the C ABI) against a plain PyTorch fp32 reference of the
same op on the same bf16-rounded operands (the GEMM cases: per element against float64, tests/test_gemm_plans_gpu.py).  Used by tests/test_kernels_gpu.py (asserting) and by
tools/gpu_check.py (report-everything mode for debugging on the GPU box)."""
import math

import torch
import torch.nn.functional as F

from fast3r_b200 import lib as L
from fast3r_b200 import ops


def rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _rand(shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def check_gemm(names):
    """The GEMM cases `names` of tests/gemm_plans.CASES, each checked per element against float64 and for its launch
    plan (tests/test_gemm_plans_gpu.run_case; it raises on a failure)."""
    from tests import gemm_plans as GP
    from tests.test_gemm_plans_gpu import run_case
    for name in names:
        i, case = next((i, c) for i, c in enumerate(GP.CASES) if c["name"] == name)
        assert GP.plan_key(case) == case["key"], (name, GP.plan_key(case), case["key"])
        run_case(case, seed=1000 + i)
    return 0.0, 0.0, {}


def attention_ref(q, k, v, scale):
    a = (q.float() @ k.float().transpose(-2, -1)) * scale
    return a.softmax(-1) @ v.float()


def check_attention(batch=2, heads=2, sq=736, skv=736, scale=0.125, seed=90, qscale=1.0):
    D = heads * 64
    q = _rand((batch * sq, D), seed, qscale)
    kv = _rand((batch * skv, 2 * D), seed + 1)
    out = torch.zeros(batch * sq, D, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(batch, heads, sq, dtype=torch.float32, device="cuda")
    ops.attention(q, kv, out, batch=batch, heads=heads, sq=sq, skv=skv, scale=scale, lse=lse)
    qh = q.reshape(batch, sq, heads, 64).transpose(1, 2)
    kh = kv[:, :D].reshape(batch, skv, heads, 64).transpose(1, 2)
    vh = kv[:, D:].reshape(batch, skv, heads, 64).transpose(1, 2)
    ref = attention_ref(qh, kh, vh, scale).transpose(1, 2).reshape(batch * sq, D)
    lref = torch.logsumexp((qh.float() @ kh.float().transpose(-2, -1)) * scale, -1)
    e = rel(out, ref)
    info = dict(lse=rel(lse, lref), nan=bool(torch.isnan(out.float()).any()))
    if e > 1e-2:  # localise: per 128-row tile / per head / per 16-col group errors
        o = out.float().reshape(batch, sq, heads, 64)
        r = ref.reshape(batch, sq, heads, 64)
        info["per_head"] = [rel(o[:, :, hh], r[:, :, hh]) for hh in range(heads)]
        info["per_qtile"] = [rel(o[0, s:s + 128], r[0, s:s + 128]) for s in range(0, min(sq, 1024), 128)]
        info["per_dgroup"] = [rel(o[..., c:c + 16], r[..., c:c + 16]) for c in range(0, 64, 16)]
    return e, 8e-3, info


def check_attention_ranges(heads=2, sq=700, chunk=736, world=4, rank=1, scale=0.16019, seed=95):
    """Sequence-parallel style: attend to the local key chunk, then to the ranges before / after it (each key-sliced),
    merge by log-sum-exp; must equal attention over all keys."""
    D = heads * 64
    skv = chunk * world
    q = _rand((sq, D), seed)
    kv = _rand((skv, 2 * D), seed + 1)
    lo, hi = rank * chunk, (rank + 1) * chunk
    ranges = [(lo, chunk)] + [r for r in ((0, lo), (hi, skv - hi)) if r[1] > 0]
    splits = [1, 2, 3][:len(ranges)]
    slots = sum(splits)
    part_o = torch.zeros(slots, sq, D, dtype=torch.float32, device="cuda")
    part_lse = torch.zeros(slots, 1, heads, sq, dtype=torch.float32, device="cuda")
    base = 0
    for (row0, n), ns in zip(ranges, splits):
        ops.attention_partial(q, kv, part_o, part_lse, part_base=base, n_split=ns, batch=1, heads=heads, sq=sq,
                              kv_rows_total=skv, kv_row0=row0, skv=n, scale=scale)
        base += ns
    out = torch.zeros(sq, D, dtype=torch.bfloat16, device="cuda")
    ops.attention_merge(part_o, part_lse, slots, out, batch=1, heads=heads, sq=sq)
    qh = q.reshape(1, sq, heads, 64).transpose(1, 2)
    kh = kv[:, :D].reshape(1, skv, heads, 64).transpose(1, 2)
    vh = kv[:, D:].reshape(1, skv, heads, 64).transpose(1, 2)
    ref = attention_ref(qh, kh, vh, scale).transpose(1, 2).reshape(sq, D)
    return rel(out, ref), 8e-3, dict(nan=bool(torch.isnan(out.float()).any()))


def check_attention_autosplit(batch=1, heads=4, sq=600, skv=4000, scale=0.16019, seed=97):
    """Few query tiles: ops.attention slices the keys (pick_kv_split) and merges; same result as one slice."""
    D = heads * 64
    q = _rand((batch * sq, D), seed)
    kv = _rand((batch * skv, 2 * D), seed + 1)
    a = torch.zeros(batch * sq, D, dtype=torch.bfloat16, device="cuda")
    b = torch.zeros_like(a)
    ops.attention(q, kv, a, batch=batch, heads=heads, sq=sq, skv=skv, scale=scale, kv_split=1)
    ns = ops.pick_kv_split(batch * heads * ((sq + 127) // 128), (skv + 127) // 128)
    ops.attention(q, kv, b, batch=batch, heads=heads, sq=sq, skv=skv, scale=scale)
    return rel(b, a), 3e-3, dict(auto_split=ns)


def check_attention_n320_slices(heads=1, sq=256, skv=235520, scale=0.16019, seed=99):
    """The N=320 key count (235 520 keys = 1 840 key blocks): one pass over all keys vs 4 key slices merged by their
    log-sum-exp - two different accumulation orders of the same softmax must agree (size-independent property)."""
    D = heads * 64
    q = _rand((sq, D), seed)
    kv = _rand((skv, 2 * D), seed + 1)
    a = torch.zeros(sq, D, dtype=torch.bfloat16, device="cuda")
    b = torch.zeros_like(a)
    ops.attention(q, kv, a, batch=1, heads=heads, sq=sq, skv=skv, scale=scale, kv_split=1)
    ops.attention(q, kv, b, batch=1, heads=heads, sq=sq, skv=skv, scale=scale, kv_split=4)
    # sanity against fp32 math on a subset of the rows
    qs = q[:32].float().reshape(32, heads, 64).transpose(0, 1)
    kh = kv[:, :D].float().reshape(skv, heads, 64).transpose(0, 1)
    vh = kv[:, D:].float().reshape(skv, heads, 64).transpose(0, 1)
    ref = (((qs @ kh.transpose(-2, -1)) * scale).softmax(-1) @ vh).transpose(0, 1).reshape(32, D)
    return max(rel(b, a), rel(a[:32], ref)), 8e-3, dict(slices_vs_single=rel(b, a), vs_fp32=rel(a[:32], ref))


def check_layernorm(rows=1000, dim=1024, eps=1e-5, seed=100):
    x = _rand((rows, dim), seed, 2.0, torch.float32) + 0.5
    w, b = _rand((dim,), seed + 1, 1.0, torch.float32), _rand((dim,), seed + 2, 1.0, torch.float32)
    out = torch.zeros(rows, dim, dtype=torch.bfloat16, device="cuda")
    ops.layernorm(x, w, b, eps, out)
    ref = F.layer_norm(x, (dim,), w, b, eps)
    o32 = torch.zeros(rows, dim, dtype=torch.float32, device="cuda")
    ops.layernorm(x, w, b, eps, o32)
    return max(rel(out, ref), rel(o32, ref) * 1000), 4e-3, dict(f32=rel(o32, ref))


def check_im2col_patch(n=3, H=64, W=96, seed=110):
    img = _rand((n, 3, H, W), seed, 1.0, torch.float32)
    out = torch.zeros(n * (H // 16) * (W // 16), 768, dtype=torch.bfloat16, device="cuda")
    ops.im2col_patch(img, out)
    ref = F.unfold(img, kernel_size=16, stride=16).transpose(1, 2).reshape(-1, 768).to(torch.bfloat16)
    return float((out.float() - ref.float()).abs().max()), 1e-9, {}


def check_im2col3x3s2(n=2, H=5, W=6, C=64, seed=120):
    x = _rand((n, H, W, C), seed)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    out = torch.zeros(n * Ho * Wo, 9 * C, dtype=torch.bfloat16, device="cuda")
    ops.im2col3x3s2(x, out, n, H, W, C, Ho, Wo)
    u = F.unfold(x.float().permute(0, 3, 1, 2), kernel_size=3, stride=2, padding=1)  # (n, C*9, L) c-major
    ref = u.reshape(n, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(n * Ho * Wo, 9 * C)
    return float((out.float() - ref).abs().max()), 1e-9, {}


def check_upsample(n=2, H=12, W=16, C=64, crop=True, seed=130):
    x = _rand((n, H, W, C), seed)
    Ho, Wo = (2 * H - 1, 2 * W) if crop else (2 * H, 2 * W)
    out = torch.zeros(n, Ho, Wo, C, dtype=torch.bfloat16, device="cuda")
    ops.upsample2x(x, out, n, H, W, C, Ho, Wo)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True)
    ref = ref[:, :, :Ho, :Wo].permute(0, 2, 3, 1)
    return rel(out, ref), 4e-3, {}


def check_cast(n=4096 * 3, seed=140):
    x = _rand((n,), seed, 1.0, torch.float32)
    out = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    ops.cast_bf16(x, out)
    return float((out.float() - x.to(torch.bfloat16).float()).abs().max()), 1e-9, {}


# ---------------------------------------------------------------- parity path (hi/lo-split bf16 products, fp32 storage)
def _pack_x3(w):  # (N, taps, K) fp32 -> bf16 [Whi | Whi | Wlo]  (same packing as fast3r_b200.model._pk)
    hi = w.to(torch.bfloat16)
    lo = (w - hi.float()).to(torch.bfloat16)
    return torch.cat([hi, hi, lo], dim=-1).contiguous()


def check_split3(rows=300, k=200, seed=200):
    x = _rand((rows, k), seed, 3.0, torch.float32)
    out = torch.zeros(rows, 3 * k, dtype=torch.bfloat16, device="cuda")
    ops.split3(x, out, relu=True)
    v = F.relu(x)
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16)
    ref = torch.cat([hi, lo, hi], -1)
    exact = float((out.float() - ref.float()).abs().max())
    recon = rel(out[:, :k].float() + out[:, k:2 * k].float(), v)
    return max(exact, recon / 1e-5 * 1e-9), 1e-9, dict(recon=recon)


def check_linear_x3(M=1000, K=1024, N=512, seed=210, act=L.ACT_NONE):
    a = _rand((M, K), seed, 1.0, torch.float32)
    w = _rand((N, 1, K), seed + 1, K ** -0.5, torch.float32)
    bias = _rand((N,), seed + 2, 1.0, torch.float32)
    out = torch.zeros(M, N, dtype=torch.float32, device="cuda")
    ops.gemm_x3(a, _pack_x3(w), w=M, bias=bias, out0=out, act=act)
    ref = (a.double() @ w[:, 0].double().T + bias.double())
    if act == L.ACT_GELU:
        ref = F.gelu(ref)
    return rel(out, ref), 3e-5, {}


def check_conv3x3_x3(nb=2, H=9, W=24, C=96, N=256, seed=220):
    x = _rand((nb, H, W, C), seed, 1.0, torch.float32)
    w = _rand((N, C, 3, 3), seed + 1, (9 * C) ** -0.5, torch.float32)
    bias = _rand((N,), seed + 2, 1.0, torch.float32)
    r0 = _rand((nb, H, W, N), seed + 3, 1.0, torch.float32)
    out = torch.zeros(nb, H, W, N, dtype=torch.float32, device="cuda")
    ops.gemm_x3(x, _pack_x3(w.permute(0, 2, 3, 1).reshape(N, 9, C)), a_relu=True, w=W, h=H, nb=nb, taps=9, bias=bias,
                out0=out, res0=r0)
    ref = F.conv2d(F.relu(x).double().permute(0, 3, 1, 2), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1) + r0
    return rel(out, ref), 3e-5, {}


def check_attention_x3(batch=2, heads=2, sq=300, skv=736, scale=0.16019, seed=230, qscale=1.0):
    D = heads * 64
    q = _rand((batch * sq, D), seed, qscale, torch.float32)
    kv = _rand((batch * skv, 2 * D), seed + 1, 1.0, torch.float32)
    out = torch.zeros(batch * sq, D, dtype=torch.float32, device="cuda")
    lse = torch.zeros(batch, heads, sq, dtype=torch.float32, device="cuda")
    ops.attention_x3(q, kv, out, batch=batch, heads=heads, sq=sq, skv=skv, scale=scale, lse=lse)
    qh = q.reshape(batch, sq, heads, 64).transpose(1, 2).double()
    kh = kv[:, :D].reshape(batch, skv, heads, 64).transpose(1, 2).double()
    vh = kv[:, D:].reshape(batch, skv, heads, 64).transpose(1, 2).double()
    sc = (qh @ kh.transpose(-2, -1)) * scale
    ref = (sc.softmax(-1) @ vh).transpose(1, 2).reshape(batch * sq, D)
    return rel(out, ref), 5e-5, dict(lse=rel(lse, torch.logsumexp(sc, -1)), nan=bool(torch.isnan(out).any()))


def check_upsample_f32(n=2, H=12, W=16, C=256, crop=True, seed=240):
    x = _rand((n, H, W, C), seed, 1.0, torch.float32)
    Ho, Wo = (2 * H - 1, 2 * W) if crop else (2 * H, 2 * W)
    out = torch.zeros(n, Ho, Wo, C, dtype=torch.float32, device="cuda")
    ops.upsample2x(x, out, n, H, W, C, Ho, Wo)
    ref = F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True)
    return rel(out, ref[:, :, :Ho, :Wo].permute(0, 2, 3, 1)), 2e-6, {}


def check_im2col_patch_f32(n=2, H=32, W=48, seed=250):
    img = _rand((n, 3, H, W), seed, 1.0, torch.float32)
    out = torch.zeros(n * (H // 16) * (W // 16), 768, dtype=torch.float32, device="cuda")
    ops.im2col_patch(img, out)
    ref = F.unfold(img, kernel_size=16, stride=16).transpose(1, 2).reshape(-1, 768)
    return float((out - ref).abs().max()), 1e-9, {}


def check_add_f32(n=4096 * 5, seed=260):
    a, b = _rand((n,), seed, 1.0, torch.float32), _rand((n,), seed + 1, 1.0, torch.float32)
    ref = a + b
    ops.add_f32(a, b)
    return float((a - ref).abs().max()), 1e-9, {}


ALL = [
    ("x3_split3", check_split3, {}),
    ("x3_linear", check_linear_x3, {}),
    ("x3_linear_gelu_tails", check_linear_x3, dict(M=333, K=256, N=96, act=L.ACT_GELU)),
    ("x3_conv3x3_c96_relu_res", check_conv3x3_x3, {}),
    ("x3_attn_tails", check_attention_x3, {}),
    ("x3_attn_128", check_attention_x3, dict(batch=1, heads=1, sq=128, skv=128, scale=0.125)),
    ("x3_attn_peaky_long", check_attention_x3, dict(batch=1, heads=2, sq=256, skv=4096, scale=0.5, qscale=3.0)),
    ("x3_upsample_f32", check_upsample_f32, {}),
    ("x3_im2col_patch_f32", check_im2col_patch_f32, {}),
    ("x3_add_f32", check_add_f32, {}),
    ("cast", check_cast, {}),
    ("layernorm_1024", check_layernorm, {}),
    ("layernorm_128", check_layernorm, dict(rows=77, dim=128, eps=1e-6)),
    ("im2col_patch", check_im2col_patch, {}),
    ("im2col3x3s2", check_im2col3x3s2, {}),
    ("upsample_crop", check_upsample, {}),
    ("upsample_full", check_upsample, dict(H=23, W=32, C=128, crop=False)),
    ("linear_small_tails", check_gemm, dict(names=["linear_small_tails"])),
    ("linear_qkv_shape", check_gemm, dict(names=["linear_qkv_shape"])),
    ("linear_bn256", check_gemm, dict(names=["linear_bn256"])),
    ("linear_resid_gelu", check_gemm, dict(names=["linear_resid_gelu", "linear_resid_gelu_out1"])),
    ("linear_resid_splitk", check_gemm, dict(names=["linear_resid_splitk", "linear_resid_splitk_out1"])),  # K slices
    ("linear_split", check_gemm, dict(names=["linear_split"])),
    ("rope_epilogue", check_gemm, dict(names=["rope_epilogue"])),
    ("idxemb_epilogue", check_gemm, dict(names=["idxemb_epilogue"])),
    ("conv1x1_tinymap", check_gemm, dict(names=["conv1x1_tinymap"])),
    ("conv3x3_w256", check_gemm, dict(names=["conv3x3_w256"])),
    ("conv3x3_w6_c96_res", check_gemm, dict(names=["conv3x3_w6_c96_res"])),
    ("conv3x3_w24_c192", check_gemm, dict(names=["conv3x3_w24_c192"])),
    ("conv3x3_w512", check_gemm, dict(names=["conv3x3_w512"])),
    ("convT_k4", check_gemm, dict(names=["convT_k4"])),
    ("convT_k2", check_gemm, dict(names=["convT_k2"])),
    ("final_fused", check_gemm, dict(names=["final_fused"])),
    ("attn_736_b2h2", check_attention, {}),
    ("attn_128", check_attention, dict(batch=1, heads=1, sq=128, skv=128)),
    ("attn_256x384", check_attention, dict(batch=1, heads=2, sq=256, skv=384)),
    ("attn_tails_1000", check_attention, dict(batch=1, heads=3, sq=1000, skv=1000, scale=0.16019)),
    ("attn_24", check_attention, dict(batch=3, heads=2, sq=24, skv=24)),
    ("attn_long_3072", check_attention, dict(batch=1, heads=2, sq=512, skv=3072, scale=0.16019)),
    ("attn_peaky", check_attention, dict(batch=1, heads=2, sq=512, skv=2048, scale=0.5, qscale=3.0)),
    ("attn_q9tiles_oddpair", check_attention, dict(batch=1, heads=2, sq=2300, skv=1000, scale=0.16019)),
    ("attn_ranges_merge", check_attention_ranges, {}),
    ("attn_ranges_merge_rank0", check_attention_ranges, dict(rank=0, world=3, chunk=500, sq=300)),
    ("attn_autosplit", check_attention_autosplit, {}),
    ("attn_skv235520_slices", check_attention_n320_slices, {}),
    # the bench regime: 23 552 keys (N=32 views) = 184 key blocks of lazy-rescale accumulation, flat and peaky scores
    ("attn_skv23552", check_attention, dict(batch=1, heads=2, sq=512, skv=23552, scale=0.16019)),
    ("attn_skv23552_peaky", check_attention, dict(batch=1, heads=1, sq=256, skv=23552, scale=0.5, qscale=3.0)),
]
